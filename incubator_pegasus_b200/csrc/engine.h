// engine.h — internal C++ view of the device engine (not part of the ABI).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/pegasus_b200.h"
#include "../host/hotkey.h"
#include "device_util.cuh"

namespace pgs {

struct Run {
    uint64_t id = 0;
    int32_t level = 0;
    pgs_run_info info{};
    // device allocations (owned)
    uint8_t *d_data = nullptr;
    uint64_t *d_blk_off = nullptr;
    uint32_t *d_blk_size = nullptr;
    uint32_t *d_blk_rec = nullptr;
    uint32_t *d_ikey_off = nullptr;
    uint8_t *d_ikeys = nullptr;
    uint32_t *d_rec_off = nullptr;
    uint32_t *d_bloom = nullptr;
    uint32_t bloom_lines = 0;
    uint64_t n_bloom_entries = 0; // user keys + distinct hash-key prefixes that went into the filter (sizes a merged run's filter)
    uint64_t data_cap = 0;
    cudaStream_t pool_stream;  // the buffers come from cudaMallocAsync on the engine's stream
    struct Engine *eng;        // large data buffers go back to the engine's spare list
    explicit Run(struct Engine *e);
    RunDev dev() const
    {
        return RunDev{d_data, d_blk_off, d_blk_size, d_blk_rec, d_ikey_off, d_ikeys, d_rec_off, d_bloom, bloom_lines, info.n_blocks, info.max_ukey_len, 0};
    }
    ~Run();
};

struct Engine {
    int device = 0;
    cudaStream_t stream = nullptr;
    pgs_engine_config cfg{};
    int sm_count = 0;
    int max_smem_optin = 0;
    uint32_t scan_static_smem = 0; // k_scan's static shared memory (lookup_init_kernels)
    uint64_t *d_crc = nullptr; // the crc64 table (2 KB) of partition-hash validation in reads and compactions
    std::atomic<uint64_t> launches{0};
    std::atomic<uint64_t> next_run_id{1};
    // reads of different host threads go to different streams (runs are complete before they become visible, so a reader
    // needs no ordering with the stream that built them); writes / uploads / compactions use `stream`
    static constexpr int kReadStreams = 8;
    cudaStream_t up_copy = nullptr;     // host -> HBM copies of run uploads (the index build follows chunk by chunk on `stream`)
    cudaStream_t rd_streams[kReadStreams] = {};
    cudaStream_t read_stream();
    // reusable pinned staging + device scratch
    std::mutex mu;
    void *h_pinned = nullptr;
    size_t h_pinned_cap = 0;
    void *pinned(size_t bytes);
    // Spare list of large block buffers.  A compaction frees a few ~GB buffers and asks for one of a different size; what
    // the stream-ordered pool does with that depends on its placement choices, and growing the pool is slow.
    // Buffers of dropped runs are therefore kept here (all uses are ordered on `stream`) and handed to the next taker.
    struct Spare { uint8_t *p; uint64_t cap; };
    std::mutex spare_mu;
    std::vector<Spare> spares;
    uint64_t spare_bytes_max = 0; // set at open from the device's memory size
    cudaError_t alloc_data(Run &r, uint64_t need); // r.d_data / r.data_cap: a kept buffer when one fits, else a new one
    void give_data(uint8_t *p, uint64_t cap);
    // pinned host staging for the small arrays of an upload (block handles in, per-block counts out): with pageable memory a
    // cudaMemcpyAsync waits for everything queued before it on its stream, which stalls the upload pipeline between runs
    struct Pin { void *p; size_t cap; };
    std::mutex pin_mu;
    std::vector<Pin> pins;
    void *take_pinned(size_t need, size_t *cap);
    void give_pinned(void *p, size_t cap);
    ~Engine();
};

struct Partition {
    Engine *eng;
    int32_t app_id, pidx;
    uint32_t data_version;
    std::mutex mu;
    std::vector<std::shared_ptr<Run>> runs; // read order: L0 newest first, then L1, L2 ...
    std::shared_ptr<Run> find(uint64_t id);
    void insert(std::shared_ptr<Run> r);
    // hot-key collectors of the replica (host/hotkey.h).  The READ collector's coarse counters of batched gets live in HBM
    // (hk_dev_buckets, hk_dev_n of them, allocated at the first capturing launch); a capturing launch holds hk_dev_mu shared
    // from its launch to the hand-over of its fine captures, analysis and STOP hold it exclusively, so no capture is lost
    // between reading the counters and zeroing them.
    HotkeyCollector hk_read{HOTKEY_READ}, hk_write{HOTKEY_WRITE};
    std::shared_mutex hk_dev_mu;
    unsigned long long *hk_dev_buckets = nullptr;
    uint32_t hk_dev_n = 0;
    ~Partition();
};

// the device half of the READ collector (lookup.cu): analysis and STOP of a partition's collectors, with its HBM counters
int32_t hotkey_analyse(Partition &p, uint32_t now);
int32_t hotkey_control(Partition &p, int32_t type, int32_t action, uint32_t now, std::string &text);
// pgs_get_batch; capture = false leaves the READ collector to the caller
int32_t get_batch(pgs_partition *ph, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                  uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used, bool capture);
// Where a scan call's answers go.  One request: its records and their bytes at kvs and arena, its resume key at resume.
// Several: the launch gives request i arena_stride bytes, kv_stride records and a resume slot of resume_stride bytes, and
// the answers come back packed -- request i's records at kvs + kv_base[i], their bytes at arena + arena_base[i] (n + 1
// entries each, may be null), its resume key at resume + i * resume_stride.  arena_cap / kv_cap bound the whole answer.
struct ScanOut {
    uint8_t *arena;
    uint64_t arena_stride, arena_cap;
    pgs_kv *kvs;
    uint32_t kv_stride;
    uint64_t kv_cap;
    uint8_t *resume;
    uint32_t resume_stride;
    uint64_t *arena_base;
    uint32_t *kv_base;
};
// range scans over parts[0] (req_part null), or forward scans over several partitions of one engine in one launch: request i
// reads partition slot req_part[i].  pinned = the runs to read instead of the partition's current ones (a parked scan context)
int32_t scan_many(pgs_partition *const *parts, uint32_t n_parts, const uint32_t *req_part, const pgs_scan_request *reqs, uint32_t n,
                  uint32_t now, pgs_scan_result *results, const ScanOut &out, const std::vector<std::shared_ptr<Run>> *pinned = nullptr);
// true when k_scan can stage one block of every current run of the partition in one request's launch; a batch with a reverse
// request gets PGS_NOT_SUPPORTED otherwise (the server folds L0 first, server.cpp)
bool scan_stages_every_run(pgs_partition *ph);

// pgs_partition_split over the runs `snap` of src (nullptr: its current runs)
int32_t partition_split(pgs_partition *src, const std::vector<std::shared_ptr<Run>> *snap, uint32_t src_count, uint32_t dst_count,
                        pgs_partition *const *dst, uint32_t n_dst, pgs_split_result *out);
// pgs_partition_split_many over the runs snaps[i] of job i's parent (snaps null: the parents' current runs)
int32_t partition_split_many(const pgs_split_job *jobs, uint32_t n, uint32_t src_count, uint32_t dst_count,
                             const std::vector<std::shared_ptr<Run>> *snaps, pgs_split_result *out);

void set_error(const char *fmt, ...);
int32_t cuda_fail(cudaError_t e, const char *what);
#define PGS_CUDA(expr)                                                                             \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) return ::pgs::cuda_fail(_e, #expr);                                 \
    } while (0)

// the device scratch and events of one launch.  They are released when the owner goes out of scope, after the launch's
// final synchronise or on an error return; buffers go back with cudaFreeAsync on the launch's stream.
struct LaunchScratch {
    cudaStream_t st;
    std::vector<void *> bufs;
    std::vector<cudaEvent_t> events;
    explicit LaunchScratch(cudaStream_t s) : st(s) {}
    LaunchScratch(const LaunchScratch &) = delete;
    LaunchScratch &operator=(const LaunchScratch &) = delete;
    ~LaunchScratch()
    {
        for (void *p : bufs) cudaFreeAsync(p, st);
        for (cudaEvent_t ev : events) cudaEventDestroy(ev);
    }
    template <class T> cudaError_t alloc(T *&p, size_t bytes)
    {
        cudaError_t e = cudaMallocAsync((void **)&p, bytes, st);
        if (e == cudaSuccess) bufs.push_back((void *)p);
        return e;
    }
    template <class T> cudaError_t upload(T *&p, const std::remove_const_t<T> *src, size_t n) // a device copy of n host elements
    {
        cudaError_t e = alloc(p, sizeof(T) * n);
        return e == cudaSuccess ? cudaMemcpyAsync((void *)p, src, sizeof(T) * n, cudaMemcpyHostToDevice, st) : e;
    }
    cudaError_t event(cudaEvent_t &ev)
    {
        cudaError_t e = cudaEventCreate(&ev);
        if (e == cudaSuccess) events.push_back(ev);
        return e;
    }
};

// The (pointer, count, fill[, out]) buffers of a launch plan (build_buffers, sort_buffers, split_buffers, ...) in S: count
// elements each, every byte set to fill unless it is kNoFill.  ce keeps the first failure; after it nothing is allocated.
inline auto scratch_buffers(LaunchScratch &S, cudaError_t &ce)
{
    return [&S, &ce](auto *&p, uint64_t count, int fill, bool = false) {
        const size_t bytes = sizeof(*p) * count;
        if (ce != cudaSuccess) return;
        ce = S.alloc(p, bytes ? bytes : 16);
        if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync((void *)p, fill, bytes, S.st);
    };
}
// The (pointer, bytes, ReadInit) buffers of a launch plan (get_buffers, scan_buffers, stage_records) in S, on its stream; ce
// keeps the first failure
inline auto device_buffers(LaunchScratch &S, cudaError_t &ce)
{
    return [&S, &ce](auto *&p, uint64_t bytes, ReadInit in) {
        if (ce == cudaSuccess) ce = S.alloc(p, bytes);
        if (ce == cudaSuccess && in.src) ce = cudaMemcpyAsync((void *)p, in.src, in.src_bytes, cudaMemcpyHostToDevice, S.st);
        if (ce == cudaSuccess && in.fill != kNoFill) ce = cudaMemsetAsync((void *)p, in.fill, bytes, S.st);
    };
}

} // namespace pgs

struct pgs_engine { pgs::Engine e; };
struct pgs_partition { pgs::Partition p; };
