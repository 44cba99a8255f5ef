// engine.h — internal C++ view of the device engine (not part of the ABI).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/pegasus_b200.h"
#include "format.h"

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
};

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

// scans an uploaded / freshly merged run's blocks on the device and fills the index + info

} // namespace pgs

struct pgs_engine { pgs::Engine e; };
struct pgs_partition { pgs::Partition p; };
