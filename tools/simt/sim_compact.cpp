// sim_compact.cpp — runs the compaction kernels (incubator_pegasus_b200/csrc/compact_kernels.cuh, the same source nvcc compiles
// for sm_90a) inside the host SIMT interpreter of simt.h.  Test / development tool: lets the CPU test-suite execute the kernels'
// logic against the oracle without a GPU.  NOT part of the product library and never a fallback for it.
#include "simt.h"

#define PGS_SIM 1
#include "../../incubator_pegasus_b200/csrc/build_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/compact_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/hotkey_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/index_kernel.cuh"
#include "../../incubator_pegasus_b200/csrc/read_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/scan_kernel.cuh"
#include "../../incubator_pegasus_b200/csrc/sort_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/split_kernels.cuh"

#include <sys/mman.h>

#include <cstdarg>
#include <memory>
#include <new>
#include <string>
#include <vector>

using namespace pgs;

// the message of a call the read launch plan refuses (the library keeps it for pgs_last_error)
void pgs::set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    fputs("sim: ", stderr);
    vfprintf(stderr, fmt, ap);
    fputc('\n', stderr);
    va_end(ap);
}

namespace {

constexpr uint32_t kSimSmemOptin = 227 * 1024; // the opt-in shared memory per CTA of an H100

// host buffers standing in for device memory: each one its own allocation of exactly the size the library allocates, so that
// AddressSanitizer checks the kernels against the library's bounds
using HostMem = std::vector<std::shared_ptr<void>>;
template <class T>
T *host_alloc(HostMem &mem, T *&p, uint64_t n, int fill)
{
    const size_t bytes = sizeof(T) * n;
    void *b = ::operator new(bytes ? bytes : 1, std::align_val_t(64));
    memset(b, fill, bytes);
    mem.emplace_back(b, [](void *x) { ::operator delete(x, std::align_val_t(64)); });
    return p = (T *)b;
}

// A run's data of kSparseLoad bytes or more (runs placed past 4 GiB) lives in an anonymous mapping, zero until written, and
// only the source pages that hold a non-zero byte are copied into it: the copy equals the caller's bytes everywhere, but the
// gigabytes of zeros in front of or between such a run's blocks cost neither host memory nor copy time.  Scratch of that size
// (a merge's key-stream bound grows with the span of its inputs, gaps included) is such a mapping too, zero rather than
// poisoned.  AddressSanitizer checks these buffers at page granularity only.
constexpr uint64_t kSparseLoad = 1ull << 30;
template <class T>
T *sparse_alloc(HostMem &mem, T *&p, uint64_t n)
{
    const uint64_t bytes = sizeof(T) * n;
    void *b = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (b == MAP_FAILED) throw std::bad_alloc();
    mem.emplace_back(b, [bytes](void *x) { munmap(x, bytes); });
    return p = (T *)b;
}
void sparse_copy(uint8_t *dst, const uint8_t *src, uint64_t n)
{
    constexpr uint64_t kPage = 4096;
    for (uint64_t o = 0; o < n; o += kPage) {
        const uint64_t len = std::min(kPage, n - o);
        const uint64_t *w = (const uint64_t *)(src + o); // src is at least 8-aligned (a numpy buffer or the library's)
        bool zero = true;
        for (uint64_t i = 0; i < len / 8 && zero; i++) zero = w[i] == 0;
        for (uint64_t i = len / 8 * 8; i < len && zero; i++) zero = src[o + i] == 0;
        if (!zero) memcpy(dst + o, src + o, len);
    }
}

// a run in host memory, with the buffer fields of the library's Run (engine.h)
struct HostRun {
    HostMem mem;
    uint8_t *d_data = nullptr, *d_ikeys = nullptr;
    uint64_t *d_blk_off = nullptr;
    uint32_t *d_blk_size = nullptr, *d_blk_rec = nullptr, *d_ikey_off = nullptr, *d_rec_off = nullptr, *d_bloom = nullptr;
    uint32_t bloom_lines = 0;
    uint64_t n_bloom_entries = 0;
    pgs_run_info info{};
    RunDev dev() const
    {
        return RunDev{d_data, d_blk_off, d_blk_size, d_blk_rec, d_ikey_off, d_ikeys, d_rec_off, d_bloom, bloom_lines, info.n_blocks, info.max_ukey_len, 0};
    }
};

// the (pointer, count, fill[, out]) buffers of a launch plan in mem at the library's sizes; what the library leaves unset
// (kNoFill) is poisoned until the kernels write it, unless the buffer takes kSparseLoad bytes or more
auto host_count_buffers(HostMem &mem)
{
    return [&mem](auto *&p, uint64_t count, int fill, bool = false) {
        if (fill == kNoFill && sizeof(*p) * count >= kSparseLoad) sparse_alloc(mem, p, count);
        else host_alloc(mem, p, count, fill == kNoFill ? 0xEE : fill);
    };
}

// the run's index and Bloom filter as pgs_run_upload builds them (engine.cu): index_scratch, pass 1, index_buffers, pass 2.
// max_blk: the run's largest block, as the library has it.  Returns the upload's status.
int32_t build_index(HostRun &r, uint32_t nb, uint32_t max_blk)
{
    HostMem scratch;
    IndexParams X{r.d_data, r.d_blk_off, r.d_blk_size, nb};
    index_scratch(X, host_count_buffers(scratch));
    *X.stats = index_stats_init();
    index_launch_pass1(X, 0, nb, nullptr);
    std::vector<uint32_t> rec_cum(nb + 1), key_cum(nb + 1);
    if (const int32_t rc = index_buffers(X, r, X.nrec, X.lastlen, *X.stats, rec_cum.data(), key_cum.data(), host_count_buffers(r.mem))) return rc;
    memcpy(r.d_blk_rec, rec_cum.data(), 4 * (nb + 1ull));
    memcpy(r.d_ikey_off, key_cum.data(), 4 * (nb + 1ull));
    index_launch_pass2(X, nullptr);
    if (X.stats->error) return (int32_t)X.stats->error;
    run_info_from_index(*X.stats, nb, r.d_blk_off[nb], max_blk, r.info);
    return PGS_OK;
}

// one run as the upload installs it (upload_stage_a of engine.cu): the handle rule, then the bytes up to the 16-aligned end of the
// last block (what the caller holds behind it stays on the host) with the product's slack, that end as blk_off[nb], the index
// and the filter.  Returns the upload's status.
int32_t load_run(HostRun &r, const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off, const uint32_t *blk_size, uint32_t nb)
{
    uint64_t last_end = 0;
    uint32_t max_blk = 0;
    if (run_handles_check(blk_off, blk_size, nb, data_bytes, last_end, max_blk) < nb) return PGS_INVALID_ARGUMENT;
    const uint64_t end = block_pad(last_end);
    if (end < kSparseLoad) memcpy(host_alloc(r.mem, r.d_data, end + 256, 0), data, std::min(data_bytes, end));
    else sparse_copy(sparse_alloc(r.mem, r.d_data, end + 256), data, std::min(data_bytes, end));
    memcpy(host_alloc(r.mem, r.d_blk_off, nb + 1, 0), blk_off, 8 * (size_t)nb);
    memcpy(host_alloc(r.mem, r.d_blk_size, nb, 0), blk_size, 4 * (size_t)nb);
    r.d_blk_off[nb] = end;
    return build_index(r, nb, max_blk);
}

uint64_t crc_tab[256];

struct Merged { // the output of the last sim_compact call
    HostRun run;
    MergeStats st{};
    uint32_t Q = 0;
} g_res;

std::vector<Merged> g_many; // the outputs of the last sim_compact_many call, one per job

struct Built { // the run of the last sim_run_build call
    HostRun run;
    uint64_t data_bytes = 0;
} g_built;

std::vector<Built> g_built_many; // the runs of the last sim_run_build_many call, one per job

struct Split { // the children of the last sim_split call
    std::vector<HostRun> child;
    std::vector<MergeStats> st;
    std::vector<uint8_t> built;
    uint32_t Q = 0;
} g_split;

std::vector<Split> g_split_many; // the children of the last sim_split_many call, one Split per parent run

} // namespace

extern "C" {

// returns a status code; the merged run stays in a static buffer until the next call (sim_result_* read it)
int32_t sim_compact(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                    const uint32_t *n_blocks, uint32_t block_size, uint32_t restart_interval, int32_t bottommost,
                    const pgs_filter_params *fp, uint32_t now, uint32_t group_lanes, uint64_t seg_weight, const uint64_t *crc_table)
{
    std::vector<HostRun> runs(k);
    MergeParams P{};
    P.k = k;
    CompactTotals T{};
    for (uint32_t i = 0; i < k; i++) {
        if (const int32_t rc = load_run(runs[i], data[i], data_bytes[i], blk_off[i], blk_size[i], n_blocks[i])) return rc;
        P.runs[i] = runs[i].dev();
        T.add(runs[i].info, runs[i].n_bloom_entries);
    }
    P.block_size = block_size;
    P.restart_interval = restart_interval;
    P.bottommost = bottommost ? 1 : 0;
    P.now = now;
    P.data_version = fp ? fp->data_version : 1;
    HostMem scratch;
    uint32_t n = 0;
    if (!compact_filter(P, fp, n)) return PGS_INVALID_ARGUMENT;
    if (n) {
        uint8_t *ops;
        memcpy(host_alloc(scratch, ops, n, 0), fp->ops, n);
        P.ops = ops;
    }
    if (P.validate_hash) {
        if (crc_table) memcpy(crc_tab, crc_table, sizeof crc_tab); else crc64_make_table(crc_tab);
        P.crc_table = (const unsigned long long *)crc_tab;
    }
    CompactGeometry geo{};
    if (group_lanes && group_lanes != 1 && group_lanes != 2 && group_lanes != 4 && group_lanes != 8 && group_lanes != 16) return PGS_INVALID_ARGUMENT;
    // seg_weight: smaller segments, so that a small test crosses many segment boundaries
    if (!compact_geometry(P, T, compact_smem_budget(kSimSmemOptin), geo, group_lanes, seg_weight)) return PGS_NOT_SUPPORTED;
    Merged &R = g_res;
    R = Merged{};
    compact_buffers(P, geo, T, R.run, [&](auto *&p, uint64_t n, int fill, bool out) { host_count_buffers(out ? R.run.mem : scratch)(p, n, fill); });
    MergeStats st = merge_stats_init();
    P.stats = &st;
    compact_launch(P, geo, 2, 2, nullptr, [](int) {});
    pgs_compact_result res{};
    R.run.n_bloom_entries = compact_result_stats(st, T.in_block_bytes, res, R.run.info);
    R.st = st;
    R.Q = P.Q;
    if (st.error) { fprintf(stderr, "sim_compact: status %u at segment %u of %u\n", st.error, st.error_seg, P.Q); return (int32_t)st.error; }
    return PGS_OK;
}

// n jobs through compact_many_geometry / compact_buffers / compact_launch_many, as pgs_compact_many runs them.  Job i merges
// k[i] runs, taken in order from the flat run arrays; bottommost[i] and fp[i] are its policy and filter.  group_lanes and
// seg_weight as sim_compact (seg_weight: the launch's one segment weight).  Returns a status; *launches = the launches made.
// Every job's output stays until the next call: sim_compact_many_select(i) makes job i's the one sim_result_* read.
int32_t sim_compact_many(uint32_t n, const uint32_t *k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off,
                         const uint32_t **blk_size, const uint32_t *n_blocks, uint32_t block_size, uint32_t restart_interval,
                         const int32_t *bottommost, const pgs_filter_params *fp, uint32_t now, uint32_t group_lanes, uint64_t seg_weight,
                         uint32_t *launches)
{
    g_many.clear();
    *launches = 0;
    uint32_t total = 0;
    for (uint32_t i = 0; i < n; i++) total += k[i];
    std::vector<HostRun> runs(total);
    for (uint32_t i = 0; i < total; i++)
        if (const int32_t rc = load_run(runs[i], data[i], data_bytes[i], blk_off[i], blk_size[i], n_blocks[i])) return rc;
    if (group_lanes && group_lanes != 1 && group_lanes != 2 && group_lanes != 4 && group_lanes != 8 && group_lanes != 16) return PGS_INVALID_ARGUMENT;
    crc64_make_table(crc_tab);
    HostMem scratch;
    std::vector<MergeParams> P(n);
    std::vector<CompactTotals> T(n);
    uint32_t any_hash = 0;
    for (uint32_t i = 0, r = 0; i < n; r += k[i], i++) {
        if (k[i] == 0) return PGS_INVALID_ARGUMENT;
        if (k[i] > kMaxRuns) return PGS_NOT_SUPPORTED;
        P[i].k = k[i];
        for (uint32_t x = 0; x < k[i]; x++) {
            P[i].runs[x] = runs[r + x].dev();
            T[i].add(runs[r + x].info, runs[r + x].n_bloom_entries);
        }
        P[i].block_size = block_size;
        P[i].restart_interval = restart_interval;
        P[i].bottommost = bottommost[i] ? 1 : 0;
        P[i].now = now;
        P[i].data_version = fp[i].data_version;
        uint32_t len = 0;
        if (!compact_filter(P[i], &fp[i], len)) return PGS_INVALID_ARGUMENT;
        if (len) {
            uint8_t *ops;
            memcpy(host_alloc(scratch, ops, len, 0), fp[i].ops, len);
            P[i].ops = ops;
        }
        if (P[i].validate_hash) { P[i].crc_table = (const unsigned long long *)crc_tab; any_hash = 1; }
    }
    MergeJobs M{};
    CompactGeometry shared{};
    std::vector<CompactGeometry> geo(n);
    if (!compact_many_geometry(P.data(), T.data(), geo.data(), n, compact_smem_budget(kSimSmemOptin), M, shared, group_lanes, seg_weight))
        return PGS_NOT_SUPPORTED;
    g_many.resize(n);
    std::vector<MergeStats> st(n, merge_stats_init());
    for (uint32_t i = 0; i < n; i++) {
        HostRun &run = g_many[i].run;
        compact_buffers(P[i], geo[i], T[i], run, [&](auto *&p, uint64_t cnt, int fill, bool out) { host_count_buffers(out ? run.mem : scratch)(p, cnt, fill); });
        P[i].stats = &st[i];
    }
    std::vector<uint32_t> seg_base(n + 1), blk_base(n + 1);
    compact_many_bases(P.data(), n, seg_base.data(), blk_base.data());
    host_alloc(scratch, M.ticket, 2, 0);
    M.job = P.data();
    M.seg_base = seg_base.data();
    M.blk_base = blk_base.data();
    M.validate_hash = any_hash;
    M.crc_table = (const unsigned long long *)crc_tab;
    *launches = compact_launch_many(M, shared, 2, 2, nullptr, [](int) {});
    for (uint32_t i = 0; i < n; i++) {
        Merged &R = g_many[i];
        pgs_compact_result res{};
        R.run.n_bloom_entries = compact_result_stats(st[i], T[i].in_block_bytes, res, R.run.info);
        R.st = st[i];
        R.Q = P[i].Q;
    }
    for (uint32_t i = 0; i < n; i++)
        if (st[i].error) { fprintf(stderr, "sim_compact_many: job %u: status %u at segment %u of %u\n", i, st[i].error, st[i].error_seg, P[i].Q); return (int32_t)st[i].error; }
    return PGS_OK;
}
// job i of the last sim_compact_many becomes the output sim_result_* read
int32_t sim_compact_many_select(uint32_t i)
{
    if (i >= g_many.size()) return PGS_INVALID_ARGUMENT;
    g_res = g_many[i];
    return PGS_OK;
}

void sim_result_sizes(uint64_t *data_bytes, uint32_t *n_blocks, uint32_t *n_segments)
{
    *data_bytes = g_res.st.tot_bytes;
    *n_blocks = (uint32_t)g_res.st.tot_blocks;
    *n_segments = g_res.Q;
}
void sim_result_copy(uint8_t *data, uint64_t *blk_off, uint32_t *blk_size, uint32_t *blk_rec, uint32_t *ikey_off, uint8_t *ikeys, uint32_t *rec_off)
{
    const HostRun &r = g_res.run;
    const uint32_t nb = (uint32_t)g_res.st.tot_blocks;
    memcpy(data, r.d_data, g_res.st.tot_bytes);
    memcpy(blk_off, r.d_blk_off, 8 * (size_t)(nb + 1));
    memcpy(blk_size, r.d_blk_size, 4 * (size_t)nb);
    if (blk_rec) memcpy(blk_rec, r.d_blk_rec, 4 * (size_t)(nb + 1));
    if (ikey_off) memcpy(ikey_off, r.d_ikey_off, 4 * (size_t)(nb + 1));
    if (ikeys) memcpy(ikeys, r.d_ikeys, g_res.st.tot_keyb);
    if (rec_off) memcpy(rec_off, r.d_rec_off, 4 * (size_t)g_res.st.tot_recs);
}
// the counters of pgs_compact_result, in its order: in_records, out_records, in_bytes, out_bytes, dropped_shadowed,
// dropped_tombstone, dropped_expired, dropped_user, dropped_stale, ttl_rewritten, + run info: tombstones, raw key, raw value,
// max_ukey, max_vlen, max_blk_size, max_blk_rec, smallest_seq, largest_seq, index key bytes
void sim_result_stats(uint64_t *o)
{
    pgs_compact_result r{};
    pgs_run_info i{};
    compact_result_stats(g_res.st, 0, r, i);
    const uint64_t v[20] = {r.in_records, r.out_records, r.in_bytes, r.out_bytes, r.dropped_shadowed, r.dropped_tombstone, r.dropped_expired,
                            r.dropped_user, r.dropped_stale, r.ttl_rewritten, i.n_tombstones, i.raw_key_bytes, i.raw_value_bytes, i.max_ukey_len,
                            i.max_value_len, i.max_block_size, i.max_block_records, i.smallest_seq, i.largest_seq, g_res.st.tot_keyb};
    memcpy(o, v, sizeof v);
}

// 1 when the merged run's Bloom filter admits the byte string (a user key or a hash-key prefix)
int32_t sim_result_bloom_check(const uint8_t *key, uint32_t len)
{
    return bloom_may_contain(g_res.run.d_bloom, g_res.run.bloom_lines, bloom_hash_bytes(key, len)) ? 1 : 0;
}

// up to cap words of a run's Bloom filter; returns its number of lines
static uint32_t copy_bloom(const HostRun &r, uint32_t *out, uint64_t cap)
{
    memcpy(out, r.d_bloom, 4 * std::min<uint64_t>(cap, (uint64_t)r.bloom_lines * 16));
    return r.bloom_lines;
}

// the Bloom filter of the last sim_compact output (the one k_emit built)
uint32_t sim_result_bloom(uint32_t *out, uint64_t cap) { return copy_bloom(g_res.run, out, cap); }

// the Bloom filter the upload builds for one run (the index build of build_index); 0 lines: a run the upload refuses
uint32_t sim_run_bloom(const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off, const uint32_t *blk_size, uint32_t n_blocks,
                       uint32_t *out, uint64_t cap)
{
    HostRun r;
    return load_run(r, data, data_bytes, blk_off, blk_size, n_blocks) == PGS_OK ? copy_bloom(r, out, cap) : 0;
}

// One run loaded as the upload loads it; returns the upload's status.  On PGS_OK: *info = its pgs_run_info (level and run id
// zero), *n_bloom_entries and *bloom_lines = the filter's sizing, and every non-null array gets what the upload left on the
// device: blk_rec[nb + 1], ikey_off[nb + 1], ikeys[ikey_off[nb]], rec_off[n_records], bloom[16 * lines] (the caller sizes them
// from its own model of the run; at most the cap of each, in elements, is written).
int32_t sim_run_index(const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off, const uint32_t *blk_size, uint32_t n_blocks,
                      pgs_run_info *info, uint64_t *n_bloom_entries, uint32_t *bloom_lines, uint32_t *blk_rec, uint32_t *ikey_off,
                      uint64_t blk_cap, uint8_t *ikeys, uint64_t ikeys_cap, uint32_t *rec_off, uint64_t rec_cap, uint32_t *bloom,
                      uint64_t bloom_cap)
{
    HostRun r;
    if (const int32_t rc = load_run(r, data, data_bytes, blk_off, blk_size, n_blocks)) return rc;
    *info = r.info;
    *n_bloom_entries = r.n_bloom_entries;
    *bloom_lines = r.bloom_lines;
    if (blk_rec) memcpy(blk_rec, r.d_blk_rec, 4 * std::min<uint64_t>(blk_cap, n_blocks + 1ull));
    if (ikey_off) memcpy(ikey_off, r.d_ikey_off, 4 * std::min<uint64_t>(blk_cap, n_blocks + 1ull));
    if (ikeys) memcpy(ikeys, r.d_ikeys, std::min<uint64_t>(ikeys_cap, r.d_ikey_off[n_blocks]));
    if (rec_off) memcpy(rec_off, r.d_rec_off, 4 * std::min<uint64_t>(rec_cap, r.d_blk_rec[n_blocks]));
    if (bloom) copy_bloom(r, bloom, bloom_cap);
    return PGS_OK;
}

static int32_t load_runs(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                      const uint32_t *n_blocks, std::vector<HostRun> &runs)
{
    runs.resize(k);
    for (uint32_t i = 0; i < k; i++)
        if (const int32_t rc = load_run(runs[i], data[i], data_bytes[i], blk_off[i], blk_size[i], n_blocks[i])) return rc;
    return PGS_OK;
}

// The run set of a read launch over the loaded runs (newest first), as the library's snapshot builds it.  compacted: the run
// of the last sim_compact call joins as the oldest run, with the index and filter k_emit wrote.  multi: the multi-partition
// shape -- slot 0 owns the runs [0, k/2), slot 1 the rest, slot 2 is an empty partition.  bloom = false: the runs' filters
// are left out.
static int32_t read_slots(const std::vector<HostRun> &runs, bool compacted, bool multi, bool bloom, ReadRunSet &R)
{
    std::vector<const HostRun *> all;
    for (const HostRun &r : runs) all.push_back(&r);
    if (compacted) {
        if (all.size() >= kMaxReadRuns || !g_res.st.tot_blocks) return PGS_INVALID_ARGUMENT;
        all.push_back(&g_res.run);
    }
    const auto half = all.begin() + all.size() / 2;
    const std::vector<std::vector<const HostRun *>> slots =
        multi ? std::vector<std::vector<const HostRun *>>{{all.begin(), half}, {half, all.end()}, {}} : std::vector<std::vector<const HostRun *>>{all};
    const int32_t rc = read_run_set(slots, multi, R);
    auto no_bloom = [](RunDev &d) { d.bloom = nullptr; d.bloom_lines = 0; };
    if (!bloom) {
        for (RunDev &d : R.packed) no_bloom(d);
        for (RunDev &d : R.rr.runs) no_bloom(d);
    }
    return rc;
}

// the buffers of a read launch (get_buffers, scan_buffers) in host memory at the library's sizes; what the library leaves
// unset is poisoned until the kernels write it
static auto host_buffers(HostMem &mem)
{
    return [&mem](auto *&p, uint64_t bytes, ReadInit in) {
        uint8_t *b;
        host_count_buffers(mem)(b, bytes, in.fill);
        if (in.src) memcpy(b, in.src, in.src_bytes);
        p = (std::remove_reference_t<decltype(p)>)b;
    };
}

// the slot of each of n requests in the multi-partition shape: request i belongs to slot i % 3
static std::vector<uint32_t> slot_of_each(uint32_t n)
{
    std::vector<uint32_t> s(n);
    for (uint32_t i = 0; i < n; i++) s[i] = i % 3;
    return s;
}

// k_get over k runs (newest first); results / arena as pgs_get_batch.  stats[0] = arena bytes, [1] = blocks probed, [2] = runs skipped.
// use_bloom: 1 = the runs' filters are used; 2 = the multi-partition shape of pgs_get_batch_multi (read_slots; key i belongs to
// slot i % 3); 4 = the last sim_compact output is the oldest run
int32_t sim_get(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                const uint32_t *n_blocks, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                uint64_t arena_cap, pgs_get_result *results, uint64_t *stats, uint32_t use_bloom)
{
    std::vector<HostRun> runs;
    if (const int32_t rc = load_runs(k, data, data_bytes, blk_off, blk_size, n_blocks, runs)) return rc;
    ReadRunSet R;
    if (const int32_t rc = read_slots(runs, use_bloom & 4, use_bloom & 2, use_bloom & 1, R)) return rc;
    GetParams P{};
    P.n = n; P.now = now; P.data_version = 1;
    ReadLaunch<GetParams> L;
    if (const int32_t rc = get_plan(P, R, kSimSmemOptin, L)) return rc;
    HostMem mem;
    get_buffers(P, R, keys, key_off, slot_of_each(n).data(), arena_cap, host_buffers(mem));
    read_launch(L, P, 2, nullptr);
    memcpy(results, P.results, sizeof(pgs_get_result) * n);
    for (int i = 0; i < 3; i++) stats[i] = P.arena_cursor[i];
    if (P.error[0]) return (int32_t)P.error[0];
    memcpy(arena, P.arena, std::min<uint64_t>(P.arena_cursor[0], P.arena_cap));
    return PGS_OK;
}

// range scans over k runs; outputs as the device side of scan_many: request i's answer at arena + i*arena_stride,
// kvs + i*kv_stride and resume + i*resume_stride (scan_output_strides rounds arena_stride up to a multiple of 16; a resume
// stride shorter than the key slot reports no resume key).  The kernel is scan_plan's choice.  lanes & 0xFF: k_scan_fwd's
// lanes per group; lanes & 0x100: the multi-partition shape of pgs_range_scan_many_multi (read_slots; request i belongs to
// slot i % 3).  pool_bytes (k_scan only): 0 = the pool the product gives a batch of n requests; otherwise at most pool_bytes,
// but never below the smallest pool (scan_min_pool: one block of every run), so that a small value forces chunks of about
// one block.  arena_base not null: the packed read-back of sim_scan_packed.
static int32_t scan_read_back(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                 const uint32_t *n_blocks, const pgs_scan_request *reqs, uint32_t n, uint32_t now, uint64_t arena_stride, uint32_t kv_stride,
                 uint8_t *arena, pgs_kv *kvs, uint8_t *resume, uint32_t resume_stride, pgs_scan_result *results, uint32_t lanes,
                 uint32_t pool_bytes, uint64_t *arena_base, uint32_t *kv_base, uint64_t arena_cap, uint64_t kv_cap)
{
    std::vector<HostRun> runs;
    if (const int32_t rc = load_runs(k, data, data_bytes, blk_off, blk_size, n_blocks, runs)) return rc;
    const ScanBatch B = flatten_scan_requests(reqs, n);
    if (B.any_reverse && lanes) return PGS_INVALID_ARGUMENT; // k_scan has no lane groups and no multi-partition shape
    ReadRunSet R;
    if (const int32_t rc = read_slots(runs, false, lanes & 0x100, true, R)) return rc;
    ScanParams P{};
    P.n = n; P.now = now; P.data_version = 1;
    if (B.need_crc) { crc64_make_table(crc_tab); P.crc_table = (const unsigned long long *)crc_tab; }
    ReadLaunch<ScanParams> L;
    if (const int32_t rc = scan_plan(P, R, B.any_reverse, kSimSmemOptin, sizeof(ScanShared), L, lanes & 0xFF, pool_bytes)) return rc;
    HostMem mem;
    const bool report_resume = scan_buffers(P, R, B, slot_of_each(n).data(), arena_stride, kv_stride, resume_stride, host_buffers(mem));
    read_launch(L, P, L.kernel == k_scan ? 3 : 2, nullptr);
    memcpy(results, P.results, sizeof(pgs_scan_result) * n);
    ScanPack K;
    std::vector<unsigned long long> ab{0, n ? results[0].arena_used : 0};
    std::vector<uint32_t> kb{0, n ? results[0].n_kvs : 0};
    if (arena_base && n > 1) {
        pack_offsets_launch(P, K, nullptr, host_buffers(mem));
        ab.assign(K.arena_base, K.arena_base + n + 1);
        kb.assign(K.kv_base, K.kv_base + n + 1);
    }
    if (P.error[0]) return (int32_t)P.error[0];
    if (arena_base && n) {
        if (ab[n] > arena_cap || kb[n] > kv_cap) return PGS_INCOMPLETE;
        if (n > 1) {
            pack_copy_launch(P, K, ab[n], kb[n], 2, nullptr, host_buffers(mem));
            memcpy(arena, K.arena, ab[n]);
            memcpy(kvs, K.kvs, sizeof(pgs_kv) * kb[n]);
        } else {
            memcpy(arena, P.arena, ab[1]);
            memcpy(kvs, P.kvs, sizeof(pgs_kv) * kb[1]);
        }
        memcpy(arena_base, ab.data(), 8 * (n + 1ull));
        memcpy(kv_base, kb.data(), 4 * (n + 1ull));
    }
    for (uint64_t i = 0; i < n; i++) {
        const pgs_scan_result &r = results[i];
        if (!arena_base) {
            memcpy(arena + i * P.arena_stride, P.arena + i * P.arena_stride, r.arena_used);
            memcpy(kvs + i * kv_stride, P.kvs + i * kv_stride, sizeof(pgs_kv) * r.n_kvs);
        }
        if (report_resume && r.iter_valid) memcpy(resume + i * resume_stride, P.resume + i * P.resume_stride, r.resume_len);
    }
    return PGS_OK;
}

int32_t sim_scan(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                 const uint32_t *n_blocks, const pgs_scan_request *reqs, uint32_t n, uint32_t now, uint64_t arena_stride, uint32_t kv_stride,
                 uint8_t *arena, pgs_kv *kvs, uint8_t *resume, uint32_t resume_stride, pgs_scan_result *results, uint32_t lanes,
                 uint32_t pool_bytes)
{
    return scan_read_back(k, data, data_bytes, blk_off, blk_size, n_blocks, reqs, n, now, arena_stride, kv_stride, arena, kvs, resume,
                          resume_stride, results, lanes, pool_bytes, nullptr, nullptr, 0, 0);
}

// sim_scan with the batch read back as scan_many reads it: request i's kvs at kvs[kv_base[i] ..) with offsets relative to
// arena + arena_base[i] (pack_offsets_launch / pack_copy_launch for n > 1, the slice itself for n == 1), and PGS_INCOMPLETE,
// with arena_base / kv_base unset, when arena_base[n] > arena_cap or kv_base[n] > kv_cap.  Resume keys as sim_scan.
int32_t sim_scan_packed(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                        const uint32_t *n_blocks, const pgs_scan_request *reqs, uint32_t n, uint32_t now, uint64_t arena_stride,
                        uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume,
                        uint32_t resume_stride, pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base, uint32_t lanes)
{
    return scan_read_back(k, data, data_bytes, blk_off, blk_size, n_blocks, reqs, n, now, arena_stride, kv_stride, arena, kvs, resume,
                          resume_stride, results, lanes, 0, arena_base, kv_base, arena_cap, kv_cap);
}

// k_pack_offsets alone (pack_offsets_launch) over n results the caller makes up: arena_base / kv_base get its n + 1 offsets
void sim_pack_offsets(const pgs_scan_result *results, uint32_t n, uint64_t *arena_base, uint32_t *kv_base)
{
    HostMem mem;
    ScanParams P{};
    P.n = n;
    memcpy(host_alloc(mem, P.results, n, 0), results, sizeof(pgs_scan_result) * n);
    ScanPack K;
    pack_offsets_launch(P, K, nullptr, host_buffers(mem));
    memcpy(arena_base, K.arena_base, 8 * (n + 1ull));
    memcpy(kv_base, K.kv_base, 4 * (n + 1ull));
}

// k_hotkey_capture over n keys of n_slots partition slots (key_part null: every key is slot 0).  Per slot: state (0 off,
// 1 coarse, 2 fine), target bucket and queue room; buckets = n_slots * n_buckets counters, accumulated into; tickets[n_slots];
// idx = the admitted fine indices, slot s at the sum of the rooms of the slots before it.  Returns the number of idx entries.
uint32_t sim_hotkey_capture(const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part, uint32_t n, uint32_t n_buckets,
                            uint32_t n_slots, const uint32_t *state, const uint32_t *target, const uint32_t *room,
                            unsigned long long *buckets, uint32_t *tickets, uint32_t *idx, uint32_t grid)
{
    HostMem mem;
    HotkeyParams P{};
    uint8_t *k;
    uint32_t *ko, *kp = nullptr, *t, *ix;
    memcpy(host_alloc(mem, k, key_off[n] + 16, 0), keys, key_off[n]); // the slack of the product's key buffer
    memcpy(host_alloc(mem, ko, n + 1, 0), key_off, 4 * (size_t)(n + 1));
    if (key_part) memcpy(host_alloc(mem, kp, n, 0), key_part, 4 * (size_t)n);
    HotkeySlotDev *sd;
    host_alloc(mem, sd, n_slots, 0);
    std::vector<unsigned long long *> bk(n_slots, nullptr);
    uint32_t total = 0;
    for (uint32_t s = 0; s < n_slots; s++) {
        if (state[s] == 1) memcpy(host_alloc(mem, bk[s], n_buckets, 0), buckets + (size_t)s * n_buckets, 8 * (size_t)n_buckets);
        sd[s] = HotkeySlotDev{bk[s], state[s], target[s], state[s] == 2 ? room[s] : 0u, total};
        total += sd[s].room;
    }
    host_alloc(mem, t, n_slots, 0);
    host_alloc(mem, ix, total, 0xEE);
    P.keys = k; P.key_off = ko; P.key_part = kp; P.n = n; P.n_buckets = n_buckets; P.slots = sd; P.tickets = t; P.idx = ix;
    if (n) PGS_LAUNCH(k_hotkey_capture, grid, kHotkeyThreads, 0, 0, P);
    for (uint32_t s = 0; s < n_slots; s++)
        if (bk[s]) memcpy(buckets + (size_t)s * n_buckets, bk[s], 8 * (size_t)n_buckets);
    memcpy(tickets, t, 4 * (size_t)n_slots);
    memcpy(idx, ix, 4 * (size_t)total);
    return total;
}

// the bucket hash of format.h, for the tests' model
uint64_t sim_hotkey_hash(const uint8_t *p, uint32_t len) { return hotkey_hash(p, len); }

// One parent run split into dst_count / src_count children through split_plan / split_buffers / split_child / split_launch,
// as pgs_partition_split runs it; want = the children that are built (bit c).  seg_weight: smaller segments (0: the product's
// default budget).  Returns a status; the children stay in a static buffer until the next call (sim_split_child_* read them),
// *dropped = the empty writes.
int32_t sim_split(const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off, const uint32_t *blk_size, uint32_t n_blocks,
                  uint32_t block_size, uint32_t restart_interval, uint32_t src_count, uint32_t dst_count, uint32_t want, uint64_t seg_weight,
                  uint64_t *dropped)
{
    HostRun in;
    if (const int32_t rc = load_run(in, data, data_bytes, blk_off, blk_size, n_blocks)) return rc;
    if (src_count == 0 || dst_count % src_count) return PGS_INVALID_ARGUMENT;
    const uint32_t NC = dst_count / src_count;
    SplitParams SP{};
    SP.M.runs[0] = in.dev();
    SP.M.block_size = block_size;
    SP.M.restart_interval = restart_interval;
    SP.M.data_version = 1;
    crc64_make_table(crc_tab);
    SP.M.crc_table = (const unsigned long long *)crc_tab;
    SP.S = NC; SP.src_count = src_count; SP.dst_count = dst_count; SP.want = want;
    CompactTotals T{};
    T.add(in.info, in.n_bloom_entries);
    const uint32_t smem = compact_smem_budget(kSimSmemOptin);
    SplitGeometry geo{};
    if (const int32_t rc = split_plan(SP, T, smem, geo, 0, seg_weight)) return rc;
    Split &R = g_split;
    R = Split{};
    R.child.resize(NC);
    R.built.assign(NC, 0);
    HostMem scratch;
    split_buffers(SP, host_count_buffers(scratch));
    for (uint32_t c = 0; c < NC; c++) SP.stats[c] = merge_stats_init();
    split_launch(SP, geo, nullptr, nullptr, 0, 2, 2, nullptr, [](int) {});
    R.st.assign(SP.stats, SP.stats + NC);
    *dropped = *SP.dropped;
    for (uint32_t c = 0; c < NC; c++)
        if (R.st[c].error) { fprintf(stderr, "sim_split: counting pass status %u (child %u)\n", R.st[c].error, c); return (int32_t)R.st[c].error; }
    std::vector<MergeParams> Pc;
    std::vector<CompactGeometry> gc;
    for (uint32_t c = 0; c < NC; c++) {
        if (!((want >> c) & 1u) || R.st[c].cnt[EV_OUT] == 0) continue;
        MergeParams P{};
        CompactGeometry g{};
        CompactTotals Tc{};
        if (!split_child(SP, R.st[c], SP.prefixes[c], smem, P, g, Tc)) return PGS_NOT_SUPPORTED;
        HostRun &run = R.child[c];
        compact_buffers(P, g, Tc, run, [&](auto *&p, uint64_t n, int fill, bool out) { if (out) host_count_buffers(run.mem)(p, n, fill); });
        split_child_scratch(SP, c, P);
        Pc.push_back(P);
        gc.push_back(g);
        R.built[c] = 1;
    }
    split_launch(SP, geo, Pc.data(), gc.data(), (uint32_t)Pc.size(), 2, 2, nullptr, [](int) {});
    R.st.assign(SP.stats, SP.stats + NC);
    R.Q = SP.M.Q;
    for (uint32_t c = 0; c < NC; c++) {
        if (R.st[c].error) { fprintf(stderr, "sim_split: status %u at segment %u (child %u)\n", R.st[c].error, R.st[c].error_seg, c); return (int32_t)R.st[c].error; }
        if (!R.built[c]) continue;
        pgs_compact_result cr{};
        R.child[c].n_bloom_entries = compact_result_stats(R.st[c], 0, cr, R.child[c].info);
    }
    return PGS_OK;
}

// child c of the last sim_split: 0 = not built (or nothing for it); else *info = its pgs_run_info, *n_segments = the parent's
// segments, *index_key_bytes = its index keys' bytes
int32_t sim_split_child_info(uint32_t c, pgs_run_info *info, uint32_t *n_segments, uint64_t *index_key_bytes)
{
    if (c >= g_split.child.size() || !g_split.built[c]) return 0;
    *info = g_split.child[c].info;
    *n_segments = g_split.Q;
    *index_key_bytes = g_split.st[c].tot_keyb;
    return 1;
}
void sim_split_child_copy(uint32_t c, uint8_t *data, uint64_t *blk_off, uint32_t *blk_size, uint32_t *blk_rec, uint32_t *ikey_off, uint8_t *ikeys)
{
    const HostRun &r = g_split.child[c];
    const uint32_t nb = r.info.n_blocks;
    memcpy(data, r.d_data, r.info.data_bytes);
    memcpy(blk_off, r.d_blk_off, 8 * (size_t)(nb + 1));
    memcpy(blk_size, r.d_blk_size, 4 * (size_t)nb);
    memcpy(blk_rec, r.d_blk_rec, 4 * (size_t)(nb + 1));
    memcpy(ikey_off, r.d_ikey_off, 4 * (size_t)(nb + 1));
    memcpy(ikeys, r.d_ikeys, g_split.st[c].tot_keyb);
}
// 1 when child c's Bloom filter admits the byte string
int32_t sim_split_child_bloom_check(uint32_t c, const uint8_t *key, uint32_t len)
{
    const HostRun &r = g_split.child[c];
    return bloom_may_contain(r.d_bloom, r.bloom_lines, bloom_hash_bytes(key, len)) ? 1 : 0;
}

// n parent runs split together into dst_count / src_count children each, through split_many_plan / split_many_buffers /
// split_many_child / split_many_launch, as pgs_partition_split_many runs them.  Run i comes from the flat arrays; want[i] = its
// built children (bit c).  seg_weight: the launch's one segment weight (0: the product's default budget).  Returns a status
// (pgs_partition_split_many's for the child-run count and the joint plan); dropped[i] = run i's empty writes, *launches = the
// launches made.  Every run's children stay until the next call: sim_split_many_select(i) makes run i's the ones
// sim_split_child_* read.
int32_t sim_split_many(uint32_t n, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                       const uint32_t *n_blocks, const uint32_t *want, uint32_t block_size, uint32_t restart_interval, uint32_t src_count,
                       uint32_t dst_count, uint64_t seg_weight, uint64_t *dropped, uint32_t *launches)
{
    g_split_many.clear();
    *launches = 0;
    if (n == 0 || src_count == 0 || dst_count % src_count) return PGS_INVALID_ARGUMENT;
    const uint32_t NC = dst_count / src_count;
    std::vector<HostRun> in(n);
    for (uint32_t i = 0; i < n; i++)
        if (const int32_t rc = load_run(in[i], data[i], data_bytes[i], blk_off[i], blk_size[i], n_blocks[i])) return rc;
    crc64_make_table(crc_tab);
    std::vector<SplitParams> SP(n);
    std::vector<CompactTotals> T(n);
    uint64_t child_runs = 0;
    for (uint32_t i = 0; i < n; i++) {
        SplitParams &s = SP[i];
        s.M.runs[0] = in[i].dev();
        s.M.block_size = block_size;
        s.M.restart_interval = restart_interval;
        s.M.data_version = 1;
        s.M.crc_table = (const unsigned long long *)crc_tab;
        s.S = NC; s.src_count = src_count; s.dst_count = dst_count; s.want = want[i];
        T[i].add(in[i].info, in[i].n_bloom_entries);
        child_runs += __builtin_popcount(want[i]);
    }
    if (child_runs > kMaxCompactJobs) return PGS_NOT_SUPPORTED;
    const uint32_t smem = compact_smem_budget(kSimSmemOptin);
    SplitJobs J{};
    MergeJobs M{};
    SplitGeometry geo{};
    if (const int32_t rc = split_many_plan(SP.data(), T.data(), n, smem, J, M, geo, 0, seg_weight)) return rc;
    HostMem scratch;
    split_many_buffers(SP.data(), n, J, host_count_buffers(scratch));
    for (uint64_t y = 0; y < (uint64_t)n * NC; y++) J.stats[y] = merge_stats_init();
    std::vector<MergeParams> MP(n);
    for (uint32_t i = 0; i < n; i++) MP[i] = SP[i].M;
    std::vector<uint32_t> seg_base(n + 1), blk_base(n + 1);
    compact_many_bases(MP.data(), n, seg_base.data(), blk_base.data());
    M.job = MP.data();
    M.seg_base = J.seg_base = seg_base.data();
    M.blk_base = blk_base.data();
    J.job = SP.data();
    J.crc_table = (const unsigned long long *)crc_tab;
    *launches += split_many_launch(J, M, geo, nullptr, CompactGeometry{}, 2, 0, nullptr, [](int) {});
    g_split_many.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        dropped[i] = J.dropped[i];
        Split &R = g_split_many[i];
        R.child.resize(NC);
        R.built.assign(NC, 0);
        R.st.assign(SP[i].stats, SP[i].stats + NC);
        R.Q = SP[i].M.Q;
        for (uint32_t c = 0; c < NC; c++)
            if (R.st[c].error) { fprintf(stderr, "sim_split_many: run %u: counting pass status %u (child %u)\n", i, R.st[c].error, c); return (int32_t)R.st[c].error; }
    }
    std::vector<MergeParams> Pc;
    std::vector<uint32_t> emit_base(1, 0);
    CompactGeometry shape{};
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++) {
            Split &R = g_split_many[i];
            if (!((want[i] >> c) & 1u) || R.st[c].cnt[EV_OUT] == 0) continue;
            MergeParams P{};
            CompactGeometry g{};
            CompactTotals Tc{};
            if (!split_many_child(SP[i], c, R.st[c], SP[i].prefixes[c], smem, P, g, Tc, Pc.empty() ? nullptr : &Pc[0], &shape)) return PGS_NOT_SUPPORTED;
            HostRun &run = R.child[c];
            compact_buffers(P, g, Tc, run, [&](auto *&p, uint64_t cnt, int fill, bool out) { if (out) host_count_buffers(run.mem)(p, cnt, fill); });
            if (Pc.empty()) shape = g;
            Pc.push_back(P);
            emit_base.push_back(emit_base.back() + P.Q);
            R.built[c] = 1;
        }
    if (!Pc.empty()) {
        MergeJobs E{};
        E.job = Pc.data();
        E.seg_base = emit_base.data();
        E.n = (uint32_t)Pc.size();
        E.Q = emit_base.back();
        E.ticket = J.ticket + 2;
        *launches += split_many_launch(J, M, geo, &E, shape, 2, 2, nullptr, [](int) {});
    }
    for (uint32_t i = 0; i < n; i++) {
        Split &R = g_split_many[i];
        R.st.assign(SP[i].stats, SP[i].stats + NC);
        for (uint32_t c = 0; c < NC; c++) {
            if (R.st[c].error) { fprintf(stderr, "sim_split_many: run %u: status %u at segment %u (child %u)\n", i, R.st[c].error, R.st[c].error_seg, c); return (int32_t)R.st[c].error; }
            if (!R.built[c]) continue;
            pgs_compact_result cr{};
            R.child[c].n_bloom_entries = compact_result_stats(R.st[c], 0, cr, R.child[c].info);
        }
    }
    return PGS_OK;
}
// run i of the last sim_split_many becomes the one sim_split_child_* read
int32_t sim_split_many_select(uint32_t i)
{
    if (i >= g_split_many.size()) return PGS_INVALID_ARGUMENT;
    g_split = g_split_many[i];
    return PGS_OK;
}

} // extern "C"

namespace {
// the build of records in internal-key order (P's inputs set) as pgs_run_build runs it: scratch, plan, blocks, then the upload's
// two index passes.  Returns pgs_run_build's status; on PGS_OK the run is g_built's.
int32_t build_sorted(BuildParams &P, HostMem &scratch, uint32_t grid_cap)
{
    Built &R = g_built;
    build_buffers(P, host_count_buffers(scratch));
    build_launch_plan(P, grid_cap, nullptr, [](int) {});
    const BuildSummary sum = *P.sum;
    if (const int32_t rc = build_status(sum.flags)) return rc;
    const uint32_t nb = (uint32_t)sum.n_blocks;
    HostRun &r = R.run;
    host_alloc(r.mem, r.d_data, sum.data_bytes + 256, 0xEE); // the library's slack, zeroed below as the library does
    memset(r.d_data + sum.data_bytes, 0, 256);
    memcpy(host_alloc(r.mem, r.d_blk_off, nb + 1, 0), P.blk_off, 8 * (size_t)(nb + 1));
    memcpy(host_alloc(r.mem, r.d_blk_size, nb, 0), P.blk_size, 4 * (size_t)nb);
    P.data = r.d_data;
    build_launch_blocks(P, nb, grid_cap, nullptr);
    R.data_bytes = sum.data_bytes;
    uint64_t end = 0;
    uint32_t max_blk = 0; // from the built handles (the library takes the summary's)
    run_handles_check(r.d_blk_off, r.d_blk_size, nb, sum.data_bytes, end, max_blk);
    if (const int32_t rc = build_index(r, nb, max_blk)) return rc;
    if (r.info.max_block_size != sum.max_blk) { fprintf(stderr, "sim_run_build: largest block %u, the index saw %u\n", sum.max_blk, r.info.max_block_size); return PGS_CORRUPTION; }
    return PGS_OK;
}
} // namespace

extern "C" {

// n flat records built into a run through build_plan / build_buffers / build_launch_plan / build_launch_blocks as pgs_run_build
// runs them, then indexed by the upload's two passes.  grid_cap: at most this many CTAs per launch (0: the product's grids).
// Returns pgs_run_build's status; on PGS_OK the run stays in a static buffer until the next call (sim_run_build_* read it).
int32_t sim_run_build(uint64_t n, const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals, const uint64_t *val_off,
                      const uint64_t *seq, const uint8_t *type, uint32_t block_size, uint32_t restart_interval, uint32_t grid_cap)
{
    g_built = Built{};
    if (n == 0) return PGS_OK;
    if (n > kBuildMaxRecords) return PGS_NOT_SUPPORTED;
    HostMem scratch;
    BuildParams P{};
    build_plan(P, (uint32_t)n, block_size, restart_interval);
    stage_records(P, n, keys, key_off, vals, val_off, seq, type, host_buffers(scratch));
    return build_sorted(P, scratch, grid_cap);
}

// n flat records in any order sorted through sort_plan / sort_buffers / sort_launch as pgs_run_build_unsorted runs them, then
// built from the sorted copy as sim_run_build builds.  Returns pgs_run_build_unsorted's status; on PGS_OK the run is read with
// sim_run_build_info / sim_run_build_copy.  *launches_out (if not null): the sort's launches.
int32_t sim_run_build_unsorted(uint64_t n, const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals, const uint64_t *val_off,
                               const uint64_t *seq, const uint8_t *type, uint32_t block_size, uint32_t restart_interval,
                               uint32_t grid_cap, uint32_t *launches_out)
{
    g_built = Built{};
    if (launches_out) *launches_out = 0;
    if (n == 0) return PGS_OK;
    if (n > kBuildMaxRecords) return sort_status_too_many(n, key_off, val_off);
    HostMem scratch;
    SortParams Q{};
    sort_plan(Q, (uint32_t)n);
    stage_records(Q, n, keys, key_off, vals, val_off, seq, type, host_buffers(scratch));
    sort_buffers(Q, key_off[n], val_off[n], host_count_buffers(scratch), host_count_buffers(scratch));
    uint32_t launches = 0;
    const int32_t rc = sort_launch(Q, grid_cap, nullptr, [&](SortSummary &s) { s = *Q.sum; return (int32_t)PGS_OK; }, launches);
    if (launches_out) *launches_out = launches;
    if (rc) return rc;
    BuildParams P{};
    build_plan(P, (uint32_t)n, block_size, restart_interval);
    build_inputs_sorted(P, Q);
    return build_sorted(P, scratch, grid_cap);
}
// the last sim_run_build's sizes and info (level and run id zero)
void sim_run_build_info(uint64_t *data_bytes, uint32_t *n_blocks, pgs_run_info *info)
{
    *data_bytes = g_built.data_bytes;
    *n_blocks = g_built.run.info.n_blocks;
    *info = g_built.run.info;
}
void sim_run_build_copy(uint8_t *data, uint64_t *blk_off, uint32_t *blk_size)
{
    const HostRun &r = g_built.run;
    memcpy(data, r.d_data, g_built.data_bytes);
    memcpy(blk_off, r.d_blk_off, 8 * (size_t)r.info.n_blocks);
    memcpy(blk_size, r.d_blk_size, 4 * (size_t)r.info.n_blocks);
}

// n jobs (their partitions unused) built through build_many_plan / build_many_stage / build_many_buffers /
// build_many_launch_plan / build_many_launch_blocks and both index passes over every run (index_launch_many), as
// pgs_run_build_many runs them.  Returns pgs_run_build_many's status and *failed_job (the lowest failing job), or PGS_OK with
// every job's run kept until the next call (sim_run_build_many_info / _copy read job j's).
int32_t sim_run_build_many(const pgs_run_build_job *jobs, uint32_t n, uint32_t block_size, uint32_t restart_interval, uint32_t grid_cap,
                           uint32_t *failed_job)
{
    g_built_many.clear();
    g_built_many.resize(n);
    *failed_job = 0;
    std::vector<const pgs_run_build_job *> J;
    std::vector<uint32_t> which;
    for (uint32_t i = 0; i < n; i++)
        if (jobs[i].n) { J.push_back(&jobs[i]); which.push_back(i); }
    const uint32_t jn = (uint32_t)J.size();
    if (!jn) return PGS_OK;
    HostMem scratch;
    std::vector<uint32_t> job_rec(jn + 1);
    std::vector<BuildJob> job(jn);
    BuildManyParams M{};
    build_many_plan(M, J.data(), jn, job_rec.data(), job.data(), block_size, restart_interval);
    build_many_stage(M, J.data(), job_rec.data(), job.data(), host_buffers(scratch), [](const void *dst, const void *src, uint64_t bytes) {
        if (bytes) memcpy((void *)dst, src, bytes);
    });
    build_many_buffers(M, host_count_buffers(scratch));
    build_many_launch_plan(M, grid_cap, nullptr, [](int) {});
    const BuildSummary sum = *M.B.sum;
    std::vector<uint32_t> nb(jn);
    std::vector<uint64_t> bytes(jn);
    for (uint32_t d = 0; d < jn; d++)
        if (const int32_t rc = build_many_job(M, sum, M.job_out, M.job_off, d, nb[d], bytes[d])) { *failed_job = which[d]; return rc; }
    const uint32_t NB = (uint32_t)sum.n_blocks;
    std::vector<BuildRunOut> outs(jn);
    for (uint32_t d = 0; d < jn; d++) {
        Built &R = g_built_many[which[d]];
        HostRun &r = R.run;
        host_alloc(r.mem, r.d_data, bytes[d] + 256, 0xEE); // the library's slack, zeroed as the library does
        memset(r.d_data + bytes[d], 0, 256);
        host_alloc(r.mem, r.d_blk_off, nb[d] + 1, 0xEE);
        host_alloc(r.mem, r.d_blk_size, nb[d], 0xEE);
        R.data_bytes = bytes[d];
        outs[d] = BuildRunOut{r.d_data, (unsigned long long *)r.d_blk_off, r.d_blk_size};
    }
    M.out = outs.data();
    build_many_launch_blocks(M, NB, grid_cap, nullptr);
    uint32_t *nrec, *lastlen;
    IndexStats *stats;
    host_count_buffers(scratch)(nrec, NB, kNoFill);
    host_count_buffers(scratch)(lastlen, NB, kNoFill);
    host_count_buffers(scratch)(stats, jn, kNoFill);
    std::vector<IndexParams> X(jn);
    for (uint32_t d = 0; d < jn; d++) {
        HostRun &r = g_built_many[which[d]].run;
        X[d] = IndexParams{r.d_data, r.d_blk_off, r.d_blk_size, nb[d]};
        X[d].nrec = nrec + M.job_out[d];
        X[d].lastlen = lastlen + M.job_out[d];
        X[d].stats = stats + d;
        stats[d] = index_stats_init();
    }
    index_launch_many<false>(X.data(), M.job_out, jn, NB, nullptr);
    for (uint32_t d = 0; d < jn; d++) {
        HostRun &r = g_built_many[which[d]].run;
        std::vector<uint32_t> rec_cum(nb[d] + 1), key_cum(nb[d] + 1);
        if (const int32_t rc = index_buffers(X[d], r, X[d].nrec, X[d].lastlen, stats[d], rec_cum.data(), key_cum.data(), host_count_buffers(r.mem))) {
            *failed_job = which[d];
            return rc;
        }
        memcpy(r.d_blk_rec, rec_cum.data(), 4 * (nb[d] + 1ull));
        memcpy(r.d_ikey_off, key_cum.data(), 4 * (nb[d] + 1ull));
    }
    index_launch_many<true>(X.data(), M.job_out, jn, NB, nullptr);
    for (uint32_t d = 0; d < jn; d++) {
        HostRun &r = g_built_many[which[d]].run;
        if (stats[d].error) { *failed_job = which[d]; return (int32_t)stats[d].error; }
        run_info_from_index(stats[d], nb[d], bytes[d], M.job_out[jn + d], r.info);
    }
    return PGS_OK;
}
// job j of the last sim_run_build_many: its sizes and info (level and run id zero), and its blocks and handles
void sim_run_build_many_info(uint32_t j, uint64_t *data_bytes, uint32_t *n_blocks, pgs_run_info *info)
{
    *data_bytes = g_built_many[j].data_bytes;
    *n_blocks = g_built_many[j].run.info.n_blocks;
    *info = g_built_many[j].run.info;
}
void sim_run_build_many_copy(uint32_t j, uint8_t *data, uint64_t *blk_off, uint32_t *blk_size)
{
    const HostRun &r = g_built_many[j].run;
    memcpy(data, r.d_data, g_built_many[j].data_bytes);
    memcpy(blk_off, r.d_blk_off, 8 * (size_t)r.info.n_blocks);
    memcpy(blk_size, r.d_blk_size, 4 * (size_t)r.info.n_blocks);
}

} // extern "C"
