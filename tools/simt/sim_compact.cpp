// sim_compact.cpp — runs the compaction kernels (incubator_pegasus_b200/csrc/compact_kernels.cuh, the same source nvcc compiles
// for sm_90a) inside the host SIMT interpreter of simt.h.  Test / development tool: lets the CPU test-suite execute the kernels'
// logic against the oracle without a GPU.  NOT part of the product library and never a fallback for it.
#include "simt.h"

#define PGS_SIM 1
#include "../../incubator_pegasus_b200/csrc/compact_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/index_kernel.cuh"
#include "../../incubator_pegasus_b200/csrc/read_kernels.cuh"
#include "../../incubator_pegasus_b200/csrc/scan_kernel.cuh"

#include <memory>
#include <new>
#include <string>
#include <vector>

using namespace pgs;

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

// the run's index and Bloom filter as pgs_run_upload builds them (engine.cu): the two passes of k_index_walk with the host
// layout between them
bool build_index(HostRun &r, uint32_t nb)
{
    std::vector<uint32_t> nrec(nb + 1), lastlen(nb + 1);
    IndexStats st{};
    st.min_seq = ~0ull;
    const uint32_t grid = (nb + kIdxWarps - 1) / kIdxWarps, smem = kIdxWarps * kIdxScratch;
    if (nb)
        PGS_LAUNCH(k_index_walk<false>, grid, kIdxWarps * 32, smem, 0, (const uint8_t *)r.d_data, (const uint64_t *)r.d_blk_off,
                   (const uint32_t *)r.d_blk_size, nb, nrec.data(), lastlen.data(), (const uint32_t *)nullptr, (uint8_t *)nullptr,
                   (const uint32_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, 0u, &st, 0u);
    if (st.error) return false;
    host_alloc(r.mem, r.d_blk_rec, nb + 1, 0);
    host_alloc(r.mem, r.d_ikey_off, nb + 1, 0);
    if (!index_layout(nrec.data(), lastlen.data(), nb, r.d_blk_rec, r.d_ikey_off)) return false;
    host_alloc(r.mem, r.d_ikeys, r.d_ikey_off[nb] + 16, 0); // the product's slack (engine.cu)
    host_alloc(r.mem, r.d_rec_off, r.d_blk_rec[nb] + 1, 0);
    r.n_bloom_entries = st.n_records + st.n_prefix;
    r.bloom_lines = bloom_lines_for(r.n_bloom_entries);
    host_alloc(r.mem, r.d_bloom, (uint64_t)r.bloom_lines * 16, 0);
    if (nb)
        PGS_LAUNCH(k_index_walk<true>, grid, kIdxWarps * 32, smem, 0, (const uint8_t *)r.d_data, (const uint64_t *)r.d_blk_off,
                   (const uint32_t *)r.d_blk_size, nb, (uint32_t *)nullptr, (uint32_t *)nullptr, (const uint32_t *)r.d_ikey_off,
                   r.d_ikeys, (const uint32_t *)r.d_blk_rec, r.d_rec_off, r.d_bloom, r.bloom_lines, &st, 0u);
    if (st.error) return false;
    uint32_t max_blk = 0;
    for (uint32_t b = 0; b < nb; b++) max_blk = std::max(max_blk, r.d_blk_size[b]);
    run_info_from_index(st, nb, r.d_blk_off[nb], max_blk, r.info);
    return true;
}

// one run as the upload installs it: its blocks with the product's slack (engine.cu, compact.cu), the 16-aligned end of the
// blocks as blk_off[nb], the index and the filter
bool load_run(HostRun &r, const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off, const uint32_t *blk_size, uint32_t nb)
{
    memcpy(host_alloc(r.mem, r.d_data, data_bytes + 256, 0), data, data_bytes);
    memcpy(host_alloc(r.mem, r.d_blk_off, nb + 1, 0), blk_off, 8 * (size_t)nb);
    memcpy(host_alloc(r.mem, r.d_blk_size, nb, 0), blk_size, 4 * (size_t)nb);
    const uint64_t end = nb ? blk_off[nb - 1] + blk_size[nb - 1] : 0;
    r.d_blk_off[nb] = (end + 15) & ~15ull;
    return build_index(r, nb);
}

uint64_t crc_tab[256];

struct Merged { // the output of the last sim_compact call
    HostRun run;
    MergeStats st{};
    uint32_t Q = 0;
} g_res;

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
        if (!load_run(runs[i], data[i], data_bytes[i], blk_off[i], blk_size[i], n_blocks[i])) return PGS_CORRUPTION;
        P.runs[i] = runs[i].dev();
        T.add(runs[i].info, runs[i].n_bloom_entries);
    }
    P.block_size = block_size;
    P.restart_interval = restart_interval;
    P.bottommost = bottommost ? 1 : 0;
    P.now = now;
    P.data_version = 1;
    HostMem scratch;
    if (const uint32_t n = compact_filter(P, fp)) {
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
    compact_buffers(P, geo, T, R.run, [&](auto *&p, uint64_t n, int fill, bool out) {
        host_alloc(out ? R.run.mem : scratch, p, n, fill == kNoFill ? 0xEE : fill); // poisoned until the kernels write it
    });
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

// the Bloom filter the upload builds for one run (k_index_walk); 0 lines: a corrupt run
uint32_t sim_run_bloom(const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off, const uint32_t *blk_size, uint32_t n_blocks,
                       uint32_t *out, uint64_t cap)
{
    HostRun r;
    return load_run(r, data, data_bytes, blk_off, blk_size, n_blocks) ? copy_bloom(r, out, cap) : 0;
}

static bool load_runs(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                      const uint32_t *n_blocks, std::vector<HostRun> &runs, ReadRuns &rr, uint32_t &max_ukey)
{
    runs.resize(k);
    rr.n = k;
    max_ukey = 0;
    for (uint32_t i = 0; i < k; i++) {
        if (!load_run(runs[i], data[i], data_bytes[i], blk_off[i], blk_size[i], n_blocks[i])) return false;
        rr.runs[i] = runs[i].dev();
        max_ukey = std::max(max_ukey, runs[i].info.max_ukey_len);
    }
    return true;
}

// k_get over k runs (newest first); results / arena as pgs_get_batch.  stats[0] = arena bytes, [1] = blocks probed, [2] = runs skipped.
// use_bloom: 1 = the runs' filters are used; 2 = the multi-partition shape (below); 4 = the last sim_compact output is the oldest run
int32_t sim_get(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                const uint32_t *n_blocks, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                uint64_t arena_cap, pgs_get_result *results, uint64_t *stats, uint32_t use_bloom)
{
    std::vector<HostRun> runs;
    GetParams P{};
    uint32_t mk = 0;
    if (!load_runs(k, data, data_bytes, blk_off, blk_size, n_blocks, runs, P.rr, mk)) return PGS_CORRUPTION;
    if (use_bloom & 4) { // the run of the last sim_compact call joins as the oldest run, with the index and filter k_emit wrote
        if (k >= kMaxReadRuns || !g_res.st.tot_blocks) return PGS_INVALID_ARGUMENT;
        P.rr.runs[k] = g_res.run.dev();
        mk = std::max(mk, g_res.run.info.max_ukey_len);
        P.rr.n = ++k;
    }
    if (!(use_bloom & 1)) for (uint32_t i = 0; i < k; i++) { P.rr.runs[i].bloom = nullptr; P.rr.runs[i].bloom_lines = 0; }
    std::vector<uint8_t> kcopy(keys, keys + key_off[n]);
    kcopy.resize(kcopy.size() + 16); // the slack of the product's key buffer
    unsigned long long cur[4] = {0, 0, 0, 0};
    uint32_t err[4] = {0, 0, 0, 0};
    P.keys = kcopy.data(); P.key_off = key_off; P.n = n; P.now = now; P.data_version = 1;
    P.results = results; P.arena = arena; P.arena_cap = arena_cap; P.arena_cursor = cur; P.error = err; P.ticket = err + 1;
    const ReadGeometry geo = get_geometry(read_key_slot(mk));
    geo.apply(P);
    // use_bloom & 2: the multi-partition shape of pgs_get_batch_multi -- slot 0 owns the runs [0, k/2), slot 1 the rest, slot 2
    // is an empty partition; key i belongs to slot i % 3
    std::vector<RunDev> packed(P.rr.runs, P.rr.runs + k);
    std::vector<uint32_t> begin = {0, k / 2, k, k}, kp(n);
    if (use_bloom & 2) {
        for (uint32_t i = 0; i < n; i++) kp[i] = i % 3;
        P.multi_runs = packed.data(); P.multi_begin = begin.data(); P.key_part = kp.data();
        multi_read_runs(packed, begin, P.rr);
    }
    if (use_bloom & 2) PGS_LAUNCH((k_get<8, true>), 2, kReadThreads, geo.dyn, 0, P);
    else PGS_LAUNCH((k_get<8, false>), 2, kReadThreads, geo.dyn, 0, P);
    stats[0] = cur[0]; stats[1] = cur[1]; stats[2] = cur[2];
    return err[0] ? (int32_t)err[0] : PGS_OK;
}

// range scans over k runs; outputs as the device side of scan_many (request i uses arena + i*arena_stride, kvs + i*kv_stride;
// scan_output_strides rounds arena_stride up to a multiple of 16).
// A batch without reverse requests runs k_scan_fwd, any other batch k_scan.  pool_bytes (k_scan only): 0 =
// the pool the product gives a batch of n requests; otherwise at most pool_bytes, but never below the smallest pool
// (scan_min_pool: one block of every run), so that a small value forces chunks of about one block.
int32_t sim_scan(uint32_t k, const uint8_t **data, const uint64_t *data_bytes, const uint64_t **blk_off, const uint32_t **blk_size,
                 const uint32_t *n_blocks, const pgs_scan_request *reqs, uint32_t n, uint32_t now, uint64_t arena_stride, uint32_t kv_stride,
                 uint8_t *arena, pgs_kv *kvs, uint8_t *resume, uint32_t resume_stride, pgs_scan_result *results, uint32_t lanes,
                 uint32_t pool_bytes)
{
    std::vector<HostRun> runs;
    ScanParams P{};
    uint32_t mk = 0;
    if (!load_runs(k, data, data_bytes, blk_off, blk_size, n_blocks, runs, P.rr, mk)) return PGS_CORRUPTION;
    const ScanBatch B = flatten_scan_requests(reqs, n);
    uint32_t err[4] = {0, 0, 0, 0};
    P.reqs = B.reqs.data(); P.blob = (const uint8_t *)B.blob.data(); P.n = n; P.now = now; P.data_version = 1;
    P.results = results; P.kvs = kvs; P.arena = arena; P.resume = resume; P.error = err; P.ticket = err + 1;
    P.KS = read_key_slot(mk);
    scan_output_strides(P, arena_stride, kv_stride, resume_stride);
    if (B.need_crc) { crc64_make_table(crc_tab); P.crc_table = (const unsigned long long *)crc_tab; }
    if (B.any_reverse) {
        if (lanes) return PGS_INVALID_ARGUMENT; // k_scan has no lane groups and no multi-partition shape
        ScanBlockBound bb;
        for (auto &r : runs) bb.add(r.info);
        uint64_t dyn = scan_dyn_bytes(k, P.KS, bb.max_blk, bb.max_rec, n, scan_max_dyn(kSimSmemOptin, sizeof(ScanShared)), &P.pool_bytes);
        if (!dyn) return PGS_NOT_SUPPORTED;
        if (pool_bytes) {
            const uint32_t fixed_dyn = (uint32_t)dyn - P.pool_bytes;
            P.pool_bytes = std::max(std::min(P.pool_bytes, pool_bytes), (uint32_t)scan_min_pool(k, P.KS, bb.max_blk, bb.max_rec));
            dyn = fixed_dyn + P.pool_bytes;
        }
        PGS_LAUNCH(k_scan, std::min(n, 3u), kScanThreads, dyn, 0, P);
        return err[0] ? (int32_t)err[0] : PGS_OK;
    }
    // lanes & 0x100: the multi-partition shape of pgs_range_scan_many_multi -- slot 0 owns the runs [0, k/2), slot 1 the rest,
    // slot 2 is an empty partition; request i belongs to slot i % 3
    const bool multi = (lanes & 0x100) != 0;
    std::vector<RunDev> packed(P.rr.runs, P.rr.runs + k);
    std::vector<uint32_t> begin = {0, k / 2, k, k}, rp(n);
    if (multi) {
        for (uint32_t i = 0; i < n; i++) rp[i] = i % 3;
        P.multi_runs = packed.data(); P.multi_begin = begin.data(); P.req_part = rp.data();
        multi_read_runs(packed, begin, P.rr);
    }
    const ReadGeometry geo = scan_fwd_geometry(P.rr.n, P.KS, lanes & 0xFF);
    if (geo.G < P.rr.n) return PGS_INVALID_ARGUMENT;
    geo.apply(P);
    PGS_LAUNCH(scan_fwd_kernel(geo.G, multi), 2, kReadThreads, geo.dyn, 0, P);
    return err[0] ? (int32_t)err[0] : PGS_OK;
}

} // extern "C"
