// lookup.cu — host side of the read path (pgs_get_batch, pgs_range_scan, pgs_range_scan_many).
//
//   k_get / k_scan_fwd (read_kernels.cuh)  point lookups and forward range scans: lane-group iterators straight over HBM.
//   k_scan (scan_kernel.cuh)  REVERSE range scans, every request of a batch that mixes directions, and forward scans
//           whose user keys are too long for k_scan_fwd: one CTA per request stages chunks of blocks of every run in shared memory.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "engine.h"
#include "read_kernels.cuh"
#include "scan_kernel.cuh"

namespace pgs {

// pack the per-request output slices densely so that one D2H copy brings a whole batch back
__global__ void k_pack_offsets(const pgs_scan_result *__restrict__ res, uint32_t n, unsigned long long *__restrict__ abase,
                               uint32_t *__restrict__ kbase)
{
    __shared__ uint32_t scratch[33];
    __shared__ unsigned long long carry_a;
    __shared__ uint32_t carry_k;
    if (threadIdx.x == 0) { carry_a = 0; carry_k = 0; }
    __syncthreads();
    for (uint32_t base = 0; base < n; base += blockDim.x) {
        uint32_t i = base + threadIdx.x;
        uint32_t a = i < n ? (uint32_t)((res[i].arena_used + 15) & ~15ull) : 0;
        uint32_t k = i < n ? res[i].n_kvs : 0;
        uint32_t ta, tk;
        uint32_t pa = block_excl_scan(a, scratch, &ta);
        uint32_t pk = block_excl_scan(k, scratch, &tk);
        if (i < n) { abase[i] = carry_a + pa; kbase[i] = carry_k + pk; }
        __syncthreads();
        if (threadIdx.x == 0) { carry_a += ta; carry_k += tk; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { abase[n] = carry_a; kbase[n] = carry_k; }
}
__global__ void k_pack_copy(const pgs_scan_result *__restrict__ res, uint32_t n, const uint8_t *__restrict__ arena,
                            unsigned long long arena_stride, const pgs_kv *__restrict__ kvs, uint32_t kv_stride,
                            const unsigned long long *__restrict__ abase, const uint32_t *__restrict__ kbase,
                            uint8_t *__restrict__ parena, pgs_kv *__restrict__ pkvs)
{
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        uint32_t chunks = (uint32_t)((res[i].arena_used + 15) >> 4);
        const uint4 *src = (const uint4 *)(arena + (size_t)i * arena_stride);
        uint4 *dst = (uint4 *)(parena + abase[i]);
        for (uint32_t c = threadIdx.x; c < chunks; c += blockDim.x) dst[c] = src[c];
        for (uint32_t k = threadIdx.x; k < res[i].n_kvs; k += blockDim.x) pkvs[kbase[i] + k] = kvs[(size_t)i * kv_stride + k];
    }
}

static uint64_t *g_crc_dev_rd[16] = {nullptr};
static std::mutex g_crc_rd_mu;
const uint64_t *crc64_table();
void set_last_read_stats(float ms, uint64_t probed, uint64_t skipped);

static int32_t snapshot_runs(Partition &part, std::vector<std::shared_ptr<Run>> &runs, ReadRuns &rr, uint32_t &KS,
                             const std::vector<std::shared_ptr<Run>> *pinned = nullptr)
{
    if (pinned) {
        runs = *pinned;
    } else {
        std::lock_guard<std::mutex> g(part.mu);
        runs = part.runs;
    }
    if (runs.size() > kMaxReadRuns) {
        set_error("read: %zu runs > %u (compact first)", runs.size(), kMaxReadRuns);
        return PGS_NOT_SUPPORTED;
    }
    rr.n = (uint32_t)runs.size();
    uint32_t mk = 0;
    for (uint32_t i = 0; i < rr.n; i++) { rr.runs[i] = runs[i]->dev(); mk = std::max(mk, runs[i]->info.max_ukey_len); }
    if (mk > kMaxUkeyLen) return PGS_NOT_SUPPORTED;
    KS = std::max(8u, (mk + 7) & ~7u);
    return PGS_OK;
}

// true when k_scan can stage one block of every current run of the partition in one request's launch; scan_launch answers
// a batch with a reverse request with PGS_NOT_SUPPORTED otherwise (the server folds L0 first, server.cpp)
bool scan_stages_every_run(Partition &part)
{
    std::vector<std::shared_ptr<Run>> runs;
    {
        std::lock_guard<std::mutex> g(part.mu);
        runs = part.runs;
    }
    if (runs.size() > kMaxReadRuns) return false;
    uint32_t mk = 0, max_blk = 0, max_rec = 0;
    for (auto &r : runs) {
        mk = std::max(mk, r->info.max_ukey_len);
        max_blk = std::max(max_blk, r->info.max_block_size);
        max_rec = std::max(max_rec, r->info.max_block_records);
    }
    cudaFuncAttributes attr;
    if (cudaSetDevice(part.eng->device) != cudaSuccess || cudaFuncGetAttributes(&attr, k_scan) != cudaSuccess) return true; // the launch reports it
    const uint64_t max_dyn = (uint64_t)part.eng->max_smem_optin - attr.sharedSizeBytes - 256;
    uint32_t pool = 0;
    return scan_dyn_bytes((uint32_t)runs.size(), std::max(8u, (mk + 7) & ~7u), max_blk, max_rec, 1, max_dyn, &pool) != 0;
}

// kernels of this file take their dynamic shared-memory size per launch; the opt-in maximum is set once per device here
// (a per-call cudaFuncSetAttribute would race between reader threads)
template <class K>
static cudaError_t allow_max_smem(K kernel, int max_smem)
{
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, kernel);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes);
}
int32_t lookup_init_kernels(int max_smem)
{
    PGS_CUDA(allow_max_smem(k_scan, max_smem));
    PGS_CUDA(cudaFuncSetAttribute(k_scan, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    PGS_CUDA(allow_max_smem(k_get<8, false>, max_smem)); PGS_CUDA(allow_max_smem(k_get<8, true>, max_smem));
    PGS_CUDA(allow_max_smem(k_scan_fwd<8, false>, max_smem)); PGS_CUDA(allow_max_smem(k_scan_fwd<8, true>, max_smem));
    PGS_CUDA(allow_max_smem(k_scan_fwd<16, false>, max_smem)); PGS_CUDA(allow_max_smem(k_scan_fwd<16, true>, max_smem));
    PGS_CUDA(allow_max_smem(k_scan_fwd<32, false>, max_smem)); PGS_CUDA(allow_max_smem(k_scan_fwd<32, true>, max_smem));
    return PGS_OK;
}

// the runs of several partitions, packed for one launch (pgs_range_scan_many_multi)
struct ScanMulti {
    std::vector<RunDev> packed;
    std::vector<uint32_t> begin;
    const uint32_t *req_part;
};

static int32_t scan_launch(Partition &part, std::vector<std::shared_ptr<Run>> &runs, ScanParams &P, const ScanMulti *multi,
                           const pgs_scan_request *reqs, uint32_t n, uint32_t now, unsigned long long arena_stride, uint32_t kv_stride,
                           uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume, uint32_t resume_stride,
                           pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base);

int32_t scan_many(Partition &part, const pgs_scan_request *reqs, uint32_t n, uint32_t now, unsigned long long arena_stride,
                  uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume,
                  uint32_t resume_stride, pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base,
                  const std::vector<std::shared_ptr<Run>> *pinned)
{
    std::vector<std::shared_ptr<Run>> runs;
    ScanParams P{};
    int32_t rc = snapshot_runs(part, runs, P.rr, P.KS, pinned);
    if (rc != PGS_OK) return rc;
    if (n == 0) return PGS_OK;
    return scan_launch(part, runs, P, nullptr, reqs, n, now, arena_stride, kv_stride, arena, arena_cap, kvs, kv_cap, resume, resume_stride,
                       results, arena_base, kv_base);
}

// forward scans over several partitions of one engine in one launch: request i reads partition slot req_part[i]
static int32_t scan_many_multi(pgs_partition *const *parts, uint32_t n_parts, const pgs_scan_request *reqs, const uint32_t *req_part, uint32_t n,
                               uint32_t now, unsigned long long arena_stride, uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs,
                               uint64_t kv_cap, uint8_t *resume, uint32_t resume_stride, pgs_scan_result *results, uint64_t *arena_base,
                               uint32_t *kv_base)
{
    Partition &part = parts[0]->p;
    std::vector<std::shared_ptr<Run>> runs; // every run a request may touch stays alive until the launch is done
    ScanParams P{};
    ScanMulti M;
    M.req_part = req_part;
    M.begin.push_back(0);
    P.KS = 8;
    uint32_t max_nr = 0;
    for (uint32_t p = 0; p < n_parts; p++) {
        Partition &pp = parts[p]->p;
        if (pp.eng != part.eng || pp.data_version != part.data_version) { set_error("range_scan_many_multi: partitions of different engines / data versions"); return PGS_INVALID_ARGUMENT; }
        std::vector<std::shared_ptr<Run>> rs;
        ReadRuns rr;
        uint32_t ks = 0;
        int32_t rc = snapshot_runs(pp, rs, rr, ks);
        if (rc != PGS_OK) return rc;
        for (uint32_t i = 0; i < rr.n; i++) M.packed.push_back(rr.runs[i]);
        M.begin.push_back((uint32_t)M.packed.size());
        runs.insert(runs.end(), rs.begin(), rs.end());
        P.KS = std::max(P.KS, ks);
        max_nr = std::max(max_nr, rr.n);
    }
    for (uint32_t i = 0; i < n; i++) {
        if (req_part[i] >= n_parts) { set_error("range_scan_many_multi: request %u names partition slot %u of %u", i, req_part[i], n_parts); return PGS_INVALID_ARGUMENT; }
        if (reqs[i].reverse) { set_error("range_scan_many_multi: reverse scans go through pgs_range_scan_many"); return PGS_NOT_SUPPORTED; }
    }
    if (n == 0) return PGS_OK;
    P.rr.n = max_nr;
    if (!M.packed.empty())
        for (uint32_t i = 0; i < kMaxReadRuns; i++) P.rr.runs[i] = M.packed[0]; // a valid dummy for idle groups
    return scan_launch(part, runs, P, &M, reqs, n, now, arena_stride, kv_stride, arena, arena_cap, kvs, kv_cap, resume, resume_stride, results,
                       arena_base, kv_base);
}

static int32_t scan_launch(Partition &part, std::vector<std::shared_ptr<Run>> &runs, ScanParams &P, const ScanMulti *multi,
                           const pgs_scan_request *reqs, uint32_t n, uint32_t now, unsigned long long arena_stride, uint32_t kv_stride,
                           uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume, uint32_t resume_stride,
                           pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base)
{
    Engine *e = part.eng;
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->read_stream();
    // flatten requests
    std::vector<ScanReqDev> dev(n);
    std::string blob;
    bool need_crc = false, any_reverse = false;
    for (uint32_t i = 0; i < n; i++) {
        const pgs_scan_request &q = reqs[i];
        ScanReqDev &d = dev[i];
        memset(&d, 0, sizeof d);
        auto put = [&](const pgs_blob &b, uint32_t &off, uint32_t &len) {
            off = (uint32_t)blob.size();
            len = b.len;
            if (b.len) blob.append((const char *)b.data, b.len);
        };
        put(q.start, d.start_off, d.start_len);
        put(q.stop, d.stop_off, d.stop_len);
        put(q.hash_filter, d.hf_off, d.hf_len);
        put(q.sort_filter, d.sf_off, d.sf_len);
        d.start_inclusive = q.start_inclusive; d.stop_inclusive = q.stop_inclusive; d.reverse = q.reverse;
        d.no_value = q.no_value; d.key_mode = q.key_mode; d.return_expire_ts = q.return_expire_ts;
        d.count_only = q.count_only; d.validate_hash = q.validate_hash; d.prefix_same_as_start = q.prefix_same_as_start;
        d.has_upper = q.reserved[0]; // iterate_upper_bound (internal flag used by sortkey_count)
        d.hash_filter_type = q.hash_filter_type; d.sort_filter_type = q.sort_filter_type;
        d.max_count = q.max_count; d.max_iter_count = q.max_iter_count; d.max_iter_size = q.max_iter_size;
        d.pidx = q.pidx; d.partition_version = q.partition_version;
        need_crc |= q.validate_hash != 0;
        any_reverse |= q.reverse != 0;
    }
    blob.append(16, '\0');
    if (resume_stride < P.KS) resume_stride = 0; // caller gave no room: resume keys are not reported
    P.n = n; P.now = now; P.data_version = part.data_version;
    P.use_tma = (e->cfg.flags & PGS_ENGINE_NO_TMA) ? 0 : 1;
    P.kv_stride = kv_stride; P.arena_stride = (arena_stride + 15) & ~15ull; P.resume_stride = resume_stride ? resume_stride : P.KS;
    if (multi ? multi->packed.empty() : P.rr.n == 0) { // empty DB: every iterator is invalid from the start
        memset(results, 0, sizeof(pgs_scan_result) * n);
        if (arena_base) for (uint32_t i = 0; i <= n; i++) arena_base[i] = 0;
        if (kv_base) for (uint32_t i = 0; i <= n; i++) kv_base[i] = 0;
        return PGS_OK;
    }

    ScanReqDev *d_reqs = nullptr; uint8_t *d_blob = nullptr, *d_arena = nullptr, *d_resume = nullptr, *d_parena = nullptr;
    pgs_scan_result *d_res = nullptr; pgs_kv *d_kvs = nullptr, *d_pkvs = nullptr; uint32_t *d_err = nullptr, *d_kbase = nullptr;
    unsigned long long *d_abase = nullptr;
    RunDev *d_multi = nullptr;
    uint32_t *d_begin = nullptr, *d_part = nullptr;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    auto cleanup = [&]() {
        if (d_multi) cudaFreeAsync(d_multi, st);
        if (d_begin) cudaFreeAsync(d_begin, st);
        if (d_part) cudaFreeAsync(d_part, st);
        cudaFreeAsync(d_reqs, st); cudaFreeAsync(d_blob, st); cudaFreeAsync(d_arena, st); cudaFreeAsync(d_resume, st);
        cudaFreeAsync(d_parena, st); cudaFreeAsync(d_res, st); cudaFreeAsync(d_kvs, st); cudaFreeAsync(d_pkvs, st);
        cudaFreeAsync(d_err, st); cudaFreeAsync(d_kbase, st); cudaFreeAsync(d_abase, st);
        if (ev_a) cudaEventDestroy(ev_a);
        if (ev_b) cudaEventDestroy(ev_b);
    };
#define CK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { cleanup(); return cuda_fail(_e, #expr); } } while (0)
    CK(cudaEventCreate(&ev_a));
    CK(cudaEventCreate(&ev_b));
    CK(cudaMallocAsync(&d_reqs, sizeof(ScanReqDev) * n, st));
    CK(cudaMallocAsync(&d_blob, blob.size(), st));
    CK(cudaMallocAsync(&d_arena, P.arena_stride * n + 16, st));
    CK(cudaMallocAsync(&d_kvs, sizeof(pgs_kv) * (size_t)kv_stride * n + 16, st));
    CK(cudaMallocAsync(&d_resume, (size_t)P.resume_stride * n + 16, st));
    CK(cudaMallocAsync(&d_res, sizeof(pgs_scan_result) * n, st));
    CK(cudaMallocAsync(&d_err, 256, st));
    CK(cudaMemcpyAsync(d_reqs, dev.data(), sizeof(ScanReqDev) * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_blob, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_err, 0, 256, st));
    if (multi) {
        CK(cudaMallocAsync(&d_multi, sizeof(RunDev) * multi->packed.size(), st));
        CK(cudaMallocAsync(&d_begin, sizeof(uint32_t) * multi->begin.size(), st));
        CK(cudaMallocAsync(&d_part, sizeof(uint32_t) * n, st));
        CK(cudaMemcpyAsync(d_multi, multi->packed.data(), sizeof(RunDev) * multi->packed.size(), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_begin, multi->begin.data(), sizeof(uint32_t) * multi->begin.size(), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_part, multi->req_part, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
        P.multi_runs = d_multi; P.multi_begin = d_begin; P.req_part = d_part;
    }
    if (need_crc) {
        std::lock_guard<std::mutex> g(g_crc_rd_mu);
        int dv = e->device & 15;
        if (!g_crc_dev_rd[dv]) {
            uint64_t *t = nullptr;
            CK(cudaMalloc(&t, 2048));
            CK(cudaMemcpy(t, crc64_table(), 2048, cudaMemcpyHostToDevice));
            g_crc_dev_rd[dv] = t;
        }
        P.crc_table = (const unsigned long long *)g_crc_dev_rd[dv];
    }
    P.reqs = d_reqs; P.blob = d_blob; P.results = d_res; P.kvs = d_kvs; P.arena = d_arena; P.resume = d_resume; P.error = d_err;
    P.ticket = d_err + 8;
    const char *pt_env = getenv("PGS_PHASE_TIMING"); // diagnostics: per-phase cycle totals of the reverse kernel on stderr
    const bool phase_timing = any_reverse && pt_env && pt_env[0] == '1';
    P.phase_cycles = phase_timing ? (unsigned long long *)(d_err + 16) : nullptr;
    // forward scans: lane-group merging iterators (read_kernels.cuh), unless the groups' key rows do not fit shared memory
    // (user keys of a few KB): then k_scan, which stages records instead of keeping one key row per run and group
    const uint32_t NR = P.rr.n, G = NR <= 8 ? 8 : NR <= 16 ? 16 : 32;
    const uint32_t fwd_ks = (P.KS + 3) & ~3u, fwd_ksw = (fwd_ks + 8) / 4 + 1;
    const uint32_t fwd_group_smem = (uint32_t)((NR * (sizeof(CurState) + fwd_ksw * 4) + 3 * fwd_ksw * 4 + 15) & ~(size_t)15);
    const uint32_t fwd_dyn = 2048 + kMaxReadRuns * (uint32_t)sizeof(RunDev) + (kReadThreads / G) * fwd_group_smem;
    const bool fwd_fits = fwd_dyn <= (uint32_t)e->max_smem_optin;
    if (!fwd_fits && multi) { cleanup(); set_error("scan: %u runs with keys of %u bytes do not fit shared memory", NR, P.KS); return PGS_NOT_SUPPORTED; }
    if (!any_reverse && fwd_fits) {
        P.KS = fwd_ks;
        P.KSW = fwd_ksw;
        P.group_smem = fwd_group_smem;
        const uint32_t dyn = fwd_dyn;
        auto kern = multi ? (G == 8 ? k_scan_fwd<8, true> : G == 16 ? k_scan_fwd<16, true> : k_scan_fwd<32, true>)
                          : (G == 8 ? k_scan_fwd<8, false> : G == 16 ? k_scan_fwd<16, false> : k_scan_fwd<32, false>);
        int occ = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (int)kReadThreads, (size_t)dyn));
        const uint32_t per_cta = kReadThreads / G;
        const uint32_t grid = std::min<uint32_t>((n + per_cta - 1) / per_cta, (uint32_t)std::max(1, occ) * e->sm_count);
        CK(cudaEventRecord(ev_a, st));
        kern<<<grid, kReadThreads, dyn, st>>>(P);
        CK(cudaEventRecord(ev_b, st));
    } else {
        // ---- reverse scans (and forward ones with long keys): the block-staging kernel ---------------------------------
        cudaFuncAttributes attr;
        CK(cudaFuncGetAttributes(&attr, k_scan));
        P.warp_scratch = 0;
        uint32_t max_blk = 0, max_rec = 0;
        for (auto &r : runs) { max_blk = std::max(max_blk, r->info.max_block_size); max_rec = std::max(max_rec, r->info.max_block_records); }
        const uint64_t max_dyn = (uint64_t)e->max_smem_optin - attr.sharedSizeBytes - 256;
        const uint64_t dyn = scan_dyn_bytes((uint32_t)runs.size(), P.KS, max_blk, max_rec, n, max_dyn, &P.pool_bytes);
        if (!dyn) {
            cleanup();
            set_error("scan: blocks too large for shared memory");
            return PGS_NOT_SUPPORTED;
        }
        int occ = 0; // resident CTAs per SM for this dynamic shared-memory size (registers count too)
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_scan, (int)kScanThreads, (size_t)dyn));
        uint32_t grid = std::min<uint32_t>(n, (uint32_t)std::max(1, occ) * e->sm_count);
        CK(cudaEventRecord(ev_a, st));
        k_scan<<<grid, kScanThreads, dyn, st>>>(P);
        CK(cudaEventRecord(ev_b, st));
        if (phase_timing) {
            unsigned long long h[16] = {0};
            cudaMemcpyAsync(h, d_err + 16, sizeof h, cudaMemcpyDeviceToHost, st);
            cudaStreamSynchronize(st);
            static const char *names[13] = {"init", "choose", "stage", "farbound", "decode1", "decode2", "window", "rank", "visible", "loop", "emit", "advance", "result"};
            unsigned long long tot = 0;
            for (int i = 0; i < 13; i++) tot += h[i];
            fprintf(stderr, "[k_scan phases] requests=%u grid=%u dyn=%llu", n, grid, (unsigned long long)dyn);
            for (int i = 0; i < 13; i++) fprintf(stderr, " %s=%.1f%%", names[i], tot ? 100.0 * (double)h[i] / (double)tot : 0.0);
            fprintf(stderr, " cycles/request=%.0f\n", n ? (double)tot / n : 0.0);
        }
    }
    e->launches++;
    uint32_t herr = 0;
    if (n == 1) {
        CK(cudaMemcpyAsync(results, d_res, sizeof(pgs_scan_result), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (!herr) {
            if (results[0].arena_used > arena_cap || results[0].n_kvs > kv_cap) { cleanup(); return PGS_INCOMPLETE; }
            if (results[0].arena_used) CK(cudaMemcpyAsync(arena, d_arena, results[0].arena_used, cudaMemcpyDeviceToHost, st));
            if (results[0].n_kvs) CK(cudaMemcpyAsync(kvs, d_kvs, sizeof(pgs_kv) * results[0].n_kvs, cudaMemcpyDeviceToHost, st));
            if (results[0].iter_valid && resume && resume_stride) CK(cudaMemcpyAsync(resume, d_resume, results[0].resume_len, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        if (arena_base) { arena_base[0] = 0; arena_base[1] = results[0].arena_used; }
        if (kv_base) { kv_base[0] = 0; kv_base[1] = results[0].n_kvs; }
    } else {
        CK(cudaMallocAsync(&d_abase, sizeof(unsigned long long) * (n + 1), st));
        CK(cudaMallocAsync(&d_kbase, sizeof(uint32_t) * (n + 1), st));
        k_pack_offsets<<<1, 1024, 0, st>>>(d_res, n, d_abase, d_kbase);
        std::vector<unsigned long long> ab(n + 1);
        std::vector<uint32_t> kb(n + 1);
        CK(cudaMemcpyAsync(ab.data(), d_abase, sizeof(unsigned long long) * (n + 1), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(kb.data(), d_kbase, sizeof(uint32_t) * (n + 1), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(results, d_res, sizeof(pgs_scan_result) * n, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        e->launches++;
        if (!herr) {
            if (ab[n] > arena_cap || kb[n] > kv_cap) { cleanup(); set_error("scan_many: output arena too small"); return PGS_INCOMPLETE; }
            CK(cudaMallocAsync(&d_parena, ab[n] + 16, st));
            CK(cudaMallocAsync(&d_pkvs, sizeof(pgs_kv) * ((size_t)kb[n] + 1), st));
            k_pack_copy<<<std::min<uint32_t>(n, 8 * e->sm_count), 128, 0, st>>>(d_res, n, d_arena, P.arena_stride, d_kvs, kv_stride, d_abase,
                                                                              d_kbase, d_parena, d_pkvs);
            e->launches++;
            if (ab[n]) CK(cudaMemcpyAsync(arena, d_parena, ab[n], cudaMemcpyDeviceToHost, st));
            if (kb[n]) CK(cudaMemcpyAsync(kvs, d_pkvs, sizeof(pgs_kv) * kb[n], cudaMemcpyDeviceToHost, st));
            if (resume && resume_stride) CK(cudaMemcpyAsync(resume, d_resume, (size_t)P.resume_stride * n, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        if (arena_base) for (uint32_t i = 0; i <= n; i++) arena_base[i] = ab[i];
        if (kv_base) for (uint32_t i = 0; i <= n; i++) kv_base[i] = kb[i];
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    set_last_read_stats(ms, 0, 0);
    cleanup();
#undef CK
    if (herr) {
        set_error("scan kernel failed with status %u", herr);
        // PGS_ABORTED = a request's output did not fit its arena / kv slice: the caller may retry with more room
        return herr == PGS_CORRUPTION ? PGS_CORRUPTION : (herr == PGS_NOT_SUPPORTED ? PGS_NOT_SUPPORTED : (herr == PGS_ABORTED ? PGS_ABORTED : PGS_IO_ERROR));
    }
    return PGS_OK;
}

} // namespace pgs

using namespace pgs;

// one get launch over the keys of one partition (parts[0], key_part null) or of several partitions of one engine
static int32_t get_batch_impl(pgs_partition *const *parts, uint32_t n_parts, const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part,
                              uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used)
{
    Partition &part = parts[0]->p;
    Engine *e = part.eng;
    if (arena_used) *arena_used = 0;
    if (n == 0) return PGS_OK;
    // pgs_get_result::value_off is 32-bit: a call uses at most the first 4 GiB - 1 of the arena.  A value that would end
    // beyond that gets PGS_INCOMPLETE like any value that does not fit, and *arena_used still reports the whole need.
    arena_cap = std::min<uint64_t>(arena_cap, UINT32_MAX);
    std::vector<std::shared_ptr<Run>> runs; // every run a key may touch stays alive until the launch is done
    GetParams P{};
    std::vector<RunDev> packed;
    std::vector<uint32_t> begin;
    if (!key_part) {
        int32_t rc = snapshot_runs(part, runs, P.rr, P.KS);
        if (rc != PGS_OK) return rc;
    } else {
        P.rr.n = 0;
        P.KS = 8;
        begin.push_back(0);
        for (uint32_t p = 0; p < n_parts; p++) {
            Partition &pp = parts[p]->p;
            if (pp.eng != e || pp.data_version != part.data_version) { set_error("get_batch_multi: partitions of different engines / data versions"); return PGS_INVALID_ARGUMENT; }
            std::vector<std::shared_ptr<Run>> rs;
            ReadRuns rr;
            uint32_t ks = 0;
            int32_t rc = snapshot_runs(pp, rs, rr, ks);
            if (rc != PGS_OK) return rc;
            for (uint32_t i = 0; i < rr.n; i++) packed.push_back(rr.runs[i]);
            begin.push_back((uint32_t)packed.size());
            runs.insert(runs.end(), rs.begin(), rs.end());
            P.KS = std::max(P.KS, ks);
        }
        for (uint32_t i = 0; i < n; i++)
            if (key_part[i] >= n_parts) { set_error("get_batch_multi: key %u names partition slot %u of %u", i, key_part[i], n_parts); return PGS_INVALID_ARGUMENT; }
        if (!packed.empty()) P.rr.runs[0] = packed[0]; // a valid dummy for idle groups
    }
    if (key_part ? packed.empty() : P.rr.n == 0) {
        for (uint32_t i = 0; i < n; i++) { memset(&results[i], 0, sizeof results[i]); results[i].status = PGS_NOT_FOUND; }
        return PGS_OK;
    }
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->read_stream();
    uint64_t key_bytes = key_off[n];
    uint8_t *d_keys = nullptr, *d_arena = nullptr;
    uint32_t *d_off = nullptr, *d_err = nullptr;
    pgs_get_result *d_res = nullptr;
    unsigned long long *d_cur = nullptr;
    RunDev *d_multi = nullptr;
    uint32_t *d_begin = nullptr, *d_part = nullptr;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    auto cleanup = [&]() {
        cudaFreeAsync(d_keys, st); cudaFreeAsync(d_arena, st); cudaFreeAsync(d_off, st); cudaFreeAsync(d_err, st);
        cudaFreeAsync(d_res, st); cudaFreeAsync(d_cur, st);
        if (d_multi) cudaFreeAsync(d_multi, st);
        if (d_begin) cudaFreeAsync(d_begin, st);
        if (d_part) cudaFreeAsync(d_part, st);
        if (ev_a) cudaEventDestroy(ev_a);
        if (ev_b) cudaEventDestroy(ev_b);
    };
#define CK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { cleanup(); return cuda_fail(_e, #expr); } } while (0)
    CK(cudaEventCreate(&ev_a));
    CK(cudaEventCreate(&ev_b));
    CK(cudaMallocAsync(&d_keys, key_bytes + 16, st));
    CK(cudaMallocAsync(&d_off, sizeof(uint32_t) * (n + 1), st));
    CK(cudaMallocAsync(&d_res, sizeof(pgs_get_result) * n, st));
    CK(cudaMallocAsync(&d_arena, arena_cap + 16, st));
    CK(cudaMallocAsync(&d_cur, 32, st));
    CK(cudaMallocAsync(&d_err, 16, st));
    CK(cudaMemcpyAsync(d_keys, keys, key_bytes, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_off, key_off, sizeof(uint32_t) * (n + 1), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_cur, 0, 32, st));
    CK(cudaMemsetAsync(d_err, 0, 16, st));
    if (key_part) {
        CK(cudaMallocAsync(&d_multi, sizeof(RunDev) * packed.size(), st));
        CK(cudaMallocAsync(&d_begin, sizeof(uint32_t) * begin.size(), st));
        CK(cudaMallocAsync(&d_part, sizeof(uint32_t) * n, st));
        CK(cudaMemcpyAsync(d_multi, packed.data(), sizeof(RunDev) * packed.size(), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_begin, begin.data(), sizeof(uint32_t) * begin.size(), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_part, key_part, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
        P.multi_runs = d_multi; P.multi_begin = d_begin; P.key_part = d_part;
    }
    P.keys = d_keys; P.key_off = d_off; P.n = n; P.now = now; P.data_version = part.data_version;
    P.results = d_res; P.arena = d_arena; P.arena_cap = arena_cap; P.arena_cursor = d_cur; P.error = d_err; P.ticket = d_err + 1;
    constexpr uint32_t G = 8;
    P.KS = (P.KS + 3) & ~3u;
    P.KSW = (P.KS + 8) / 4 + 1;
    P.group_smem = (uint32_t)((sizeof(CurState) + 2 * P.KSW * 4 + 15) & ~(size_t)15);
    const uint32_t dyn = kMaxReadRuns * (uint32_t)sizeof(RunDev) + (kReadThreads / G) * P.group_smem;
    if (dyn > (uint32_t)e->max_smem_optin) { cleanup(); return PGS_NOT_SUPPORTED; }
    int occ = 0;
    auto kern = key_part ? k_get<G, true> : k_get<G, false>;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (int)kReadThreads, (size_t)dyn));
    const uint32_t per_cta = kReadThreads / G;
    const uint32_t grid = std::min<uint32_t>((n + per_cta - 1) / per_cta, (uint32_t)std::max(1, occ) * e->sm_count);
    CK(cudaEventRecord(ev_a, st));
    kern<<<grid, kReadThreads, dyn, st>>>(P);
    CK(cudaEventRecord(ev_b, st));
    e->launches++;
    uint32_t herr = 0;
    unsigned long long cur3[3] = {0, 0, 0};
    CK(cudaMemcpyAsync(results, d_res, sizeof(pgs_get_result) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(cur3, d_cur, 24, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    set_last_read_stats(ms, cur3[1], cur3[2]);
    const unsigned long long used = cur3[0];
    if (arena_used) *arena_used = used;
    if (!herr && used) {
        CK(cudaMemcpyAsync(arena, d_arena, std::min<unsigned long long>(used, arena_cap), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    cleanup();
#undef CK
    if (herr) { set_error("get kernel failed with status %u", herr); return herr == PGS_CORRUPTION ? PGS_CORRUPTION : PGS_IO_ERROR; }
    return used > arena_cap ? PGS_INCOMPLETE : PGS_OK;
}

extern "C" int32_t pgs_get_batch(pgs_partition *ph, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                                 uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used)
{
    if (!ph || (n && (!keys || !key_off || !results))) return PGS_INVALID_ARGUMENT;
    return get_batch_impl(&ph, 1, keys, key_off, nullptr, n, now, arena, arena_cap, results, arena_used);
}

extern "C" int32_t pgs_get_batch_multi(pgs_partition *const *parts, uint32_t n_parts, const uint8_t *keys, const uint32_t *key_off,
                                       const uint32_t *key_part, uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap,
                                       pgs_get_result *results, uint64_t *arena_used)
{
    if (!parts || !n_parts || (n && (!keys || !key_off || !key_part || !results))) return PGS_INVALID_ARGUMENT;
    for (uint32_t p = 0; p < n_parts; p++)
        if (!parts[p]) return PGS_INVALID_ARGUMENT;
    return get_batch_impl(parts, n_parts, keys, key_off, key_part, n, now, arena, arena_cap, results, arena_used);
}

extern "C" int32_t pgs_range_scan(pgs_partition *ph, const pgs_scan_request *req, uint32_t now, uint8_t *arena,
                                  uint64_t arena_cap, pgs_kv *kvs, uint32_t kv_cap, uint8_t *resume_key,
                                  uint32_t resume_cap, pgs_scan_result *out)
{
    if (!ph || !req || !out) return PGS_INVALID_ARGUMENT;
    return scan_many(ph->p, req, 1, now, arena_cap, kv_cap, arena, arena_cap, kvs, kv_cap, resume_key, resume_cap, out, nullptr, nullptr, nullptr);
}

extern "C" int32_t pgs_range_scan_many(pgs_partition *ph, const pgs_scan_request *reqs, uint32_t n, uint32_t now,
                                       uint64_t arena_stride, uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap,
                                       pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume_keys, uint32_t resume_stride,
                                       pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base)
{
    if (!ph || (n && (!reqs || !results))) return PGS_INVALID_ARGUMENT;
    return scan_many(ph->p, reqs, n, now, arena_stride, kv_stride, arena, arena_cap, kvs, kv_cap, resume_keys, resume_stride, results,
                     arena_base, kv_base, nullptr);
}

extern "C" int32_t pgs_range_scan_many_multi(pgs_partition *const *parts, uint32_t n_parts, const pgs_scan_request *reqs, const uint32_t *req_part,
                                             uint32_t n, uint32_t now, uint64_t arena_stride, uint32_t kv_stride, uint8_t *arena,
                                             uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume_keys, uint32_t resume_stride,
                                             pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base)
{
    if (!parts || !n_parts || (n && (!reqs || !req_part || !results))) return PGS_INVALID_ARGUMENT;
    for (uint32_t p = 0; p < n_parts; p++)
        if (!parts[p]) return PGS_INVALID_ARGUMENT;
    return scan_many_multi(parts, n_parts, reqs, req_part, n, now, arena_stride, kv_stride, arena, arena_cap, kvs, kv_cap, resume_keys,
                           resume_stride, results, arena_base, kv_base);
}
