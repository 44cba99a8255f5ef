// lookup.cu — host side of the read path (pgs_get_batch, pgs_range_scan, pgs_range_scan_many).
//
//   k_get / k_scan_fwd (read_kernels.cuh)  point lookups and forward range scans: lane-group iterators straight over HBM.
//   k_scan (scan_kernel.cuh)  REVERSE range scans, every request of a batch that mixes directions, and forward scans
//           whose user keys are too long for k_scan_fwd: one CTA per request stages chunks of blocks of every run in shared memory.
#include <algorithm>
#include <cstring>

#include "engine.h"
#include "hotkey_kernels.cuh"
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
    KS = read_key_slot(mk);
    return PGS_OK;
}

// the runs of several partitions of one engine, packed for one launch: partition slot s reads packed[begin[s] .. begin[s + 1])
struct MultiRuns {
    std::vector<std::shared_ptr<Run>> runs; // every run a request may touch stays alive until the launch is done
    std::vector<RunDev> packed;
    std::vector<uint32_t> begin{0};
};
// what: the ABI call, for the error message
static int32_t snapshot_multi(pgs_partition *const *parts, uint32_t n_parts, const char *what, MultiRuns &M, ReadRuns &rr, uint32_t &KS)
{
    const Partition &part = parts[0]->p;
    KS = 8;
    for (uint32_t p = 0; p < n_parts; p++) {
        Partition &pp = parts[p]->p;
        if (pp.eng != part.eng || pp.data_version != part.data_version) { set_error("%s: partitions of different engines / data versions", what); return PGS_INVALID_ARGUMENT; }
        std::vector<std::shared_ptr<Run>> rs;
        ReadRuns one;
        uint32_t ks = 0;
        int32_t rc = snapshot_runs(pp, rs, one, ks);
        if (rc != PGS_OK) return rc;
        M.packed.insert(M.packed.end(), one.runs, one.runs + one.n);
        M.begin.push_back((uint32_t)M.packed.size());
        M.runs.insert(M.runs.end(), rs.begin(), rs.end());
        KS = std::max(KS, ks);
    }
    multi_read_runs(M.packed, M.begin, rr);
    return PGS_OK;
}

// the dynamic shared memory of a k_scan launch of n_req requests over these runs on the current device (scan_dyn_bytes: 0 when
// one block of every run does not fit); *pool = its staging pool
static cudaError_t scan_launch_dyn(const Engine &e, const std::vector<std::shared_ptr<Run>> &runs, uint32_t KS, uint32_t n_req,
                                   uint64_t &dyn, uint32_t *pool)
{
    cudaFuncAttributes attr;
    const cudaError_t rc = cudaFuncGetAttributes(&attr, k_scan);
    if (rc != cudaSuccess) return rc;
    ScanBlockBound bb;
    for (auto &r : runs) bb.add(r->info);
    dyn = scan_dyn_bytes((uint32_t)runs.size(), KS, bb.max_blk, bb.max_rec, n_req, scan_max_dyn(e.max_smem_optin, attr.sharedSizeBytes), pool);
    return cudaSuccess;
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
    uint32_t mk = 0;
    for (auto &r : runs) mk = std::max(mk, r->info.max_ukey_len);
    uint64_t dyn = 0; uint32_t pool = 0;
    if (cudaSetDevice(part.eng->device) != cudaSuccess || scan_launch_dyn(*part.eng, runs, read_key_slot(mk), 1, dyn, &pool) != cudaSuccess)
        return true; // the launch reports it
    return dyn != 0;
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
    for (uint32_t G : kScanFwdGs)
        for (bool multi : {false, true}) PGS_CUDA(allow_max_smem(scan_fwd_kernel(G, multi), max_smem));
    return PGS_OK;
}

static int32_t scan_launch(Partition &part, const std::vector<std::shared_ptr<Run>> &runs, ScanParams &P, const MultiRuns *multi,
                           const uint32_t *req_part, const pgs_scan_request *reqs, uint32_t n, uint32_t now, unsigned long long arena_stride,
                           uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume,
                           uint32_t resume_stride, pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base);

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
    return scan_launch(part, runs, P, nullptr, nullptr, reqs, n, now, arena_stride, kv_stride, arena, arena_cap, kvs, kv_cap, resume,
                       resume_stride, results, arena_base, kv_base);
}

// forward scans over several partitions of one engine in one launch: request i reads partition slot req_part[i]
static int32_t scan_many_multi(pgs_partition *const *parts, uint32_t n_parts, const pgs_scan_request *reqs, const uint32_t *req_part, uint32_t n,
                               uint32_t now, unsigned long long arena_stride, uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs,
                               uint64_t kv_cap, uint8_t *resume, uint32_t resume_stride, pgs_scan_result *results, uint64_t *arena_base,
                               uint32_t *kv_base)
{
    ScanParams P{};
    MultiRuns M;
    int32_t rc = snapshot_multi(parts, n_parts, "range_scan_many_multi", M, P.rr, P.KS);
    if (rc != PGS_OK) return rc;
    for (uint32_t i = 0; i < n; i++) {
        if (req_part[i] >= n_parts) { set_error("range_scan_many_multi: request %u names partition slot %u of %u", i, req_part[i], n_parts); return PGS_INVALID_ARGUMENT; }
        if (reqs[i].reverse) { set_error("range_scan_many_multi: reverse scans go through pgs_range_scan_many"); return PGS_NOT_SUPPORTED; }
    }
    if (n == 0) return PGS_OK;
    return scan_launch(parts[0]->p, M.runs, P, &M, req_part, reqs, n, now, arena_stride, kv_stride, arena, arena_cap, kvs, kv_cap, resume,
                       resume_stride, results, arena_base, kv_base);
}

static int32_t scan_launch(Partition &part, const std::vector<std::shared_ptr<Run>> &runs, ScanParams &P, const MultiRuns *multi,
                           const uint32_t *req_part, const pgs_scan_request *reqs, uint32_t n, uint32_t now, unsigned long long arena_stride,
                           uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume,
                           uint32_t resume_stride, pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base)
{
    Engine *e = part.eng;
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->read_stream();
    const ScanBatch B = flatten_scan_requests(reqs, n);
    if (!scan_output_strides(P, arena_stride, kv_stride, resume_stride)) resume_stride = 0; // caller gave no room for resume keys
    P.n = n; P.now = now; P.data_version = part.data_version;
    if (multi ? multi->packed.empty() : P.rr.n == 0) { // empty DB: every iterator is invalid from the start
        memset(results, 0, sizeof(pgs_scan_result) * n);
        if (arena_base) for (uint32_t i = 0; i <= n; i++) arena_base[i] = 0;
        if (kv_base) for (uint32_t i = 0; i <= n; i++) kv_base[i] = 0;
        return PGS_OK;
    }

    LaunchScratch S(st);
    cudaEvent_t ev_a, ev_b;
    PGS_CUDA(S.event(ev_a));
    PGS_CUDA(S.event(ev_b));
    PGS_CUDA(S.upload(P.reqs, B.reqs.data(), n));
    PGS_CUDA(S.upload(P.blob, (const uint8_t *)B.blob.data(), B.blob.size()));
    PGS_CUDA(S.alloc(P.arena, P.arena_stride * n + 16));
    PGS_CUDA(S.alloc(P.kvs, sizeof(pgs_kv) * (size_t)kv_stride * n + 16));
    PGS_CUDA(S.alloc(P.resume, (size_t)P.resume_stride * n + 16));
    PGS_CUDA(S.alloc(P.results, sizeof(pgs_scan_result) * n));
    PGS_CUDA(S.alloc(P.error, 16));
    PGS_CUDA(cudaMemsetAsync(P.error, 0, 16, st));
    if (multi) {
        PGS_CUDA(S.upload(P.multi_runs, multi->packed.data(), multi->packed.size()));
        PGS_CUDA(S.upload(P.multi_begin, multi->begin.data(), multi->begin.size()));
        PGS_CUDA(S.upload(P.req_part, req_part, n));
    }
    if (B.need_crc) P.crc_table = (const unsigned long long *)e->d_crc;
    P.ticket = P.error + 1;
    // forward scans: lane-group merging iterators (read_kernels.cuh), unless the groups' key rows do not fit shared memory
    // (user keys of a few KB): then k_scan, which stages records instead of keeping one key row per run and group
    const ReadGeometry fwd = scan_fwd_geometry(P.rr.n, P.KS);
    const bool fwd_fits = fwd.dyn <= (uint32_t)e->max_smem_optin;
    if (!fwd_fits && multi) { set_error("scan: %u runs with keys of %u bytes do not fit shared memory", P.rr.n, P.KS); return PGS_NOT_SUPPORTED; }
    if (!B.any_reverse && fwd_fits) {
        fwd.apply(P);
        const scan_fwd_kernel_t kern = scan_fwd_kernel(fwd.G, multi != nullptr);
        int occ = 0;
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (int)kReadThreads, (size_t)fwd.dyn));
        const uint32_t per_cta = kReadThreads / fwd.G;
        const uint32_t grid = std::min<uint32_t>((n + per_cta - 1) / per_cta, (uint32_t)std::max(1, occ) * e->sm_count);
        PGS_CUDA(cudaEventRecord(ev_a, st));
        kern<<<grid, kReadThreads, fwd.dyn, st>>>(P);
        PGS_CUDA(cudaEventRecord(ev_b, st));
    } else {
        // ---- reverse scans (and forward ones with long keys): the block-staging kernel ---------------------------------
        uint64_t dyn = 0;
        PGS_CUDA(scan_launch_dyn(*e, runs, P.KS, n, dyn, &P.pool_bytes));
        if (!dyn) {
            set_error("scan: blocks too large for shared memory");
            return PGS_NOT_SUPPORTED;
        }
        int occ = 0; // resident CTAs per SM for this dynamic shared-memory size (registers count too)
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_scan, (int)kScanThreads, (size_t)dyn));
        uint32_t grid = std::min<uint32_t>(n, (uint32_t)std::max(1, occ) * e->sm_count);
        PGS_CUDA(cudaEventRecord(ev_a, st));
        k_scan<<<grid, kScanThreads, dyn, st>>>(P);
        PGS_CUDA(cudaEventRecord(ev_b, st));
    }
    e->launches++;
    uint32_t herr = 0;
    if (n == 1) {
        PGS_CUDA(cudaMemcpyAsync(results, P.results, sizeof(pgs_scan_result), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(&herr, P.error, 4, cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaStreamSynchronize(st));
        if (!herr) {
            if (results[0].arena_used > arena_cap || results[0].n_kvs > kv_cap) return PGS_INCOMPLETE;
            if (results[0].arena_used) PGS_CUDA(cudaMemcpyAsync(arena, P.arena, results[0].arena_used, cudaMemcpyDeviceToHost, st));
            if (results[0].n_kvs) PGS_CUDA(cudaMemcpyAsync(kvs, P.kvs, sizeof(pgs_kv) * results[0].n_kvs, cudaMemcpyDeviceToHost, st));
            if (results[0].iter_valid && resume && resume_stride) PGS_CUDA(cudaMemcpyAsync(resume, P.resume, results[0].resume_len, cudaMemcpyDeviceToHost, st));
            PGS_CUDA(cudaStreamSynchronize(st));
        }
        if (arena_base) { arena_base[0] = 0; arena_base[1] = results[0].arena_used; }
        if (kv_base) { kv_base[0] = 0; kv_base[1] = results[0].n_kvs; }
    } else {
        unsigned long long *d_abase = nullptr;
        uint32_t *d_kbase = nullptr;
        PGS_CUDA(S.alloc(d_abase, sizeof(unsigned long long) * (n + 1)));
        PGS_CUDA(S.alloc(d_kbase, sizeof(uint32_t) * (n + 1)));
        k_pack_offsets<<<1, 1024, 0, st>>>(P.results, n, d_abase, d_kbase);
        std::vector<unsigned long long> ab(n + 1);
        std::vector<uint32_t> kb(n + 1);
        PGS_CUDA(cudaMemcpyAsync(ab.data(), d_abase, sizeof(unsigned long long) * (n + 1), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(kb.data(), d_kbase, sizeof(uint32_t) * (n + 1), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(results, P.results, sizeof(pgs_scan_result) * n, cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(&herr, P.error, 4, cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaStreamSynchronize(st));
        e->launches++;
        if (!herr) {
            if (ab[n] > arena_cap || kb[n] > kv_cap) { set_error("scan_many: output arena too small"); return PGS_INCOMPLETE; }
            uint8_t *d_parena = nullptr;
            pgs_kv *d_pkvs = nullptr;
            PGS_CUDA(S.alloc(d_parena, ab[n] + 16));
            PGS_CUDA(S.alloc(d_pkvs, sizeof(pgs_kv) * ((size_t)kb[n] + 1)));
            k_pack_copy<<<std::min<uint32_t>(n, 8 * e->sm_count), 128, 0, st>>>(P.results, n, P.arena, P.arena_stride, P.kvs, kv_stride, d_abase,
                                                                              d_kbase, d_parena, d_pkvs);
            e->launches++;
            if (ab[n]) PGS_CUDA(cudaMemcpyAsync(arena, d_parena, ab[n], cudaMemcpyDeviceToHost, st));
            if (kb[n]) PGS_CUDA(cudaMemcpyAsync(kvs, d_pkvs, sizeof(pgs_kv) * kb[n], cudaMemcpyDeviceToHost, st));
            if (resume && resume_stride) PGS_CUDA(cudaMemcpyAsync(resume, P.resume, (size_t)P.resume_stride * n, cudaMemcpyDeviceToHost, st));
            PGS_CUDA(cudaStreamSynchronize(st));
        }
        if (arena_base) for (uint32_t i = 0; i <= n; i++) arena_base[i] = ab[i];
        if (kv_base) for (uint32_t i = 0; i <= n; i++) kv_base[i] = kb[i];
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    set_last_read_stats(ms, 0, 0);
    if (herr) {
        set_error("scan kernel failed with status %u", herr);
        // PGS_ABORTED = a request's output did not fit its arena / kv slice: the caller may retry with more room
        return herr == PGS_CORRUPTION ? PGS_CORRUPTION : (herr == PGS_NOT_SUPPORTED ? PGS_NOT_SUPPORTED : (herr == PGS_ABORTED ? PGS_ABORTED : PGS_IO_ERROR));
    }
    return PGS_OK;
}

// ---- hot-key capture of batched gets (hotkey_kernels.cuh) ------------------------------------------------------------------
Partition::~Partition()
{
    if (hk_dev_buckets) { cudaSetDevice(eng->device); cudaFree(hk_dev_buckets); }
}

int32_t hotkey_control(Partition &p, int32_t type, int32_t action, uint32_t now, std::string &text)
{
    if (action != HOTKEY_START && action != HOTKEY_STOP && action != HOTKEY_QUERY) { text = "invalid detect_action"; return HOTKEY_INVALID_PARAMETERS; }
    if (type != HOTKEY_READ && type != HOTKEY_WRITE) { text = "invalid hotkey_type"; return HOTKEY_INVALID_PARAMETERS; }
    if (type == HOTKEY_WRITE) return p.hk_write.control(action, now, text);
    std::unique_lock<std::shared_mutex> g(p.hk_dev_mu);
    if (action == HOTKEY_START && p.hk_read.state() == HOTKEY_STOPPED) { // the device counters start from zero
        const uint32_t nb = p.hk_read.config().buckets;
        cudaError_t e = cudaSetDevice(p.eng->device);
        if (e == cudaSuccess && p.hk_dev_buckets && p.hk_dev_n != nb) { cudaFree(p.hk_dev_buckets); p.hk_dev_buckets = nullptr; }
        if (e == cudaSuccess && !p.hk_dev_buckets) e = cudaMalloc((void **)&p.hk_dev_buckets, sizeof(unsigned long long) * nb);
        if (e == cudaSuccess) { p.hk_dev_n = nb; e = cudaMemset(p.hk_dev_buckets, 0, sizeof(unsigned long long) * nb); }
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { cuda_fail(e, "hotkey counters"); text = std::string("hotkey counters: ") + cudaGetErrorString(e); return HOTKEY_INVALID_STATE; }
    }
    return p.hk_read.control(action, now, text);
}

int32_t hotkey_analyse(Partition &p, uint32_t now)
{
    p.hk_write.analyse(now);
    std::unique_lock<std::shared_mutex> g(p.hk_dev_mu); // no capturing launch is in flight
    std::vector<uint64_t> dev;
    if (p.hk_dev_buckets && p.hk_read.state() == HOTKEY_COARSE) { // read and zero the counters with one small copy each way
        PGS_CUDA(cudaSetDevice(p.eng->device));
        dev.resize(p.hk_dev_n);
        PGS_CUDA(cudaMemcpy(dev.data(), p.hk_dev_buckets, sizeof(unsigned long long) * p.hk_dev_n, cudaMemcpyDeviceToHost));
        PGS_CUDA(cudaMemset(p.hk_dev_buckets, 0, sizeof(unsigned long long) * p.hk_dev_n));
        PGS_CUDA(cudaDeviceSynchronize());
    }
    p.hk_read.analyse(now, &dev);
    return PGS_OK;
}

// The READ collectors a get launch captures into: the distinct partitions of the call with an active collector, locked
// shared (hk_dev_mu) until the fine captures are handed over, and one slot descriptor per partition slot of the launch.
struct HotkeyCapture {
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    std::vector<HotkeySlotDev> slots;
    std::vector<Partition *> slot_part;
    uint32_t total_room = 0;
    bool any = false;
    uint32_t n_buckets = 0;

    void open(pgs_partition *const *parts, uint32_t n_parts)
    {
        bool active = false;
        for (uint32_t s = 0; s < n_parts; s++) active |= parts[s]->p.hk_read.active();
        if (!active) return; // no detection: nothing is locked, uploaded or launched
        std::vector<Partition *> locked;
        slots.assign(n_parts, HotkeySlotDev{nullptr, 0, 0, 0, 0});
        slot_part.assign(n_parts, nullptr);
        for (uint32_t s = 0; s < n_parts; s++) {
            Partition &pp = parts[s]->p;
            if (!pp.hk_read.active()) continue;
            if (std::find(locked.begin(), locked.end(), &pp) == locked.end()) { locks.emplace_back(pp.hk_dev_mu); locked.push_back(&pp); }
            const HotkeyCollector::Phase ph = pp.hk_read.device_phase();
            // every collector of one engine shares the bucket count of its options; a slot with another count is left out
            if (ph.state == HOTKEY_STOPPED || !pp.hk_dev_buckets || (n_buckets && pp.hk_dev_n != n_buckets)) continue;
            n_buckets = pp.hk_dev_n;
            HotkeySlotDev &d = slots[s];
            d.state = ph.state;
            if (ph.state == HOTKEY_COARSE) d.buckets = pp.hk_dev_buckets;
            else { d.target = ph.target; d.room = ph.room; d.idx_base = total_room; total_room += ph.room; }
            slot_part[s] = &pp;
            any = true;
        }
    }
    // keys the memtable-less shortcut answers without a launch (a partition with no runs): captured on the host
    void capture_on_host(const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part, uint32_t n)
    {
        for (uint32_t i = 0; any && i < n; i++)
            if (Partition *pp = slot_part[key_part ? key_part[i] : 0])
                pp->hk_read.capture_raw_key(std::string_view((const char *)keys + key_off[i], key_off[i + 1] - key_off[i]), 1);
    }
    // the fine captures of a finished launch: the first min(ticket, room) admitted keys of every fine slot
    void hand_over(const uint8_t *keys, const uint32_t *key_off, const std::vector<uint32_t> &tickets, const std::vector<uint32_t> &idx)
    {
        for (uint32_t s = 0; s < slots.size(); s++) {
            if (slots[s].state != HOTKEY_FINE) continue;
            const uint32_t m = std::min(tickets[s], slots[s].room);
            std::vector<std::string> hks;
            for (uint32_t j = 0; j < m; j++) {
                const uint32_t q = idx[slots[s].idx_base + j];
                const KeyParts k = split_key(keys + key_off[q], key_off[q + 1] - key_off[q]);
                hks.emplace_back((const char *)k.hk, k.hkl);
            }
            slot_part[s]->hk_read.add_fine_keys(hks);
        }
    }
};

} // namespace pgs

using namespace pgs;

// one get launch over the keys of one partition (parts[0], key_part null) or of several partitions of one engine
static int32_t get_batch_impl(pgs_partition *const *parts, uint32_t n_parts, const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part,
                              uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used,
                              bool capture = true)
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
    MultiRuns M;
    int32_t rc = key_part ? snapshot_multi(parts, n_parts, "get_batch_multi", M, P.rr, P.KS) : snapshot_runs(part, runs, P.rr, P.KS);
    if (rc != PGS_OK) return rc;
    for (uint32_t i = 0; key_part && i < n; i++)
        if (key_part[i] >= n_parts) { set_error("get_batch_multi: key %u names partition slot %u of %u", i, key_part[i], n_parts); return PGS_INVALID_ARGUMENT; }
    HotkeyCapture hk;
    if (capture) hk.open(parts, key_part ? n_parts : 1);
    if (key_part ? M.packed.empty() : P.rr.n == 0) {
        for (uint32_t i = 0; i < n; i++) { memset(&results[i], 0, sizeof results[i]); results[i].status = PGS_NOT_FOUND; }
        hk.capture_on_host(keys, key_off, key_part, n);
        return PGS_OK;
    }
    const ReadGeometry geo = get_geometry(P.KS);
    if (geo.dyn > (uint32_t)e->max_smem_optin) return PGS_NOT_SUPPORTED;
    geo.apply(P);
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->read_stream();
    const uint64_t key_bytes = key_off[n];
    LaunchScratch S(st);
    cudaEvent_t ev_a, ev_b;
    uint8_t *d_keys = nullptr;
    PGS_CUDA(S.event(ev_a));
    PGS_CUDA(S.event(ev_b));
    PGS_CUDA(S.alloc(d_keys, key_bytes + 16));
    PGS_CUDA(cudaMemcpyAsync(d_keys, keys, key_bytes, cudaMemcpyHostToDevice, st));
    PGS_CUDA(S.upload(P.key_off, key_off, n + 1));
    PGS_CUDA(S.alloc(P.results, sizeof(pgs_get_result) * n));
    PGS_CUDA(S.alloc(P.arena, arena_cap + 16));
    PGS_CUDA(S.alloc(P.arena_cursor, 32));
    PGS_CUDA(S.alloc(P.error, 16));
    PGS_CUDA(cudaMemsetAsync(P.arena_cursor, 0, 32, st));
    PGS_CUDA(cudaMemsetAsync(P.error, 0, 16, st));
    if (key_part) {
        PGS_CUDA(S.upload(P.multi_runs, M.packed.data(), M.packed.size()));
        PGS_CUDA(S.upload(P.multi_begin, M.begin.data(), M.begin.size()));
        PGS_CUDA(S.upload(P.key_part, key_part, n));
    }
    P.keys = d_keys; P.n = n; P.now = now; P.data_version = part.data_version;
    P.arena_cap = arena_cap; P.ticket = P.error + 1;
    int occ = 0;
    auto kern = key_part ? k_get<8, true> : k_get<8, false>;
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (int)kReadThreads, (size_t)geo.dyn));
    const uint32_t per_cta = kReadThreads / geo.G;
    const uint32_t grid = std::min<uint32_t>((n + per_cta - 1) / per_cta, (uint32_t)std::max(1, occ) * e->sm_count);
    PGS_CUDA(cudaEventRecord(ev_a, st));
    kern<<<grid, kReadThreads, geo.dyn, st>>>(P);
    PGS_CUDA(cudaEventRecord(ev_b, st));
    e->launches++;
    // hot-key capture (only while a slot's READ collector is active): its fine tickets and indices come back with the results
    std::vector<uint32_t> hk_tickets, hk_idx;
    if (hk.any) {
        HotkeyParams H{};
        H.keys = d_keys; H.key_off = P.key_off; H.key_part = key_part ? P.key_part : nullptr; H.n = n; H.n_buckets = hk.n_buckets;
        const uint32_t n_slots = (uint32_t)hk.slots.size();
        PGS_CUDA(S.upload(H.slots, hk.slots.data(), n_slots));
        PGS_CUDA(S.alloc(H.tickets, sizeof(uint32_t) * (n_slots + (size_t)hk.total_room)));
        PGS_CUDA(cudaMemsetAsync(H.tickets, 0, sizeof(uint32_t) * n_slots, st));
        H.idx = H.tickets + n_slots;
        const uint32_t hgrid = std::min<uint32_t>((n + kHotkeyThreads - 1) / kHotkeyThreads, 8u * e->sm_count);
        k_hotkey_capture<<<hgrid, kHotkeyThreads, 0, st>>>(H);
        e->launches++;
        hk_tickets.resize(n_slots + (size_t)hk.total_room);
        PGS_CUDA(cudaMemcpyAsync(hk_tickets.data(), H.tickets, sizeof(uint32_t) * hk_tickets.size(), cudaMemcpyDeviceToHost, st));
    }
    uint32_t herr = 0;
    unsigned long long cur3[3] = {0, 0, 0};
    PGS_CUDA(cudaMemcpyAsync(results, P.results, sizeof(pgs_get_result) * n, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(cur3, P.arena_cursor, 24, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(&herr, P.error, 4, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaStreamSynchronize(st));
    if (hk.any && hk.total_room) {
        hk_idx.assign(hk_tickets.begin() + hk.slots.size(), hk_tickets.end());
        hk_tickets.resize(hk.slots.size());
        hk.hand_over(keys, key_off, hk_tickets, hk_idx);
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    set_last_read_stats(ms, cur3[1], cur3[2]);
    const unsigned long long used = cur3[0];
    if (arena_used) *arena_used = used;
    if (!herr && used) {
        PGS_CUDA(cudaMemcpyAsync(arena, P.arena, std::min<unsigned long long>(used, arena_cap), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaStreamSynchronize(st));
    }
    if (herr) { set_error("get kernel failed with status %u", herr); return herr == PGS_CORRUPTION ? PGS_CORRUPTION : PGS_IO_ERROR; }
    return used > arena_cap ? PGS_INCOMPLETE : PGS_OK;
}

// pgs_get_batch, with the READ collector's capture switched on or off (handlers that capture with their own weights)
int32_t pgs::get_batch(pgs_partition *ph, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                       uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used, bool capture)
{
    if (!ph || (n && (!keys || !key_off || !results))) return PGS_INVALID_ARGUMENT;
    return get_batch_impl(&ph, 1, keys, key_off, nullptr, n, now, arena, arena_cap, results, arena_used, capture);
}

extern "C" int32_t pgs_get_batch(pgs_partition *ph,const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
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
