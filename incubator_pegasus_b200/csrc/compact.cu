// compact.cu — host side of level compaction (pgs_compact): picks the input runs, allocates and launches the plan of
// compact_kernels.cuh (k_plan -> k_seg_bounds -> k_seg_layout -> k_walk -> k_seg_scan -> k_emit) on the engine stream, times it
// and installs the merged run.  Replaces DB::CompactRange / the background compaction job (src/server/pegasus_server_impl.cpp:3373-3394).
// Also the host side of pgs_partition_split (split_kernels.cuh), which launches k_seg_scan and k_emit per child: the kernels of
// both live in this one translation unit.
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include <cstring>

#include "engine.h"
#include "split_kernels.cuh"

namespace pgs {
// the opt-in shared-memory maximum of the compaction kernels, once per device (a per-call cudaFuncSetAttribute would race)
int32_t compact_init_kernels(int max_smem)
{
    cudaFuncAttributes a;
    for (uint32_t G : kWalkGs) {
        PGS_CUDA(cudaFuncGetAttributes(&a, walk_kernel(G)));
        PGS_CUDA(cudaFuncSetAttribute(walk_kernel(G), cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes));
    }
    PGS_CUDA(cudaFuncGetAttributes(&a, k_emit));
    PGS_CUDA(cudaFuncSetAttribute(k_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes));
    for (uint32_t G : kWalkGs) {
        PGS_CUDA(cudaFuncGetAttributes(&a, walk_many_kernel(G)));
        PGS_CUDA(cudaFuncSetAttribute(walk_many_kernel(G), cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes));
    }
    PGS_CUDA(cudaFuncGetAttributes(&a, k_emit_many));
    PGS_CUDA(cudaFuncSetAttribute(k_emit_many, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes));
    return PGS_OK;
}
} // namespace pgs

using namespace pgs;

extern "C" int32_t pgs_compact(pgs_partition *ph, const uint64_t *run_ids, uint32_t k, int32_t out_level,
                               int32_t bottommost, const pgs_filter_params *fp, uint32_t now,
                               pgs_compact_result *out)
{
    return pgs_compact_ex(ph, run_ids, k, out_level, bottommost, fp, now, 0, out);
}

extern "C" int32_t pgs_compact_ex(pgs_partition *ph, const uint64_t *run_ids, uint32_t k, int32_t out_level,
                                  int32_t bottommost, const pgs_filter_params *fp, uint32_t now, uint32_t flags,
                                  pgs_compact_result *out)
{
    if (!ph || !run_ids || k == 0 || out_level < 0) return PGS_INVALID_ARGUMENT;
    Partition &part = ph->p;
    Engine *e = part.eng;
    pgs_compact_result res{};
    std::vector<std::shared_ptr<Run>> in;
    {
        std::lock_guard<std::mutex> g(part.mu);
        for (uint32_t i = 0; i < k; i++) {
            auto r = part.find(run_ids[i]);
            if (!r) { set_error("compact: unknown run %llu", (unsigned long long)run_ids[i]); return PGS_NOT_FOUND; }
            for (auto &x : in) if (x == r) return PGS_INVALID_ARGUMENT;
            in.push_back(r);
        }
        if (bottommost < 0) { // true iff every run outside the input set is newer than every input
            size_t first_in = part.runs.size();
            for (size_t i = 0; i < part.runs.size(); i++)
                if (std::find(in.begin(), in.end(), part.runs[i]) != in.end()) { first_in = i; break; }
            bottommost = 1;
            for (size_t i = first_in; i < part.runs.size(); i++)
                if (std::find(in.begin(), in.end(), part.runs[i]) == in.end()) bottommost = 0;
        }
    }
    if (k > kMaxRuns) { set_error("compact: %u runs > %u per merge", k, kMaxRuns); return PGS_NOT_SUPPORTED; }
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;

    MergeParams P{};
    P.k = k;
    CompactTotals T{};
    for (uint32_t i = 0; i < k; i++) {
        P.runs[i] = in[i]->dev();
        const pgs_run_info &fi = in[i]->info;
        T.add(fi, in[i]->n_bloom_entries);
        if (fi.n_blocks >= (1u << 28) || fi.data_bytes >= (1ull << 40)) return PGS_NOT_SUPPORTED;
    }
    if (T.max_ukey > kMaxUkeyLen) { set_error("compact: user key of %u bytes > %u", T.max_ukey, kMaxUkeyLen); return PGS_NOT_SUPPORTED; }
    P.block_size = e->cfg.block_size;
    P.restart_interval = e->cfg.restart_interval;
    P.bottommost = bottommost ? 1 : 0;
    P.now = now;
    P.data_version = part.data_version;
    uint32_t ops_len = 0;
    if (!compact_filter(P, fp, ops_len)) { set_error("compact: malformed ops table of %u bytes", fp->ops_len); return PGS_INVALID_ARGUMENT; }
    if (P.validate_hash) P.crc_table = (const unsigned long long *)e->d_crc;
    CompactGeometry geo{};
    uint32_t force_G = 0; // diagnostics: PGS_WALK_G = lanes per merge group (1, 2, 4, 8, 16)
    if (const char *ev = getenv("PGS_WALK_G")) { const int v = atoi(ev); if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) force_G = (uint32_t)v; }
    const uint32_t smem = compact_smem_budget((uint32_t)e->max_smem_optin);
    bool geo_ok = compact_geometry(P, T, smem, geo, force_G);
    if (geo_ok) { // second pass: the segment budget follows from how many groups the device runs at once
        int occ = 0;
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, walk_kernel(geo.G), (int)kWalkThreads, (size_t)geo.walk_dyn));
        const uint64_t groups = (uint64_t)std::max(1, occ) * e->sm_count * (kWalkThreads / geo.G);
        geo_ok = compact_geometry(P, T, smem, geo, geo.G, 0, groups);
    }
    if (!geo_ok) {
        set_error("compact: input too large for one merge launch (keys of %u bytes, %llu records)", T.max_ukey, (unsigned long long)T.n_rec);
        return PGS_NOT_SUPPORTED;
    }

    LaunchScratch S(st);
    auto outr = std::make_shared<Run>(e);
    outr->level = out_level;
    cudaError_t ce = cudaSuccess;
    compact_buffers(P, geo, T, *outr, [&](auto *&p, uint64_t n, int fill, bool out) {
        const size_t bytes = sizeof(*p) * n;
        if (ce != cudaSuccess) return;
        if ((void *)&p == (void *)&outr->d_data) ce = e->alloc_data(*outr, bytes); // from the spare list when one fits
        else ce = out ? cudaMallocAsync((void **)&p, bytes, st) : S.alloc(p, bytes); // ~Run frees the run's buffers
        if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, bytes, st);
    });
    PGS_CUDA(ce);
    MergeStats hs = merge_stats_init();
    PGS_CUDA(S.upload(P.stats, &hs, 1));
    if (ops_len) PGS_CUDA(S.upload(P.ops, fp->ops, ops_len));

    cudaEvent_t ev[4];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    int occ_w = 0, occ_e = 0;
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_w, walk_kernel(geo.G), (int)kWalkThreads, (size_t)geo.walk_dyn));
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_e, k_emit, (int)(geo.emit_warps * 32), (size_t)geo.emit_dyn));
    const uint32_t launches = compact_launch(P, geo, (uint64_t)std::max(1, occ_w) * e->sm_count, (uint64_t)std::max(1, occ_e) * e->sm_count,
                                             st, [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
    e->launches += launches;
    PGS_CUDA(ce);
    PGS_CUDA(cudaMemcpyAsync(&hs, P.stats, sizeof hs, cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return cuda_fail(se, "compaction kernels");
    float ms_total = 0, ms_merge = 0, ms_walk = 0, ms_emit = 0;
    cudaEventElapsedTime(&ms_total, ev[0], ev[3]);
    cudaEventElapsedTime(&ms_merge, ev[1], ev[3]);
    cudaEventElapsedTime(&ms_walk, ev[1], ev[2]);
    cudaEventElapsedTime(&ms_emit, ev[2], ev[3]);
    if (hs.error) {
        set_error("compaction kernel failed with status %u at segment %u of %u", hs.error, hs.error_seg, P.Q);
        return (int32_t)hs.error;
    }
    outr->n_bloom_entries = compact_result_stats(hs, T.in_block_bytes, res, outr->info);
    outr->info.level = out_level;
    res.n_tiles = P.Q; res.n_launches = launches;
    res.device_ms = ms_total; res.merge_kernel_ms = ms_merge;
    res.walk_ms = ms_walk; res.emit_ms = ms_emit;
    {
        std::lock_guard<std::mutex> g(part.mu);
        if (!(flags & PGS_COMPACT_KEEP_INPUTS))
            for (auto &r : in) part.runs.erase(std::find(part.runs.begin(), part.runs.end(), r));
        if (hs.tot_blocks > 0 && !(flags & PGS_COMPACT_DISCARD_OUTPUT)) {
            outr->id = e->next_run_id++;
            outr->info.run_id = outr->id;
            part.insert(outr);
            res.new_run_id = outr->id;
        }
    }
    if (out) *out = res;
    return PGS_OK;
}

// ---- pgs_compact_many --------------------------------------------------------------------------------------------------------
// The jobs of many partitions planned together (compact_many_geometry) and launched once (compact_launch_many).  The jobs'
// scratch shares one allocation; each merged run keeps buffers of its own, as pgs_compact's does.
extern "C" int32_t pgs_compact_many(const pgs_compact_job *jobs, uint32_t n, uint32_t now, uint32_t flags, pgs_compact_result *out)
{
    if (n == 0) return PGS_OK;
    if (!jobs) { set_error("compact_many: %u jobs and no job array", n); return PGS_INVALID_ARGUMENT; }
    if (n > kMaxCompactJobs) { set_error("compact_many: %u jobs > %u per call", n, kMaxCompactJobs); return PGS_NOT_SUPPORTED; }
    Engine *e = nullptr;
    std::vector<Partition *> parts(n);
    for (uint32_t i = 0; i < n; i++) {
        const pgs_compact_job &J = jobs[i];
        if (!J.part || !J.run_ids || J.k == 0 || J.out_level < 0) {
            set_error("compact_many: job %u: no partition, no runs or a negative output level", i);
            return PGS_INVALID_ARGUMENT;
        }
        parts[i] = &J.part->p;
        if (!e) e = parts[i]->eng;
        if (parts[i]->eng != e) { set_error("compact_many: job %u: its partition is on another engine than job 0's", i); return PGS_INVALID_ARGUMENT; }
    }
    std::vector<Partition *> order = parts; // the install locks them in this order
    std::sort(order.begin(), order.end());
    for (uint32_t i = 1; i < n; i++)
        if (order[i] == order[i - 1]) {
            const uint32_t j = (uint32_t)(std::find(parts.begin(), parts.end(), order[i]) - parts.begin());
            set_error("compact_many: job %u: its partition is in another job too", j);
            return PGS_INVALID_ARGUMENT;
        }

    // the inputs and the bottommost rule of every job, as pgs_compact_ex finds them
    std::vector<std::vector<std::shared_ptr<Run>>> in(n);
    std::vector<int32_t> bottom(n);
    for (uint32_t i = 0; i < n; i++) {
        const pgs_compact_job &J = jobs[i];
        Partition &part = *parts[i];
        std::lock_guard<std::mutex> g(part.mu);
        for (uint32_t x = 0; x < J.k; x++) {
            auto r = part.find(J.run_ids[x]);
            if (!r) { set_error("compact_many: job %u: unknown run %llu", i, (unsigned long long)J.run_ids[x]); return PGS_NOT_FOUND; }
            for (auto &y : in[i])
                if (y == r) { set_error("compact_many: job %u: run %llu given twice", i, (unsigned long long)J.run_ids[x]); return PGS_INVALID_ARGUMENT; }
            in[i].push_back(r);
        }
        bottom[i] = J.bottommost;
        if (bottom[i] < 0) {
            size_t first_in = part.runs.size();
            for (size_t x = 0; x < part.runs.size(); x++)
                if (std::find(in[i].begin(), in[i].end(), part.runs[x]) != in[i].end()) { first_in = x; break; }
            bottom[i] = 1;
            for (size_t x = first_in; x < part.runs.size(); x++)
                if (std::find(in[i].begin(), in[i].end(), part.runs[x]) == in[i].end()) bottom[i] = 0;
        }
    }
    std::vector<MergeParams> P(n);
    std::vector<CompactTotals> T(n);
    std::vector<uint32_t> ops_len(n);
    uint64_t ops_total = 0;
    uint32_t any_hash = 0;
    for (uint32_t i = 0; i < n; i++) {
        const pgs_compact_job &J = jobs[i];
        if (J.k > kMaxRuns) { set_error("compact_many: job %u: %u runs > %u per merge", i, J.k, kMaxRuns); return PGS_NOT_SUPPORTED; }
        MergeParams &p = P[i];
        p.k = J.k;
        for (uint32_t x = 0; x < J.k; x++) {
            p.runs[x] = in[i][x]->dev();
            const pgs_run_info &fi = in[i][x]->info;
            T[i].add(fi, in[i][x]->n_bloom_entries);
            if (fi.n_blocks >= (1u << 28) || fi.data_bytes >= (1ull << 40)) { set_error("compact_many: job %u: a run too large for a merge", i); return PGS_NOT_SUPPORTED; }
        }
        if (T[i].max_ukey > kMaxUkeyLen) { set_error("compact_many: job %u: user key of %u bytes > %u", i, T[i].max_ukey, kMaxUkeyLen); return PGS_NOT_SUPPORTED; }
        p.block_size = e->cfg.block_size;
        p.restart_interval = e->cfg.restart_interval;
        p.bottommost = bottom[i] ? 1 : 0;
        p.now = now;
        p.data_version = parts[i]->data_version;
        if (!compact_filter(p, J.fp, ops_len[i])) { set_error("compact_many: job %u: malformed ops table of %u bytes", i, J.fp->ops_len); return PGS_INVALID_ARGUMENT; }
        if (p.validate_hash) { p.crc_table = (const unsigned long long *)e->d_crc; any_hash = 1; }
        ops_total += (ops_len[i] + 15) & ~15u;
    }
    MergeJobs M{};
    CompactGeometry shared{};
    std::vector<CompactGeometry> geo(n);
    uint32_t force_G = 0; // diagnostics: PGS_WALK_G, as pgs_compact_ex
    if (const char *ev = getenv("PGS_WALK_G")) { const int v = atoi(ev); if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) force_G = (uint32_t)v; }
    const uint32_t smem = compact_smem_budget((uint32_t)e->max_smem_optin);
    bool geo_ok = compact_many_geometry(P.data(), T.data(), geo.data(), n, smem, M, shared, force_G);
    if (geo_ok) { // second pass: the segment weight follows from how many groups the device runs at once
        int occ = 0;
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, walk_many_kernel(shared.G), (int)kWalkThreads, (size_t)shared.walk_dyn));
        const uint64_t groups = (uint64_t)std::max(1, occ) * e->sm_count * (kWalkThreads / shared.G);
        geo_ok = compact_many_geometry(P.data(), T.data(), geo.data(), n, smem, M, shared, shared.G, 0, groups);
    }
    if (!geo_ok) {
        uint32_t widest = 0;
        for (auto &t : T) widest = std::max(widest, t.max_ukey);
        set_error("compact_many: %u jobs (user keys up to %u bytes) do not fit one merge launch; split the call", n, widest);
        return PGS_NOT_SUPPORTED;
    }

    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    LaunchScratch S(st);
    // the merged runs' buffers, one set per job; the scratch of every job is laid out in one allocation, grouped by fill byte
    struct Slice { void **p; uint64_t bytes; int fill; };
    std::vector<Slice> slices;
    std::vector<std::shared_ptr<Run>> outr(n);
    cudaError_t ce = cudaSuccess;
    for (uint32_t i = 0; i < n; i++) {
        outr[i] = std::make_shared<Run>(e);
        outr[i]->level = jobs[i].out_level;
        Run &r = *outr[i];
        compact_buffers(P[i], geo[i], T[i], r, [&](auto *&p, uint64_t cnt, int fill, bool is_out) {
            const size_t bytes = sizeof(*p) * cnt;
            if (!is_out) { slices.push_back(Slice{(void **)&p, bytes, fill}); return; }
            if (ce != cudaSuccess) return;
            if ((void *)&p == (void *)&r.d_data) ce = e->alloc_data(r, bytes);
            else ce = cudaMallocAsync((void **)&p, bytes, st); // ~Run frees the run's buffers
            if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, bytes, st);
        });
    }
    PGS_CUDA(ce);
    slices.push_back(Slice{(void **)&M.ticket, 2 * sizeof(uint32_t), 0});
    std::vector<int> fills;
    for (auto &s : slices)
        if (std::find(fills.begin(), fills.end(), s.fill) == fills.end()) fills.push_back(s.fill);
    std::vector<uint64_t> offs(slices.size());
    std::vector<std::pair<uint64_t, uint64_t>> fill_range(fills.size());
    uint64_t arena_bytes = 0;
    for (size_t f = 0; f < fills.size(); f++) {
        fill_range[f].first = arena_bytes;
        for (size_t x = 0; x < slices.size(); x++)
            if (slices[x].fill == fills[f]) { offs[x] = arena_bytes; arena_bytes += (std::max<uint64_t>(slices[x].bytes, 16) + 255) & ~255ull; }
        fill_range[f].second = arena_bytes;
    }
    uint8_t *arena = nullptr;
    PGS_CUDA(S.alloc(arena, arena_bytes));
    for (size_t f = 0; f < fills.size(); f++)
        if (fills[f] != kNoFill) PGS_CUDA(cudaMemsetAsync(arena + fill_range[f].first, fills[f], fill_range[f].second - fill_range[f].first, st));
    for (size_t x = 0; x < slices.size(); x++) *slices[x].p = arena + offs[x];

    // the job table: MergeParams[n] | MergeStats[n] | seg_base[n + 1] | blk_base[n + 1] | the ops tables, in one upload
    const uint64_t o_stats = sizeof(MergeParams) * (uint64_t)n, o_seg = (o_stats + sizeof(MergeStats) * (uint64_t)n + 15) & ~15ull;
    const uint64_t o_blk = (o_seg + 4ull * (n + 1) + 15) & ~15ull, o_ops = (o_blk + 4ull * (n + 1) + 15) & ~15ull;
    const uint64_t tab_bytes = o_ops + ops_total;
    uint8_t *tab = nullptr;
    PGS_CUDA(S.alloc(tab, tab_bytes));
    std::vector<uint8_t> h(tab_bytes, 0);
    uint64_t ops_at = o_ops;
    for (uint32_t i = 0; i < n; i++) {
        P[i].stats = (MergeStats *)(tab + o_stats) + i;
        if (ops_len[i]) {
            memcpy(h.data() + ops_at, jobs[i].fp->ops, ops_len[i]);
            P[i].ops = tab + ops_at;
            ops_at += (ops_len[i] + 15) & ~15u;
        }
        const MergeStats s0 = merge_stats_init();
        memcpy(h.data() + o_stats + sizeof(MergeStats) * i, &s0, sizeof s0);
    }
    memcpy(h.data(), P.data(), sizeof(MergeParams) * (size_t)n);
    compact_many_bases(P.data(), n, (uint32_t *)(h.data() + o_seg), (uint32_t *)(h.data() + o_blk));
    PGS_CUDA(cudaMemcpyAsync(tab, h.data(), tab_bytes, cudaMemcpyHostToDevice, st));
    M.job = (const MergeParams *)tab;
    M.seg_base = (const uint32_t *)(tab + o_seg);
    M.blk_base = (const uint32_t *)(tab + o_blk);
    M.validate_hash = any_hash;
    M.crc_table = (const unsigned long long *)e->d_crc;

    cudaEvent_t ev[4];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    int occ_w = 0, occ_e = 0;
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_w, walk_many_kernel(shared.G), (int)kWalkThreads, (size_t)shared.walk_dyn));
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_e, k_emit_many, (int)(shared.emit_warps * 32), (size_t)shared.emit_dyn));
    const uint32_t launches = compact_launch_many(M, shared, (uint64_t)std::max(1, occ_w) * e->sm_count, (uint64_t)std::max(1, occ_e) * e->sm_count,
                                                  st, [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
    e->launches += launches;
    PGS_CUDA(ce);
    std::vector<MergeStats> hs(n);
    PGS_CUDA(cudaMemcpyAsync(hs.data(), tab + o_stats, sizeof(MergeStats) * (size_t)n, cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return cuda_fail(se, "multi-job compaction kernels");
    for (uint32_t i = 0; i < n; i++)
        if (hs[i].error) {
            set_error("compact_many: job %u: compaction kernel failed with status %u at segment %u of %u", i, hs[i].error, hs[i].error_seg, P[i].Q);
            return (int32_t)hs[i].error;
        }
    float ms_total = 0, ms_merge = 0, ms_walk = 0, ms_emit = 0;
    cudaEventElapsedTime(&ms_total, ev[0], ev[3]);
    cudaEventElapsedTime(&ms_merge, ev[1], ev[3]);
    cudaEventElapsedTime(&ms_walk, ev[1], ev[2]);
    cudaEventElapsedTime(&ms_emit, ev[2], ev[3]);
    std::vector<pgs_compact_result> res(n);
    for (uint32_t i = 0; i < n; i++) {
        outr[i]->n_bloom_entries = compact_result_stats(hs[i], T[i].in_block_bytes, res[i], outr[i]->info);
        outr[i]->info.level = jobs[i].out_level;
        res[i].n_tiles = P[i].Q; res[i].n_launches = launches;
        res[i].device_ms = ms_total; res[i].merge_kernel_ms = ms_merge;
        res[i].walk_ms = ms_walk; res[i].emit_ms = ms_emit;
    }
    // all partitions or none: every lock is held (in address order) from the check that the inputs are still there to the install
    std::vector<std::unique_lock<std::mutex>> held;
    for (Partition *p : order) held.emplace_back(p->mu);
    for (uint32_t i = 0; i < n; i++)
        for (auto &r : in[i])
            if (std::find(parts[i]->runs.begin(), parts[i]->runs.end(), r) == parts[i]->runs.end()) {
                set_error("compact_many: job %u: run %llu left the partition during the merge", i, (unsigned long long)r->id);
                return PGS_ABORTED;
            }
    for (uint32_t i = 0; i < n; i++) {
        Partition &part = *parts[i];
        if (!(flags & PGS_COMPACT_KEEP_INPUTS))
            for (auto &r : in[i]) part.runs.erase(std::find(part.runs.begin(), part.runs.end(), r));
        if (hs[i].tot_blocks > 0 && !(flags & PGS_COMPACT_DISCARD_OUTPUT)) {
            outr[i]->id = e->next_run_id++;
            outr[i]->info.run_id = outr[i]->id;
            part.insert(outr[i]);
            res[i].new_run_id = outr[i]->id;
        }
    }
    if (out) memcpy(out, res.data(), sizeof(pgs_compact_result) * (size_t)n);
    return PGS_OK;
}

// ---- pgs_partition_split ------------------------------------------------------------------------------------------------------
// Plans and launches split_kernels.cuh once per parent run on the engine stream, and installs every child's runs together once
// all of them were built.  Replaces local_partition_split's per-record loop (src/shell/commands/local_partition_split.cpp:238-283)
// and the whole-checkpoint copy of the online split manager.

namespace pgs {
// the opt-in shared-memory maximum of the split walkers, once per device
int32_t split_init_kernels(int max_smem)
{
    cudaFuncAttributes a;
    for (uint32_t G : kSplitGs)
        for (bool w : {false, true}) {
            PGS_CUDA(cudaFuncGetAttributes(&a, split_kernel(G, w)));
            PGS_CUDA(cudaFuncSetAttribute(split_kernel(G, w), cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes));
            PGS_CUDA(cudaFuncGetAttributes(&a, split_many_kernel(G, w)));
            PGS_CUDA(cudaFuncSetAttribute(split_many_kernel(G, w), cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes));
        }
    return PGS_OK;
}

namespace {

// one parent run split into its children's runs (out[c], null where child c gets nothing or is not built)
int32_t split_run(Engine *e, const Run &in, const SplitParams &proto, std::vector<std::shared_ptr<Run>> &out, pgs_split_result &res)
{
    const uint32_t NC = proto.S;
    cudaStream_t st = e->stream;
    SplitParams SP = proto;
    SP.M.runs[0] = in.dev();
    CompactTotals T{};
    T.add(in.info, in.n_bloom_entries);
    if (in.info.n_blocks >= (1u << 28) || in.info.data_bytes >= (1ull << 40)) return PGS_NOT_SUPPORTED;
    const uint32_t smem = compact_smem_budget((uint32_t)e->max_smem_optin);
    SplitGeometry geo{};
    int32_t rc = split_plan(SP, T, smem, geo);
    int occ_w = 0;
    if (rc == PGS_OK) { // second pass: segments sized by the groups the device runs at once
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_w, split_kernel(geo.G, false), (int)kSplitThreads, (size_t)geo.walk_dyn));
        const uint64_t groups = (uint64_t)std::max(1, occ_w) * e->sm_count * (kSplitThreads / geo.G);
        rc = split_plan(SP, T, smem, geo, groups);
    }
    if (rc != PGS_OK) {
        set_error("partition_split: a run with user keys of %u bytes into %u children is not supported", T.max_ukey, NC);
        return rc;
    }
    const uint64_t walk_ctas = (uint64_t)std::max(1, occ_w) * e->sm_count;

    LaunchScratch S(st);
    cudaError_t ce = cudaSuccess;
    split_buffers(SP, scratch_buffers(S, ce));
    PGS_CUDA(ce);
    std::vector<MergeStats> hs(NC, merge_stats_init());
    PGS_CUDA(cudaMemcpyAsync(SP.stats, hs.data(), sizeof(MergeStats) * NC, cudaMemcpyHostToDevice, st));
    cudaEvent_t ev[5];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    res.n_launches += split_launch(SP, geo, nullptr, nullptr, 0, walk_ctas, 0, st, [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
    PGS_CUDA(ce);
    std::vector<unsigned long long> prefixes(NC);
    unsigned long long dropped = 0;
    PGS_CUDA(cudaMemcpyAsync(hs.data(), SP.stats, sizeof(MergeStats) * NC, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(prefixes.data(), SP.prefixes, 8 * NC, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(&dropped, SP.dropped, 8, cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return cuda_fail(se, "split counting pass");
    for (uint32_t c = 0; c < NC; c++)
        if (hs[c].error) { set_error("partition_split: counting pass failed with status %u (child %u)", hs[c].error, c); return (int32_t)hs[c].error; }

    // the children's outputs, sized by what the counting pass found
    std::vector<MergeParams> Pc;
    std::vector<CompactGeometry> gc;
    std::vector<uint32_t> which;
    out.assign(NC, nullptr);
    for (uint32_t c = 0; c < NC; c++) {
        if (!((SP.want >> c) & 1u) || hs[c].cnt[EV_OUT] == 0) continue;
        MergeParams P{};
        CompactGeometry g{};
        CompactTotals Tc{};
        if (!split_child(SP, hs[c], prefixes[c], smem, P, g, Tc)) { set_error("partition_split: child %u's run is too large", c); return PGS_NOT_SUPPORTED; }
        auto r = std::make_shared<Run>(e);
        r->level = in.level;
        compact_buffers(P, g, Tc, *r, [&](auto *&p, uint64_t n, int fill, bool is_out) {
            const size_t bytes = sizeof(*p) * n;
            if (!is_out || ce != cudaSuccess) return; // the scratch is the split's
            if ((void *)&p == (void *)&r->d_data) ce = e->alloc_data(*r, bytes);
            else ce = cudaMallocAsync((void **)&p, bytes, st); // ~Run frees the run's buffers
            if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, bytes, st);
        });
        PGS_CUDA(ce);
        split_child_scratch(SP, c, P);
        Pc.push_back(P);
        gc.push_back(g);
        which.push_back(c);
        out[c] = r;
    }
    int occ_e = 1;
    if (!gc.empty())
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_e, k_emit, (int)(gc[0].emit_warps * 32), (size_t)gc[0].emit_dyn));
    res.n_launches += split_launch(SP, geo, Pc.data(), gc.data(), (uint32_t)Pc.size(), walk_ctas, (uint64_t)std::max(1, occ_e) * e->sm_count, st,
                                   [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[2 + i], st); });
    PGS_CUDA(ce);
    PGS_CUDA(cudaMemcpyAsync(hs.data(), SP.stats, sizeof(MergeStats) * NC, cudaMemcpyDeviceToHost, st));
    se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return cuda_fail(se, "split writing pass");
    for (uint32_t c = 0; c < NC; c++)
        if (hs[c].error) { set_error("partition_split: writing pass failed with status %u at segment %u (child %u)", hs[c].error, hs[c].error_seg, c); return (int32_t)hs[c].error; }
    float ms_count = 0, ms_walk = 0, ms_emit = 0;
    cudaEventElapsedTime(&ms_count, ev[0], ev[1]);
    cudaEventElapsedTime(&ms_walk, ev[2], ev[4]);
    cudaEventElapsedTime(&ms_emit, ev[4], ev[3]);
    res.count_ms += ms_count; res.walk_ms += ms_walk; res.emit_ms += ms_emit;
    for (uint32_t c : which) {
        Run &r = *out[c];
        pgs_compact_result cr{};
        r.n_bloom_entries = compact_result_stats(hs[c], 0, cr, r.info);
        r.info.level = in.level;
    }
    res.in_records += in.info.n_records;
    res.in_bytes += in.info.raw_key_bytes + in.info.raw_value_bytes;
    res.dropped_empty += dropped;
    return PGS_OK;
}

} // namespace

namespace {
// pgs_partition_split's argument checks: the counts, src's index, and every destination (want = bit i for a built child i)
int32_t split_dests(pgs_partition *src, uint32_t src_count, uint32_t dst_count, pgs_partition *const *dst, uint32_t n_dst, uint32_t &want)
{
    if (!src || !dst || src_count == 0 || dst_count <= src_count || dst_count % src_count) {
        set_error("partition_split: dst_count %u is not src_count %u times a power of two", dst_count, src_count);
        return PGS_INVALID_ARGUMENT;
    }
    const uint32_t NC = dst_count / src_count;
    Partition &part = src->p;
    Engine *e = part.eng;
    if ((NC & (NC - 1)) || n_dst != NC || part.pidx < 0 || (uint32_t)part.pidx >= src_count) {
        set_error("partition_split: %u destinations for %u -> %u partitions of index %d", n_dst, src_count, dst_count, part.pidx);
        return PGS_INVALID_ARGUMENT;
    }
    want = 0;
    for (uint32_t i = 0; i < NC; i++) {
        if (!dst[i]) continue;
        Partition &c = dst[i]->p;
        bool empty;
        {
            std::lock_guard<std::mutex> g(c.mu);
            empty = c.runs.empty();
        }
        // the children may belong to another app (the offline split writes a new table); their index is the parent's + i * src_count
        if (dst[i] == src || c.eng != e || !empty || (int64_t)c.pidx != (int64_t)part.pidx + (int64_t)i * src_count) {
            set_error("partition_split: destination %u is not an empty partition of index %lld on the source's engine", i,
                      (long long)part.pidx + (long long)i * src_count);
            return PGS_INVALID_ARGUMENT;
        }
        for (uint32_t j = 0; j < i; j++)
            if (dst[j] == dst[i]) { set_error("partition_split: destination %u given twice", i); return PGS_INVALID_ARGUMENT; }
        if (c.data_version != part.data_version) {
            set_error("partition_split: destination data_version %u != %u", c.data_version, part.data_version);
            return PGS_NOT_SUPPORTED;
        }
        want |= 1u << (i & 31);
    }
    if (NC > kSplitMaxChildren) { set_error("partition_split: %u children > %u", NC, kSplitMaxChildren); return PGS_NOT_SUPPORTED; }
    return PGS_OK;
}
} // namespace

// pgs_partition_split over the runs `snap` of src (nullptr: its current runs); pgs_rrdb_split passes the snapshot it took
// under the replica's writer lock
int32_t partition_split(pgs_partition *src, const std::vector<std::shared_ptr<Run>> *snap, uint32_t src_count, uint32_t dst_count,
                        pgs_partition *const *dst, uint32_t n_dst, pgs_split_result *out)
{
    uint32_t want = 0;
    if (const int32_t rc = split_dests(src, src_count, dst_count, dst, n_dst, want)) return rc;
    const uint32_t NC = dst_count / src_count;
    Partition &part = src->p;
    Engine *e = part.eng;
    std::vector<std::shared_ptr<Run>> runs;
    if (snap) runs = *snap;
    else {
        std::lock_guard<std::mutex> g(part.mu);
        runs = part.runs;
    }
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    SplitParams proto{};
    proto.M.block_size = e->cfg.block_size;
    proto.M.restart_interval = e->cfg.restart_interval;
    proto.M.data_version = part.data_version;
    proto.M.crc_table = (const unsigned long long *)e->d_crc;
    proto.S = NC;
    proto.src_count = src_count;
    proto.dst_count = dst_count;
    proto.want = want;

    pgs_split_result res{};
    LaunchScratch S(st);
    cudaEvent_t t0, t1;
    PGS_CUDA(S.event(t0));
    PGS_CUDA(S.event(t1));
    PGS_CUDA(cudaEventRecord(t0, st));
    std::vector<std::vector<std::shared_ptr<Run>>> built(NC); // the children's runs in the parent's order
    for (const auto &r : runs) {
        if (r->info.n_records == 0 || r->info.n_blocks == 0) continue;
        std::vector<std::shared_ptr<Run>> parts;
        if (const int32_t rc = split_run(e, *r, proto, parts, res)) return rc; // what was built so far is dropped
        for (uint32_t c = 0; c < NC; c++)
            if (parts[c]) built[c].push_back(parts[c]);
    }
    PGS_CUDA(cudaEventRecord(t1, st));
    PGS_CUDA(cudaEventSynchronize(t1));
    cudaEventElapsedTime(&res.device_ms, t0, t1);
    res.kernel_ms = res.count_ms + res.walk_ms + res.emit_ms;
    // all children, or none: every child's lock is held (in address order) from the check to the install
    std::vector<Partition *> kids;
    for (uint32_t c = 0; c < NC; c++)
        if (dst[c]) kids.push_back(&dst[c]->p);
    std::sort(kids.begin(), kids.end());
    std::vector<std::unique_lock<std::mutex>> held;
    for (Partition *k : kids) held.emplace_back(k->mu);
    for (Partition *k : kids)
        if (!k->runs.empty()) { set_error("partition_split: destination %d took runs during the split", k->pidx); return PGS_ABORTED; }
    for (uint32_t c = 0; c < NC; c++) {
        if (!dst[c]) continue;
        pgs_split_child_result &cr = res.child[c];
        for (auto &r : built[c]) {
            r->id = e->next_run_id++;
            r->info.run_id = r->id;
            cr.records += r->info.n_records;
            cr.tombstones += r->info.n_tombstones;
            cr.raw_bytes += r->info.raw_key_bytes + r->info.raw_value_bytes;
            cr.block_bytes += r->info.data_bytes;
            cr.runs++;
        }
        dst[c]->p.runs = built[c];
    }
    e->launches += res.n_launches;
    if (out) *out = res;
    return PGS_OK;
}

// ---- pgs_partition_split_many -------------------------------------------------------------------------------------------------
// Every run of every parent planned together (split_many_plan) and launched once per phase (split_many_launch).  The parent
// runs' scratch shares one allocation; each child run keeps buffers of its own, as pgs_partition_split's do.
int32_t partition_split_many(const pgs_split_job *jobs, uint32_t n, uint32_t src_count, uint32_t dst_count,
                             const std::vector<std::shared_ptr<Run>> *snaps, pgs_split_result *out)
{
    if (n == 0) return PGS_OK;
    if (!jobs) { set_error("partition_split_many: %u jobs and no job array", n); return PGS_INVALID_ARGUMENT; }
    if (n > PGS_SPLIT_MANY_MAX_JOBS) { set_error("partition_split_many: %u jobs > %u per call", n, PGS_SPLIT_MANY_MAX_JOBS); return PGS_NOT_SUPPORTED; }
    const uint32_t n_dst = src_count ? dst_count / src_count : 0;
    std::vector<uint32_t> want(n);
    Engine *e = nullptr;
    for (uint32_t i = 0; i < n; i++) {
        if (const int32_t rc = split_dests(jobs[i].src, src_count, dst_count, jobs[i].dst, n_dst, want[i])) {
            const std::string why = pgs_last_error();
            set_error("partition_split_many: job %u: %s", i, why.c_str());
            return rc;
        }
        if (!e) e = jobs[i].src->p.eng;
        if (jobs[i].src->p.eng != e) { set_error("partition_split_many: job %u: its parent is on another engine than job 0's", i); return PGS_INVALID_ARGUMENT; }
    }
    const uint32_t NC = n_dst;
    // every partition in one job only: a parent is no other job's parent or child, a child no other job's child
    std::vector<std::pair<Partition *, uint32_t>> seen;
    for (uint32_t i = 0; i < n; i++) {
        seen.emplace_back(&jobs[i].src->p, i);
        for (uint32_t c = 0; c < NC; c++)
            if (jobs[i].dst[c]) seen.emplace_back(&jobs[i].dst[c]->p, i);
    }
    std::sort(seen.begin(), seen.end());
    for (size_t x = 1; x < seen.size(); x++)
        if (seen[x].first == seen[x - 1].first) {
            set_error("partition_split_many: job %u: a partition of job %u is in job %u too", std::max(seen[x].second, seen[x - 1].second),
                      std::min(seen[x].second, seen[x - 1].second), std::max(seen[x].second, seen[x - 1].second));
            return PGS_INVALID_ARGUMENT;
        }

    // the parent runs, job by job in each parent's order; run x belongs to job run_job[x]
    std::vector<std::shared_ptr<Run>> in;
    std::vector<uint32_t> run_job;
    uint64_t child_runs = 0, emit_segments = 0;
    for (uint32_t i = 0; i < n; i++) {
        std::vector<std::shared_ptr<Run>> runs;
        if (snaps) runs = snaps[i];
        else {
            std::lock_guard<std::mutex> g(jobs[i].src->p.mu);
            runs = jobs[i].src->p.runs;
        }
        for (auto &r : runs) {
            if (r->info.n_records == 0 || r->info.n_blocks == 0) continue;
            if (r->info.n_blocks >= (1u << 28) || r->info.data_bytes >= (1ull << 40)) {
                set_error("partition_split_many: job %u: run %llu is too large for a split", i, (unsigned long long)r->id);
                return PGS_NOT_SUPPORTED;
            }
            in.push_back(r);
            run_job.push_back(i);
            child_runs += __builtin_popcount(want[i]);
        }
    }
    if (child_runs > kMaxCompactJobs) {
        set_error("partition_split_many: %llu child runs > %u per call; split the call", (unsigned long long)child_runs, kMaxCompactJobs);
        return PGS_NOT_SUPPORTED;
    }
    const uint32_t nr = (uint32_t)in.size();
    std::vector<SplitParams> SP(nr);
    std::vector<CompactTotals> T(nr);
    for (uint32_t x = 0; x < nr; x++) {
        SplitParams &s = SP[x];
        s.M.runs[0] = in[x]->dev();
        s.M.block_size = e->cfg.block_size;
        s.M.restart_interval = e->cfg.restart_interval;
        s.M.data_version = jobs[run_job[x]].src->p.data_version;
        s.M.crc_table = (const unsigned long long *)e->d_crc;
        s.S = NC;
        s.src_count = src_count;
        s.dst_count = dst_count;
        s.want = want[run_job[x]];
        T[x].add(in[x]->info, in[x]->n_bloom_entries);
    }
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    const uint32_t smem = compact_smem_budget((uint32_t)e->max_smem_optin);
    SplitJobs J{};
    MergeJobs M{};
    SplitGeometry geo{};
    int occ_w = 0;
    if (nr) {
        int32_t rc = split_many_plan(SP.data(), T.data(), nr, smem, J, M, geo);
        if (rc == PGS_OK) { // second pass: segments sized by the groups the device runs at once
            PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_w, split_many_kernel(geo.G, false), (int)kSplitThreads, (size_t)geo.walk_dyn));
            const uint64_t groups = (uint64_t)std::max(1, occ_w) * e->sm_count * (kSplitThreads / geo.G);
            rc = split_many_plan(SP.data(), T.data(), nr, smem, J, M, geo, groups);
        }
        for (uint32_t x = 0; x < nr && rc == PGS_OK; x++) emit_segments += (uint64_t)SP[x].M.Q * __builtin_popcount(SP[x].want);
        if (rc == PGS_OK && emit_segments > 0x7FFFFFF0ull) rc = PGS_NOT_SUPPORTED;
        if (rc != PGS_OK) {
            uint32_t widest = 0;
            for (auto &t : T) widest = std::max(widest, t.max_ukey);
            set_error("partition_split_many: %u parent runs (user keys up to %u bytes) into %u children do not fit one launch; split the call", nr, widest, NC);
            return rc;
        }
    }

    pgs_split_result all{}; // the call's timings and launches
    LaunchScratch S(st);
    cudaEvent_t t0, t1, ev[5];
    PGS_CUDA(S.event(t0));
    PGS_CUDA(S.event(t1));
    for (auto &x : ev) PGS_CUDA(S.event(x));
    PGS_CUDA(cudaEventRecord(t0, st));
    std::vector<MergeStats> hs((size_t)nr * NC, merge_stats_init());
    std::vector<unsigned long long> prefixes((size_t)nr * NC), dropped(nr);
    std::vector<std::vector<std::shared_ptr<Run>>> outs(nr, std::vector<std::shared_ptr<Run>>(NC));
    cudaError_t ce = cudaSuccess;
    if (nr) {
        // the scratch in one allocation grouped by fill byte: one pass of split_many_buffers sizes it, a second hands it out
        std::vector<std::pair<uint64_t, int>> sl;
        split_many_buffers(SP.data(), nr, J, [&](auto *&p, uint64_t cnt, int fill, bool) { sl.emplace_back(sizeof(*p) * cnt, fill); p = nullptr; });
        std::vector<int> fills;
        for (auto &s : sl)
            if (std::find(fills.begin(), fills.end(), s.second) == fills.end()) fills.push_back(s.second);
        std::vector<uint64_t> offs(sl.size());
        std::vector<std::pair<uint64_t, uint64_t>> fill_range(fills.size());
        uint64_t arena_bytes = 0;
        for (size_t f = 0; f < fills.size(); f++) {
            fill_range[f].first = arena_bytes;
            for (size_t x = 0; x < sl.size(); x++)
                if (sl[x].second == fills[f]) { offs[x] = arena_bytes; arena_bytes += (std::max<uint64_t>(sl[x].first, 16) + 255) & ~255ull; }
            fill_range[f].second = arena_bytes;
        }
        uint8_t *arena = nullptr;
        PGS_CUDA(S.alloc(arena, arena_bytes));
        for (size_t f = 0; f < fills.size(); f++)
            if (fills[f] != kNoFill) PGS_CUDA(cudaMemsetAsync(arena + fill_range[f].first, fills[f], fill_range[f].second - fill_range[f].first, st));
        size_t at = 0;
        split_many_buffers(SP.data(), nr, J, [&](auto *&p, uint64_t, int, bool) { *(void **)&p = arena + offs[at++]; });
        PGS_CUDA(cudaMemcpyAsync(J.stats, hs.data(), sizeof(MergeStats) * hs.size(), cudaMemcpyHostToDevice, st));

        // the job tables: MergeParams[nr] (the planner's) | SplitParams[nr] | seg_base[nr + 1] | blk_base[nr + 1], in one upload
        std::vector<MergeParams> MP(nr);
        for (uint32_t x = 0; x < nr; x++) MP[x] = SP[x].M;
        const uint64_t o_split = (sizeof(MergeParams) * (uint64_t)nr + 15) & ~15ull;
        const uint64_t o_seg = (o_split + sizeof(SplitParams) * (uint64_t)nr + 15) & ~15ull, o_blk = (o_seg + 4ull * (nr + 1) + 15) & ~15ull;
        const uint64_t tab_bytes = o_blk + 4ull * (nr + 1);
        std::vector<uint8_t> h(tab_bytes, 0);
        memcpy(h.data(), MP.data(), sizeof(MergeParams) * (size_t)nr);
        memcpy(h.data() + o_split, SP.data(), sizeof(SplitParams) * (size_t)nr);
        compact_many_bases(MP.data(), nr, (uint32_t *)(h.data() + o_seg), (uint32_t *)(h.data() + o_blk));
        uint8_t *tab = nullptr;
        PGS_CUDA(S.upload(tab, h.data(), tab_bytes));
        M.job = (const MergeParams *)tab;
        M.seg_base = J.seg_base = (const uint32_t *)(tab + o_seg);
        M.blk_base = (const uint32_t *)(tab + o_blk);
        J.job = (const SplitParams *)(tab + o_split);
        J.crc_table = (const unsigned long long *)e->d_crc;

        // counting phase, then one read-back of every (job, child) counter, prefix count and dropped count
        const uint64_t walk_ctas = (uint64_t)std::max(1, occ_w) * e->sm_count;
        all.n_launches += split_many_launch(J, M, geo, nullptr, CompactGeometry{}, walk_ctas, 0, st,
                                            [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
        PGS_CUDA(ce);
        PGS_CUDA(cudaMemcpyAsync(hs.data(), J.stats, sizeof(MergeStats) * hs.size(), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(prefixes.data(), J.prefixes, 8 * prefixes.size(), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(dropped.data(), J.dropped, 8 * dropped.size(), cudaMemcpyDeviceToHost, st));
        cudaError_t se = cudaStreamSynchronize(st);
        if (se != cudaSuccess) return cuda_fail(se, "multi-job split counting pass");
        for (size_t y = 0; y < hs.size(); y++)
            if (hs[y].error) {
                set_error("partition_split_many: job %u: counting pass failed with status %u (child %u)", run_job[y / NC], hs[y].error, (uint32_t)(y % NC));
                return (int32_t)hs[y].error;
            }

        // the children's outputs, sized by what the counting pass found; every (parent run, built child) is a job of k_emit_many
        std::vector<MergeParams> Pc;
        std::vector<uint32_t> emit_base(1, 0);
        CompactGeometry shape{};
        for (uint32_t x = 0; x < nr; x++)
            for (uint32_t c = 0; c < NC; c++) {
                const size_t y = (size_t)x * NC + c;
                if (!((SP[x].want >> c) & 1u) || hs[y].cnt[EV_OUT] == 0) continue;
                MergeParams P{};
                CompactGeometry g{};
                CompactTotals Tc{};
                if (!split_many_child(SP[x], c, hs[y], prefixes[y], smem, P, g, Tc, Pc.empty() ? nullptr : &Pc[0], &shape)) {
                    set_error("partition_split_many: job %u: child %u's run is too large, or not of the launch's shape", run_job[x], c);
                    return PGS_NOT_SUPPORTED;
                }
                auto r = std::make_shared<Run>(e);
                r->level = in[x]->level;
                compact_buffers(P, g, Tc, *r, [&](auto *&p, uint64_t cnt, int fill, bool is_out) {
                    const size_t bytes = sizeof(*p) * cnt;
                    if (!is_out || ce != cudaSuccess) return; // the scratch is the split's
                    if ((void *)&p == (void *)&r->d_data) ce = e->alloc_data(*r, bytes);
                    else ce = cudaMallocAsync((void **)&p, bytes, st); // ~Run frees the run's buffers
                    if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, bytes, st);
                });
                PGS_CUDA(ce);
                if (Pc.empty()) shape = g;
                Pc.push_back(P);
                emit_base.push_back(emit_base.back() + P.Q);
                outs[x][c] = r;
            }
        if (!Pc.empty()) { // writing phase
            const uint32_t nc = (uint32_t)Pc.size();
            const uint64_t o_base = (sizeof(MergeParams) * (uint64_t)nc + 15) & ~15ull;
            std::vector<uint8_t> hc(o_base + 4ull * (nc + 1), 0);
            memcpy(hc.data(), Pc.data(), sizeof(MergeParams) * (size_t)nc);
            memcpy(hc.data() + o_base, emit_base.data(), 4ull * (nc + 1));
            uint8_t *ctab = nullptr;
            PGS_CUDA(S.upload(ctab, hc.data(), hc.size()));
            MergeJobs E{};
            E.job = (const MergeParams *)ctab;
            E.seg_base = (const uint32_t *)(ctab + o_base);
            E.n = nc;
            E.Q = emit_base.back();
            E.ticket = J.ticket + 2;
            int occ_e = 0;
            PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_e, k_emit_many, (int)(shape.emit_warps * 32), (size_t)shape.emit_dyn));
            all.n_launches += split_many_launch(J, M, geo, &E, shape, walk_ctas, (uint64_t)std::max(1, occ_e) * e->sm_count, st,
                                                [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[2 + i], st); });
            PGS_CUDA(ce);
            PGS_CUDA(cudaMemcpyAsync(hs.data(), J.stats, sizeof(MergeStats) * hs.size(), cudaMemcpyDeviceToHost, st));
            se = cudaStreamSynchronize(st);
            if (se != cudaSuccess) return cuda_fail(se, "multi-job split writing pass");
            for (size_t y = 0; y < hs.size(); y++)
                if (hs[y].error) {
                    set_error("partition_split_many: job %u: writing pass failed with status %u at segment %u (child %u)", run_job[y / NC], hs[y].error,
                              hs[y].error_seg, (uint32_t)(y % NC));
                    return (int32_t)hs[y].error;
                }
            float ms_walk = 0, ms_emit = 0;
            cudaEventElapsedTime(&ms_walk, ev[2], ev[4]);
            cudaEventElapsedTime(&ms_emit, ev[4], ev[3]);
            all.walk_ms = ms_walk;
            all.emit_ms = ms_emit;
        }
        cudaEventElapsedTime(&all.count_ms, ev[0], ev[1]);
    }
    PGS_CUDA(cudaEventRecord(t1, st));
    PGS_CUDA(cudaEventSynchronize(t1));
    cudaEventElapsedTime(&all.device_ms, t0, t1);
    all.kernel_ms = all.count_ms + all.walk_ms + all.emit_ms;

    std::vector<pgs_split_result> res(n, all);
    for (uint32_t x = 0; x < nr; x++) {
        pgs_split_result &r = res[run_job[x]];
        r.in_records += in[x]->info.n_records;
        r.in_bytes += in[x]->info.raw_key_bytes + in[x]->info.raw_value_bytes;
        r.dropped_empty += dropped[x];
        for (uint32_t c = 0; c < NC; c++)
            if (outs[x][c]) {
                Run &o = *outs[x][c];
                pgs_compact_result cr{};
                o.n_bloom_entries = compact_result_stats(hs[(size_t)x * NC + c], 0, cr, o.info);
                o.info.level = in[x]->level;
            }
    }
    // all children of all jobs, or none: every child's lock is held (in address order) from the check to the last install
    std::vector<Partition *> kids;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++)
            if (jobs[i].dst[c]) kids.push_back(&jobs[i].dst[c]->p);
    std::sort(kids.begin(), kids.end());
    std::vector<std::unique_lock<std::mutex>> held;
    for (Partition *k : kids) held.emplace_back(k->mu);
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++)
            if (jobs[i].dst[c] && !jobs[i].dst[c]->p.runs.empty()) {
                set_error("partition_split_many: job %u: destination %u took runs during the split", i, c);
                return PGS_ABORTED;
            }
    std::vector<std::vector<std::shared_ptr<Run>>> built((size_t)n * NC); // job i's child c at i * NC + c, in the parent's run order
    for (uint32_t x = 0; x < nr; x++)
        for (uint32_t c = 0; c < NC; c++)
            if (outs[x][c]) built[(size_t)run_job[x] * NC + c].push_back(outs[x][c]);
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++) {
            if (!jobs[i].dst[c]) continue;
            pgs_split_child_result &cr = res[i].child[c];
            auto &b = built[(size_t)i * NC + c];
            for (auto &r : b) {
                r->id = e->next_run_id++;
                r->info.run_id = r->id;
                cr.records += r->info.n_records;
                cr.tombstones += r->info.n_tombstones;
                cr.raw_bytes += r->info.raw_key_bytes + r->info.raw_value_bytes;
                cr.block_bytes += r->info.data_bytes;
                cr.runs++;
            }
            jobs[i].dst[c]->p.runs = b;
        }
    e->launches += all.n_launches;
    if (out) memcpy(out, res.data(), sizeof(pgs_split_result) * (size_t)n);
    return PGS_OK;
}
} // namespace pgs

using namespace pgs;

extern "C" int32_t pgs_partition_split(pgs_partition *src, uint32_t src_count, uint32_t dst_count, pgs_partition *const *dst, uint32_t n_dst,
                                       pgs_split_result *out)
{
    return partition_split(src, nullptr, src_count, dst_count, dst, n_dst, out);
}

extern "C" int32_t pgs_partition_split_many(const pgs_split_job *jobs, uint32_t n, uint32_t src_count, uint32_t dst_count, pgs_split_result *out)
{
    return partition_split_many(jobs, n, src_count, dst_count, nullptr, out);
}
