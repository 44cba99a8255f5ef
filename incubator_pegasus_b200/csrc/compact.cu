// compact.cu — host side of level compaction (pgs_compact): picks the input runs, allocates and launches the plan of
// compact_kernels.cuh (k_plan -> k_seg_bounds -> k_seg_layout -> k_walk -> k_seg_scan -> k_emit) on the engine stream, times it
// and installs the merged run.  Replaces DB::CompactRange / the background compaction job (src/server/pegasus_server_impl.cpp:3373-3394).
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "compact_kernels.cuh"
#include "engine.h"

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
    const uint32_t ops_len = compact_filter(P, fp);
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
