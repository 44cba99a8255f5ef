// compact.cu — host side of level compaction (pgs_compact): sizes the scratch, launches
// k_plan -> k_seg_bounds -> k_seg_layout -> k_walk -> k_seg_scan -> k_emit (compact_kernels.cuh) on the engine stream and installs the
// merged run.  Replaces DB::CompactRange / the background compaction job (src/server/pegasus_server_impl.cpp:3373-3394).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

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
    std::vector<uint8_t> ops_host;
    if (fp) {
        P.enabled = fp->enabled;
        P.validate_hash = fp->validate_hash;
        P.default_ttl = fp->default_ttl;
        P.pidx = fp->pidx;
        P.partition_version = fp->partition_version;
        if (fp->ops && fp->ops_len >= 4) {
            memcpy(&P.n_ops, fp->ops, 4);
            ops_host.assign(fp->ops, fp->ops + fp->ops_len);
        }
    }
    CompactGeometry geo{};
    uint32_t force_G = 0; // diagnostics: PGS_WALK_G = lanes per merge group (1, 2, 4, 8, 16)
    if (const char *ev = getenv("PGS_WALK_G")) { const int v = atoi(ev); if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) force_G = (uint32_t)v; }
    bool geo_ok = compact_geometry(P, T, (uint32_t)e->max_smem_optin - 1024, geo, force_G);
    if (geo_ok) { // second pass: the segment budget follows from how many groups the device runs at once
        int occ = 0;
        PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, walk_kernel(geo.G), (int)kWalkThreads, (size_t)geo.walk_dyn));
        const uint64_t groups = (uint64_t)std::max(1, occ) * e->sm_count * (kWalkThreads / geo.G);
        geo_ok = compact_geometry(P, T, (uint32_t)e->max_smem_optin - 1024, geo, geo.G, 0, groups);
    }
    if (!geo_ok) {
        set_error("compact: input too large for one merge launch (keys of %u bytes, %llu records)", T.max_ukey, (unsigned long long)T.n_rec);
        return PGS_NOT_SUPPORTED;
    }
    const uint64_t Q = P.Q;

    auto outr = std::make_shared<Run>();
    outr->level = out_level;
    outr->data_cap = geo.out_cap + 256;
    LaunchScratch S(st);
    outr->pool_stream = st;
    outr->eng = e;
    { uint64_t cap = 0; outr->d_data = outr->data_cap >= (64ull << 20) ? e->take_data(outr->data_cap, &cap) : nullptr; if (outr->d_data) outr->data_cap = cap; }
    if (!outr->d_data) PGS_CUDA(cudaMallocAsync(&outr->d_data, outr->data_cap, st));
    PGS_CUDA(cudaMallocAsync(&outr->d_blk_off, sizeof(uint64_t) * (geo.blk_cap + 1), st));
    PGS_CUDA(cudaMallocAsync(&outr->d_blk_size, sizeof(uint32_t) * (geo.blk_cap + 1), st));
    PGS_CUDA(cudaMallocAsync(&outr->d_blk_rec, sizeof(uint32_t) * (geo.blk_cap + 1), st));
    PGS_CUDA(cudaMallocAsync(&outr->d_ikey_off, sizeof(uint32_t) * (geo.blk_cap + 1), st));
    PGS_CUDA(cudaMallocAsync(&outr->d_ikeys, geo.ikey_cap, st));
    PGS_CUDA(cudaMallocAsync(&outr->d_rec_off, sizeof(uint32_t) * (T.n_rec + 1), st));
    outr->bloom_lines = bloom_lines_for(T.bloom_entries);
    PGS_CUDA(cudaMallocAsync(&outr->d_bloom, (size_t)outr->bloom_lines * 64, st));
    PGS_CUDA(cudaMemsetAsync(outr->d_bloom, 0, (size_t)outr->bloom_lines * 64, st));
    PGS_CUDA(S.alloc(P.split_pos, sizeof(uint32_t) * (Q + 1) * k));
    PGS_CUDA(S.alloc(P.split_ref, sizeof(uint32_t) * (Q + 1)));
    PGS_CUDA(S.alloc(P.ticket, 256));
    PGS_CUDA(S.alloc(P.seg, sizeof(SegLayout) * Q));
    PGS_CUDA(S.alloc(P.agg, sizeof(SegAgg) * Q));
    PGS_CUDA(S.alloc(P.base, sizeof(SegBase) * Q));
    PGS_CUDA(S.alloc(P.desc, sizeof(Desc) * P.desc_cap));
    PGS_CUDA(S.alloc(P.heads, P.head_cap + 64));
    PGS_CUDA(cudaMemsetAsync(P.split_pos, 0xFF, sizeof(uint32_t) * (Q + 1) * k, st));
    PGS_CUDA(cudaMemsetAsync(P.split_ref, 0xFF, sizeof(uint32_t) * (Q + 1), st));
    PGS_CUDA(cudaMemsetAsync(P.ticket, 0, 256, st));
    PGS_CUDA(cudaMemsetAsync(P.agg, 0, sizeof(SegAgg) * Q, st));
    MergeStats hs{};
    hs.error_seg = 0xFFFFFFFFu;
    PGS_CUDA(S.upload(P.stats, &hs, 1));
    if (!ops_host.empty()) {
        uint8_t *d_ops = nullptr;
        PGS_CUDA(S.upload(d_ops, ops_host.data(), ops_host.size()));
        P.ops = d_ops;
    }
    if (P.validate_hash) P.crc_table = (const unsigned long long *)e->d_crc;
    P.out_data = outr->d_data;
    P.out_blk_off = (unsigned long long *)outr->d_blk_off;
    P.out_blk_size = outr->d_blk_size;
    P.out_blk_rec = outr->d_blk_rec;
    P.out_ikey_off = outr->d_ikey_off;
    P.out_ikeys = outr->d_ikeys;
    P.out_rec_off = outr->d_rec_off;
    P.out_bloom = outr->d_bloom;
    P.out_bloom_lines = outr->bloom_lines;

    cudaEvent_t ev[4];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    walk_kernel_t walk = walk_kernel(geo.G);
    int occ_w = 0, occ_e = 0;
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_w, walk, (int)kWalkThreads, (size_t)geo.walk_dyn));
    PGS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_e, k_emit, (int)(geo.emit_warps * 32), (size_t)geo.emit_dyn));
    const uint32_t seg_per_cta_w = kWalkThreads / geo.G;
    const uint32_t grid_w = (uint32_t)std::min<uint64_t>((Q + seg_per_cta_w - 1) / seg_per_cta_w, (uint64_t)std::max(1, occ_w) * e->sm_count);
    const uint32_t grid_e = (uint32_t)std::min<uint64_t>((Q + geo.emit_warps - 1) / geo.emit_warps, (uint64_t)std::max(1, occ_e) * e->sm_count);
    PGS_CUDA(cudaEventRecord(ev[0], st));
    k_plan<<<(uint32_t)((T.total_blocks + 255) / 256), 256, 0, st>>>(P);
    k_seg_bounds<<<(uint32_t)((Q + 255) / 256), 256, 0, st>>>(P);
    k_seg_layout<<<1, 1024, 0, st>>>(P);
    PGS_CUDA(cudaEventRecord(ev[1], st));
    walk<<<grid_w, kWalkThreads, geo.walk_dyn, st>>>(P);
    PGS_CUDA(cudaEventRecord(ev[2], st));
    k_seg_scan<<<1, 1024, 0, st>>>(P);
    k_emit<<<grid_e, geo.emit_warps * 32, geo.emit_dyn, st>>>(P);
    PGS_CUDA(cudaEventRecord(ev[3], st));
    e->launches += 6;
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
    res.n_tiles = P.Q; res.n_launches = 6;
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
