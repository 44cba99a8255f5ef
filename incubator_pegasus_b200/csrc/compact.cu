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
    split_buffers(SP, [&](auto *&p, uint64_t n, int fill, bool) {
        const size_t bytes = sizeof(*p) * n;
        if (ce != cudaSuccess) return;
        ce = S.alloc(p, bytes ? bytes : 16);
        if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, bytes, st);
    });
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

// pgs_partition_split over the runs `snap` of src (nullptr: its current runs); pgs_rrdb_split passes the snapshot it took
// under the replica's writer lock
int32_t partition_split(pgs_partition *src, const std::vector<std::shared_ptr<Run>> *snap, uint32_t src_count, uint32_t dst_count,
                        pgs_partition *const *dst, uint32_t n_dst, pgs_split_result *out)
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
    uint32_t want = 0;
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
} // namespace pgs

using namespace pgs;

extern "C" int32_t pgs_partition_split(pgs_partition *src, uint32_t src_count, uint32_t dst_count, pgs_partition *const *dst, uint32_t n_dst,
                                       pgs_split_result *out)
{
    return partition_split(src, nullptr, src_count, dst_count, dst, n_dst, out);
}
