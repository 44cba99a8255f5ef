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

namespace pgs {
namespace {

// PGS_WALK_G (diagnostics): the lanes per merge group of every compaction's walk, 1, 2, 4, 8 or 16 (0: the planner's choice)
uint32_t walk_g_override()
{
    const char *ev = getenv("PGS_WALK_G");
    const int v = ev ? atoi(ev) : 0;
    return v == 1 || v == 2 || v == 4 || v == 8 || v == 16 ? (uint32_t)v : 0u;
}

// A compaction job's k input runs, looked up by id under part's lock, and the bottommost < 0 rule: true iff every run outside
// the inputs is newer than every input.  Refuses an unknown run and a run given twice, with a message that starts with who.
int32_t compact_inputs(Partition &part, const uint64_t *run_ids, uint32_t k, int32_t &bottommost, std::vector<std::shared_ptr<Run>> &in,
                       const char *who)
{
    std::lock_guard<std::mutex> g(part.mu);
    for (uint32_t i = 0; i < k; i++) {
        auto r = part.find(run_ids[i]);
        if (!r) { set_error("%s unknown run %llu", who, (unsigned long long)run_ids[i]); return PGS_NOT_FOUND; }
        if (std::find(in.begin(), in.end(), r) != in.end()) { set_error("%s run %llu given twice", who, (unsigned long long)run_ids[i]); return PGS_INVALID_ARGUMENT; }
        in.push_back(r);
    }
    if (bottommost < 0) {
        size_t first_in = part.runs.size();
        for (size_t i = 0; i < part.runs.size(); i++)
            if (std::find(in.begin(), in.end(), part.runs[i]) != in.end()) { first_in = i; break; }
        bottommost = 1;
        for (size_t i = first_in; i < part.runs.size(); i++)
            if (std::find(in.begin(), in.end(), part.runs[i]) == in.end()) bottommost = 0;
    }
    return PGS_OK;
}

// n finished merges installed, all or none (many: with pgs_compact_many's messages).  Every partition's lock is held from the
// check that each job's inputs in[i] are still in parts[i] (PGS_ABORTED otherwise: pgs_run_drop took one during the merge) to
// the last install.  Job i's inputs leave unless KEEP_INPUTS, its output outr[i] goes in unless it is empty or DISCARD_OUTPUT,
// and out[i] (if out) = res's launches and times with job i's counters, segments and new run id.
int32_t compact_install(uint32_t n, Partition *const *parts, const std::vector<std::shared_ptr<Run>> *in, const std::shared_ptr<Run> *outr,
                        const MergeStats *hs, const MergeParams *P, const CompactTotals *T, const pgs_compact_result &res, uint32_t flags,
                        bool many, pgs_compact_result *out)
{
    Engine *e = parts[0]->eng;
    std::vector<pgs_compact_result> r(n, res);
    for (uint32_t i = 0; i < n; i++) {
        outr[i]->n_bloom_entries = compact_result_stats(hs[i], T[i].in_block_bytes, r[i], outr[i]->info);
        outr[i]->info.level = outr[i]->level;
        r[i].n_tiles = P[i].Q;
    }
    const auto held = lock_partitions(std::vector<Partition *>(parts, parts + n));
    for (uint32_t i = 0; i < n; i++)
        for (auto &x : in[i])
            if (std::find(parts[i]->runs.begin(), parts[i]->runs.end(), x) == parts[i]->runs.end()) {
                if (many) set_error("compact_many: job %u: run %llu left the partition during the merge", i, (unsigned long long)x->id);
                else set_error("compact: run %llu left the partition during the merge", (unsigned long long)x->id);
                return PGS_ABORTED;
            }
    for (uint32_t i = 0; i < n; i++) {
        Partition &part = *parts[i];
        if (!(flags & PGS_COMPACT_KEEP_INPUTS))
            for (auto &x : in[i]) part.runs.erase(std::find(part.runs.begin(), part.runs.end(), x));
        if (hs[i].tot_blocks > 0 && !(flags & PGS_COMPACT_DISCARD_OUTPUT)) {
            outr[i]->id = e->next_run_id++;
            outr[i]->info.run_id = outr[i]->id;
            part.insert(outr[i]);
            r[i].new_run_id = outr[i]->id;
        }
    }
    if (out) memcpy(out, r.data(), sizeof(pgs_compact_result) * (size_t)n);
    return PGS_OK;
}

} // namespace
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
    Partition &part = ph->p, *parts = &part;
    Engine *e = part.eng;
    std::vector<std::shared_ptr<Run>> in;
    if (const int32_t rc = compact_inputs(part, run_ids, k, bottommost, in, "compact:")) return rc;
    MergeParams P{};
    CompactTotals T{};
    uint32_t ops_len = 0;
    if (const int32_t rc = compact_job_params(P, T, k, [&](uint32_t i) -> const Run & { return *in[i]; }, e->cfg.block_size, e->cfg.restart_interval,
                                              bottommost, now, part.data_version, fp, (const unsigned long long *)e->d_crc, ops_len, "compact:"))
        return rc;
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    CompactGeometry geo{};
    const uint32_t smem = compact_smem_budget((uint32_t)e->max_smem_optin);
    Resident walk{};
    bool geo_ok = compact_geometry(P, T, smem, geo, walk_g_override());
    if (geo_ok) { // second pass: the segment budget follows from how many groups the device runs at once
        PGS_CUDA(resident(*e, walk_kernel(geo.G), kWalkThreads, geo.G, geo.walk_dyn, walk));
        geo_ok = compact_geometry(P, T, smem, geo, geo.G, 0, walk.groups);
    }
    if (!geo_ok) {
        set_error("compact: input too large for one merge launch (keys of %u bytes, %llu records)", T.max_ukey, (unsigned long long)T.n_rec);
        return PGS_NOT_SUPPORTED;
    }

    LaunchScratch S(st);
    auto outr = std::make_shared<Run>(e);
    outr->level = out_level;
    cudaError_t ce = cudaSuccess;
    auto keep = run_buffers(e, *outr, ce);
    auto scratch = scratch_buffers(S, ce);
    compact_buffers(P, geo, T, *outr, [&](auto *&p, uint64_t n, int fill, bool is_out) { if (is_out) keep(p, n, fill); else scratch(p, n, fill); });
    PGS_CUDA(ce);
    MergeStats hs = merge_stats_init();
    PGS_CUDA(S.upload(P.stats, &hs, 1));
    if (ops_len) PGS_CUDA(S.upload(P.ops, fp->ops, ops_len));

    cudaEvent_t ev[4];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    Resident emit{};
    PGS_CUDA(resident(*e, k_emit, geo.emit_warps * 32, 32, geo.emit_dyn, emit));
    const uint32_t launches = compact_launch(P, geo, walk.ctas, emit.ctas, st, [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
    e->launches += launches;
    PGS_CUDA(ce);
    PGS_CUDA(cudaMemcpyAsync(&hs, P.stats, sizeof hs, cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return cuda_fail(se, "compaction kernels");
    pgs_compact_result res{};
    res.n_launches = launches;
    cudaEventElapsedTime(&res.device_ms, ev[0], ev[3]);
    cudaEventElapsedTime(&res.merge_kernel_ms, ev[1], ev[3]);
    cudaEventElapsedTime(&res.walk_ms, ev[1], ev[2]);
    cudaEventElapsedTime(&res.emit_ms, ev[2], ev[3]);
    if (hs.error) {
        set_error("compaction kernel failed with status %u at segment %u of %u", hs.error, hs.error_seg, P.Q);
        return (int32_t)hs.error;
    }
    return compact_install(1, &parts, &in, &outr, &hs, &P, &T, res, flags, false, out);
}

// ---- pgs_compact_many --------------------------------------------------------------------------------------------------------
// The jobs of many partitions planned together (compact_many_geometry) and launched once (compact_launch_many).  The jobs'
// scratch shares one allocation; each merged run keeps buffers of its own, as pgs_compact's does.
extern "C" int32_t pgs_compact_many(const pgs_compact_job *jobs, uint32_t n, uint32_t now, uint32_t flags, pgs_compact_result *out)
{
    if (n == 0) return PGS_OK;
    if (!jobs) { set_error("compact_many: %u jobs and no job array", n); return PGS_INVALID_ARGUMENT; }
    if (n > kMaxCompactJobs) { set_error("compact_many: %u jobs > %u per call", n, kMaxCompactJobs); return PGS_NOT_SUPPORTED; }
    JobPartitions set;
    std::vector<Partition *> parts(n);
    for (uint32_t i = 0; i < n; i++) {
        const pgs_compact_job &J = jobs[i];
        if (!J.part || !J.run_ids || J.k == 0 || J.out_level < 0) {
            set_error("compact_many: job %u: no partition, no runs or a negative output level", i);
            return PGS_INVALID_ARGUMENT;
        }
        parts[i] = &J.part->p;
        if (!set.add(*parts[i], i)) { set_error("compact_many: job %u: its partition is on another engine than job 0's", i); return PGS_INVALID_ARGUMENT; }
    }
    uint32_t a = 0, b = 0;
    if (set.twice(a, b)) { set_error("compact_many: job %u: its partition is in another job too", a); return PGS_INVALID_ARGUMENT; }
    Engine *e = set.e;
    char who_buf[40];
    auto who = [&](uint32_t i) { snprintf(who_buf, sizeof who_buf, "compact_many: job %u:", i); return who_buf; };

    // the inputs and the bottommost rule of every job, then every job's limits and filter, as pgs_compact_ex checks them
    std::vector<std::vector<std::shared_ptr<Run>>> in(n);
    std::vector<int32_t> bottom(n);
    for (uint32_t i = 0; i < n; i++) {
        bottom[i] = jobs[i].bottommost;
        if (const int32_t rc = compact_inputs(*parts[i], jobs[i].run_ids, jobs[i].k, bottom[i], in[i], who(i))) return rc;
    }
    std::vector<MergeParams> P(n);
    std::vector<CompactTotals> T(n);
    std::vector<uint32_t> ops_len(n);
    uint32_t any_hash = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (const int32_t rc = compact_job_params(P[i], T[i], jobs[i].k, [&](uint32_t x) -> const Run & { return *in[i][x]; }, e->cfg.block_size,
                                                  e->cfg.restart_interval, bottom[i], now, parts[i]->data_version, jobs[i].fp,
                                                  (const unsigned long long *)e->d_crc, ops_len[i], who(i)))
            return rc;
        if (P[i].validate_hash) any_hash = 1;
    }
    MergeJobs M{};
    CompactGeometry shared{};
    std::vector<CompactGeometry> geo(n);
    const uint32_t smem = compact_smem_budget((uint32_t)e->max_smem_optin);
    Resident walk{};
    bool geo_ok = compact_many_geometry(P.data(), T.data(), geo.data(), n, smem, M, shared, walk_g_override());
    if (geo_ok) { // second pass: the segment weight follows from how many groups the device runs at once
        PGS_CUDA(resident(*e, walk_many_kernel(shared.G), kWalkThreads, shared.G, shared.walk_dyn, walk));
        geo_ok = compact_many_geometry(P.data(), T.data(), geo.data(), n, smem, M, shared, shared.G, 0, walk.groups);
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
    // the merged runs' buffers, one set per job; the scratch of every job in one allocation
    ScratchArena arena;
    std::vector<std::shared_ptr<Run>> outr(n);
    cudaError_t ce = cudaSuccess;
    for (uint32_t i = 0; i < n; i++) {
        outr[i] = std::make_shared<Run>(e);
        outr[i]->level = jobs[i].out_level;
        auto keep = run_buffers(e, *outr[i], ce);
        compact_buffers(P[i], geo[i], T[i], *outr[i], [&](auto *&p, uint64_t cnt, int fill, bool is_out) { if (is_out) keep(p, cnt, fill); else arena(p, cnt, fill); });
    }
    PGS_CUDA(ce);
    arena(M.ticket, 2, 0);
    PGS_CUDA(arena.place(S));

    // the job table: MergeParams[n] | MergeStats[n] | seg_base[n + 1] | blk_base[n + 1] | the ops tables
    JobTable tab;
    const uint64_t o_job = tab.add<MergeParams>(n), o_stats = tab.add<MergeStats>(n);
    const uint64_t o_seg = tab.add<uint32_t>(n + 1), o_blk = tab.add<uint32_t>(n + 1);
    std::vector<uint64_t> o_ops(n);
    for (uint32_t i = 0; i < n; i++)
        if (ops_len[i]) o_ops[i] = tab.add<uint8_t>(ops_len[i]);
    PGS_CUDA(tab.alloc(S));
    for (uint32_t i = 0; i < n; i++) {
        P[i].stats = tab.dev<MergeStats>(o_stats) + i;
        tab.host<MergeStats>(o_stats)[i] = merge_stats_init();
        if (ops_len[i]) {
            memcpy(tab.host<uint8_t>(o_ops[i]), jobs[i].fp->ops, ops_len[i]);
            P[i].ops = tab.dev<uint8_t>(o_ops[i]);
        }
    }
    memcpy(tab.host<MergeParams>(o_job), P.data(), sizeof(MergeParams) * (size_t)n);
    compact_many_bases(P.data(), n, tab.host<uint32_t>(o_seg), tab.host<uint32_t>(o_blk));
    PGS_CUDA(tab.upload(st));
    M.job = tab.dev<MergeParams>(o_job);
    M.seg_base = tab.dev<uint32_t>(o_seg);
    M.blk_base = tab.dev<uint32_t>(o_blk);
    M.validate_hash = any_hash;
    M.crc_table = (const unsigned long long *)e->d_crc;

    cudaEvent_t ev[4];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    Resident emit{};
    PGS_CUDA(resident(*e, k_emit_many, shared.emit_warps * 32, 32, shared.emit_dyn, emit));
    const uint32_t launches = compact_launch_many(M, shared, walk.ctas, emit.ctas, st, [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
    e->launches += launches;
    PGS_CUDA(ce);
    std::vector<MergeStats> hs(n);
    PGS_CUDA(cudaMemcpyAsync(hs.data(), tab.dev<MergeStats>(o_stats), sizeof(MergeStats) * (size_t)n, cudaMemcpyDeviceToHost, st));
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) return cuda_fail(se, "multi-job compaction kernels");
    for (uint32_t i = 0; i < n; i++)
        if (hs[i].error) {
            set_error("compact_many: job %u: compaction kernel failed with status %u at segment %u of %u", i, hs[i].error, hs[i].error_seg, P[i].Q);
            return (int32_t)hs[i].error;
        }
    pgs_compact_result res{};
    res.n_launches = launches;
    cudaEventElapsedTime(&res.device_ms, ev[0], ev[3]);
    cudaEventElapsedTime(&res.merge_kernel_ms, ev[1], ev[3]);
    cudaEventElapsedTime(&res.walk_ms, ev[1], ev[2]);
    cudaEventElapsedTime(&res.emit_ms, ev[2], ev[3]);
    return compact_install(n, parts.data(), in.data(), outr.data(), hs.data(), P.data(), T.data(), res, flags, true, out);
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
    Resident walk{};
    int32_t rc = split_plan(SP, T, smem, geo);
    if (rc == PGS_OK) { // second pass: segments sized by the groups the device runs at once
        PGS_CUDA(resident(*e, split_kernel(geo.G, false), kSplitThreads, geo.G, geo.walk_dyn, walk));
        rc = split_plan(SP, T, smem, geo, walk.groups);
    }
    if (rc != PGS_OK) {
        set_error("partition_split: a run with user keys of %u bytes into %u children is not supported", T.max_ukey, NC);
        return rc;
    }

    LaunchScratch S(st);
    cudaError_t ce = cudaSuccess;
    split_buffers(SP, scratch_buffers(S, ce));
    PGS_CUDA(ce);
    std::vector<MergeStats> hs(NC, merge_stats_init());
    PGS_CUDA(cudaMemcpyAsync(SP.stats, hs.data(), sizeof(MergeStats) * NC, cudaMemcpyHostToDevice, st));
    cudaEvent_t ev[5];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    res.n_launches += split_launch(SP, geo, nullptr, nullptr, 0, walk.ctas, 0, st, [&](int i) { if (ce == cudaSuccess) ce = cudaEventRecord(ev[i], st); });
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
        auto keep = run_buffers(e, *r, ce);
        compact_buffers(P, g, Tc, *r, [&](auto *&p, uint64_t n, int fill, bool is_out) { if (is_out) keep(p, n, fill); }); // the scratch is the split's
        PGS_CUDA(ce);
        split_child_scratch(SP, c, P);
        Pc.push_back(P);
        gc.push_back(g);
        which.push_back(c);
        out[c] = r;
    }
    Resident emit{};
    if (!gc.empty()) PGS_CUDA(resident(*e, k_emit, gc[0].emit_warps * 32, 32, gc[0].emit_dyn, emit));
    res.n_launches += split_launch(SP, geo, Pc.data(), gc.data(), (uint32_t)Pc.size(), walk.ctas, emit.ctas, st,
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

// The children of n split jobs installed, all or none (many: with pgs_partition_split_many's messages).  rows[i][c] = job i's
// child c (null: not built), built[i * NC + c] = its runs in the parent's order.  Every child's lock is held from the check that
// none took runs during the split (PGS_ABORTED otherwise) to the last install; each run gets its id and res[i].child[c] counts it.
int32_t split_install(Engine *e, pgs_partition *const *const *rows, uint32_t n, uint32_t NC, const std::vector<std::vector<std::shared_ptr<Run>>> &built,
                      pgs_split_result *res, bool many)
{
    std::vector<Partition *> kids;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++)
            if (rows[i][c]) kids.push_back(&rows[i][c]->p);
    const auto held = lock_partitions(kids);
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++)
            if (rows[i][c] && !rows[i][c]->p.runs.empty()) {
                if (many) set_error("partition_split_many: job %u: destination %u took runs during the split", i, c);
                else set_error("partition_split: destination %d took runs during the split", rows[i][c]->p.pidx);
                return PGS_ABORTED;
            }
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t c = 0; c < NC; c++) {
            if (!rows[i][c]) continue;
            pgs_split_child_result &cr = res[i].child[c];
            const auto &b = built[(size_t)i * NC + c];
            for (auto &r : b) {
                r->id = e->next_run_id++;
                r->info.run_id = r->id;
                cr.records += r->info.n_records;
                cr.tombstones += r->info.n_tombstones;
                cr.raw_bytes += r->info.raw_key_bytes + r->info.raw_value_bytes;
                cr.block_bytes += r->info.data_bytes;
                cr.runs++;
            }
            rows[i][c]->p.runs = b;
        }
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
    if (const int32_t rc = split_install(e, &dst, 1, NC, built, &res, false)) return rc;
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
    const uint32_t NC = src_count ? dst_count / src_count : 0;
    std::vector<uint32_t> want(n);
    // every partition in one job only: a parent is no other job's parent or child, a child no other job's child
    JobPartitions set;
    for (uint32_t i = 0; i < n; i++) {
        if (const int32_t rc = split_dests(jobs[i].src, src_count, dst_count, jobs[i].dst, NC, want[i])) {
            const std::string why = pgs_last_error();
            set_error("partition_split_many: job %u: %s", i, why.c_str());
            return rc;
        }
        if (!set.add(jobs[i].src->p, i)) { set_error("partition_split_many: job %u: its parent is on another engine than job 0's", i); return PGS_INVALID_ARGUMENT; }
        for (uint32_t c = 0; c < NC; c++)
            if (jobs[i].dst[c]) set.add(jobs[i].dst[c]->p, i); // on the parent's engine (split_dests)
    }
    uint32_t a = 0, b = 0;
    if (set.twice(a, b)) { set_error("partition_split_many: job %u: a partition of job %u is in job %u too", b, a, b); return PGS_INVALID_ARGUMENT; }
    Engine *e = set.e;

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
    Resident walk{};
    if (nr) {
        int32_t rc = split_many_plan(SP.data(), T.data(), nr, smem, J, M, geo);
        if (rc == PGS_OK) { // second pass: segments sized by the groups the device runs at once
            PGS_CUDA(resident(*e, split_many_kernel(geo.G, false), kSplitThreads, geo.G, geo.walk_dyn, walk));
            rc = split_many_plan(SP.data(), T.data(), nr, smem, J, M, geo, walk.groups);
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
        ScratchArena arena; // the scratch in one allocation
        split_many_buffers(SP.data(), nr, J, arena);
        PGS_CUDA(arena.place(S));
        PGS_CUDA(cudaMemcpyAsync(J.stats, hs.data(), sizeof(MergeStats) * hs.size(), cudaMemcpyHostToDevice, st));

        // the job tables: MergeParams[nr] (the planner's) | SplitParams[nr] | seg_base[nr + 1] | blk_base[nr + 1]
        JobTable tab;
        const uint64_t o_job = tab.add<MergeParams>(nr), o_split = tab.add<SplitParams>(nr);
        const uint64_t o_seg = tab.add<uint32_t>(nr + 1), o_blk = tab.add<uint32_t>(nr + 1);
        split_many_tables(SP.data(), nr, J, tab.host<MergeParams>(o_job), tab.host<uint32_t>(o_seg), tab.host<uint32_t>(o_blk));
        memcpy(tab.host<SplitParams>(o_split), SP.data(), sizeof(SplitParams) * (size_t)nr);
        PGS_CUDA(tab.alloc(S));
        PGS_CUDA(tab.upload(st));
        M.job = tab.dev<MergeParams>(o_job);
        M.seg_base = J.seg_base = tab.dev<uint32_t>(o_seg);
        M.blk_base = tab.dev<uint32_t>(o_blk);
        J.job = tab.dev<SplitParams>(o_split);
        J.crc_table = (const unsigned long long *)e->d_crc;

        // counting phase, then one read-back of every (job, child) counter, prefix count and dropped count
        all.n_launches += split_many_launch(J, M, geo, nullptr, CompactGeometry{}, walk.ctas, 0, st,
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
        std::vector<uint32_t> emit_base;
        CompactGeometry shape{};
        uint64_t at = 0;
        const bool sized = split_many_children(SP.data(), nr, hs.data(), prefixes.data(), smem, Pc, emit_base, shape, at,
                                               [&](uint32_t x, uint32_t c, MergeParams &P, const CompactGeometry &g, const CompactTotals &Tc) {
                                                   auto r = std::make_shared<Run>(e);
                                                   r->level = in[x]->level;
                                                   auto keep = run_buffers(e, *r, ce);
                                                   compact_buffers(P, g, Tc, *r, [&](auto *&p, uint64_t cnt, int fill, bool is_out) { if (is_out) keep(p, cnt, fill); });
                                                   outs[x][c] = r;
                                                   return ce == cudaSuccess;
                                               });
        PGS_CUDA(ce);
        if (!sized) {
            set_error("partition_split_many: job %u: child %u's run is too large, or not of the launch's shape", run_job[at / NC], (uint32_t)(at % NC));
            return PGS_NOT_SUPPORTED;
        }
        if (!Pc.empty()) { // writing phase
            const uint32_t nc = (uint32_t)Pc.size();
            JobTable ctab;
            const uint64_t o_pc = ctab.add<MergeParams>(nc), o_base = ctab.add<uint32_t>(nc + 1);
            memcpy(ctab.host<MergeParams>(o_pc), Pc.data(), sizeof(MergeParams) * (size_t)nc);
            memcpy(ctab.host<uint32_t>(o_base), emit_base.data(), 4ull * (nc + 1));
            PGS_CUDA(ctab.alloc(S));
            PGS_CUDA(ctab.upload(st));
            MergeJobs E{};
            E.job = ctab.dev<MergeParams>(o_pc);
            E.seg_base = ctab.dev<uint32_t>(o_base);
            E.n = nc;
            E.Q = emit_base.back();
            E.ticket = J.ticket + 2;
            Resident emit{};
            PGS_CUDA(resident(*e, k_emit_many, shape.emit_warps * 32, 32, shape.emit_dyn, emit));
            all.n_launches += split_many_launch(J, M, geo, &E, shape, walk.ctas, emit.ctas, st,
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
            cudaEventElapsedTime(&all.walk_ms, ev[2], ev[4]);
            cudaEventElapsedTime(&all.emit_ms, ev[4], ev[3]);
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
    std::vector<std::vector<std::shared_ptr<Run>>> built((size_t)n * NC); // job i's child c at i * NC + c, in the parent's run order
    for (uint32_t x = 0; x < nr; x++)
        for (uint32_t c = 0; c < NC; c++)
            if (outs[x][c]) built[(size_t)run_job[x] * NC + c].push_back(outs[x][c]);
    std::vector<pgs_partition *const *> rows(n);
    for (uint32_t i = 0; i < n; i++) rows[i] = jobs[i].dst;
    if (const int32_t rc = split_install(e, rows.data(), n, NC, built, res.data(), true)) return rc;
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
