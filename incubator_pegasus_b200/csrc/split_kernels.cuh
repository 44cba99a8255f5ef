// split_kernels.cuh — partition split on the GPU (host side: pgs_partition_split in compact.cu): every record of a parent run goes to the child partition its key's
// pegasus_key_hash names, and each child gets one run at the parent run's level, with its own blocks, index and Bloom filter.
//
// Replaces (reference file:line):
//   local_partition_split's per-record loop ............. src/shell/commands/local_partition_split.cpp:238-283
//   the split manager's copy_checkpoint_to_dir / storage_apply_checkpoint pair (replica_split_manager.cpp:278), which copies
//   the whole parent into the child
//
// Shape of the computation (per parent run; byte work bound by HBM):
//   k_plan, k_seg_bounds, k_seg_layout   compaction's planner with k = 1: segments of whole user keys, a descriptor and
//                 key-stream region per segment bounded by its input slice (compact_kernels.cuh)
//   k_split_walk<count>   one lane group per segment decodes the run's entries in order (the cursor of group.cuh), computes
//                 the crc64 of a hash key once for its consecutive records, and runs, per child, the writer state k_walk keeps
//                 for its one output (shared prefix with the child's previous record, block fill, restart countdown, big-entry
//                 flag) with k_walk's block-cut rule.  It counts per (segment, child) records and key-stream bytes and adds up
//                 each child's record statistics: they size the children's outputs exactly.
//   k_split_walk<write>   the same walk again; each segment's region is divided among the children by the counts, and every
//                 record leaves as a Desc + key-stream record of its child in the format k_walk hands to k_emit.
//   k_seg_scan, k_emit    unchanged, once per child over that child's segment aggregates, descriptors and key stream.
// pgs_partition_split_many runs the same steps over every run of many parents at once: the *_many planner kernels, then
// k_split_walk_many<count / write> over the launch's segment list, then k_seg_scan_many and k_emit_many over every built child
// (the end of this file).
// Nothing is filtered: versions, tombstones, trailers and values stay as they are.  Records with an empty user key (the empty
// write) are dropped and counted.
#pragma once
#include "compact_kernels.cuh"

namespace pgs {

// The most children of one split: each lane group keeps a SplitChild (128 bytes) per child in shared memory, so 32 children
// cost 4 KB per group, and with 4096-byte user keys (four key rows of ~4 KB) a CTA of 4 groups of 32 lanes still fits twice
// per SM.
constexpr uint32_t kSplitMaxChildren = 32;
constexpr uint32_t kSplitThreads = 128;

struct SplitCount { // what one segment gives one child: records, key-stream bytes (counting pass)
    uint32_t n, ks;
};

// a child's writer state inside the segment a group walks (shared memory; lane 0 of the group writes, all lanes read)
struct __align__(16) SplitChild {
    unsigned long long out_bytes, b_key, b_val, m_seq, m_seq_inv;
    unsigned long long d_off, k_off; // writing pass: where its descriptors and key stream of this segment start
    uint32_t n, kpos;                // records and key-stream bytes so far
    uint32_t blk_n, blk_bytes, to_restart, nrest, prev_big; // the open block (as k_walk keeps it)
    uint32_t n_blocks, keyb, lenA;   // closed blocks, their index-key bytes, the last record's user-key length
    uint32_t lcp;                    // bytes the current key shares with the child's last record (the minimum along the way)
    uint32_t n_tomb, m_ukey, m_vlen, m_bsize, m_brec, n_prefix, pad;
};
static_assert(sizeof(SplitChild) == 128, "SplitChild");

struct SplitParams {
    MergeParams M;         // the plan over the parent run (k = 1), its scratch; M.stats = stats
    uint32_t S;            // children
    uint32_t src_count, dst_count;
    uint32_t want;         // bit c: child c is built (records of the others are skipped)
    uint32_t group_smem;   // one group's shared memory: child states | cursor | four key rows
    SplitCount *cnt;       // [Q * S]
    SegLayout *lay;        // [S * Q]: child c's segment q at c * Q + q (k_emit's P.seg of the child), as are agg and base
    SegAgg *agg;
    SegBase *base;
    MergeStats *stats;     // [S]
    unsigned long long *prefixes; // [S] hash-key prefixes each child's Bloom filter takes
    unsigned long long *dropped;  // [1] empty writes
};

struct SplitGeometry {
    CompactGeometry cg; // the planner's (and the children's k_emit shape)
    uint32_t G, walk_dyn;
};

PGS_HD uint32_t split_group_smem(uint32_t S, uint32_t KSW)
{
    return (S * (uint32_t)sizeof(SplitChild) + (((uint32_t)sizeof(CurState) + 15) & ~15u) + 16 * KSW + 15) & ~15u;
}
PGS_HD uint64_t split_dyn_smem(uint32_t G, uint32_t group_smem) { return 2048 + (uint64_t)(kSplitThreads / G) * group_smem; }

// the plan of one parent run (S.M.runs[0], S.M.block_size, S.M.restart_interval and S.S set): segments, scratch bounds, the
// walker's lanes per group.  walk_groups = groups the device runs at once (0: not known yet).  Returns a status.
inline int32_t split_plan(SplitParams &S, const CompactTotals &T, uint32_t max_smem, SplitGeometry &geo, uint64_t walk_groups = 0,
                          uint64_t force_weight = 0)
{
    if (S.S < 2 || S.S > kSplitMaxChildren) return PGS_NOT_SUPPORTED;
    S.M.k = 1;
    if (T.max_ukey > kMaxUkeyLen || !compact_geometry(S.M, T, max_smem, geo.cg, 0, force_weight, walk_groups)) return PGS_NOT_SUPPORTED;
    S.group_smem = split_group_smem(S.S, S.M.KSW);
    geo.G = 0;
    for (uint32_t G = 4; G <= 32 && !geo.G; G *= 2) // the narrowest group whose CTA fits shared memory twice per SM (or once)
        if (split_dyn_smem(G, S.group_smem) <= max_smem / 2) geo.G = G;
    for (uint32_t G = 4; G <= 32 && !geo.G; G *= 2)
        if (split_dyn_smem(G, S.group_smem) <= max_smem) geo.G = G;
    if (!geo.G) return PGS_NOT_SUPPORTED;
    geo.walk_dyn = (uint32_t)split_dyn_smem(geo.G, S.group_smem);
    return PGS_OK;
}

// The per-segment scratch of one parent run's split (its plan, descriptors, key stream and the children's segment tables), as
// compact_buffers hands it out: buf(pointer, elements, fill, out = false).
template <class F>
inline void split_scratch(SplitParams &S, F &&buf)
{
    const uint64_t Q = S.M.Q, C = S.S;
    buf(S.M.split_pos, Q + 1, 0xFF, false);
    buf(S.M.split_ref, Q + 1, 0xFF, false);
    buf(S.M.seg, Q, kNoFill, false);
    buf(S.M.desc, S.M.desc_cap, kNoFill, false);
    buf(S.M.kstream, S.M.ks_cap + 64, kNoFill, false);
    buf(S.cnt, Q * C, 0, false);
    buf(S.lay, C * Q, kNoFill, false);
    buf(S.agg, C * Q, 0, false); // a child that gets nothing from a segment has an empty aggregate
    buf(S.base, C * Q, kNoFill, false);
}
// The scratch of one parent run's split: split_scratch, the tickets and the children's counters.
template <class F>
inline void split_buffers(SplitParams &S, F &&buf)
{
    const uint64_t C = S.S;
    split_scratch(S, buf);
    buf(S.M.ticket, 4 + 2 * C, 0, false); // [0] counting walk, [2] writing walk, 4 + 2c: child c's k_emit (its ticket[1])
    buf(S.stats, C, kNoFill, false); // the caller sets every child's to merge_stats_init()
    buf(S.prefixes, C, 0, false);
    buf(S.dropped, 1, 0, false);
    S.M.stats = S.stats;
}

// Child c's k_seg_scan / k_emit parameters from what the counting pass found (st = its MergeStats, prefixes = its new hash-key
// prefixes): the parent's segments and block shape, an output sized by the child's own totals (T), the split's scratch.  The
// child's run buffers come from compact_buffers(Pc, geo, T, run, buf) with buf allocating only `out` buffers, then
// split_child_scratch.  false: not supported.
inline bool split_child(const SplitParams &S, const MergeStats &st, unsigned long long prefixes, uint32_t max_smem, MergeParams &Pc,
                        CompactGeometry &geo, CompactTotals &T)
{
    Pc = S.M;
    T = CompactTotals{};
    T.max_ukey = S.M.KS; // the parent's key rows: the same key-stream stage and block buffer as the walker planned with
    T.n_rec = st.cnt[EV_OUT];
    T.raw_key = st.bytes[SB_OUT_KEY];
    T.raw_val = st.bytes[SB_OUT_VAL];
    T.bloom_entries = T.n_rec + prefixes;
    return compact_geometry(Pc, T, max_smem, geo, 0, 0, 0, S.M.Q) && Pc.block_size == S.M.block_size && Pc.blk_buf == S.M.blk_buf;
}
inline void split_child_scratch(const SplitParams &S, uint32_t c, MergeParams &Pc)
{
    const uint64_t Q = S.M.Q;
    Pc.seg = S.lay + c * Q;
    Pc.agg = S.agg + c * Q;
    Pc.base = S.base + c * Q;
    Pc.desc = S.M.desc;
    Pc.kstream = S.M.kstream;
    Pc.ticket = S.M.ticket + 4 + 2 * c;
    Pc.stats = S.stats + c;
}

// ------------------------------------------------------------------------------------------------
// k_split_walk
// ------------------------------------------------------------------------------------------------
PGS_DEV uint32_t row_byte(const uint32_t *row, uint32_t i) { return (row[i >> 2] >> (8 * (i & 3))) & 0xffu; }
// the leading bytes of a user key pegasus_key_hash depends on: 2 + the hash key (clamped as split_key clamps it), or the
// whole key when the hash key is empty (the sort key is hashed then); by_hk tells which
PGS_DEV uint32_t hash_span(const uint32_t *row, uint32_t ulen, bool &by_hk)
{
    uint32_t hkl = ulen >= 2 ? (row_byte(row, 0) << 8) | row_byte(row, 1) : 0u;
    if (hkl + 2 > ulen) hkl = ulen >= 2 ? ulen - 2 : 0u;
    by_hk = hkl != 0;
    return hkl ? 2 + hkl : ulen;
}

// One segment per group, the groups of a warp in lock step (group.cuh): every collective is reached by all 32 lanes.
template <uint32_t G, bool WRITE>
PGS_DEV void split_segment(const SplitParams &S, const Grp<G> &g, bool seg_en, uint32_t q, CurState *C, uint32_t *row, uint32_t *prow,
                           uint32_t *rowLO, uint32_t *rowHI, SplitChild *ch, const unsigned long long *crc)
{
    const MergeParams &P = S.M;
    const RunDev &r = P.runs[0];
    const uint32_t NC = S.S, KS = P.KS, RI = P.restart_interval, BS = P.block_size, Q = P.Q;
    const bool first = q == 0, last = q == Q - 1;
    uint32_t err = 0;

    // ---- boundary keys (U_lo, U_hi], the children's states ---------------------------------------------------------------
    uint32_t ulo_len = 0, uhi_len = 0;
    if (seg_en) {
        for (uint32_t which = 0; which < 2; which++) {
            if (which == 0 ? first : last) continue;
            const uint32_t ref = P.split_ref[q + which], b = ref & 0x0FFFFFFFu;
            if (ref == 0xFFFFFFFFu || (ref >> 28) != 0 || b >= r.nb) { err = PGS_ABORTED; break; }
            const uint32_t off = r.ikey_off[b], len = r.ikey_off[b + 1] - off;
            if (len > KS) { err = PGS_ABORTED; break; }
            uint8_t *dst = (uint8_t *)(which == 0 ? rowLO : rowHI);
#pragma unroll 1
            for (uint32_t i = g.gl; i < len; i += G) dst[i] = r.ikeys[off + i];
            if (which == 0) ulo_len = len; else uhi_len = len;
        }
        for (uint32_t c = g.gl; c < NC; c += G) {
            SplitChild z;
            memset(&z, 0, sizeof z);
            ch[c] = z;
        }
    }
    g.sync();
    if (WRITE && seg_en && g.gl == 0) { // the segment's region, divided among the children by the counting pass
        unsigned long long d = P.seg[q].desc_off, k = P.seg[q].ks_off;
        for (uint32_t c = 0; c < NC; c++) {
            const SplitCount n = S.cnt[(size_t)q * NC + c];
            ch[c].d_off = d; ch[c].k_off = k;
            SegLayout L;
            L.desc_off = d; L.ks_off = k;
            S.lay[(size_t)c * Q + q] = L;
            d += n.n; k += n.ks;
        }
    }
    g.sync();

    // ---- open the cursor, skip what belongs to the previous segment ----------------------------------------------------------
    uint32_t lo = 0, hi_ex = 0, chk = 0, dpos = 0;
    if (seg_en && !err && !seg_slice(P, q, 0, lo, hi_ex, chk)) err = PGS_ABORTED;
    {
        const bool en = seg_en && !err;
        const uint32_t e1 = cur_open<G>(g, en, r, C, row, KS, lo, hi_ex, chk);
        if (en) err = e1;
    }
#pragma unroll 1
    for (;;) {
        const bool sk = seg_en && !err && !first && C->live;
        const int c = row_cmp(g, sk, row, sk ? C->klen - 8 : 0u, rowLO, ulo_len, dpos);
        const bool more = sk && c <= 0;
        if (!g.any(more)) break;
        const uint32_t e2 = cur_next<G>(g, more, r, C, row, KS);
        if (more) err = e2;
    }

    // ---- the records of the segment, in order ------------------------------------------------------------------------------
    bool done = !seg_en, have_prev = false, have_hash = false, p_by_hk = false;
    uint32_t plen = 0, pspan = 0, child = 0, n_empty = 0;
#pragma unroll 1
    for (;;) {
        bool act = !done && !err && C->live;
        const uint32_t ulen = act ? C->klen - 8 : 0u;
        const bool hi = act && !last && C->b >= C->chk_from; // past the upper bound: the next segment's
        const int chi = row_cmp(g, hi, row, ulen, rowHI, uhi_len, dpos);
        if (hi && chi > 0) act = false;
        if (!act) done = true;
        if (!g.any(act)) break;
        // (1) what the key shares with the run's previous record, exactly: the entry's `shared` field, checked at the byte it
        // ends in front of (a restart point stores 0, another writer may store less than the exact length)
        uint32_t L = 0, from = 0;
        bool need = false;
        if (act && have_prev) {
            const uint32_t m = ulen < plen ? ulen : plen;
            from = C->shared < m ? C->shared : m;
            if (from < m && row_byte(row, from) == row_byte(prow, from)) need = true;
            else L = from;
        }
        if (g.any(need)) {
            uint32_t dp = 0;
            row_cmp(g, need, row, ulen, prow, plen, dp, from);
            if (need) L = dp;
        }
        // (2) the child: the hash is computed again only when the bytes it reads changed
        const bool empty = act && ulen == 0;
        if (empty) n_empty++;
        if (act && !empty) {
            bool by_hk = false;
            const uint32_t span = hash_span(row, ulen, by_hk);
            if (!(have_hash && have_prev && by_hk == p_by_hk && span == pspan && L >= span)) {
                const uint64_t h = dev_key_hash(crc, (const uint8_t *)row, ulen);
                child = (uint32_t)((h % S.dst_count) / S.src_count);
                have_hash = true;
            }
            p_by_hk = by_hk;
            pspan = span;
        }
        // (3) every child's prefix with its last record shrinks to what this key shares with the previous one
        if (act)
            for (uint32_t c = g.gl; c < NC; c += G)
                if (ch[c].lcp > L) ch[c].lcp = L;
        g.sync();
        // (4) the record joins its child's output: k_walk's writer state and block-cut rule (compact_kernels.cuh, merge loop (3))
        const bool route = act && !empty && ((S.want >> child) & 1u);
        SplitChild w;
        uint32_t aux = 0, e = 0, flags = 0, vlen = 0, tr_lo = 0, tr_hi = 0;
        uint32_t *sp = nullptr;
        if (route) {
            w = ch[child];
            vlen = C->vlen; tr_lo = C->tr_lo; tr_hi = C->tr_hi;
            aux = w.n ? w.lcp : 0u;
            bool restart = w.to_restart == 0;
            uint32_t shared = restart ? 0u : aux, kd = ulen - shared;
            e = entry_head_len(shared, kd, vlen) + vlen;
            if (vlen > 0xFFF00000u) err = PGS_NOT_SUPPORTED; // entry sizes are 32-bit
            if (w.blk_n > 0 && (w.prev_big || block_bytes(w.blk_bytes + e, w.nrest + (restart ? 1u : 0u)) > BS)) {
                const uint32_t size = block_bytes(w.blk_bytes, w.nrest);
                w.out_bytes += block_span(size);
                w.n_blocks++;
                w.keyb += w.lenA;
                if (size > w.m_bsize) w.m_bsize = size;
                if (w.blk_n > w.m_brec) w.m_brec = w.blk_n;
                w.blk_n = 0; w.blk_bytes = 0; w.nrest = 0;
                restart = true; kd = ulen;
                e = entry_head_len(0u, kd, vlen) + vlen;
            }
            if (w.blk_n == 0) flags |= DF_NEWBLOCK;
            const bool big = e + 8 > P.blk_buf; // a block of its own in k_emit
            if (big) flags |= DF_BIG;
            if (WRITE) sp = reinterpret_cast<uint32_t *>(P.kstream + w.k_off + w.kpos);
            w.blk_n++;
            w.blk_bytes += e;
            if (restart) { w.nrest++; w.to_restart = RI; }
            w.to_restart--;
            w.prev_big = big ? 1u : 0u;
            const unsigned long long seq = ((unsigned long long)tr_hi << 24) | (tr_lo >> 8);
            if ((tr_lo & 0xffu) == PGS_TYPE_DELETION) w.n_tomb++;
            w.b_key += ulen;
            w.b_val += vlen;
            if (ulen > w.m_ukey) w.m_ukey = ulen;
            if (vlen > w.m_vlen) w.m_vlen = vlen;
            if (seq > w.m_seq) w.m_seq = seq;
            if (~seq > w.m_seq_inv) w.m_seq_inv = ~seq;
            const uint32_t pl = hashkey_prefix_len((const uint8_t *)row, ulen); // k_emit's bloom_add takes the prefix when aux < pl
            if (pl && aux < pl) w.n_prefix++;
            w.kpos += ks_record(0u, ulen);
            w.lenA = ulen;
            w.lcp = ulen;
        }
        g.sync(); // every lane has read the child's state
        if (route) {
            if (g.gl == 0) {
                if (WRITE) {
                    Desc d;
                    d.loc = desc_loc(cur_base(C) + C->voff, 0, ulen, flags);
                    d.vlen = vlen;
                    d.aux = aux;
                    *reinterpret_cast<uint4 *>(&P.desc[w.d_off + w.n]) = *reinterpret_cast<const uint4 *>(&d);
                    sp[0] = tr_lo;
                    sp[1] = tr_hi;
                }
                w.n++;
                ch[child] = w;
            }
            if (WRITE)
#pragma unroll 1
                for (uint32_t wd = g.gl; 4 * wd < ulen; wd += G) sp[2 + wd] = row[wd];
        }
        // (5) the previous key for the next record: from the first word the cursor may change (bytes below `shared` stay)
        if (act) {
            const uint32_t keep = have_prev ? (C->shared < plen ? C->shared : plen) : 0u;
#pragma unroll 1
            for (uint32_t wd = (keep >> 2) + g.gl; 4 * wd < ulen; wd += G) prow[wd] = row[wd];
            plen = ulen;
            have_prev = true;
        }
        g.sync();
        const uint32_t e3 = cur_next<G>(g, act && !err, r, C, row, KS);
        if (act && !err) err = e3;
    }

    // ---- the children's last blocks, what the segment gave each child --------------------------------------------------------
    if (seg_en) {
        for (uint32_t c = g.gl; c < NC; c += G) {
            SplitChild w = ch[c];
            if (!err && w.blk_n > 0) {
                const uint32_t size = block_bytes(w.blk_bytes, w.nrest);
                w.out_bytes += block_span(size);
                w.n_blocks++;
                w.keyb += w.lenA;
                if (size > w.m_bsize) w.m_bsize = size;
                if (w.blk_n > w.m_brec) w.m_brec = w.blk_n;
            }
            if (err) {
                atomicMax(&S.stats[c].error, err);
                atomicMin(&S.stats[c].error_seg, q);
                continue;
            }
            if (!WRITE) {
                SplitCount n;
                n.n = w.n; n.ks = w.kpos;
                S.cnt[(size_t)q * NC + c] = n;
                if (!w.n) continue;
                MergeStats &st = S.stats[c];
                atomicAdd(&st.cnt[EV_IN], (unsigned long long)w.n);
                atomicAdd(&st.cnt[EV_OUT], (unsigned long long)w.n);
                if (w.n_tomb) atomicAdd(&st.cnt[EV_OUT_TOMB], (unsigned long long)w.n_tomb);
                atomicAdd(&st.bytes[SB_IN], w.b_key + w.b_val);
                atomicAdd(&st.bytes[SB_OUT], w.b_key + w.b_val);
                atomicAdd(&st.bytes[SB_OUT_KEY], w.b_key);
                atomicAdd(&st.bytes[SB_OUT_VAL], w.b_val);
                atomicMax(&st.mx[SM_UKEY], (unsigned long long)w.m_ukey);
                atomicMax(&st.mx[SM_VLEN], (unsigned long long)w.m_vlen);
                atomicMax(&st.mx[SM_MAX_SEQ], w.m_seq);
                atomicMax(&st.mx[SM_MIN_SEQ_INV], w.m_seq_inv);
                atomicMax(&st.mx[SM_BLK_SIZE], (unsigned long long)w.m_bsize);
                atomicMax(&st.mx[SM_BLK_REC], (unsigned long long)w.m_brec);
                if (w.n_prefix) atomicAdd(&S.prefixes[c], (unsigned long long)w.n_prefix);
            } else {
                const SplitCount n = S.cnt[(size_t)q * NC + c];
                if (n.n != w.n || n.ks != w.kpos) { // the two passes disagree
                    atomicMax(&S.stats[c].error, (uint32_t)PGS_CORRUPTION);
                    atomicMin(&S.stats[c].error_seg, q);
                    continue;
                }
                SegAgg a;
                a.out_bytes = w.out_bytes; a.n_entries = w.n; a.n_blocks = w.n_blocks; a.keyb = w.keyb; a.ks_bytes = w.kpos; a.last_klen = w.lenA;
                a.pad = 0;
                S.agg[(size_t)c * Q + q] = a;
            }
        }
        if (!WRITE && !err && n_empty && g.gl == 0) atomicAdd(S.dropped, (unsigned long long)n_empty);
    }
    g.sync();
}

template <uint32_t G, bool WRITE>
__global__ void __launch_bounds__(kSplitThreads) k_split_walk(const __grid_constant__ SplitParams S)
{
    PGS_SMEM_DYN(dyn);
    const Grp<G> g;
    constexpr uint32_t NGW = 32 / G; // groups per warp
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long *crc = (unsigned long long *)dyn; // pegasus_key_hash's table, 2 KB
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) crc[i] = S.M.crc_table[i];
    if (__syncthreads_or(S.M.stats->error != 0)) return; // the planner rejected the layout
    const uint32_t gi = warp * NGW + g.shift / G;
    uint8_t *gs = dyn + 2048 + (size_t)gi * S.group_smem;
    SplitChild *ch = (SplitChild *)gs;
    CurState *C = (CurState *)(gs + (size_t)S.S * sizeof(SplitChild));
    uint32_t *row = (uint32_t *)((uint8_t *)C + ((sizeof(CurState) + 15) & ~(size_t)15));
    uint32_t *prow = row + S.M.KSW, *rowLO = prow + S.M.KSW, *rowHI = rowLO + S.M.KSW;
#pragma unroll 1
    for (;;) {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(S.M.ticket + (WRITE ? 2 : 0), NGW);
        t0 = __shfl_sync(kFull, t0, 0);
        if (t0 >= S.M.Q) break;
        const uint32_t q = t0 + g.shift / G;
        split_segment<G, WRITE>(S, g, q < S.M.Q, q < S.M.Q ? q : 0u, C, row, prow, rowLO, rowHI, ch, crc);
    }
}

typedef void (*split_kernel_t)(const SplitParams);
constexpr uint32_t kSplitGs[] = {4, 8, 16, 32};
inline split_kernel_t split_kernel(uint32_t G, bool write)
{
    switch (G) {
    case 4: return write ? k_split_walk<4, true> : k_split_walk<4, false>;
    case 8: return write ? k_split_walk<8, true> : k_split_walk<8, false>;
    case 16: return write ? k_split_walk<16, true> : k_split_walk<16, false>;
    default: return write ? k_split_walk<32, true> : k_split_walk<32, false>;
    }
}

// The launches of one parent run's split on stream st.  children == nullptr: the counting phase (k_plan, k_seg_bounds,
// k_seg_layout, k_split_walk<count>).  Otherwise the writing phase: k_split_walk<write>, then k_seg_scan and k_emit of each of
// the n_children children (their parameters from split_child).  walk_ctas / emit_ctas = CTAs the device runs at once.  mark(i)
// is called before the first launch (0), after the last (1) and, in the writing phase, after k_split_walk<write> (2).  Returns the number of launches.
template <class Mark>
inline uint32_t split_launch(const SplitParams &S, const SplitGeometry &geo, const MergeParams *children, const CompactGeometry *child_geo,
                             uint32_t n_children, uint64_t walk_ctas, uint64_t emit_ctas, cudaStream_t st, Mark &&mark)
{
    const uint32_t seg_per_cta = kSplitThreads / geo.G;
    const uint32_t grid_w = (uint32_t)std::min<uint64_t>((S.M.Q + seg_per_cta - 1) / seg_per_cta, walk_ctas);
    uint32_t n = 0;
    mark(0);
    if (!children) {
        PGS_LAUNCH(k_plan, (S.M.total_blocks + 255ull) / 256, 256, 0, st, S.M);
        PGS_LAUNCH(k_seg_bounds, (S.M.Q + 255ull) / 256, 256, 0, st, S.M);
        PGS_LAUNCH(k_seg_layout, 1, 1024, 0, st, S.M);
        PGS_LAUNCH(split_kernel(geo.G, false), grid_w, kSplitThreads, geo.walk_dyn, st, S);
        n = 4;
    } else {
        PGS_LAUNCH(split_kernel(geo.G, true), grid_w, kSplitThreads, geo.walk_dyn, st, S);
        mark(2);
        n = 1;
        for (uint32_t i = 0; i < n_children; i++) {
            const MergeParams &Pc = children[i];
            const uint32_t grid_e = (uint32_t)std::min<uint64_t>((Pc.Q + child_geo[i].emit_warps - 1) / child_geo[i].emit_warps, emit_ctas);
            PGS_LAUNCH(k_seg_scan, 1, 1024, 0, st, Pc);
            PGS_LAUNCH(k_emit, grid_e, child_geo[i].emit_warps * 32, child_geo[i].emit_dyn, st, Pc);
            n += 2;
        }
    }
    mark(1);
    return n;
}

// ================================================================================================================================
// Several splits in one launch (pgs_partition_split_many): every run of every parent partition of one engine is a job, planned
// with k = 1 by compaction's multi-job planner (compact_many_geometry, k_plan_many, k_seg_bounds_many, k_seg_layout_many), so
// one segment weight cuts every run.  k_split_walk_many numbers the jobs' segments one after the other, as k_walk_many does,
// and runs split_segment on each segment's job.  Every (parent run, built child) pair is then one job of k_seg_scan_many and
// k_emit_many.  The jobs share the launch's shape: the child count S (one app's split per call), and the key rows of the
// widest user key of any job, so that one group_smem serves the walker and every child's k_emit has the same stages.
// ================================================================================================================================
struct SplitJobs {
    const SplitParams *job;   // [n] in device memory
    const uint32_t *seg_base; // [n + 1]: job j's segments are the launch's segments [seg_base[j], seg_base[j + 1])
    uint32_t n, Q;
    uint32_t S, KSW, group_smem; // every job's
    const unsigned long long *crc_table;
    uint32_t *ticket;             // [0] counting walk, [1] writing walk, [2..3] the children's MergeJobs::ticket
    MergeStats *stats;            // [n * S]: job j's children at j * S (its SplitParams::stats), as are prefixes
    unsigned long long *prefixes; // [n * S]
    unsigned long long *dropped;  // [n]
};

// k_split_walk over the segments of every job.  The groups of a warp may draw segments of different jobs: a group reads its
// job's SplitParams (and the run table inside it) through the L1 cache, where k_split_walk has its one job as a kernel
// parameter.  A job whose plan failed is not walked.
template <uint32_t G, bool WRITE>
__global__ void __launch_bounds__(kSplitThreads) k_split_walk_many(const __grid_constant__ SplitJobs J)
{
    PGS_SMEM_DYN(dyn);
    const Grp<G> g;
    constexpr uint32_t NGW = 32 / G; // groups per warp
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long *crc = (unsigned long long *)dyn; // pegasus_key_hash's table, 2 KB
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) crc[i] = J.crc_table[i];
    __syncthreads();
    const uint32_t gi = warp * NGW + g.shift / G;
    uint8_t *gs = dyn + 2048 + (size_t)gi * J.group_smem;
    SplitChild *ch = (SplitChild *)gs;
    CurState *C = (CurState *)(gs + (size_t)J.S * sizeof(SplitChild));
    uint32_t *row = (uint32_t *)((uint8_t *)C + ((sizeof(CurState) + 15) & ~(size_t)15));
    uint32_t *prow = row + J.KSW, *rowLO = prow + J.KSW, *rowHI = rowLO + J.KSW;
#pragma unroll 1
    for (;;) {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(J.ticket + (WRITE ? 1 : 0), NGW);
        t0 = __shfl_sync(kFull, t0, 0);
        if (t0 >= J.Q) break;
        const uint32_t q = t0 + g.shift / G;
        const uint32_t j = q < J.Q ? job_of(J.seg_base, J.n, q) : 0u;
        const SplitParams &S = J.job[j];
        const uint32_t failed = g.shfl(g.gl == 0 ? S.M.stats->error : 0u, 0); // one lane reads the flag for the group
        const bool en = q < J.Q && failed == 0;
        split_segment<G, WRITE>(S, g, en, en ? q - J.seg_base[j] : 0u, C, row, prow, rowLO, rowHI, ch, crc);
    }
}

typedef void (*split_many_kernel_t)(const SplitJobs);
inline split_many_kernel_t split_many_kernel(uint32_t G, bool write)
{
    switch (G) {
    case 4: return write ? k_split_walk_many<4, true> : k_split_walk_many<4, false>;
    case 8: return write ? k_split_walk_many<8, true> : k_split_walk_many<8, false>;
    case 16: return write ? k_split_walk_many<16, true> : k_split_walk_many<16, false>;
    default: return write ? k_split_walk_many<32, true> : k_split_walk_many<32, false>;
    }
}

// The joint plan of n parent runs (host side).  S[i] holds job i's run (M.runs[0]), block_size, restart_interval, S, counts and
// want; T[i] its run's totals.  compact_many_geometry sizes every job's key rows by the widest user key and cuts every run by
// one segment weight from the whole launch's weight (walk_groups = split groups the device runs at once, 0: not known yet;
// force_weight overrides it); then the narrowest split group that fits, as split_plan chooses it.  J and M (the planner
// kernels' jobs) get the launch's counts and shape, no pointers.  Returns a status: PGS_NOT_SUPPORTED when the jobs do not fit
// one launch (the caller can split them).
inline int32_t split_many_plan(SplitParams *S, const CompactTotals *T, uint32_t n, uint32_t max_smem, SplitJobs &J, MergeJobs &M,
                               SplitGeometry &geo, uint64_t walk_groups = 0, uint64_t force_weight = 0)
{
    if (n == 0 || n > kMaxCompactJobs) return PGS_NOT_SUPPORTED;
    const uint32_t NC = S[0].S;
    if (NC < 2 || NC > kSplitMaxChildren) return PGS_NOT_SUPPORTED;
    std::vector<MergeParams> P(n);
    std::vector<CompactGeometry> cg(n);
    for (uint32_t i = 0; i < n; i++) {
        if (S[i].S != NC) return PGS_INVALID_ARGUMENT;
        if (T[i].max_ukey > kMaxUkeyLen) return PGS_NOT_SUPPORTED;
        S[i].M.k = 1;
        P[i] = S[i].M;
    }
    if (!compact_many_geometry(P.data(), T, cg.data(), n, max_smem, M, geo.cg, 0, force_weight, walk_groups)) return PGS_NOT_SUPPORTED;
    for (uint32_t i = 0; i < n; i++) {
        S[i].M = P[i];
        S[i].group_smem = split_group_smem(NC, P[i].KSW);
    }
    const uint32_t group_smem = S[0].group_smem;
    geo.G = 0;
    for (uint32_t G = 4; G <= 32 && !geo.G; G *= 2) // as split_plan
        if (split_dyn_smem(G, group_smem) <= max_smem / 2) geo.G = G;
    for (uint32_t G = 4; G <= 32 && !geo.G; G *= 2)
        if (split_dyn_smem(G, group_smem) <= max_smem) geo.G = G;
    if (!geo.G) return PGS_NOT_SUPPORTED;
    geo.walk_dyn = (uint32_t)split_dyn_smem(geo.G, group_smem);
    J.n = n;
    J.Q = M.Q;
    J.S = NC;
    J.KSW = S[0].M.KSW;
    J.group_smem = group_smem;
    return PGS_OK;
}

// The scratch of a joint split, every buffer through buf(pointer, elements, fill, out = false) as split_buffers hands them out.
// buf may place them later (the library's one allocation): nothing here reads a pointer it was given.
template <class F>
inline void split_many_buffers(SplitParams *S, uint32_t n, SplitJobs &J, F &&buf)
{
    const uint64_t C = J.S;
    buf(J.ticket, 4, 0, false);
    buf(J.stats, n * C, kNoFill, false); // the caller sets every one to merge_stats_init()
    buf(J.prefixes, n * C, 0, false);
    buf(J.dropped, n, 0, false);
    for (uint32_t i = 0; i < n; i++) split_scratch(S[i], buf);
}

// The counting phase's tables of a joint split, once split_many_buffers' buffers are placed: every job gets its slice of the
// launch's counters, job[i] = S[i].M (the planner kernels' jobs), and seg_base / blk_base their prefixes (compact_many_bases).
inline void split_many_tables(SplitParams *S, uint32_t n, const SplitJobs &J, MergeParams *job, uint32_t *seg_base, uint32_t *blk_base)
{
    const uint64_t C = J.S;
    for (uint32_t i = 0; i < n; i++) {
        S[i].stats = J.stats + i * C;
        S[i].prefixes = J.prefixes + i * C;
        S[i].dropped = J.dropped + i;
        S[i].M.stats = S[i].stats;
        S[i].M.ticket = nullptr; // the launch's tickets are J's
        job[i] = S[i].M;
    }
    compact_many_bases(job, n, seg_base, blk_base);
}

// Child c of job S's k_seg_scan_many / k_emit_many parameters: split_child and split_child_scratch, and the emit shape every
// child of the launch shares (shape = the first child's; false: this child's differs, or split_child refuses it).
inline bool split_many_child(const SplitParams &S, uint32_t c, const MergeStats &st, unsigned long long prefixes, uint32_t max_smem,
                             MergeParams &Pc, CompactGeometry &geo, CompactTotals &T, const MergeParams *shape, const CompactGeometry *shape_geo)
{
    if (!split_child(S, st, prefixes, max_smem, Pc, geo, T)) return false;
    split_child_scratch(S, c, Pc);
    Pc.ticket = nullptr; // k_emit_many draws from MergeJobs::ticket
    return !shape || (Pc.KS == shape->KS && Pc.blk_buf == shape->blk_buf && Pc.emit_warp_smem == shape->emit_warp_smem &&
                      Pc.emit_obuf == shape->emit_obuf && Pc.ks_stage == shape->ks_stage && geo.emit_warps == shape_geo->emit_warps &&
                      geo.emit_dyn == shape_geo->emit_dyn);
}

// The children of a joint split after its counting pass (st, prefixes: [n * S] as read back): every (job x, child c) that is
// built and got records, in that order, becomes one job of k_emit_many -- Pc its parameters, emit_base [Pc.size() + 1] the
// prefixes of their segments, shape the emit shape they share.  out(x, c, P, geo, T) gives the child's run its buffers
// (compact_buffers' `out` ones) and returns false to stop.  Returns false when a child is refused (at = x * S + c) or out stopped.
template <class Out>
inline bool split_many_children(const SplitParams *S, uint32_t n, const MergeStats *st, const unsigned long long *prefixes, uint32_t max_smem,
                                std::vector<MergeParams> &Pc, std::vector<uint32_t> &emit_base, CompactGeometry &shape, uint64_t &at, Out &&out)
{
    const uint32_t NC = n ? S[0].S : 0;
    emit_base.assign(1, 0);
    for (uint32_t x = 0; x < n; x++)
        for (uint32_t c = 0; c < NC; c++) {
            at = (uint64_t)x * NC + c;
            if (!((S[x].want >> c) & 1u) || st[at].cnt[EV_OUT] == 0) continue;
            MergeParams P{};
            CompactGeometry g{};
            CompactTotals T{};
            if (!split_many_child(S[x], c, st[at], prefixes[at], max_smem, P, g, T, Pc.empty() ? nullptr : &Pc[0], &shape)) return false;
            if (!out(x, c, P, g, T)) return false;
            if (Pc.empty()) shape = g;
            Pc.push_back(P);
            emit_base.push_back(emit_base.back() + P.Q);
        }
    return true;
}

// The launches of a joint split on stream st.  emit == nullptr: the counting phase (k_plan_many, k_seg_bounds_many,
// k_seg_layout_many over the planner's jobs M, then k_split_walk_many<count>).  Otherwise the writing phase:
// k_split_walk_many<write>, then k_seg_scan_many and k_emit_many over the children (*emit, every child's shape emit_geo).
// walk_ctas / emit_ctas = CTAs the device runs at once.  mark(i) as split_launch.  Returns the number of launches.
template <class Mark>
inline uint32_t split_many_launch(const SplitJobs &J, const MergeJobs &M, const SplitGeometry &geo, const MergeJobs *emit,
                                  const CompactGeometry &emit_geo, uint64_t walk_ctas, uint64_t emit_ctas, cudaStream_t st, Mark &&mark)
{
    const uint32_t seg_per_cta = kSplitThreads / geo.G;
    const uint32_t grid_w = (uint32_t)std::min<uint64_t>((J.Q + seg_per_cta - 1) / seg_per_cta, walk_ctas);
    uint32_t n = 0;
    mark(0);
    if (!emit) {
        PGS_LAUNCH(k_plan_many, std::max(1ull, (M.total_blocks + 255ull) / 256), 256, 0, st, M);
        PGS_LAUNCH(k_seg_bounds_many, (M.Q + 255ull) / 256, 256, 0, st, M);
        PGS_LAUNCH(k_seg_layout_many, M.n, 1024, 0, st, M);
        PGS_LAUNCH(split_many_kernel(geo.G, false), grid_w, kSplitThreads, geo.walk_dyn, st, J);
        n = 4;
    } else {
        PGS_LAUNCH(split_many_kernel(geo.G, true), grid_w, kSplitThreads, geo.walk_dyn, st, J);
        mark(2);
        const uint32_t grid_e = (uint32_t)std::min<uint64_t>((emit->Q + emit_geo.emit_warps - 1) / emit_geo.emit_warps, emit_ctas);
        PGS_LAUNCH(k_seg_scan_many, emit->n, 1024, 0, st, *emit);
        PGS_LAUNCH(k_emit_many, grid_e, emit_geo.emit_warps * 32, emit_geo.emit_dyn, st, *emit);
        n = 3;
    }
    mark(1);
    return n;
}

} // namespace pgs
