// compact_kernels.cuh — level compaction on the GPU: k-way merge of HBM-resident sorted runs with
// KeyWithTTLCompactionFilter fused into the merge loop.
//
// Replaces (reference file:line):
//   DB::CompactRange / background compaction job ....... src/server/pegasus_server_impl.cpp:3373-3394
//   RocksDB MergingIterator + CompactionIterator + BlockBasedTableBuilder (v8.5.3, not in tree;
//   semantics restated in SURVEY.md Appendix A)
//   KeyWithTTLCompactionFilter::Filter .................. src/server/key_ttl_compaction_filter.h:55-121
//   compaction_operation / compaction_filter_rule ....... src/server/compaction_operation.cpp:33-113,
//                                                         src/server/compaction_filter_rule.cpp:31-90
//
// Shape of the computation (byte/integer work bound by HBM, no tensor cores):
//   k_plan        one thread per input block ranks the block's last user key against every run's block index
//                 => cumulative weight of everything <= that key.  Keys where the weight crosses a multiple of the
//                 segment budget become segment boundaries: segment q = user keys in (U_q, U_q+1], a contiguous
//                 block range per run.  All versions of a user key fall into one segment.
//   k_walk        the merge itself.  A *group* of G lanes (4 by default, 1 to 16) owns one segment and walks it
//                 sequentially like RocksDB's MergingIterator + CompactionIterator: one cursor per run, whose next entry's
//                 head (header, key delta, trailer, expire_ts) is fetched into a 96-byte shared-memory window while the
//                 current one is handled, in the same block or across into the next (group.cuh, kHeadWin), so a merge step
//                 waits for no global load of its own; the current keys in shared-memory rows compared with one ballot, newest
//                 version wins, tombstone / bottommost rules, Filter() per surviving value, prefix compression against the
//                 previous survivor, 4 KB block cuts.  It copies no values: per survivor it emits a 16-byte descriptor
//                 (where the value lives, lengths, flags) and a key-stream record (trailer | rewritten expire_ts | user key).
//                 32/G groups share a warp in lock step; there is no block-wide barrier anywhere.
//   k_seg_scan    exclusive prefix of the per-segment output sizes (bytes, blocks, records, index-key bytes).
//   k_emit        one warp per segment builds the output blocks in batches of up to 32 entries, one thread per entry:
//                 a batch's key-stream records and values arrive in shared-memory stages by bulk TMA copies (one wait per
//                 batch), entry heads and values are assembled byte-exact in an output buffer together with the restart
//                 arrays and padding of the blocks that close, and each batch leaves with one bulk TMA store; the new
//                 run's index and Bloom filter are written alongside.
//   Output blocks stay contiguous and in key order; every segment starts a new block.
#pragma once
#include <algorithm>

#include "group.cuh"

namespace pgs {

constexpr uint32_t kSegRecCost = 256;          // planner weight = block bytes + 256 per record
constexpr uint64_t kSegWeight = 128ull << 10;  // default segment budget (about 240 records of 300 bytes)
constexpr uint64_t kSegWeightMax = 4ull << 20, kSegWeightMin = 16ull << 10;   // bounds of the wave-fitted budget
constexpr uint32_t kWalkThreads = 128;
constexpr uint32_t kEmitThreads = 128;

enum : uint32_t { DF_NEWBLOCK = 1, DF_REWRITE = 2, DF_BIG = 4 };

// ---- what k_walk hands to k_emit ---------------------------------------------------------------------------------------------
// One descriptor per surviving record.
struct __align__(16) Desc {
    unsigned long long loc; // bits 0..39 byte offset of the value inside its run, 40..43 run, 44..59 user-key bytes, 60..63 DF_*
    uint32_t vlen;          // value bytes to copy (0 for a tombstone)
    uint32_t aux;           // bytes the user key shares with the previous survivor of the segment
};
static_assert(sizeof(Desc) == 16, "Desc");
PGS_HD unsigned long long desc_loc(unsigned long long voff, unsigned long long run, unsigned long long ulen, unsigned long long flags)
{
    return voff | (run << 40) | (ulen << 44) | (flags << 60);
}
PGS_HD unsigned long long desc_voff(unsigned long long loc) { return loc & ((1ull << 40) - 1); }
PGS_HD uint32_t desc_run(unsigned long long loc) { return (uint32_t)(loc >> 40) & 15u; }
PGS_HD uint32_t desc_ulen(unsigned long long loc) { return (uint32_t)(loc >> 44) & 0xffffu; }
PGS_HD uint32_t desc_flags(unsigned long long loc) { return (uint32_t)(loc >> 60); }

// One record per survivor in its segment's key stream: trailer (8 bytes) | the rewritten expire_ts (BE32, only with DF_REWRITE) |
// the whole user key, padded to 4 bytes.  k_emit builds the entry head, the index key and the Bloom filter bits from it.
PGS_HD uint32_t ks_fixed(uint32_t flags) { return (flags & DF_REWRITE) ? 12u : 8u; }
PGS_HD uint32_t ks_record(uint32_t flags, uint32_t ulen) { return ks_fixed(flags) + ((ulen + 3) & ~3u); }
// the key-stream bytes planned per input record for user keys of at most KS bytes (more than ks_record(DF_REWRITE, KS))
PGS_HD uint32_t ks_record_bound(uint32_t KS) { return 15 + KS + 8 + 4; }

// An output block: entries, then the restart array (one 4-byte offset per restart point) and its 4-byte count, padded to
// kBlockAlign.  An entry is varint shared | varint non_shared (= key delta + 8) | varint value length | key delta | trailer | value.
PGS_HD uint32_t entry_head_len(uint32_t shared, uint32_t kd, uint32_t vlen) { return varint_len(shared) + varint_len(kd + 8) + varint_len(vlen) + kd + 8; }
PGS_HD uint32_t block_bytes(uint32_t entry_bytes, uint32_t nrest) { return entry_bytes + 4 * (nrest + 1); }
PGS_HD uint32_t block_span(uint32_t size) { return (size + kBlockAlign - 1) & ~(kBlockAlign - 1); }
PGS_HD uint32_t restart_count(uint32_t n, uint32_t RI) { return (n + RI - 1) / RI; } // restart points of n entries
// the three varints of an entry head at p; returns their bytes
PGS_DEV uint32_t put_entry_varints(uint8_t *p, uint32_t shared, uint32_t kd, uint32_t vlen)
{
    uint32_t n = put_varint32_s(p, shared);
    n += put_varint32_s(p + n, kd + 8);
    return n + put_varint32_s(p + n, vlen);
}

struct SegLayout { // where a segment's scratch lives (k_seg_layout)
    unsigned long long desc_off; // index of its first descriptor
    unsigned long long ks_off;   // byte offset of its key stream
};
struct __align__(16) SegAgg { // what a segment produced (k_walk)
    unsigned long long out_bytes; // sum of 16-aligned block sizes
    uint32_t n_entries, n_blocks, keyb, ks_bytes, last_klen, pad;
};
struct __align__(16) SegBase { // exclusive prefixes over the segments (k_seg_scan)
    unsigned long long bytes;
    uint32_t blocks, recs, keyb, pad;
};

// counters of one compaction.  k_walk keeps them in registers per group, adds them up per CTA in shared memory and adds the
// CTA's totals here.
struct MergeStats {
    unsigned long long cnt[16];  // EV_*
    unsigned long long bytes[4]; // SB_*
    unsigned long long mx[8];    // SM_* (maxima; the smallest sequence number is kept as the maximum of its complement)
    unsigned long long tot_bytes, tot_blocks, tot_recs, tot_keyb; // k_seg_scan
    uint32_t error, error_seg;
};
enum { EV_IN = 0, EV_OUT, EV_SHADOW, EV_TOMB, EV_EXPIRED, EV_USER, EV_STALE, EV_TTL, EV_OUT_TOMB, EV_BLOOM_KEY, EV_BLOOM_PREFIX };
enum { SB_IN = 0, SB_OUT, SB_OUT_KEY, SB_OUT_VAL };
enum { SM_UKEY = 0, SM_VLEN, SM_MAX_SEQ, SM_MIN_SEQ_INV, SM_BLK_SIZE, SM_BLK_REC };

struct MergeParams {
    RunDev runs[kMaxRuns];
    uint32_t k;
    // plan
    uint32_t *split_pos; // [(Q+1)*k]
    uint32_t *split_ref; // [Q+1]  run<<28 | block
    uint32_t Q;
    unsigned long long tile_weight;
    uint32_t rec_cost;
    uint32_t total_blocks;
    // scratch
    SegLayout *seg;
    SegAgg *agg;
    SegBase *base;
    Desc *desc;
    uint8_t *kstream; // the segments' key streams
    unsigned long long desc_cap, ks_cap;
    uint32_t *ticket; // [0] k_walk, [1] k_emit
    uint32_t KS;      // user-key capacity of a key row (multiple of 4)
    uint32_t KSW;     // 32-bit words per key row
    uint32_t group_smem, emit_warp_smem, emit_obuf, blk_buf, ks_stage;
    // filter + policy
    uint32_t now, enabled, validate_hash, data_version, default_ttl;
    int32_t pidx, partition_version;
    const uint8_t *ops;
    uint32_t n_ops;
    uint32_t bottommost, block_size, restart_interval;
    const unsigned long long *crc_table;
    // output run
    uint8_t *out_data;
    unsigned long long out_cap;
    unsigned long long *out_blk_off;
    uint32_t *out_blk_size, *out_blk_rec, *out_ikey_off, *out_rec_off;
    uint8_t *out_ikeys;
    uint32_t out_blk_cap, out_ikey_cap;
    unsigned long long out_rec_cap;
    uint32_t *out_bloom; // the new run's Bloom filter (zeroed by the host), out_bloom_lines lines of 64 bytes
    uint32_t out_bloom_lines;
    MergeStats *stats;
    uint32_t emit_vstage; // k_emit's value stage per warp (bytes)
};

// ---- launch geometry and buffer bounds (host side; shared with the CPU simulation driver under tools/simt) -----------------
struct CompactTotals { // sums / maxima over the input runs' pgs_run_info
    uint32_t max_ukey, max_blk, max_blk_rec;
    uint64_t total_blocks, n_rec, raw_key, raw_val, in_block_bytes;
    uint64_t bloom_entries; // sizes the output's Bloom filter
    // n_bloom_entries: what went into the input's filter (0: not known, two per record are assumed)
    void add(const pgs_run_info &fi, uint64_t n_bloom_entries)
    {
        max_ukey = std::max(max_ukey, fi.max_ukey_len);
        max_blk = std::max(max_blk, fi.max_block_size);
        max_blk_rec = std::max(max_blk_rec, fi.max_block_records);
        total_blocks += fi.n_blocks;
        n_rec += fi.n_records;
        raw_key += fi.raw_key_bytes;
        raw_val += fi.raw_value_bytes;
        in_block_bytes += fi.data_bytes;
        bloom_entries += n_bloom_entries ? n_bloom_entries : 2 * fi.n_records;
    }
};
// a finished merge's counters as pgs_compact_result reports them, and the merged run's pgs_run_info (without level and run
// id); returns the entries of the merged run's Bloom filter
inline uint64_t compact_result_stats(const MergeStats &s, uint64_t in_block_bytes, pgs_compact_result &res, pgs_run_info &info)
{
    res.in_records = s.cnt[EV_IN]; res.out_records = s.cnt[EV_OUT];
    res.in_bytes = s.bytes[SB_IN]; res.out_bytes = s.bytes[SB_OUT];
    res.in_block_bytes = in_block_bytes; res.out_block_bytes = s.tot_bytes;
    res.dropped_shadowed = s.cnt[EV_SHADOW]; res.dropped_tombstone = s.cnt[EV_TOMB];
    res.dropped_expired = s.cnt[EV_EXPIRED]; res.dropped_user = s.cnt[EV_USER]; res.dropped_stale = s.cnt[EV_STALE];
    res.ttl_rewritten = s.cnt[EV_TTL];
    info.n_blocks = (uint32_t)s.tot_blocks;
    info.n_records = s.tot_recs;
    info.n_tombstones = s.cnt[EV_OUT_TOMB];
    info.data_bytes = s.tot_bytes;
    info.raw_key_bytes = s.bytes[SB_OUT_KEY];
    info.raw_value_bytes = s.bytes[SB_OUT_VAL];
    info.max_ukey_len = (uint32_t)s.mx[SM_UKEY];
    info.max_value_len = (uint32_t)s.mx[SM_VLEN];
    info.max_block_size = (uint32_t)s.mx[SM_BLK_SIZE];
    info.max_block_records = (uint32_t)s.mx[SM_BLK_REC];
    info.smallest_seq = s.tot_recs ? (~s.mx[SM_MIN_SEQ_INV] & ((1ull << 56) - 1)) : ~0ull;
    info.largest_seq = s.mx[SM_MAX_SEQ];
    return s.cnt[EV_BLOOM_KEY] + s.cnt[EV_BLOOM_PREFIX];
}
struct CompactGeometry {
    uint32_t G, walk_dyn, emit_warps, emit_dyn;
    uint64_t blk_cap, out_cap, ikey_cap;
};
struct WalkCtaStats { // k_walk's per-CTA totals, shared memory
    uint32_t cnt[12];
    unsigned long long bytes[4];
    unsigned long long mx[6];
};
// k_walk's CTA-wide shared memory in front of the groups': crc table (2 KB), run table, WalkCtaStats
constexpr uint32_t kWalkFixedSmem = 2048 + kMaxRuns * (uint32_t)sizeof(RunDev) + (uint32_t)sizeof(WalkCtaStats);
// Behind the groups' states and key rows: each group's head windows (group.cuh, kHeadWin), one per run, 16-aligned.  The
// extra 16 bytes per group put the windows of the groups of a warp in different banks.
PGS_HD uint32_t walk_win_stride(uint32_t k) { return k * kHeadWin + 16; }
PGS_HD uint32_t walk_win_off(uint32_t G, uint32_t group_smem) { return (kWalkFixedSmem + (kWalkThreads / G) * group_smem + 15) & ~15u; }
PGS_HD uint64_t walk_dyn_smem(uint32_t G, uint32_t group_smem, uint32_t k)
{
    return walk_win_off(G, group_smem) + (uint64_t)(kWalkThreads / G) * walk_win_stride(k);
}
// k_walk_many (several jobs per launch) has no CTA-wide run table: a group reads its job's runs through the cache, and keeps
// its counters in a WalkCtaStats of its own, which it hands to its job's MergeStats after every segment.  Its layout: crc table
// (2 KB) | one WalkCtaStats per group | the groups' states and key rows | their head windows.
PGS_HD uint32_t walk_many_fixed_smem(uint32_t G) { return 2048 + (kWalkThreads / G) * (uint32_t)sizeof(WalkCtaStats); }
PGS_HD uint32_t walk_many_win_off(uint32_t G, uint32_t group_smem) { return (walk_many_fixed_smem(G) + (kWalkThreads / G) * group_smem + 15) & ~15u; }
PGS_HD uint64_t walk_many_dyn_smem(uint32_t G, uint32_t group_smem, uint32_t k)
{
    return walk_many_win_off(G, group_smem) + (uint64_t)(kWalkThreads / G) * walk_win_stride(k);
}
// k_emit's shared memory per warp, every part 16-aligned: output buffer (ob) | key-stream stage (ks) | value stage (vs) | the
// stages' mbarrier | restart offsets.  The 32 bytes behind each buffer take the whole 16-byte chunks read or written past its end.
PGS_HD uint32_t emit_vs_off(uint32_t ob, uint32_t ks) { return ob + 32 + ks + 32; }
PGS_HD uint32_t emit_bar_off(uint32_t ob, uint32_t ks, uint32_t vs) { return emit_vs_off(ob, ks) + vs + 32; }
PGS_HD uint32_t emit_rst_off(uint32_t ob, uint32_t ks, uint32_t vs) { return emit_bar_off(ob, ks, vs) + 16; }
// The output buffer for a block buffer of bb bytes: at least one entry + the restart array of the block it closes, normally
// 8 KB (a batch of ~28 entries).  The value stage is as large: it holds the 16-byte span of any entry's value (at most bb + 30
// bytes) and rarely ends a batch before the output buffer does.  Returns k_emit's shared memory per warp (bb, ks < 2^24).
PGS_HD uint32_t emit_warp_layout(uint32_t bb, uint32_t RI, uint32_t ks, uint32_t &ob)
{
    const uint32_t rst = 4 * (bb / (11 * RI) + 4); // the restart offsets of an open block (entries of at least 11 bytes)
    const uint32_t ob_min = bb + rst + 256;
    ob = ob_min < 8192 ? 8192u : ((ob_min + 15) & ~15u);
    return (emit_rst_off(ob, ks, ob) + rst + 15) & ~15u;
}
// fills the derived fields of P (P.k, P.block_size, P.restart_interval must be set); false = not supported
constexpr uint32_t kWalkMinG = 4; // default lanes per merge group (see group.cuh)
// walk_groups = merge groups the device runs at the same time (0: not known yet, the default segment budget is used);
// force_Q = the segment count of a plan made elsewhere (a partition split's child is emitted over its parent's segments);
// many = the shared memory of k_walk_many rather than k_walk's
inline bool compact_geometry(MergeParams &P, const CompactTotals &T, uint32_t max_smem, CompactGeometry &geo, uint32_t force_G = 0,
                             uint64_t force_weight = 0, uint64_t walk_groups = 0, uint32_t force_Q = 0, bool many = false)
{
    const uint32_t k = P.k;
    auto walk_dyn_smem = [many](uint32_t G, uint32_t group_smem, uint32_t k) {
        return many ? walk_many_dyn_smem(G, group_smem, k) : pgs::walk_dyn_smem(G, group_smem, k);
    };
    P.total_blocks = (uint32_t)T.total_blocks;
    P.KS = T.max_ukey < 4 ? 4u : ((T.max_ukey + 3) & ~3u);
    P.KSW = (P.KS + 8) / 4 + 1;
    // one group's shared memory: cursor states + key rows; an odd number of words, so that the groups of a warp start in
    // different banks
    P.group_smem = (uint32_t)(k * sizeof(CurState) + (size_t)(k + 4) * P.KSW * 4);
    if ((P.group_smem / 4) % 2 == 0) P.group_smem += 4;
    // lanes per group: the narrowest shape whose CTA fits shared memory twice per SM (or once); force_G overrides (diagnostics)
    geo.G = 0;
    for (uint32_t G = force_G ? force_G : kWalkMinG; G <= 16 && !geo.G; G *= 2) {
        const uint64_t dyn = walk_dyn_smem(G, P.group_smem, k);
        if (dyn <= max_smem / 2 || (force_G && dyn <= max_smem)) geo.G = G;
    }
    for (uint32_t G = kWalkMinG; G <= 16 && !geo.G; G *= 2)
        if (walk_dyn_smem(G, P.group_smem, k) <= max_smem) geo.G = G;
    if (!geo.G) return false;
    geo.walk_dyn = (uint32_t)walk_dyn_smem(geo.G, P.group_smem, k);
    const uint32_t hs = (2 * P.KS + 64 + 15) & ~15u;
    P.ks_stage = hs < 2048 ? 2048u : hs;
    // k_emit per warp (emit_warp_layout): output buffer, key-stream stage, value stage, the stages' mbarrier, the restart offsets
    // of the open block.  An entry that does not fit a block buffer gets a block of its own, written in place.
    const uint32_t RI = P.restart_interval;
    uint32_t blk_buf = (uint32_t)std::min<uint64_t>((P.block_size + 24ull + 15) & ~15ull, max_smem & ~15u), ob = 0;
    if (P.ks_stage > max_smem || emit_warp_layout(blk_buf, RI, P.ks_stage, ob) > max_smem) {
        // huge block_size: cut smaller blocks, to the largest block buffer whose warp fits shared memory
        uint32_t lo = 0, hi = blk_buf / 16; // lo * 16 fits (or is 0), hi * 16 does not
        while (hi - lo > 1) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (emit_warp_layout(mid * 16, RI, P.ks_stage, ob) <= max_smem) lo = mid; else hi = mid;
        }
        if (lo * 16 < 1024) return false;
        blk_buf = lo * 16;
        if (P.block_size > blk_buf - 24) P.block_size = blk_buf - 24;
    }
    P.blk_buf = blk_buf;
    P.emit_warp_smem = emit_warp_layout(blk_buf, RI, P.ks_stage, P.emit_obuf);
    P.emit_vstage = P.emit_obuf;
    // warps per CTA: the most (up to 4) that fit shared memory once, unless CTAs that fit twice per SM run more warps in all
    // (large blocks: two CTAs of 3 warps rather than one of 4)
    const uint32_t w_once = std::min(max_smem / P.emit_warp_smem, kEmitThreads / 32);
    const uint32_t w_twice = std::min((max_smem / 2) / P.emit_warp_smem, kEmitThreads / 32);
    geo.emit_warps = 2 * w_twice > w_once ? w_twice : w_once;
    if (geo.emit_warps == 0) return false;
    geo.emit_dyn = geo.emit_warps * P.emit_warp_smem;
    // segments
    P.rec_cost = kSegRecCost;
    const uint64_t W_total = T.in_block_bytes + T.n_rec * P.rec_cost;
    P.tile_weight = kSegWeight;
    if (walk_groups) {
        // A group walks its segments one after the other and a segment is a sequential job: the walk takes (waves of
        // segments) x (time of a segment), and a last, partly filled wave costs as much as a full one.  Size the segments
        // so that they fill a whole number of waves -- one wave whenever a segment stays under kSegWeightMax: every segment
        // pays for opening its cursors and skipping into its range, so fewer and longer ones are cheaper.  Small inputs
        // get one wave of short segments.
        const uint64_t waves = (W_total + kSegWeightMax * walk_groups - 1) / (kSegWeightMax * walk_groups);
        const uint64_t slots = (waves ? waves : 1) * walk_groups;
        uint64_t w = (W_total + slots - 1) / slots;
        w += w / 64; // the planner cuts at block boundaries: keep the segment count just under the slot count
        P.tile_weight = w < kSegWeightMin ? kSegWeightMin : w;
    }
    if (force_weight) P.tile_weight = force_weight;
    uint64_t Q = (W_total + P.tile_weight - 1) / P.tile_weight;
    if (Q == 0) Q = 1;
    if (force_Q) Q = force_Q;
    if (Q > 0x7FFFFFF0ull) return false;
    P.Q = (uint32_t)Q;
    // output capacity (every segment starts a new block; two neighbouring blocks of a segment hold more than block_size bytes)
    const uint64_t raw_total = T.raw_key + T.raw_val + 23 * T.n_rec;
    geo.blk_cap = 2 * (raw_total / P.block_size) + Q + 2;
    uint64_t out_cap = raw_total + 19 * geo.blk_cap + 4 * (T.n_rec / RI + geo.blk_cap) + 256;
    geo.out_cap = (out_cap + 255) & ~255ull;
    uint64_t ik = geo.blk_cap * (uint64_t)(T.max_ukey ? T.max_ukey : 1);
    if (ik > T.raw_key) ik = T.raw_key;
    geo.ikey_cap = ik + 16;
    if (geo.blk_cap > 0xFFFFFFF0ull || geo.ikey_cap > 0xFFFFFFF0ull || T.n_rec > 0xFFFFFFF0ull) return false;
    P.out_cap = geo.out_cap;
    P.out_blk_cap = (uint32_t)geo.blk_cap;
    P.out_ikey_cap = (uint32_t)geo.ikey_cap;
    P.out_rec_cap = T.n_rec;
    // scratch: the blocks on a segment boundary are read by both neighbours
    const uint64_t Nb = T.n_rec + Q * k * (uint64_t)T.max_blk_rec;
    const uint64_t Bb = T.in_block_bytes + Q * k * ((uint64_t)T.max_blk + 16);
    const uint64_t per_rec = ks_record_bound(P.KS);
    P.desc_cap = Nb + 1;
    P.ks_cap = Nb * per_rec + (2 * (Bb + Nb * per_rec) / P.block_size + 2 * Q + 2) * (uint64_t)(P.KS + 8) + 64 * Q + 64;
    P.out_bloom_lines = bloom_lines_for(T.bloom_entries);
    return true;
}

// the shared memory a compaction launch is planned for: the device's opt-in maximum per CTA less 1 KB (226 KB on an H100)
inline uint32_t compact_smem_budget(uint32_t max_smem_optin) { return max_smem_optin - 1024; }

// the filter and policy fields of P from the caller's filter parameters (nullptr: no filter); ops_len = how many bytes of
// fp->ops the launch needs in device memory at P.ops (0: no user ops).  Returns false, and nothing may be launched, when
// fp->ops is not a well-formed ops table (ops_table_valid).
inline bool compact_filter(MergeParams &P, const pgs_filter_params *fp, uint32_t &ops_len)
{
    ops_len = 0;
    if (!fp) return true;
    P.enabled = fp->enabled;
    P.validate_hash = fp->validate_hash;
    P.default_ttl = fp->default_ttl;
    P.pidx = fp->pidx;
    P.partition_version = fp->partition_version;
    if (!fp->ops || fp->ops_len == 0) return true;
    if (!ops_table_valid(fp->ops, fp->ops_len)) return false;
    memcpy(&P.n_ops, fp->ops, 4);
    ops_len = fp->ops_len;
    return true;
}

// One compaction job's MergeParams and CompactTotals from its k input runs (run(i): the i-th, with dev(), info and
// n_bloom_entries), the engine's block shape, the merge's policy and the filter fp (nullptr: none; the crc table is set when it
// validates hashes).  Refuses more than kMaxRuns runs, a run of 2^28 blocks or 2^40 bytes and a user key over kMaxUkeyLen
// (PGS_NOT_SUPPORTED), then a malformed ops table (PGS_INVALID_ARGUMENT), with a message that starts with who.  ops_len as
// compact_filter.
template <class RunAt>
inline int32_t compact_job_params(MergeParams &P, CompactTotals &T, uint32_t k, RunAt &&run, uint32_t block_size, uint32_t restart_interval,
                                  int32_t bottommost, uint32_t now, uint32_t data_version, const pgs_filter_params *fp,
                                  const unsigned long long *crc_table, uint32_t &ops_len, const char *who)
{
    if (k > kMaxRuns) { set_error("%s %u runs > %u per merge", who, k, kMaxRuns); return PGS_NOT_SUPPORTED; }
    P.k = k;
    for (uint32_t i = 0; i < k; i++) {
        const auto &r = run(i);
        P.runs[i] = r.dev();
        T.add(r.info, r.n_bloom_entries);
        if (r.info.n_blocks >= (1u << 28) || r.info.data_bytes >= (1ull << 40)) { set_error("%s a run too large for a merge", who); return PGS_NOT_SUPPORTED; }
    }
    if (T.max_ukey > kMaxUkeyLen) { set_error("%s user key of %u bytes > %u", who, T.max_ukey, kMaxUkeyLen); return PGS_NOT_SUPPORTED; }
    P.block_size = block_size;
    P.restart_interval = restart_interval;
    P.bottommost = bottommost ? 1 : 0;
    P.now = now;
    P.data_version = data_version;
    if (!compact_filter(P, fp, ops_len)) { set_error("%s malformed ops table of %u bytes", who, fp->ops_len); return PGS_INVALID_ARGUMENT; }
    if (P.validate_hash) P.crc_table = crc_table;
    return PGS_OK;
}

// Every buffer of one launch: buf(pointer, elements, fill, out) allocates the elements and, unless fill is kNoFill, sets each
// byte to fill before the first kernel.  The scratch (out = false) lives as long as the launch; the merged run's buffers
// (out = true) are fields of `run` (the library's Run, or the simulator's host copy), which outlives it.  P points at all of them.
template <class R, class F>
inline void compact_buffers(MergeParams &P, const CompactGeometry &geo, const CompactTotals &T, R &run, F &&buf)
{
    const uint64_t Q = P.Q, nb = geo.blk_cap + 1;
    buf(P.split_pos, (Q + 1) * P.k, 0xFF, false); // no boundary yet (seg_slice)
    buf(P.split_ref, Q + 1, 0xFF, false);
    buf(P.ticket, 64, 0, false);
    buf(P.seg, Q, kNoFill, false);
    buf(P.agg, Q, 0, false);                      // a walk that did not run produced nothing
    buf(P.base, Q, kNoFill, false);
    buf(P.desc, P.desc_cap, kNoFill, false);
    buf(P.kstream, P.ks_cap + 64, kNoFill, false);
    buf(run.d_data, geo.out_cap + 256, kNoFill, true);
    buf(run.d_blk_off, nb, kNoFill, true);
    buf(run.d_blk_size, nb, kNoFill, true);
    buf(run.d_blk_rec, nb, kNoFill, true);
    buf(run.d_ikey_off, nb, kNoFill, true);
    buf(run.d_ikeys, geo.ikey_cap, kNoFill, true);
    buf(run.d_rec_off, T.n_rec + 1, kNoFill, true);
    buf(run.d_bloom, (uint64_t)P.out_bloom_lines * 16, 0, true); // k_emit only sets bits
    run.bloom_lines = P.out_bloom_lines;
    P.out_data = run.d_data;
    P.out_blk_off = (unsigned long long *)run.d_blk_off;
    P.out_blk_size = run.d_blk_size;
    P.out_blk_rec = run.d_blk_rec;
    P.out_ikey_off = run.d_ikey_off;
    P.out_ikeys = run.d_ikeys;
    P.out_rec_off = run.d_rec_off;
    P.out_bloom = run.d_bloom;
}
// what P.stats holds before the first kernel: no error, no failing segment
inline MergeStats merge_stats_init()
{
    MergeStats s{};
    s.error_seg = 0xFFFFFFFFu;
    return s;
}

// ------------------------------------------------------------------------------------------------
// k_plan
// ------------------------------------------------------------------------------------------------
PGS_DEV unsigned long long run_weight(const RunDev &r, uint32_t pos, uint32_t rec_cost)
{
    return r.blk_off[pos] + (unsigned long long)r.blk_rec[pos] * rec_cost;
}

// input block gt (over all of P's runs, < P.total_blocks): the segment boundaries its last user key sets
PGS_DEV void plan_block(const MergeParams &P, uint32_t gt)
{
    uint32_t i = 0, b = gt;
    while (b >= P.runs[i].nb) { b -= P.runs[i].nb; i++; }
    const RunDev &ri = P.runs[i];
    const uint8_t *U = ri.ikeys + ri.ikey_off[b];
    uint32_t ulen = ri.ikey_off[b + 1] - ri.ikey_off[b];
    uint32_t pos[kMaxRuns];
    unsigned long long Wb = 0, W = 0, W0 = 0;
    for (uint32_t j = 0; j < P.k; j++) {
        const RunDev &rj = P.runs[j];
        W0 += run_weight(rj, 0, P.rec_cost);
        uint32_t lo = 0, hi = rj.nb; // upper bound: #blocks with last key <= U
        if (j == i) { // the key's own run: its block, and the blocks after it that end with the same user key (older versions)
            lo = b + 1;
            while (lo < rj.nb && cmp_bytes4(rj.ikeys + rj.ikey_off[lo], rj.ikey_off[lo + 1] - rj.ikey_off[lo], U, ulen) == 0) lo++;
            hi = lo;
        }
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            const uint8_t *kp = rj.ikeys + rj.ikey_off[mid];
            uint32_t kl = rj.ikey_off[mid + 1] - rj.ikey_off[mid];
            if (cmp_bytes4(kp, kl, U, ulen) <= 0) lo = mid + 1; else hi = mid;
        }
        uint32_t ub = lo, lb = lo;
        while (lb > 0) {
            const uint8_t *kp = rj.ikeys + rj.ikey_off[lb - 1];
            uint32_t kl = rj.ikey_off[lb] - rj.ikey_off[lb - 1];
            if (cmp_bytes4(kp, kl, U, ulen) != 0) break;
            lb--;
        }
        pos[j] = ub;
        W += run_weight(rj, ub, P.rec_cost);
        Wb += run_weight(rj, lb, P.rec_cost);
    }
    // the weight starts at the runs' first blocks, not at zero: a run's first block may lie anywhere in its data (an upload
    // takes any offsets), so the block of the smallest last key (every lb at 0) also bounds the segments in front of it
    unsigned long long q_lo = Wb == W0 ? 1 : Wb / P.tile_weight + 1, q_hi = W / P.tile_weight;
    if (q_hi > P.Q - 1) q_hi = P.Q - 1;
    for (unsigned long long q = q_lo; q <= q_hi; q++) {
        for (uint32_t j = 0; j < P.k; j++) P.split_pos[q * P.k + j] = pos[j];
        P.split_ref[q] = (i << 28) | b;
    }
}

__global__ void __launch_bounds__(256) k_plan(const __grid_constant__ MergeParams P)
{
    uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    if (gt >= P.total_blocks) return;
    plan_block(P, gt);
}

// slice of run j that segment q may touch: blocks [lo, hi_ex); blocks >= chk may hold keys above the upper bound
PGS_DEV bool seg_slice(const MergeParams &P, uint32_t q, uint32_t j, uint32_t &lo, uint32_t &hi_ex, uint32_t &chk)
{
    const RunDev &r = P.runs[j];
    const bool first = q == 0, last = q == P.Q - 1;
    lo = first ? 0 : P.split_pos[(size_t)q * P.k + j];
    const uint32_t hi = last ? r.nb : P.split_pos[(size_t)(q + 1) * P.k + j];
    if (lo == 0xFFFFFFFFu || hi == 0xFFFFFFFFu || lo > r.nb || hi > r.nb || lo > hi) { lo = hi_ex = 0; chk = 0; return false; }
    hi_ex = last ? r.nb : (hi + 1 < r.nb ? hi + 1 : r.nb);
    chk = last ? 0xFFFFFFFFu : hi;
    return true;
}

// upper bound of a segment's key stream, from its input slice: records and block bytes it may read
PGS_HD unsigned long long ks_bound(unsigned long long n_in, unsigned long long in_bytes, uint32_t KS, uint32_t block_size)
{
    const unsigned long long per_rec = ks_record_bound(KS);
    unsigned long long blocks = 2 * (in_bytes + n_in * per_rec) / block_size + 2;
    if (blocks > n_in + 1) blocks = n_in + 1;
    return (n_in * per_rec + blocks * (unsigned long long)(KS + 8) + 64 + 15) & ~15ull; // key-stream records are stored as words
}

// ------------------------------------------------------------------------------------------------
// k_seg_bounds + k_seg_layout: where each segment's descriptor array and key stream live.  One thread per segment computes
// the bounds of what it may emit (from its input slice); one CTA turns them into offsets with an exclusive scan.
// ------------------------------------------------------------------------------------------------
PGS_DEV void seg_bound(const MergeParams &P, uint32_t q)
{
    unsigned long long n_in = 0, in_bytes = 0;
    bool ok = true;
    for (uint32_t j = 0; j < P.k; j++) {
        uint32_t lo, hi_ex, chk;
        ok &= seg_slice(P, q, j, lo, hi_ex, chk);
        n_in += P.runs[j].blk_rec[hi_ex] - P.runs[j].blk_rec[lo];
        in_bytes += P.runs[j].blk_off[hi_ex] - P.runs[j].blk_off[lo];
    }
    if (!ok) { atomicMax(&P.stats->error, (uint32_t)PGS_ABORTED); atomicMin(&P.stats->error_seg, q); }
    P.seg[q].desc_off = n_in;
    P.seg[q].ks_off = ks_bound(n_in, in_bytes, P.KS, P.block_size);
}
__global__ void __launch_bounds__(256) k_seg_bounds(const __grid_constant__ MergeParams P)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= P.Q) return;
    seg_bound(P, q);
}

// the whole CTA: P's segment bounds become offsets
PGS_DEV void seg_layout(const MergeParams &P)
{
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    cta_excl_scan<2>(P.Q, [&](uint32_t q, unsigned long long (&v)[2]) { v[0] += P.seg[q].desc_off; v[1] += P.seg[q].ks_off; }, q0, q1, pre, tot);
    if (threadIdx.x == 0 && (tot[0] > P.desc_cap || tot[1] > P.ks_cap)) { atomicMax(&P.stats->error, (uint32_t)PGS_ABORTED); atomicMin(&P.stats->error_seg, 0u); }
    for (uint32_t q = q0; q < q1; q++) {
        const unsigned long long a = P.seg[q].desc_off, b = P.seg[q].ks_off;
        P.seg[q].desc_off = pre[0];
        P.seg[q].ks_off = pre[1];
        pre[0] += a;
        pre[1] += b;
    }
}
__global__ void __launch_bounds__(1024) k_seg_layout(const __grid_constant__ MergeParams P) { seg_layout(P); }

// ------------------------------------------------------------------------------------------------
// compaction filter on the device
// ------------------------------------------------------------------------------------------------
// user_specified_operation_filter: key_ttl_compaction_filter.h:94-108 over the binary ops table.
// Every op sees the value as of entry (entry_ts); returns true when a delete op fired.
static __device__ __noinline__ bool dev_user_ops(const MergeParams &P, const uint8_t *ukey, uint32_t klen, uint32_t entry_ts, uint32_t &new_ts,
                                                bool &changed)
{
    const KeyParts k = split_key(ukey, klen);
    const uint8_t *p = P.ops + 4;
    for (uint32_t o = 0; o < P.n_ops; o++) {
        uint32_t op_type = p[0], ttl_type = p[1], n_rules = le16(p + 2), ttl_value = le32(p + 4);
        p += 8;
        bool all = n_rules > 0; // all_rules_match: empty rule set => false (compaction_operation.cpp:37-39)
        for (uint32_t r = 0; r < n_rules; r++) {
            uint32_t rt = p[0], mt = p[1], pl = le16(p + 2), start_ttl = le32(p + 4), stop_ttl = le32(p + 8);
            const uint8_t *pat = p + 12;
            p += 12 + ((pl + 3) & ~3u);
            if (!all) continue;
            bool m; // string_pattern_match: compaction_filter_rule.cpp:31-54 (an empty pattern never matches)
            if (rt == RULE_HASHKEY) m = pl != 0 && pattern_match(mt, pat, pl, k.hk, k.hkl);
            else if (rt == RULE_SORTKEY) m = pl != 0 && pattern_match(mt, pat, pl, k.sk, k.skl);
            else { // ttl_range_rule::match, compaction_filter_rule.cpp:76-90 (u32 arithmetic)
                if (entry_ts == 0 && start_ttl == 0 && stop_ttl == 0) m = true;
                else m = (uint32_t)(start_ttl + P.now) <= entry_ts && (uint32_t)(stop_ttl + P.now) >= entry_ts;
            }
            all = m;
        }
        if (!all) continue;
        if (op_type == OP_DELETE) return true; // delete_key::filter
        // update_ttl::filter, compaction_operation.cpp:77-113
        uint32_t ts;
        if (ttl_type == TTL_FROM_NOW) ts = P.now + ttl_value;
        else if (ttl_type == TTL_FROM_CURRENT) { if (entry_ts == 0) continue; ts = ttl_value + entry_ts; }
        else if (ttl_type == TTL_TIMESTAMP) ts = ttl_value - kEpochBegin;
        else continue;
        new_ts = ts;
        changed = true;
    }
    return false;
}

// pegasus_key_hash out of line: the walker's registers stay those of its common path
static __device__ __noinline__ uint64_t dev_key_hash(const unsigned long long *tab, const uint8_t *key, uint32_t len)
{
    return pegasus_key_hash(tab, key, len);
}

// KeyWithTTLCompactionFilter::Filter (key_ttl_compaction_filter.h:55-92).  expire_ts = the value's BE32 header field.
// returns 0 keep, 1 expired, 2 user op, 3 stale split data
PGS_DEV uint32_t dev_filter(const MergeParams &P, const unsigned long long *crc_tab, const uint8_t *ukey, uint32_t klen,
                            uint32_t expire_ts, uint32_t vlen, uint32_t &new_ts, bool &changed)
{
    changed = false;
    if (!P.enabled || klen < 2 || vlen < 4) return 0;
    if (P.default_ttl != 0 && expire_ts == 0) {
        expire_ts = P.now + P.default_ttl;
        new_ts = expire_ts;
        changed = true;
    }
    if (P.n_ops) {
        if (dev_user_ops(P, ukey, klen, expire_ts, new_ts, changed)) return 2;
    }
    if (ts_expired(P.now, expire_ts)) return 1;
    // check_if_stale_split_data (key_ttl_compaction_filter.h:114-121): only a valid partition version checks the key's hash
    if (P.validate_hash && P.partition_version >= 0 && P.pidx <= P.partition_version) {
        const uint64_t h = dev_key_hash(crc_tab, ukey, klen);
        if ((long long)(h & (unsigned long long)(long long)P.partition_version) != (long long)P.pidx) return 3;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// k_walk
// ------------------------------------------------------------------------------------------------
// Group-uniform running statistics of a group (every lane computes the same values); flushed into the CTA's totals (shared
// memory) and from there into MergeStats.
struct WalkAcc {
    uint32_t e0, e1, e2;  // event counters, 8 bits each: EV_ 0..3, 4..7, 8..11
    uint32_t n;           // records since the last flush of e0..e2 (at most 255)
    unsigned long long b_in, b_key, b_val;
    uint32_t m_ukey, m_vlen, m_bsize, m_brec;
    unsigned long long m_seq, m_seq_inv;
};
PGS_DEV uint32_t spread4(uint32_t x) { return (x * 0x00204081u) & 0x01010101u; } // bits 0..3 -> the low bit of bytes 0..3
PGS_DEV void acc_flush_events(WalkAcc &acc, WalkCtaStats *cta, bool lane0)
{
    if (lane0) {
#pragma unroll
        for (uint32_t i = 0; i < 12; i++) {
            const uint32_t v = ((i < 4 ? acc.e0 : i < 8 ? acc.e1 : acc.e2) >> (8 * (i & 3))) & 0xffu;
            if (v) atomicAdd(&cta->cnt[i], v);
        }
    }
    acc.e0 = acc.e1 = acc.e2 = 0; acc.n = 0;
}

// the merge order of a group's cursors: run indices as 4-bit fields, position 0 = the smallest head
PGS_DEV uint32_t ord_at(unsigned long long o, uint32_t i) { return (uint32_t)(o >> (4 * i)) & 15u; }
PGS_DEV unsigned long long ord_insert(unsigned long long o, uint32_t pos, uint32_t run)
{
    const unsigned long long low = (1ull << (4 * pos)) - 1ull;
    return (o & low) | ((unsigned long long)run << (4 * pos)) | ((o & ~low) << 4);
}
PGS_DEV unsigned long long ord_head_to(unsigned long long o, uint32_t pos) // the head moves behind the entries 1..pos
{
    const unsigned long long low = (1ull << (4 * pos)) - 1ull, c = o & 15ull, rest = o >> 4;
    return (rest & low) | (c << (4 * pos)) | ((rest & ~low) << 4);
}

// What neighbours in the merge order share: field i (16 bits) = bytes the user keys at positions i and i + 1 have in common,
// kLcpUnknown when not known; positions past the fourth are never known (deep stacks fall back to whole compares).
constexpr uint32_t kLcpUnknown = 0xFFFFu;
PGS_DEV uint32_t adj_get(unsigned long long a, uint32_t i) { return i < 4 ? (uint32_t)(a >> (16 * i)) & 0xFFFFu : kLcpUnknown; }
PGS_DEV unsigned long long adj_set(unsigned long long a, uint32_t i, uint32_t v)
{
    if (i >= 4) return a;
    if (v > kLcpUnknown) v = kLcpUnknown;
    return (a & ~(0xFFFFull << (16 * i))) | ((unsigned long long)v << (16 * i));
}
// the head leaves position 0 and lands behind the entries 1..pos: the fields before it move down, lo / hi are what it shares
// with its new neighbours
PGS_DEV unsigned long long adj_head_to(unsigned long long a, uint32_t pos, uint32_t lo, uint32_t hi)
{
    unsigned long long n = ~0ull;
#pragma unroll
    for (uint32_t i = 0; i < 4; i++) {
        uint32_t v;
        if (i + 1 < pos) v = adj_get(a, i + 1);
        else if (i + 1 == pos) v = lo;
        else if (i == pos) v = hi;
        else v = adj_get(a, i);
        n = adj_set(n, i, v);
    }
    return n;
}

// One segment per group, all groups of the warp in lock step (see group.cuh): every statement outside an `if (en...)` body is
// executed by all 32 lanes; `act` marks the groups that still have records.
// MANY: the groups of a warp may walk segments of different jobs (k_walk_many), whose run counts differ; the cursors are
// opened in a loop of k_open (warp-uniform, at least every group's P.k) steps, and a group takes part in those past its P.k
// with nothing enabled.
template <uint32_t G, bool MANY = false>
PGS_DEV void walk_segment(const MergeParams &P, const RunDev *runs, const Grp<G> &g, bool seg_en, uint32_t q, CurState *cs, uint32_t *rows,
                          uint8_t *wins, const unsigned long long *crc, WalkAcc &acc, WalkCtaStats *cta, uint32_t k_open = 0)
{
    const uint32_t k = P.k, KS = P.KS, KSW = P.KSW, RI = P.restart_interval, BS = P.block_size;
    uint32_t *rowA = rows + k * KSW, *rowB = rowA + KSW, *rowLO = rowB + KSW, *rowHI = rowLO + KSW;
    const bool first = q == 0, last = q == P.Q - 1;
    uint32_t err = 0;

    // ---- boundary keys (U_lo, U_hi] --------------------------------------------------------------------------------
    uint32_t ulo_len = 0, uhi_len = 0;
    if (seg_en) {
        for (uint32_t which = 0; which < 2; which++) {
            if (which == 0 ? first : last) continue;
            const uint32_t ref = P.split_ref[q + which];
            const uint32_t run = ref >> 28, b = ref & 0x0FFFFFFFu;
            if (ref == 0xFFFFFFFFu || run >= k || b >= runs[run].nb) { err = PGS_ABORTED; break; }
            const uint32_t off = runs[run].ikey_off[b], len = runs[run].ikey_off[b + 1] - off;
            if (len > KS) { err = PGS_ABORTED; break; }
            uint8_t *dst = (uint8_t *)(which == 0 ? rowLO : rowHI);
            const uint8_t *src = runs[run].ikeys + off;
#pragma unroll 1
            for (uint32_t i = g.gl; i < len; i += G) dst[i] = src[i];
            if (which == 0) ulo_len = len; else uhi_len = len;
        }
    }
    g.sync();

    // ---- open one cursor per run, skip what belongs to the previous segment ---------------------------------------------
    uint32_t live = 0;
    unsigned long long order = 0; // entries 0..live-1: the group's runs in merge order
    uint32_t dpos = 0;
#pragma unroll 1
    for (uint32_t j = 0; j < (MANY ? k_open : k); j++) {
        const bool run_en = seg_en && (!MANY || j < k); // (a group past its own runs takes part with nothing enabled)
        const bool en = run_en && !err;
        uint32_t lo = 0, hi_ex = 0, chk = 0;
        if (en && !seg_slice(P, q, j, lo, hi_ex, chk)) err = PGS_ABORTED;
        CurState *C = &cs[j];
        uint32_t *row = rows + j * KSW;
        const uint32_t e1 = cur_open<G, true>(g, en && !err, runs[j], C, row, KS, lo, hi_ex, chk, wins + j * kHeadWin);
        if (en && !err) err = e1;
#pragma unroll 1
        for (;;) { // records at or below U_lo belong to the previous segment
            const bool sk = run_en && !err && !first && C->live;
            const int c = row_cmp(g, sk, row, sk ? C->klen - 8 : 0u, rowLO, ulo_len, dpos);
            const bool more = sk && c <= 0;
            if (!g.any(more)) break;
            const uint32_t e2 = cur_next<G, true>(g, more, runs[j], C, row, KS, wins + j * kHeadWin);
            if (more) err = e2;
        }
        const bool hi = run_en && !err && C->live && !last && C->b >= C->chk_from;
        const int ch = row_cmp(g, hi, row, hi ? C->klen - 8 : 0u, rowHI, uhi_len, dpos);
        g.sync();
        if (hi && ch > 0 && g.gl == 0) C->live = 0;
        g.sync();
        // insert into the order
        const bool ins = run_en && !err && C->live;
        uint32_t pos = live;
        bool searching = ins;
#pragma unroll 1
        for (uint32_t i = 0; g.any(searching && i < live); i++) {
            const bool e = searching && i < live;
            const bool bf = head_before(g, e, cs, rows, KSW, j, ord_at(order, i), dpos);
            if (e && bf) { pos = i; searching = false; }
        }
        if (ins) { order = ord_insert(order, pos, j); live++; }
    }
    unsigned long long adj = ~0ull; // see adj_get
#pragma unroll 1
    for (uint32_t i = 0; g.any(seg_en && !err && i + 1 < live) && i < 4; i++) {
        const bool e = seg_en && !err && i + 1 < live;
        uint32_t dp = 0;
        head_before(g, e, cs, rows, KSW, ord_at(order, i), ord_at(order, i + 1), dp);
        if (e) adj = adj_set(adj, i, dp);
    }

    // ---- the merge loop --------------------------------------------------------------------------------------------------
    Desc *desc = seg_en ? P.desc + P.seg[q].desc_off : nullptr;
    uint8_t *kstream = seg_en ? P.kstream + P.seg[q].ks_off : nullptr;
    uint32_t n_out = 0, kpos = 0;                        // descriptors / key-stream bytes written
    uint32_t blk_n = 0, blk_bytes = 0;                   // entries and entry bytes of the open output block
    uint32_t to_restart = 0, nrest = 0;                  // entries until the next restart point, restart points so far (no divisions in the loop)
    uint32_t n_blocks = 0, keyb = 0, lenA = 0;
    unsigned long long out_bytes = 0;
    bool have_head = false, head_in_A = false, prev_big = false;
    uint32_t hi_run = 0xffu, hi_l = 0, hi_ulen = 0, sw_lcp = kLcpUnknown; // the run whose last key was compared with the upper bound, and the bytes it shared with it
    uint32_t head_len = 0, last_run = 0xffu, lcpA = 0; // lcpA: bytes the head shares with A (the last survivor's key)
    auto close_block = [&]() { // bookkeeping of a finished block (k_emit derives the same numbers)
        const uint32_t size = block_bytes(blk_bytes, nrest);
        out_bytes += block_span(size);
        n_blocks++;
        keyb += lenA;
        if (size > acc.m_bsize) acc.m_bsize = size;
        if (blk_n > acc.m_brec) acc.m_brec = blk_n;
    };
#pragma unroll 1
    for (;;) {
        const bool act = seg_en && live > 0 && !err;
        if (!g.any(act)) break;
        const uint32_t c = (uint32_t)order & 15u;
        CurState *C = &cs[c];
        uint32_t *row = rows + c * KSW;
        uint32_t ulen = 0, vlen = 0, type = 0, tr_lo = 0, tr_hi = 0;
        if (act) { ulen = C->klen - 8; vlen = C->vlen; tr_lo = C->tr_lo; tr_hi = C->tr_hi; type = tr_lo & 0xffu; }
        uint32_t ev = act ? 1u << EV_IN : 0u; // what happened to this record, one bit per counter
        // (1) an older version of the user key that was just handled?  The record before this one carried the head's user key;
        // when it came from the same run, the entry's `shared` field is a known common prefix: all of the key (a shadow, no
        // compare), or it ends in front of a byte that differs (one byte to look at; a block writer that stored less than
        // the exact shared length falls through to the compare).
        uint32_t lcp_head = 0, from = 0;
        const bool cmp1 = act && have_head;
        const uint32_t *hrow = head_in_A ? rowA : rowB;
        bool from_exact = false;
        if (cmp1 && last_run == c) { from = C->shared < ulen ? C->shared : ulen; if (from > head_len) from = head_len; }
        else if (cmp1 && sw_lcp != kLcpUnknown) { // the old runner-up leads now: the order knew what it shared with the old head
            from = sw_lcp < ulen ? sw_lcp : ulen;
            if (from > head_len) from = head_len;
            from_exact = true;
        } else if (cmp1 && last_run != 0xffu && cs[last_run].live) {
            // another run leads now: head <= this key <= the key the head's run moved on to, so this key shares with the
            // head at least what that one does
            const uint32_t ls = cs[last_run].shared, lu = cs[last_run].klen - 8;
            from = ls < lu ? ls : lu;
            if (from > ulen) from = ulen;
            if (from > head_len) from = head_len;
        }
        bool shadow = cmp1 && from == ulen && ulen == head_len;
        bool cmp1b = cmp1 && !shadow;
        if (cmp1b && from_exact) { lcp_head = from; cmp1b = false; }
        if (cmp1b && last_run == c) {
            if (from == ulen || from == head_len) { lcp_head = from; cmp1b = false; } // one key is a proper prefix of the other
            else if (((row[from >> 2] ^ hrow[from >> 2]) >> (8 * (from & 3))) & 0xffu) { lcp_head = from; cmp1b = false; }
        }
        if (g.any(cmp1b)) {
            const int c1 = row_cmp(g, cmp1b, row, ulen, hrow, head_len, lcp_head, from);
            if (cmp1b && c1 == 0) shadow = true;
        }
        if (shadow) lcp_head = ulen;
        // (2) newest version of a user key: CompactionIterator rules + KeyWithTTLCompactionFilter::Filter
        bool keep = false, tomb = false, rewrite = false;
        uint32_t nts = 0, vlen_out = vlen;
        if (act) {
            if (shadow) ev |= 1u << EV_SHADOW;
            else if (type == PGS_TYPE_VALUE) {
                bool changed;
                const uint32_t ets = __byte_perm(C->ets_le, 0, 0x0123);
                const uint32_t why = dev_filter(P, crc, (const uint8_t *)row, ulen, ets, vlen, nts, changed);
                if (why) {
                    ev |= why == 1 ? 1u << EV_EXPIRED : (why == 2 ? 1u << EV_USER : 1u << EV_STALE);
                    // Decision::kRemove turns the entry into a deletion; it disappears only at the bottommost level
                    if (!P.bottommost) { keep = tomb = true; vlen_out = 0; }
                } else {
                    keep = true;
                    if (changed) { rewrite = true; ev |= 1u << EV_TTL; }
                }
            } else if (type == PGS_TYPE_DELETION) {
                if (P.bottommost) ev |= 1u << EV_TOMB; else keep = tomb = true;
            } else {
                keep = true;
            }
        }
        // (3) prefix compression against the previous survivor A.  Keys arrive in ascending order, so the prefix shared with A
        // is the minimum over the heads in between: lcp(K, A) = min(lcp(K, head), lcp(head, A)) -- no compare.
        bool restart = to_restart == 0;
        const uint32_t lcp_KA = !have_head ? 0u : head_in_A ? lcp_head : (lcp_head < lcpA ? lcp_head : lcpA);
        uint32_t shared = keep && !restart ? lcp_KA : 0u;
        uint32_t *kdst = nullptr;
        if (keep) {
            const uint32_t otype = tomb ? (uint32_t)PGS_TYPE_DELETION : type;
            const bool zero_seq = P.bottommost && otype == PGS_TYPE_VALUE;
            const uint32_t otr_lo = zero_seq ? otype : ((tr_lo & ~0xffu) | otype), otr_hi = zero_seq ? 0u : tr_hi;
            if (vlen_out > 0xFFF00000u) err = PGS_NOT_SUPPORTED; // entry sizes are 32-bit below
            uint32_t kd = ulen - shared;
            // entry_head_len + value and ks_record below, written out: through the helpers ptxas schedules this loop differently
            uint32_t e = varint_len(shared) + varint_len(kd + 8) + varint_len(vlen_out) + kd + 8 + vlen_out;
            uint32_t flags = 0;
            // block cut: the entry (and the restart array it may extend) must fit the block
            if (blk_n > 0 && (prev_big || block_bytes(blk_bytes + e, nrest + (restart ? 1u : 0u)) > BS)) {
                close_block();
                blk_n = 0; blk_bytes = 0; nrest = 0;
                restart = true; shared = 0; kd = ulen;
                e = 1 + varint_len(kd + 8) + varint_len(vlen_out) + kd + 8 + vlen_out;
            }
            if (blk_n == 0) flags |= DF_NEWBLOCK;
            const bool big = e + 8 > P.blk_buf; // does not fit the block buffer of k_emit: a block of its own, written in place
            if (big) flags |= DF_BIG;
            if (rewrite) flags |= DF_REWRITE;
            // the survivor's key-stream record (ks_record)
            uint32_t *sp = reinterpret_cast<uint32_t *>(kstream + kpos);
            const uint32_t fixed = rewrite ? 3u : 2u; // words
#pragma unroll
            for (uint32_t i = g.gl; i < 3; i += G)
                if (i < fixed) sp[i] = i == 0 ? otr_lo : i == 1 ? otr_hi : __byte_perm(nts, 0, 0x0123); // BE32 in memory
            kdst = sp + fixed; // the key words follow below, together with the copy that becomes the new A
            kpos += 4 * fixed + ((ulen + 3) & ~3u);
            if (g.gl == 0) {
                Desc d;
                d.loc = desc_loc(cur_base(C) + C->voff, c, ulen, flags);
                d.vlen = vlen_out;
                d.aux = lcp_KA;
                *reinterpret_cast<uint4 *>(&desc[n_out]) = *reinterpret_cast<const uint4 *>(&d);
            }
            n_out++;
            blk_n++;
            blk_bytes += e;
            if (restart) { nrest++; to_restart = RI; }
            to_restart--;
            prev_big = big;
            ev |= 1u << EV_OUT;
            if (otype == PGS_TYPE_DELETION) ev |= 1u << EV_OUT_TOMB;
            // maxima and byte sums of the output (sequence numbers are 56 bits)
            const unsigned long long seq = ((unsigned long long)otr_hi << 24) | (otr_lo >> 8);
            if (ulen > acc.m_ukey) acc.m_ukey = ulen;
            if (vlen_out > acc.m_vlen) acc.m_vlen = vlen_out;
            if (seq > acc.m_seq) acc.m_seq = seq;
            if (~seq > acc.m_seq_inv) acc.m_seq_inv = ~seq;
            acc.b_key += ulen;
            acc.b_val += vlen_out;
        }
        // counters
        if (act) acc.b_in += ulen + vlen;
        acc.e0 += spread4(ev & 15u);
        acc.e1 += spread4((ev >> 4) & 15u);
        acc.e2 += spread4((ev >> 8) & 15u);
        if (++acc.n == 255) acc_flush_events(acc, cta, g.gl == 0);
        g.sync(); // every lane has read the previous survivor's key
        if (act && !shadow) { // the new head: a survivor goes to A and to its stream record, a dropped head to B
            uint32_t *dst = keep ? rowA : rowB;
#pragma unroll 1
            for (uint32_t w = g.gl; 4 * w < ulen; w += G) { const uint32_t x = row[w]; dst[w] = x; if (keep) kdst[w] = x; }
            if (keep) { lenA = ulen; lcpA = ulen; } else lcpA = lcp_KA; // lcp(new head, A)
            head_in_A = keep;
            have_head = true;
            head_len = ulen;
        }
        last_run = c;
        g.sync();
        // (4) advance the cursor and restore the merge order
        const uint32_t e3 = cur_next<G, true>(g, act && !err, runs[c], C, row, KS, wins + c * kHeadWin);
        if (act && !err) err = e3;
        const bool adv = act && !err;
        bool alive = adv && C->live != 0;
        // Upper bound of the segment.  The key before this one (same run) was below the bound and shared hi_l bytes with it: a
        // key that shares more than hi_l bytes with its predecessor stands in the same relation; one that shares fewer rose
        // above the bound at that byte (checked: a block writer may have stored less than the exact shared length).
        const bool hi = alive && !last && C->b >= C->chk_from;
        bool hi_cmp = hi;
        uint32_t hi_from = 0;
        if (hi && hi_run == c) {
            const uint32_t sh_c = C->shared, ul = C->klen - 8;
            // (`shared` counts internal-key bytes: it says something about user keys only inside the predecessor's user key)
            if (sh_c > hi_l) { if (hi_l < hi_ulen) hi_cmp = false; }
            else if (sh_c == hi_l) { if (hi_l <= ul) hi_from = hi_l; }
            else if (sh_c < ul && ((row[sh_c >> 2] >> (8 * (sh_c & 3))) & 0xffu) > ((rowHI[sh_c >> 2] >> (8 * (sh_c & 3))) & 0xffu)) { alive = false; hi_cmp = false; }
        }
        if (g.any(hi_cmp)) {
            uint32_t dp = 0;
            const int ch = row_cmp(g, hi_cmp, row, hi_cmp ? C->klen - 8 : 0u, rowHI, uhi_len, dp, hi_from);
            if (hi_cmp) { if (ch > 0) alive = false; else hi_l = dp; }
        }
        if (hi && alive) { hi_run = c; hi_ulen = C->klen - 8; } else if (hi_run == c) hi_run = 0xffu;
        // Restore the merge order.  Keys are sorted, so what this key shares with a neighbour follows from what it shares with
        // the one before and what those two share (adj): more -> it sorts before the neighbour, less -> after it (the byte is
        // checked: a block writer may have stored less than the exact shared length), the same -> compare from that byte on.
        sw_lcp = live > 1 ? adj_get(adj, 0) : kLcpUnknown; // what the record just handled shares with the runner-up: needed if that one takes over
        bool searching = adv && alive && live > 1;
        uint32_t cur = 0; // bytes this key shares with the entry examined last (first: its predecessor in the run, the old head)
        if (searching) {
            const uint32_t ku = C->klen - 8;
            cur = C->shared < ku ? C->shared : ku;
            if (cur > ulen) cur = ulen;
            const uint32_t a0 = adj_get(adj, 0);
            if (a0 != kLcpUnknown && cur > a0) searching = false; // stays in front, shares with the runner-up what its predecessor did
        }
        uint32_t pos = 0, nxt = kLcpUnknown;
        const bool reorder = searching;
#pragma unroll 1
        for (uint32_t i = 1; g.any(searching && i < live); i++) {
            const bool e = searching && i < live;
            const uint32_t r = ord_at(order, i);
            const uint32_t a_i = adj_get(adj, i - 1);
            bool need = e, bf = false;
            uint32_t from = 0, d = 0;
            if (e && a_i != kLcpUnknown) {
                if (cur > a_i) { bf = true; d = a_i; need = false; }
                else if (cur == a_i) from = cur;
                else if (cur < C->klen - 8 && ((row[cur >> 2] >> (8 * (cur & 3))) & 0xffu) > ((rows[r * KSW + (cur >> 2)] >> (8 * (cur & 3))) & 0xffu)) { d = cur; need = false; }
            }
            if (g.any(need)) {
                const bool bfc = head_before(g, need, cs, rows, KSW, c, r, dpos, from);
                if (need) { bf = bfc; d = dpos; }
            }
            if (e) {
                if (bf) { nxt = d; searching = false; }
                else { pos = i; cur = d; }
            }
        }
        if (adv && !alive) { // drop the exhausted run
            order >>= 4;
            adj = (adj >> 16) | (0xFFFFull << 48);
            live--;
            last_run = 0xffu;
        } else if (reorder) {
            if (pos > 0) { order = ord_head_to(order, pos); adj = adj_head_to(adj, pos, cur, nxt); }
            else adj = adj_set(adj, 0, nxt);
        }
    }
    if (seg_en) {
        if (!err && blk_n > 0) close_block();
        if (err) {
            if (g.gl == 0) { atomicMax(&P.stats->error, err); atomicMin(&P.stats->error_seg, q); }
            n_out = 0; n_blocks = 0; keyb = 0; out_bytes = 0; kpos = 0; lenA = 0;
        }
        if (g.gl == 0) {
            SegAgg a;
            a.out_bytes = out_bytes; a.n_entries = n_out; a.n_blocks = n_blocks; a.keyb = keyb; a.ks_bytes = kpos; a.last_klen = lenA; a.pad = 0;
            P.agg[q] = a;
        }
    }
    g.sync();
}

template <uint32_t G>
__global__ void __launch_bounds__(kWalkThreads, 4) k_walk(const __grid_constant__ MergeParams P)
{
    PGS_SMEM_DYN(dyn);
    const Grp<G> g;
    constexpr uint32_t NGW = 32 / G; // groups per warp
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // CTA-wide shared memory: crc table (2 KB, only filled when the stale-split check is on), the run table (the groups of a
    // warp work on different runs at the same time: a per-lane index into kernel parameters would serialise), the CTA's totals
    unsigned long long *crc = (unsigned long long *)dyn;
    RunDev *runs = (RunDev *)(dyn + 2048);
    WalkCtaStats *cta = (WalkCtaStats *)(dyn + 2048 + kMaxRuns * sizeof(RunDev));
    if (P.validate_hash)
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) crc[i] = P.crc_table[i];
    for (uint32_t i = threadIdx.x; i < kMaxRuns; i += blockDim.x) runs[i] = P.runs[i < P.k ? i : 0];
    for (uint32_t i = threadIdx.x; i < sizeof(WalkCtaStats) / 4; i += blockDim.x) ((uint32_t *)cta)[i] = 0;
    if (__syncthreads_or(P.stats->error != 0)) return; // the planner rejected the layout: the output is discarded
    const uint32_t gi = warp * NGW + g.shift / G; // the group inside the CTA
    uint8_t *gs = dyn + kWalkFixedSmem + (size_t)gi * P.group_smem;
    CurState *cs = (CurState *)gs;
    uint32_t *rows = (uint32_t *)(gs + (size_t)P.k * sizeof(CurState));
    uint8_t *wins = dyn + walk_win_off(G, P.group_smem) + (size_t)gi * walk_win_stride(P.k);
    WalkAcc acc;
    acc.e0 = acc.e1 = acc.e2 = acc.n = 0;
    acc.b_in = acc.b_key = acc.b_val = 0;
    acc.m_ukey = acc.m_vlen = acc.m_bsize = acc.m_brec = 0;
    acc.m_seq = acc.m_seq_inv = 0;
#pragma unroll 1
    for (;;) {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(P.ticket, NGW);
        t0 = __shfl_sync(kFull, t0, 0);
        if (t0 >= P.Q) break;
        const uint32_t q = t0 + g.shift / G;
        walk_segment<G>(P, runs, g, q < P.Q, q < P.Q ? q : 0u, cs, rows, wins, crc, acc, cta);
    }
    // statistics: group -> CTA (shared-memory atomics) -> MergeStats
    acc_flush_events(acc, cta, g.gl == 0);
    if (g.gl == 0) {
        if (acc.b_in) atomicAdd(&cta->bytes[SB_IN], acc.b_in);
        if (acc.b_key + acc.b_val) atomicAdd(&cta->bytes[SB_OUT], acc.b_key + acc.b_val);
        if (acc.b_key) atomicAdd(&cta->bytes[SB_OUT_KEY], acc.b_key);
        if (acc.b_val) atomicAdd(&cta->bytes[SB_OUT_VAL], acc.b_val);
        if (acc.m_ukey) atomicMax(&cta->mx[SM_UKEY], (unsigned long long)acc.m_ukey);
        if (acc.m_vlen) atomicMax(&cta->mx[SM_VLEN], (unsigned long long)acc.m_vlen);
        if (acc.m_seq) atomicMax(&cta->mx[SM_MAX_SEQ], acc.m_seq);
        if (acc.m_seq_inv) atomicMax(&cta->mx[SM_MIN_SEQ_INV], acc.m_seq_inv);
        if (acc.m_bsize) atomicMax(&cta->mx[SM_BLK_SIZE], (unsigned long long)acc.m_bsize);
        if (acc.m_brec) atomicMax(&cta->mx[SM_BLK_REC], (unsigned long long)acc.m_brec);
    }
    __syncthreads();
    const uint32_t t = threadIdx.x;
    if (t < 12 && cta->cnt[t]) atomicAdd(&P.stats->cnt[t], (unsigned long long)cta->cnt[t]);
    if (t >= 32 && t < 36 && cta->bytes[t - 32]) atomicAdd(&P.stats->bytes[t - 32], cta->bytes[t - 32]);
    if (t >= 64 && t < 70 && cta->mx[t - 64]) atomicMax(&P.stats->mx[t - 64], cta->mx[t - 64]);
}

// ------------------------------------------------------------------------------------------------
// k_seg_scan: one CTA; exclusive prefixes of the segments' output sizes, totals, index sentinels
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_seg_scan(const __grid_constant__ MergeParams P)
{
    uint32_t q0, q1;
    unsigned long long pre[4], tot[4];
    cta_excl_scan<4>(P.Q, [&](uint32_t q, unsigned long long (&v)[4]) {
        const SegAgg a = P.agg[q];
        v[0] += a.out_bytes; v[1] += a.n_blocks; v[2] += a.n_entries; v[3] += a.keyb;
    }, q0, q1, pre, tot);
    const uint32_t tid = threadIdx.x;
    for (uint32_t q = q0; q < q1; q++) {
        const SegAgg a = P.agg[q];
        SegBase b;
        b.bytes = pre[0]; b.blocks = (uint32_t)pre[1]; b.recs = (uint32_t)pre[2]; b.keyb = (uint32_t)pre[3]; b.pad = 0;
        P.base[q] = b;
        pre[0] += a.out_bytes; pre[1] += a.n_blocks; pre[2] += a.n_entries; pre[3] += a.keyb;
    }
    if (tid == 0) {
        P.stats->tot_bytes = tot[0]; P.stats->tot_blocks = tot[1]; P.stats->tot_recs = tot[2]; P.stats->tot_keyb = tot[3];
        if (tot[0] > P.out_cap || tot[1] > P.out_blk_cap || tot[2] > P.out_rec_cap || tot[3] > P.out_ikey_cap) {
            atomicMax(&P.stats->error, (uint32_t)PGS_ABORTED);
        } else { // sentinels of the new run's index
            P.out_blk_off[tot[1]] = tot[0];
            P.out_blk_rec[tot[1]] = (uint32_t)tot[2];
            P.out_ikey_off[tot[1]] = (uint32_t)tot[3];
        }
    }
}
// k_seg_scan's body for one job of a multi-job launch (k_seg_scan_many), by the whole CTA.  k_seg_scan keeps its own copy of
// these lines: moved into a function they schedule differently, and the single-partition kernels keep their machine code.
PGS_DEV void seg_scan(const MergeParams &P)
{
    uint32_t q0, q1;
    unsigned long long pre[4], tot[4];
    cta_excl_scan<4>(P.Q, [&](uint32_t q, unsigned long long (&v)[4]) {
        const SegAgg a = P.agg[q];
        v[0] += a.out_bytes; v[1] += a.n_blocks; v[2] += a.n_entries; v[3] += a.keyb;
    }, q0, q1, pre, tot);
    const uint32_t tid = threadIdx.x;
    for (uint32_t q = q0; q < q1; q++) {
        const SegAgg a = P.agg[q];
        SegBase b;
        b.bytes = pre[0]; b.blocks = (uint32_t)pre[1]; b.recs = (uint32_t)pre[2]; b.keyb = (uint32_t)pre[3]; b.pad = 0;
        P.base[q] = b;
        pre[0] += a.out_bytes; pre[1] += a.n_blocks; pre[2] += a.n_entries; pre[3] += a.keyb;
    }
    if (tid == 0) {
        P.stats->tot_bytes = tot[0]; P.stats->tot_blocks = tot[1]; P.stats->tot_recs = tot[2]; P.stats->tot_keyb = tot[3];
        if (tot[0] > P.out_cap || tot[1] > P.out_blk_cap || tot[2] > P.out_rec_cap || tot[3] > P.out_ikey_cap) {
            atomicMax(&P.stats->error, (uint32_t)PGS_ABORTED);
        } else { // sentinels of the new run's index
            P.out_blk_off[tot[1]] = tot[0];
            P.out_blk_rec[tot[1]] = (uint32_t)tot[2];
            P.out_ikey_off[tot[1]] = (uint32_t)tot[3];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// k_emit
// ------------------------------------------------------------------------------------------------
// One 16-byte chunk of a byte stream at destination alignment: the stream continues from aligned source chunk P into C and
// starts `a` bytes (0..15) into P.  Select network + funnel shifts: no indexed registers, the same code for every lane.
PGS_DEV uint4 realign16(uint4 Pc, uint4 Cc, uint32_t a)
{
    uint32_t w0 = Pc.x, w1 = Pc.y, w2 = Pc.z, w3 = Pc.w, w4 = Cc.x, w5 = Cc.y, w6 = Cc.z, w7 = Cc.w;
    if (a & 4) { w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6; w6 = w7; }
    if (a & 8) { w0 = w2; w1 = w3; w2 = w4; w3 = w5; w4 = w6; }
    const uint32_t bs = (a & 3) * 8;
    return make_uint4(__funnelshift_r(w0, w1, bs), __funnelshift_r(w1, w2, bs), __funnelshift_r(w2, w3, bs), __funnelshift_r(w3, w4, bs));
}
// store the bytes [lo, hi) of a 16-byte chunk held in registers to a 16-aligned shared-memory chunk (its neighbours own the rest)
PGS_DEV void store_chunk_part(uint8_t *dst16, uint4 v, uint32_t lo, uint32_t hi)
{
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (uint32_t j = 0; j < 4; j++) {
        const uint32_t b0 = 4 * j, b1 = 4 * j + 4;
        if (lo <= b0 && b1 <= hi) *reinterpret_cast<uint32_t *>(dst16 + b0) = w[j];
        else if (lo < b1 && b0 < hi) {
#pragma unroll
            for (uint32_t b = 0; b < 4; b++)
                if (b0 + b >= lo && b0 + b < hi) dst16[b0 + b] = (uint8_t)(w[j] >> (8 * b));
        }
    }
}
// one THREAD copies n bytes inside shared memory, from src (any alignment, readable in whole 16-byte chunks from the chunk before
// the one src lies in) to obuf16 + doff (any alignment): 16-byte loads and stores, byte-exact at both ends, four loads at a time.
PGS_DEV void thread_copy_s2s(uint8_t *obuf16, uint32_t doff, const uint8_t *src, uint32_t n)
{
    if (n == 0) return;
    const uint32_t x0 = doff & ~15u;                   // first destination chunk
    const uint8_t *A = src - (doff - x0);              // source byte that lands on destination offset x0 (may precede src)
    const uint32_t a = (uint32_t)((uintptr_t)A & 15);
    const uint4 *sp = reinterpret_cast<const uint4 *>(A - a);
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    uint4 Pc = sp[0];
    const uint32_t end = doff + n;
#pragma unroll 1
    for (uint32_t x = x0; x < end; x += 64) {
        uint4 nx[4];                                   // (reads at most the chunk after the one of src's last byte)
#pragma unroll
        for (uint32_t j = 0; j < 4; j++) nx[j] = x + 16 * j < end ? sp[j + 1] : zero;
        sp += 4;
#pragma unroll
        for (uint32_t j = 0; j < 4; j++) {
            const uint32_t xx = x + 16 * j;
            if (xx < end) {
                const uint4 o = realign16(j == 0 ? Pc : nx[j - 1], nx[j], a);
                const uint32_t lo = xx < doff ? doff - xx : 0u, hi = end - xx < 16 ? end - xx : 16u;
                if (lo == 0 && hi == 16) *reinterpret_cast<uint4 *>(obuf16 + xx) = o;
                else store_chunk_part(obuf16 + xx, o, lo, hi);
            }
        }
        Pc = nx[3];
    }
}

// the Bloom hash of a key held as 32-bit words (4-byte aligned, any address space), one thread: same function as bloom_hash_row
PGS_DEV unsigned long long bloom_hash_words(const uint32_t *w32, uint32_t len)
{
    uint32_t ha = 0, hb = 0;
#pragma unroll 1
    for (uint32_t w = 0; 4 * w < len; w++) {
        uint32_t x = w32[w];
        if (len - 4 * w < 4) x &= (1u << (8 * (len - 4 * w))) - 1u;
        bloom_word(x, w, ha, hb);
    }
    return bloom_finish(ha, hb, len);
}
// one thread copies n bytes between two shared-memory buffers of any alignment: words where the destination allows, the
// source re-aligned with a funnel shift (reads up to 3 bytes past the source's end: stages carry slack)
PGS_DEV void copy_bytes_s2s(uint8_t *dst, const uint8_t *src, uint32_t n)
{
    while (n && ((uintptr_t)dst & 3)) { *dst++ = *src++; n--; }
    const uint32_t *sw = reinterpret_cast<const uint32_t *>((uintptr_t)src & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)((uintptr_t)src & 3) * 8;
    uint32_t w0 = sw[0];
#pragma unroll 1
    for (; n >= 4; n -= 4) {
        const uint32_t w1 = *++sw;
        *reinterpret_cast<uint32_t *>(dst) = __funnelshift_r(w0, w1, sh);
        w0 = w1;
        dst += 4;
    }
    if (n) {
        const uint32_t v = __funnelshift_r(w0, sh ? sw[1] : 0u, sh);
        for (uint32_t i = 0; i < n; i++) dst[i] = (uint8_t)(v >> (8 * i));
    }
}

// k_emit: one warp per segment, one THREAD per entry.  A batch of up to 32 descriptors is laid out with warp scans (block
// membership, restart points, entry sizes, offsets inside the block, block starts, places in the stages).  As soon as the batch
// is fixed its key-stream records and values are brought into the stages by bulk copies that complete on one mbarrier, so the
// batch waits for global memory once.  Then every thread builds its entry's head from its key-stream record (varints | key
// bytes after the shared prefix | trailer), copies the value from the value stage into the warp's output buffer and adds the
// key (and a new hash-key prefix) to the run's Bloom filter; the threads standing on a block boundary finish the previous
// block (restart array, padding, index entry); the batch's bytes leave with one bulk TMA store, which the next batch waits
// for only when it writes the output buffer after its own stages have landed.  Blocks of a segment are adjacent in the output
// run, so a batch's bytes are one contiguous range; the partial 16-byte chunk at its end is carried into the next batch.

// a warp's shared memory, its lane, and what it added to the filter (counted by lane 0)
struct EmitWarp {
    uint8_t *obuf;   // emit_obuf + 32 bytes: the output buffer
    uint8_t *stage;  // ks_stage + 32 bytes: the key-stream records of a batch
    uint8_t *vstage; // emit_vstage + 32 bytes: the values of a batch, each in the 16-byte-aligned span that covers it
    uint64_t *bar;   // the mbarrier the bulk copies into both stages complete on
    uint32_t *rst;   // restart offsets of the open block (it may span batches)
    uint32_t lane, lt; // lt: the lanes before mine
    uint32_t RI, OB, VS; // restart interval, output buffer bytes, value stage bytes
    uint32_t phase;  // the barrier's phase the next batch waits for
    uint32_t n_bloom_keys, n_bloom_prefixes;
};
PGS_DEV void emit_warp(EmitWarp &W, const MergeParams &P, uint8_t *ws, uint32_t lane)
{
    W.obuf = ws;
    W.RI = P.restart_interval;
    W.OB = P.emit_obuf;
    W.VS = P.emit_vstage;
    W.stage = ws + W.OB + 32;
    W.vstage = ws + emit_vs_off(W.OB, P.ks_stage);
    W.bar = (uint64_t *)(ws + emit_bar_off(W.OB, P.ks_stage, W.VS));
    W.rst = (uint32_t *)(ws + emit_rst_off(W.OB, P.ks_stage, W.VS));
    W.lane = lane;
    W.lt = (1u << lane) - 1u;
    W.phase = 0;
    W.n_bloom_keys = W.n_bloom_prefixes = 0;
    if (lane == 0) { mbar_init(W.bar, 1); mbar_fence_init(); }
    __syncwarp();
}

// what a warp carries across the batches of a segment (warp-uniform, except cv: each lane holds its own byte of the carry)
struct EmitSeg {
    const Desc *desc;
    const uint8_t *ks;              // the segment's key stream
    uint32_t n;                     // its entries
    unsigned long long blk_start;   // global offset of the open block (of the segment's first block before it opens)
    uint32_t fill, blk_n, blk_rec0; // entry bytes / entries of the open block, its first record
    bool open;
    uint32_t blk_idx, rec_idx, keyb, kpos; // the next block, record and index-key byte; the next record in the key stream
    uint32_t carry;                 // the bytes of the partial 16-byte chunk in front of the write position
    uint8_t cv;                     // PER LANE: its byte number `lane` (lane < carry), which obuf_reclaim puts back at obuf[lane]
    uint32_t last_key_off, last_ulen; // the previous entry's user key in the key stream (the index key of a block it ends)
};
PGS_DEV void emit_seg(EmitSeg &S, const MergeParams &P, uint32_t q, const SegAgg &A, const SegBase &B)
{
    S.desc = P.desc + P.seg[q].desc_off;
    S.ks = P.kstream + P.seg[q].ks_off;
    S.n = A.n_entries;
    S.blk_start = B.bytes;
    S.fill = 0; S.blk_n = 0; S.blk_rec0 = B.recs;
    S.open = false;
    S.blk_idx = B.blocks; S.rec_idx = B.recs; S.keyb = B.keyb; S.kpos = 0;
    S.carry = 0; S.cv = 0;
    S.last_key_off = 0; S.last_ulen = 0;
}

// finish the open block outside a batch (whole warp): restart array (offsets kept in rst), count and padding go to `at`
// (where byte `fill` of the block lives: obuf + carry, or global memory for a block written in place), index entry
PGS_DEV void close_open(const MergeParams &P, EmitSeg &S, const EmitWarp &W, const uint8_t *key, uint32_t klen, uint8_t *at, uint32_t nrest)
{
    const uint32_t lane = W.lane;
    const uint32_t size = block_bytes(S.fill, nrest);
    const uint32_t asz = block_span(size);
    __syncwarp();
    for (uint32_t i = lane; i < 4 * (nrest + 1); i += 32) {
        const uint32_t v = (i >> 2) < nrest ? W.rst[i >> 2] : nrest;
        at[i] = (uint8_t)(v >> (8 * (i & 3)));
    }
    for (uint32_t i = size - S.fill + lane; i < asz - S.fill; i += 32) at[i] = 0;
    if (lane == 0) {
        P.out_blk_off[S.blk_idx] = S.blk_start;
        P.out_blk_size[S.blk_idx] = size;
        P.out_blk_rec[S.blk_idx] = S.blk_rec0;
        P.out_ikey_off[S.blk_idx] = S.keyb;
    }
    for (uint32_t i = lane; i < klen; i += 32) P.out_ikeys[S.keyb + i] = key[i];
    S.keyb += klen;
    S.blk_idx++;
    S.blk_start += asz;
    S.fill = 0; S.blk_n = 0; S.open = false;
}
// send obuf[0, bytes) to the run at the 16-aligned global offset gpos (bytes % 16 == 0) without waiting: obuf_reclaim waits
// until the store has read it
PGS_DEV void flush(const MergeParams &P, const EmitWarp &W, unsigned long long gpos, uint32_t bytes)
{
    __syncwarp();
    if (bytes) {
        fence_proxy_async();
        __syncwarp();
        if (W.lane == 0) { tma_store_1d(P.out_data + gpos, W.obuf, bytes); tma_store_commit(); }
    }
}
// before the next write into obuf: wait until the last store has read it (lane 0 issued it), put the carried bytes back in front
PGS_DEV void obuf_reclaim(const EmitSeg &S, const EmitWarp &W)
{
    if (W.lane == 0) tma_store_wait_read0();
    __syncwarp();
    if (W.lane < S.carry) W.obuf[W.lane] = S.cv;
}
// close the open block and send what obuf still holds of it
PGS_DEV void finish_open(const MergeParams &P, EmitSeg &S, const EmitWarp &W)
{
    obuf_reclaim(S, W);
    const unsigned long long obase = S.blk_start + S.fill - S.carry;
    close_open(P, S, W, S.ks + S.last_key_off, S.last_ulen, W.obuf + S.carry, restart_count(S.blk_n, W.RI));
    flush(P, W, obase, (uint32_t)(S.blk_start - obase));
    S.carry = 0;
}
// one thread: the key (and its hash-key prefix when the previous survivor did not share it) goes into the filter; returns
// whether the prefix went in
PGS_DEV bool bloom_add(const MergeParams &P, const uint32_t *key32, uint32_t ulen, uint32_t lcp)
{
    if (!P.out_bloom_lines) return false;
    const unsigned long long hk = bloom_hash_words(key32, ulen);
#pragma unroll
    for (uint32_t i = 0; i < 6; i++) bloom_add_bit(P.out_bloom, P.out_bloom_lines, hk, i);
    const uint32_t pl = hashkey_prefix_len((const uint8_t *)key32, ulen);
    if (!pl || lcp >= pl) return false;
    const unsigned long long hp = bloom_hash_words(key32, pl);
#pragma unroll
    for (uint32_t i = 0; i < 6; i++) bloom_add_bit(P.out_bloom, P.out_bloom_lines, hp, i);
    return true;
}

// one lane's entry of a batch (lane i: entry e0 + i) and the batch layout as far as it has been computed
struct EmitBatch {
    unsigned long long loc;               // my descriptor
    uint32_t fl, ulen, vl, lcp;
    bool have;                            // there is an entry e0 + lane
    // batch_fit
    bool cand, mine, is_restart;          // before the first oversized entry; in the batch; a restart point
    int h, ph;                            // the lane of the head (first entry) of my block, of the head before me (-1: none)
    uint32_t hm_all, cnt;                 // the heads among the candidates; the entries of the batch (lanes 0..cnt-1)
    uint32_t n_i, sh_out, kd, hl, sz, sb; // my index in my block, shared / non-shared key bytes, head and entry bytes, record bytes
    uint32_t ps_incl, ss_incl;            // entry / record bytes of the lanes at or before me
    uint32_t vs, vs_incl;                 // the 16-byte span that covers my value (0: no value); spans of the lanes at or before me
    // stage_batch
    uint32_t total_s;                     // the batch's key-stream bytes
    const uint8_t *staged;                // the batch's first record in the stage
    // batch_offsets
    bool closes;                          // I am a head that closes the block before me
    uint32_t hm, fill_i, base_i, o_i;     // the heads of the batch; my offset in my block; my block's start from blk_start; my offset in obuf
    uint32_t T, nrest_c, size_c, asz_c;   // the block I close: entry bytes, restart points, size, aligned size
    uint32_t span_incl, nclose_incl, kb_incl; // aligned bytes / count / index-key bytes of the blocks closed at or before me
    uint32_t rec_off_i, key_off_i, pk_off, pk_len; // my record and key in the stage; the key of the entry before me
    unsigned long long obase;             // the global offset of obuf[0]
};

// An entry larger than a block buffer (DF_BIG, lane 0's; fl = its flags): a block of its own, written in place by the whole warp.
PGS_DEV void emit_big(const MergeParams &P, EmitSeg &S, EmitWarp &W, const EmitBatch &b, uint32_t fl)
{
    const uint32_t lane = W.lane;
    const unsigned long long loc = __shfl_sync(kFull, b.loc, 0);
    const uint32_t vl = __shfl_sync(kFull, b.vl, 0), ulen = __shfl_sync(kFull, b.ulen, 0), lcp = __shfl_sync(kFull, b.lcp, 0);
    const uint8_t *rec = S.ks + S.kpos; // its key-stream record, read from global memory
    const uint32_t fixed = ks_fixed(fl);
    const uint8_t *key = rec + fixed;
    if (S.open) finish_open(P, S, W); // the block in front of it
    const uint8_t *vsrc = P.runs[desc_run(loc)].data + desc_voff(loc);
    uint8_t *o = P.out_data + S.blk_start;
    uint32_t hv = 0;
    if (lane == 0) { // a restart point: nothing shared
        hv = put_entry_varints(o, 0u, ulen, vl);
        const bool np = bloom_add(P, reinterpret_cast<const uint32_t *>(key), ulen, lcp);
        W.n_bloom_keys += P.out_bloom_lines ? 1u : 0u;
        W.n_bloom_prefixes += np ? 1u : 0u;
    }
    hv = __shfl_sync(kFull, hv, 0);
    const uint32_t hl = hv + ulen + 8;
    for (uint32_t x = lane; x < ulen; x += 32) o[hv + x] = key[x];
    if (lane < 8) o[hv + ulen + lane] = rec[lane]; // trailer
    for (uint32_t x = lane; x < vl; x += 32) o[hl + x] = vsrc[x];
    if ((fl & DF_REWRITE) && vl >= 4 && lane < 4) o[hl + lane] = rec[8 + lane];
    if (lane == 0) { W.rst[0] = 0; P.out_rec_off[S.rec_idx] = 0; }
    S.fill = hl + vl; S.blk_n = 1; S.blk_rec0 = S.rec_idx; S.open = true;
    close_open(P, S, W, key, ulen, o + S.fill, 1u); // the block's last user key is this entry's
    S.last_key_off = S.kpos + fixed; S.last_ulen = ulen;
    S.rec_idx++; S.kpos += ks_record(fl, ulen);
}

// ---- the batch phases, in the order k_emit calls them ---------------------------------------------------------------------------
// my descriptor: fetched with the batch before (dn, when this batch starts at dn_e0), or read now
PGS_DEV void batch_desc(EmitBatch &b, const EmitSeg &S, const EmitWarp &W, uint32_t e0, const uint4 &dn, uint32_t dn_e0)
{
    const uint32_t idx = e0 + W.lane;
    Desc d;
    d.loc = 0; d.vlen = 0; d.aux = 0;
    if (dn_e0 == e0) *reinterpret_cast<uint4 *>(&d) = dn;
    else if (idx < S.n) *reinterpret_cast<uint4 *>(&d) = *reinterpret_cast<const uint4 *>(&S.desc[idx]);
    b.have = idx < S.n;
    b.loc = d.loc; b.fl = desc_flags(d.loc); b.ulen = desc_ulen(d.loc); b.vl = d.vlen; b.lcp = d.aux;
}
// Layout and fit.  Block membership and restart points follow from the flags alone; the batch = the entries before the first
// oversized one that fit the output buffer and the stage.  Returns its entry count (0: not even one fits).
PGS_DEV uint32_t batch_fit(const MergeParams &P, const EmitSeg &S, const EmitWarp &W, EmitBatch &b)
{
    const uint32_t lane = W.lane, lt = W.lt, RI = W.RI;
    const uint32_t bigmask = __ballot_sync(kFull, b.have && (b.fl & DF_BIG));
    b.cand = b.have && !(bigmask & (lt | (1u << lane)));
    b.hm_all = __ballot_sync(kFull, b.cand && (b.fl & DF_NEWBLOCK));
    const uint32_t at_or_before = b.hm_all & (lt | (1u << lane)), before = b.hm_all & lt;
    b.h = at_or_before ? 31 - __clz((int)at_or_before) : -1;
    b.ph = before ? 31 - __clz((int)before) : -1;
    b.n_i = b.h >= 0 ? lane - (uint32_t)b.h : S.blk_n + lane;
    b.is_restart = b.n_i % RI == 0;
    b.sh_out = b.is_restart ? 0u : (b.lcp < b.ulen ? b.lcp : b.ulen);
    b.kd = b.ulen - b.sh_out;
    b.hl = entry_head_len(b.sh_out, b.kd, b.vl);
    b.sz = b.cand ? b.hl + b.vl : 0u;
    b.sb = b.cand ? ks_record(b.fl, b.ulen) : 0u;
    const unsigned long long voff = desc_voff(b.loc);
    b.vs = b.cand && b.vl ? (uint32_t)(((voff + b.vl + 15) & ~15ull) - (voff & ~15ull)) : 0u;
    b.ps_incl = warp_incl_scan(b.sz, lane);
    b.ss_incl = warp_incl_scan(b.sb, lane);
    b.vs_incl = warp_incl_scan(b.vs, lane);
    // room: the entries, the restart arrays and paddings of the blocks that close here (the carried block brings its earlier
    // restart points along), the carried partial chunk
    const uint32_t room = S.carry + 32 * (lane + 1) + 64 + (S.open ? 4 * restart_count(S.blk_n, RI) : 0u);
    const bool fits = b.cand && room + b.ps_incl <= W.OB && b.ss_incl <= P.ks_stage && b.vs_incl <= W.VS;
    b.cnt = (uint32_t)__popc(__ballot_sync(kFull, fits)); // monotone: lanes 0..cnt-1
    b.mine = lane < b.cnt;
    return b.cnt;
}
// Fetch the next batch's descriptors; start the bulk copies of this batch into the stages, all completing on the warp's
// barrier: lane 0 copies the 16-byte-aligned range that covers the batch's key-stream records, every lane of the batch the span
// of its value (both read up to 15 bytes before and after what they cover, inside the allocation and its slack).  The barrier
// expects the bytes of all of them before any is issued.
PGS_DEV void stage_batch(const MergeParams &P, const EmitSeg &S, const EmitWarp &W, EmitBatch &b, uint32_t e0, uint4 &dn, uint32_t &dn_e0)
{
    dn_e0 = e0 + b.cnt;
    dn = dn_e0 + W.lane < S.n ? *reinterpret_cast<const uint4 *>(&S.desc[dn_e0 + W.lane]) : make_uint4(0u, 0u, 0u, 0u);
    b.total_s = __shfl_sync(kFull, b.ss_incl, (int)b.cnt - 1);
    const uint32_t total_v = __shfl_sync(kFull, b.vs_incl, (int)b.cnt - 1);
    const uint8_t *src = S.ks + S.kpos;
    const uint32_t a = (uint32_t)((uintptr_t)src & 15), ks_bytes = (a + b.total_s + 15) & ~15u;
    fence_proxy_async(); // the last batch's reads of the stages come before the copies that overwrite them
    if (W.lane == 0) mbar_expect_tx(W.bar, ks_bytes + total_v);
    __syncwarp();
    if (W.lane == 0) tma_load_1d(W.stage, src - a, ks_bytes, W.bar);
    if (b.mine && b.vs) {
        const unsigned long long voff = desc_voff(b.loc);
        tma_load_1d(W.vstage + (b.vs_incl - b.vs), P.runs[desc_run(b.loc)].data + (voff & ~15ull), b.vs, W.bar);
    }
}
// Offsets and block starts: where my entry goes, the block a head closes, the index key of that block (the user key of the
// entry before the head).
PGS_DEV void batch_offsets(const MergeParams &P, const EmitSeg &S, const EmitWarp &W, EmitBatch &b)
{
    const uint32_t lane = W.lane, lt = W.lt, RI = W.RI;
    b.hm = b.cnt >= 32 ? b.hm_all : b.hm_all & ((1u << b.cnt) - 1u);
    const bool head = b.mine && (b.fl & DF_NEWBLOCK);
    const uint32_t ps = b.ps_incl - b.sz; // entry bytes of the batch before me
    const uint32_t ps_h = __shfl_sync(kFull, ps, b.h >= 0 ? b.h : 0), ps_ph = __shfl_sync(kFull, ps, b.ph >= 0 ? b.ph : 0);
    b.fill_i = b.h >= 0 ? ps - ps_h : S.fill + ps;
    b.closes = head && (b.ph >= 0 || S.open);
    b.T = b.ph >= 0 ? ps - ps_ph : S.fill + ps;
    const uint32_t NN = b.ph >= 0 ? lane - (uint32_t)b.ph : S.blk_n + lane;
    b.nrest_c = b.closes ? restart_count(NN, RI) : 0u;
    b.size_c = block_bytes(b.T, b.nrest_c);
    b.asz_c = b.closes ? block_span(b.size_c) : 0u;
    b.span_incl = warp_incl_scan(b.asz_c, lane);
    const uint32_t span_h = __shfl_sync(kFull, b.span_incl, b.h >= 0 ? b.h : 0);
    b.base_i = b.h >= 0 ? span_h : 0u;
    b.nclose_incl = (uint32_t)__popc(__ballot_sync(kFull, b.closes) & (lt | (1u << lane)));
    b.rec_off_i = b.ss_incl - b.sb;
    b.key_off_i = b.rec_off_i + ks_fixed(b.fl);
    b.pk_off = __shfl_up_sync(kFull, b.key_off_i, 1);
    const uint32_t pk_len_l = __shfl_up_sync(kFull, b.ulen, 1);
    b.pk_len = lane == 0 ? S.last_ulen : pk_len_l;
    b.kb_incl = warp_incl_scan(b.closes ? b.pk_len : 0u, lane);
    b.obase = S.blk_start + S.fill - S.carry;
    b.o_i = (uint32_t)(S.blk_start + b.base_i + b.fill_i - b.obase);
}
// Restart points: into obuf when my block closes in this batch, else into rst; my entry's offset into the index.  When the
// carried block closes here, its restart offsets from earlier batches leave rst first: the block that opens after it in this
// batch puts its own into rst.
PGS_DEV void restart_points(const MergeParams &P, const EmitSeg &S, const EmitWarp &W, const EmitBatch &b)
{
    const uint32_t lane = W.lane, lt = W.lt, RI = W.RI;
    const uint32_t first_close = __ffs((int)__ballot_sync(kFull, b.closes)) - 1; // lane of the first closing head (or ~0)
    if (S.open && first_close < 32) {
        const uint32_t Tc = __shfl_sync(kFull, b.T, (int)first_close);
        const uint32_t have_r = restart_count(S.blk_n, RI); // restart points recorded before this batch
        const uint32_t ro = (uint32_t)(S.blk_start - b.obase) + Tc;
        for (uint32_t i = lane; i < 4 * have_r; i += 32) W.obuf[ro + i] = (uint8_t)(W.rst[i >> 2] >> (8 * (i & 3)));
        __syncwarp();
    }
    const uint32_t after = b.hm & ~(lt | (1u << lane));
    const int nh = after ? __ffs((int)after) - 1 : -1;                  // the head that closes my block inside this batch
    const uint32_t T_mine = __shfl_sync(kFull, b.T, nh >= 0 ? nh : 0); // my block's entry bytes, when it closes here
    const uint32_t r_i = b.n_i / RI;
    if (b.mine && b.is_restart) {
        if (nh >= 0) {
            const uint32_t ro = (uint32_t)(S.blk_start + b.base_i - b.obase) + T_mine + 4 * r_i;
            W.obuf[ro] = (uint8_t)b.fill_i; W.obuf[ro + 1] = (uint8_t)(b.fill_i >> 8); W.obuf[ro + 2] = (uint8_t)(b.fill_i >> 16); W.obuf[ro + 3] = (uint8_t)(b.fill_i >> 24);
        } else W.rst[r_i] = b.fill_i;
    }
    if (b.mine) P.out_rec_off[S.rec_idx + lane] = b.fill_i;
}
// One thread per entry: head, value, filter bits.
PGS_DEV void write_entries(const MergeParams &P, EmitWarp &W, const EmitBatch &b)
{
    bool new_prefix = false;
    if (b.mine) {
        const uint8_t *rec = b.staged + b.rec_off_i;
        const uint8_t *key = b.staged + b.key_off_i;
        uint8_t *dst = W.obuf + b.o_i;
        const uint32_t p = put_entry_varints(dst, b.sh_out, b.kd, b.vl);
        copy_bytes_s2s(dst + p, key + b.sh_out, b.kd);
        copy_bytes_s2s(dst + p + b.kd, rec, 8u);
        // from its span in the value stage (the chunk in front of a span is the one before it, or the key-stream stage's slack)
        thread_copy_s2s(W.obuf, b.o_i + b.hl, W.vstage + (b.vs_incl - b.vs) + (uint32_t)(desc_voff(b.loc) & 15), b.vl);
        if ((b.fl & DF_REWRITE) && b.vl >= 4) { dst[b.hl] = rec[8]; dst[b.hl + 1] = rec[9]; dst[b.hl + 2] = rec[10]; dst[b.hl + 3] = rec[11]; }
        new_prefix = bloom_add(P, reinterpret_cast<const uint32_t *>(key), b.ulen, b.lcp);
    }
    const uint32_t np = (uint32_t)__popc(__ballot_sync(kFull, new_prefix));
    if (P.out_bloom_lines) { W.n_bloom_keys += b.cnt; W.n_bloom_prefixes += np; }
}
// The heads finish the blocks that end in front of them (their restart offsets are in place): count, padding, index entry
// and index key.
PGS_DEV void close_blocks(const MergeParams &P, const EmitSeg &S, const EmitWarp &W, const EmitBatch &b)
{
    const uint32_t lane = W.lane;
    if (b.closes) {
        const uint32_t bstart = (uint32_t)(S.blk_start - b.obase) + (b.span_incl - b.asz_c); // obuf offset of the block I close
        uint32_t p = bstart + b.T + 4 * b.nrest_c;
        W.obuf[p] = (uint8_t)b.nrest_c; W.obuf[p + 1] = (uint8_t)(b.nrest_c >> 8); W.obuf[p + 2] = (uint8_t)(b.nrest_c >> 16); W.obuf[p + 3] = (uint8_t)(b.nrest_c >> 24);
        for (p += 4; p < bstart + b.asz_c; p++) W.obuf[p] = 0;
        const uint32_t bi = S.blk_idx + b.nclose_incl - 1;
        P.out_blk_off[bi] = S.blk_start + (b.span_incl - b.asz_c);
        P.out_blk_size[bi] = b.size_c;
        P.out_blk_rec[bi] = b.ph >= 0 ? S.rec_idx + (uint32_t)b.ph : S.blk_rec0;
        P.out_ikey_off[bi] = S.keyb + b.kb_incl - b.pk_len;
    }
    // the closed blocks' index keys: the whole warp copies one key at a time
    uint32_t cm = __ballot_sync(kFull, b.closes);
    while (cm) {
        const int L = __ffs((int)cm) - 1;
        cm &= cm - 1;
        const uint32_t klen_b = __shfl_sync(kFull, b.pk_len, L), ko_b = S.keyb + __shfl_sync(kFull, b.kb_incl, L) - klen_b;
        const uint32_t poff = __shfl_sync(kFull, b.pk_off, L);
        const uint8_t *pk = L == 0 ? S.ks + S.last_key_off : b.staged + poff; // staged, or the last entry of the batch before
        for (uint32_t x = lane; x < klen_b; x += 32) P.out_ikeys[ko_b + x] = pk[x];
    }
}
// Carry the state over to the next batch, send the batch's whole 16-byte chunks, keep the partial one in the lanes' cv.
PGS_DEV void carry_over(const MergeParams &P, EmitSeg &S, const EmitWarp &W, const EmitBatch &b)
{
    const uint32_t lane = W.lane;
    const uint32_t lastl = b.cnt - 1;
    const uint32_t l_base = __shfl_sync(kFull, b.base_i, (int)lastl), l_fill = __shfl_sync(kFull, b.fill_i + b.sz, (int)lastl);
    const uint32_t l_n = __shfl_sync(kFull, b.n_i, (int)lastl) + 1;
    const int l_h = __shfl_sync(kFull, b.h, (int)lastl);
    const uint32_t n_closed = (uint32_t)__popc(__ballot_sync(kFull, b.closes));
    const uint32_t kb_total = __shfl_sync(kFull, b.kb_incl, 31);
    S.last_key_off = S.kpos + __shfl_sync(kFull, b.key_off_i, (int)lastl);
    S.last_ulen = __shfl_sync(kFull, b.ulen, (int)lastl);
    if (l_h >= 0) S.blk_rec0 = S.rec_idx + (uint32_t)l_h;
    S.blk_start += l_base; S.fill = l_fill; S.blk_n = l_n; S.open = true;
    S.blk_idx += n_closed; S.keyb += kb_total; S.rec_idx += b.cnt; S.kpos += b.total_s;
    const unsigned long long wpos = S.blk_start + S.fill;
    const uint32_t used = (uint32_t)(wpos - b.obase), whole = used & ~15u;
    flush(P, W, b.obase, whole);
    S.carry = used - whole;
    S.cv = lane < S.carry ? W.obuf[whole + lane] : (uint8_t)0;
}

// segment q of P, by the whole warp: its blocks, index entries and Bloom filter bits.  This is k_emit's loop body, which k_emit
// keeps written out for the same reason as k_seg_scan (k_emit_many calls this one).
PGS_DEV void emit_segment(const MergeParams &P, EmitWarp &W, uint32_t q)
{
    const uint32_t lane = W.lane;
    const SegAgg A = P.agg[q];
    if (A.n_entries == 0) return;
    const SegBase B = P.base[q];
    EmitSeg S;
    emit_seg(S, P, q, A, B);
    uint32_t err = 0;
    uint4 dn = make_uint4(0u, 0u, 0u, 0u); // the next batch's descriptors, fetched while this batch's values are copied
    uint32_t dn_e0 = 0xFFFFFFFFu;
    for (uint32_t e0 = 0; e0 < S.n && !err;) {
        EmitBatch b;
        batch_desc(b, S, W, e0, dn, dn_e0);
        const uint32_t first_fl = __shfl_sync(kFull, b.fl, 0);
        if (first_fl & DF_BIG) { emit_big(P, S, W, b, first_fl); e0++; continue; }
        if (batch_fit(P, S, W, b) == 0) { err = PGS_ABORTED; break; }
        stage_batch(P, S, W, b, e0, dn, dn_e0);
        batch_offsets(P, S, W, b);
        mbar_wait(W.bar, W.phase); // the one wait of a batch for global memory
        W.phase ^= 1;
        b.staged = W.stage + ((uintptr_t)(S.ks + S.kpos) & 15);
        obuf_reclaim(S, W);
        restart_points(P, S, W, b);
        write_entries(P, W, b);
        __syncwarp();
        close_blocks(P, S, W, b);
        carry_over(P, S, W, b);
        e0 += b.cnt;
    }
    if (!err && S.open) finish_open(P, S, W); // the segment's last block
    if (!err && (S.blk_start != B.bytes + A.out_bytes || S.blk_idx != B.blocks + A.n_blocks || S.keyb != B.keyb + A.keyb)) err = PGS_CORRUPTION; // the two passes disagree
    if (err && lane == 0) { atomicMax(&P.stats->error, err); atomicMin(&P.stats->error_seg, q); }
}

// three CTAs per SM: what shared memory allows with an 8 KB output buffer and an 8 KB value stage per warp
__global__ void __launch_bounds__(kEmitThreads, 3) k_emit(const __grid_constant__ MergeParams P)
{
    PGS_SMEM_DYN(dyn);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (__shfl_sync(kFull, P.stats->error, 0)) return; // the plan or the walk failed: the output is discarded
    EmitWarp W;
    emit_warp(W, P, dyn + (size_t)warp * P.emit_warp_smem, lane);
    for (;;) {
        uint32_t q = 0;
        if (lane == 0) q = atomicAdd(P.ticket + 1, 1u);
        q = __shfl_sync(kFull, q, 0);
        if (q >= P.Q) break;
        const SegAgg A = P.agg[q];
        if (A.n_entries == 0) continue;
        const SegBase B = P.base[q];
        EmitSeg S;
        emit_seg(S, P, q, A, B);
        uint32_t err = 0;
        uint4 dn = make_uint4(0u, 0u, 0u, 0u); // the next batch's descriptors, fetched while this batch's values are copied
        uint32_t dn_e0 = 0xFFFFFFFFu;
        for (uint32_t e0 = 0; e0 < S.n && !err;) {
            EmitBatch b;
            batch_desc(b, S, W, e0, dn, dn_e0);
            const uint32_t first_fl = __shfl_sync(kFull, b.fl, 0);
            if (first_fl & DF_BIG) { emit_big(P, S, W, b, first_fl); e0++; continue; }
            if (batch_fit(P, S, W, b) == 0) { err = PGS_ABORTED; break; }
            stage_batch(P, S, W, b, e0, dn, dn_e0);
            batch_offsets(P, S, W, b);
            mbar_wait(W.bar, W.phase); // the one wait of a batch for global memory
            W.phase ^= 1;
            b.staged = W.stage + ((uintptr_t)(S.ks + S.kpos) & 15);
            obuf_reclaim(S, W);
            restart_points(P, S, W, b);
            write_entries(P, W, b);
            __syncwarp();
            close_blocks(P, S, W, b);
            carry_over(P, S, W, b);
            e0 += b.cnt;
        }
        if (!err && S.open) finish_open(P, S, W); // the segment's last block
        if (!err && (S.blk_start != B.bytes + A.out_bytes || S.blk_idx != B.blocks + A.n_blocks || S.keyb != B.keyb + A.keyb)) err = PGS_CORRUPTION; // the two passes disagree
        if (err && lane == 0) { atomicMax(&P.stats->error, err); atomicMin(&P.stats->error_seg, q); }
    }
    if (lane == 0) {
        tma_store_wait_all();
        if (W.n_bloom_keys) atomicAdd(&P.stats->cnt[EV_BLOOM_KEY], (unsigned long long)W.n_bloom_keys);
        if (W.n_bloom_prefixes) atomicAdd(&P.stats->cnt[EV_BLOOM_PREFIX], (unsigned long long)W.n_bloom_prefixes);
    }
}

// the k_walk instantiation for G lanes per merge group (host side)
typedef void (*walk_kernel_t)(const MergeParams);
constexpr uint32_t kWalkGs[] = {1, 2, 4, 8, 16};
inline walk_kernel_t walk_kernel(uint32_t G)
{
    switch (G) {
    case 1: return k_walk<1>;
    case 2: return k_walk<2>;
    case 4: return k_walk<4>;
    case 8: return k_walk<8>;
    default: return k_walk<16>;
    }
}

// The six kernels of one compaction on stream st.  k_walk and k_emit loop over the segments: walk_ctas / emit_ctas = how many
// of their CTAs the device runs at once.  mark(i) is called before k_plan (0), after k_seg_layout (1), after k_walk (2) and
// after k_emit (3).  Returns the number of launches.
template <class Mark>
inline uint32_t compact_launch(const MergeParams &P, const CompactGeometry &geo, uint64_t walk_ctas, uint64_t emit_ctas, cudaStream_t st,
                               Mark &&mark)
{
    const walk_kernel_t walk = walk_kernel(geo.G);
    const uint32_t seg_per_cta = kWalkThreads / geo.G;
    const uint32_t grid_w = (uint32_t)std::min<uint64_t>((P.Q + seg_per_cta - 1) / seg_per_cta, walk_ctas);
    const uint32_t grid_e = (uint32_t)std::min<uint64_t>((P.Q + geo.emit_warps - 1) / geo.emit_warps, emit_ctas);
    mark(0);
    PGS_LAUNCH(k_plan, (P.total_blocks + 255ull) / 256, 256, 0, st, P);
    PGS_LAUNCH(k_seg_bounds, (P.Q + 255ull) / 256, 256, 0, st, P);
    PGS_LAUNCH(k_seg_layout, 1, 1024, 0, st, P);
    mark(1);
    PGS_LAUNCH(walk, grid_w, kWalkThreads, geo.walk_dyn, st, P);
    mark(2);
    PGS_LAUNCH(k_seg_scan, 1, 1024, 0, st, P);
    PGS_LAUNCH(k_emit, grid_e, geo.emit_warps * 32, geo.emit_dyn, st, P);
    mark(3);
    return 6;
}

// ================================================================================================================================
// Several compactions in one launch (pgs_compact_many): the jobs of many partitions of one engine share one plan and one set of
// six launches.  Every job keeps its own MergeParams -- runs, policy and filter, scratch, output run, MergeStats -- in device
// memory; the launch numbers the jobs' segments one after the other (job j owns the launch's segments [seg_base[j],
// seg_base[j + 1])) and k_plan's threads likewise over the jobs' input blocks.  A kernel maps its global index to (job, local
// index) with job_of and runs the single-job code on that job's parameters: k_plan, k_seg_bounds and k_walk's segment walk are
// the same device functions as in the single launch, k_seg_layout and k_seg_scan give every job a CTA of its own, k_emit's
// warps draw global segments.  What the jobs share is the launch's shape: the widest user key sizes every job's key rows and
// k_emit's stages, the deepest job sizes the groups' cursor states, and one segment weight cuts every job (compact_many_geometry).
// ================================================================================================================================
constexpr uint32_t kMaxCompactJobs = 4096; // jobs of one multi-job launch

struct MergeJobs {
    const MergeParams *job;   // [n] in device memory
    const uint32_t *seg_base; // [n + 1]: job j's segments are the launch's segments [seg_base[j], seg_base[j + 1])
    const uint32_t *blk_base; // [n + 1]: job j's input blocks are k_plan's threads [blk_base[j], blk_base[j + 1])
    uint32_t n, Q, total_blocks;
    uint32_t k_max;           // the deepest job: every group's cursor states and head windows are sized for it
    uint32_t group_smem;      // one group's shared memory (every job's P.group_smem)
    uint32_t validate_hash;   // some job checks partition hashes: k_walk_many loads the crc table
    const unsigned long long *crc_table;
    uint32_t *ticket;         // [0] k_walk_many, [1] k_emit_many
};

__global__ void __launch_bounds__(256) k_plan_many(const __grid_constant__ MergeJobs M)
{
    const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    if (gt >= M.total_blocks) return;
    const uint32_t j = job_of(M.blk_base, M.n, gt);
    plan_block(M.job[j], gt - M.blk_base[j]); // ranked against its own job's runs, cut by the launch's one segment weight
}

__global__ void __launch_bounds__(256) k_seg_bounds_many(const __grid_constant__ MergeJobs M)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= M.Q) return;
    const uint32_t j = job_of(M.seg_base, M.n, q);
    seg_bound(M.job[j], q - M.seg_base[j]);
}

// one CTA per job: a segmented scan of the launch's segment list, each job's offsets from its own scratch's start
__global__ void __launch_bounds__(1024) k_seg_layout_many(const __grid_constant__ MergeJobs M) { seg_layout(M.job[blockIdx.x]); }
__global__ void __launch_bounds__(1024) k_seg_scan_many(const __grid_constant__ MergeJobs M) { seg_scan(M.job[blockIdx.x]); }

// A group's counters after a segment of a multi-job launch go to that segment's job: the events it kept in gst (its own
// WalkCtaStats, only its lane 0 touches it) and in acc, the byte sums and maxima in acc.  acc and gst start over.
PGS_DEV void walk_stats_flush(WalkAcc &acc, WalkCtaStats *gst, MergeStats *st, bool lane0)
{
    acc_flush_events(acc, gst, lane0);
    if (lane0) {
        for (uint32_t i = 0; i < 12; i++)
            if (gst->cnt[i]) { atomicAdd(&st->cnt[i], (unsigned long long)gst->cnt[i]); gst->cnt[i] = 0; }
        if (acc.b_in) atomicAdd(&st->bytes[SB_IN], acc.b_in);
        if (acc.b_key + acc.b_val) atomicAdd(&st->bytes[SB_OUT], acc.b_key + acc.b_val);
        if (acc.b_key) atomicAdd(&st->bytes[SB_OUT_KEY], acc.b_key);
        if (acc.b_val) atomicAdd(&st->bytes[SB_OUT_VAL], acc.b_val);
        if (acc.m_ukey) atomicMax(&st->mx[SM_UKEY], (unsigned long long)acc.m_ukey);
        if (acc.m_vlen) atomicMax(&st->mx[SM_VLEN], (unsigned long long)acc.m_vlen);
        if (acc.m_seq) atomicMax(&st->mx[SM_MAX_SEQ], acc.m_seq);
        if (acc.m_seq_inv) atomicMax(&st->mx[SM_MIN_SEQ_INV], acc.m_seq_inv);
        if (acc.m_bsize) atomicMax(&st->mx[SM_BLK_SIZE], (unsigned long long)acc.m_bsize);
        if (acc.m_brec) atomicMax(&st->mx[SM_BLK_REC], (unsigned long long)acc.m_brec);
    }
    acc.b_in = acc.b_key = acc.b_val = 0;
    acc.m_ukey = acc.m_vlen = acc.m_bsize = acc.m_brec = 0;
    acc.m_seq = acc.m_seq_inv = 0;
}

// k_walk over the segments of every job.  The groups of a warp may draw segments of different jobs, so there is no CTA-wide
// run table: a group reads its job's run table (MergeParams::runs) through the L1 cache -- a few hundred bytes per job, the
// same lines for the whole segment -- where k_walk copies its one table into shared memory.
template <uint32_t G>
__global__ void __launch_bounds__(kWalkThreads, 4) k_walk_many(const __grid_constant__ MergeJobs M)
{
    PGS_SMEM_DYN(dyn);
    const Grp<G> g;
    constexpr uint32_t NGW = 32 / G; // groups per warp
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gi = warp * NGW + g.shift / G; // the group inside the CTA
    unsigned long long *crc = (unsigned long long *)dyn;
    WalkCtaStats *gst = (WalkCtaStats *)(dyn + 2048) + gi;
    if (M.validate_hash)
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) crc[i] = M.crc_table[i];
    for (uint32_t i = g.gl; i < sizeof(WalkCtaStats) / 4; i += G) ((uint32_t *)gst)[i] = 0;
    __syncthreads();
    uint8_t *gs = dyn + walk_many_fixed_smem(G) + (size_t)gi * M.group_smem;
    CurState *cs = (CurState *)gs;
    uint32_t *rows = (uint32_t *)(gs + (size_t)M.k_max * sizeof(CurState));
    uint8_t *wins = dyn + walk_many_win_off(G, M.group_smem) + (size_t)gi * walk_win_stride(M.k_max);
    WalkAcc acc;
    acc.e0 = acc.e1 = acc.e2 = acc.n = 0;
    acc.b_in = acc.b_key = acc.b_val = 0;
    acc.m_ukey = acc.m_vlen = acc.m_bsize = acc.m_brec = 0;
    acc.m_seq = acc.m_seq_inv = 0;
#pragma unroll 1
    for (;;) {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(M.ticket, NGW);
        t0 = __shfl_sync(kFull, t0, 0);
        if (t0 >= M.Q) break;
        const uint32_t q = t0 + g.shift / G;
        const uint32_t j = q < M.Q ? job_of(M.seg_base, M.n, q) : 0u;
        const MergeParams &P = M.job[j];
        // a job whose plan failed is not walked (its output is discarded); one lane reads the flag for the whole group
        const uint32_t failed = g.shfl(g.gl == 0 ? P.stats->error : 0u, 0);
        const bool en = q < M.Q && failed == 0;
        walk_segment<G, true>(P, P.runs, g, en, en ? q - M.seg_base[j] : 0u, cs, rows, wins, crc, acc, gst, M.k_max);
        walk_stats_flush(acc, gst, P.stats, en && g.gl == 0);
    }
}

// k_emit over the segments of every job: a warp draws global segments and writes each into its own job's run, index and
// Bloom filter; the filter counts go to that job's MergeStats after every segment
__global__ void __launch_bounds__(kEmitThreads, 3) k_emit_many(const __grid_constant__ MergeJobs M)
{
    PGS_SMEM_DYN(dyn);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const MergeParams &P0 = M.job[0]; // the stages' layout is the launch's, the same in every job
    EmitWarp W;
    emit_warp(W, P0, dyn + (size_t)warp * P0.emit_warp_smem, lane);
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(M.ticket + 1, 1u);
        t = __shfl_sync(kFull, t, 0);
        if (t >= M.Q) break;
        const uint32_t j = job_of(M.seg_base, M.n, t);
        const MergeParams &P = M.job[j];
        if (__shfl_sync(kFull, lane == 0 ? P.stats->error : 0u, 0)) continue; // its plan or walk failed: discarded
        emit_segment(P, W, t - M.seg_base[j]);
        if (lane == 0) {
            if (W.n_bloom_keys) atomicAdd(&P.stats->cnt[EV_BLOOM_KEY], (unsigned long long)W.n_bloom_keys);
            if (W.n_bloom_prefixes) atomicAdd(&P.stats->cnt[EV_BLOOM_PREFIX], (unsigned long long)W.n_bloom_prefixes);
        }
        W.n_bloom_keys = W.n_bloom_prefixes = 0;
    }
    if (lane == 0) tma_store_wait_all();
}

typedef void (*walk_many_kernel_t)(const MergeJobs);
inline walk_many_kernel_t walk_many_kernel(uint32_t G)
{
    switch (G) {
    case 1: return k_walk_many<1>;
    case 2: return k_walk_many<2>;
    case 4: return k_walk_many<4>;
    case 8: return k_walk_many<8>;
    default: return k_walk_many<16>;
    }
}

// The joint plan of n jobs (host side).  P[i] holds job i's k, runs, block_size, restart_interval, policy and filter fields,
// T[i] its totals.  The widest user key sizes every job's key rows and k_emit's stages, the deepest job every group's cursor
// states, and one segment weight is sized from the whole launch's weight (walk_groups and force_* as in compact_geometry).
// Then every job gets its own segments and output bounds (geo[i]); shared = the launch's walk and emit shape.  M gets the
// launch's counts and shape, no pointers.  false: the jobs do not fit one launch (the caller can split them).
inline bool compact_many_geometry(MergeParams *P, const CompactTotals *T, CompactGeometry *geo, uint32_t n, uint32_t max_smem,
                                  MergeJobs &M, CompactGeometry &shared, uint32_t force_G = 0, uint64_t force_weight = 0,
                                  uint64_t walk_groups = 0)
{
    if (n == 0 || n > kMaxCompactJobs) return false;
    CompactTotals J{};
    uint32_t k_max = 0;
    for (uint32_t i = 0; i < n; i++) {
        J.max_ukey = std::max(J.max_ukey, T[i].max_ukey);
        J.max_blk = std::max(J.max_blk, T[i].max_blk);
        J.max_blk_rec = std::max(J.max_blk_rec, T[i].max_blk_rec);
        J.total_blocks += T[i].total_blocks;
        J.n_rec += T[i].n_rec;
        J.raw_key += T[i].raw_key;
        J.raw_val += T[i].raw_val;
        J.in_block_bytes += T[i].in_block_bytes;
        J.bloom_entries += T[i].bloom_entries;
        k_max = std::max(k_max, P[i].k);
    }
    MergeParams L = P[0];
    L.k = k_max;
    if (!compact_geometry(L, J, max_smem, shared, force_G, force_weight, walk_groups, 0, true)) return false;
    uint64_t Q = 0, blocks = 0;
    for (uint32_t i = 0; i < n; i++) {
        CompactTotals t = T[i];
        t.max_ukey = J.max_ukey; // the key rows of the widest key
        if (!compact_geometry(P[i], t, max_smem, geo[i], shared.G, L.tile_weight, 0, 0, true)) return false;
        if (P[i].KS != L.KS || P[i].blk_buf != L.blk_buf || P[i].emit_warp_smem != L.emit_warp_smem || P[i].block_size != L.block_size) return false;
        P[i].group_smem = L.group_smem;
        Q += P[i].Q;
        blocks += P[i].total_blocks;
    }
    if (Q > 0x7FFFFFF0ull || blocks > 0xFFFFFFF0ull) return false;
    M.n = n;
    M.Q = (uint32_t)Q;
    M.total_blocks = (uint32_t)blocks;
    M.k_max = k_max;
    M.group_smem = L.group_smem;
    return true;
}
// the exclusive prefixes of the jobs' segments and input blocks (n + 1 entries each)
inline void compact_many_bases(const MergeParams *P, uint32_t n, uint32_t *seg_base, uint32_t *blk_base)
{
    seg_base[0] = blk_base[0] = 0;
    for (uint32_t i = 0; i < n; i++) {
        seg_base[i + 1] = seg_base[i] + P[i].Q;
        blk_base[i + 1] = blk_base[i] + P[i].total_blocks;
    }
}

// The six kernels of a multi-job compaction on stream st, as compact_launch (the same marks, the same launch count).
template <class Mark>
inline uint32_t compact_launch_many(const MergeJobs &M, const CompactGeometry &geo, uint64_t walk_ctas, uint64_t emit_ctas, cudaStream_t st,
                                    Mark &&mark)
{
    const walk_many_kernel_t walk = walk_many_kernel(geo.G);
    const uint32_t seg_per_cta = kWalkThreads / geo.G;
    const uint32_t grid_w = (uint32_t)std::min<uint64_t>((M.Q + seg_per_cta - 1) / seg_per_cta, walk_ctas);
    const uint32_t grid_e = (uint32_t)std::min<uint64_t>((M.Q + geo.emit_warps - 1) / geo.emit_warps, emit_ctas);
    mark(0);
    PGS_LAUNCH(k_plan_many, std::max(1ull, (M.total_blocks + 255ull) / 256), 256, 0, st, M);
    PGS_LAUNCH(k_seg_bounds_many, (M.Q + 255ull) / 256, 256, 0, st, M);
    PGS_LAUNCH(k_seg_layout_many, M.n, 1024, 0, st, M);
    mark(1);
    PGS_LAUNCH(walk, grid_w, kWalkThreads, geo.walk_dyn, st, M);
    mark(2);
    PGS_LAUNCH(k_seg_scan_many, M.n, 1024, 0, st, M);
    PGS_LAUNCH(k_emit_many, grid_e, geo.emit_warps * 32, geo.emit_dyn, st, M);
    mark(3);
    return 6;
}

} // namespace pgs
