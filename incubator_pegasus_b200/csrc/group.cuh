// group.cuh — lane-group primitives shared by the compaction walker and the read kernels.
//
// A *group* is G consecutive lanes of a warp (G = 1, 2, 4, 8, 16 or 32) that together run one sequential iterator over sorted
// runs: group-uniform scalars (offsets, lengths, counters) are computed redundantly by every lane, the bytes of a key
// are spread over the lanes (lane L owns the 32-bit words L, L+G, ... of a key row in shared memory) and compared with
// one ballot.  The 32/G groups of a warp run in LOCK STEP on different data: control flow around every collective is
// warp-uniform (loops run while any group still needs them, per-group work is switched on and off with an `en`
// predicate), so all shuffles / ballots use the constant full mask -- a collective with a run-time lane mask costs a
// MATCH.ANY + REDUX convergence check per call and lets the groups drift apart.
// G = 1 is the degenerate case: one thread per iterator, no collectives at all, so its control flow may diverge freely (the
// hardware serialises the paths); the same source serves both shapes.
// This is the GPU shape of RocksDB's DataBlockIter / MergingIterator (v8.5.3, not in the reference tree; SURVEY.md
// Appendix A): the per-record decode chain stays sequential, the parallelism comes from thousands of independent groups.
#pragma once
#include "../../include/pegasus_b200.h"
#include "device_util.cuh"

namespace pgs {

template <uint32_t G>
struct Grp {
    static constexpr uint32_t kLow = G == 32 ? 0xffffffffu : ((1u << (G & 31)) - 1u);
    uint32_t gl;    // lane inside the group
    uint32_t shift; // first lane of the group inside the warp
    PGS_DEV Grp()
    {
        const uint32_t lane = threadIdx.x & 31;
        gl = lane & (G - 1);
        shift = lane & ~(G - 1);
    }
    // every lane of the warp executes these together; the result is the own group's
    PGS_DEV uint32_t ballot(bool p) const { return (__ballot_sync(kFull, p) >> shift) & kLow; }
    template <class T> PGS_DEV T shfl(T v, uint32_t src) const { return __shfl_sync(kFull, v, (int)(src & (G - 1)), (int)G); }
    template <class T> PGS_DEV T shfl_down(T v, uint32_t d) const { return __shfl_down_sync(kFull, v, d, (int)G); }
    template <class T> PGS_DEV T shfl_up(T v, uint32_t d) const { return __shfl_up_sync(kFull, v, d, (int)G); }
    PGS_DEV static bool any(bool p) { return __any_sync(kFull, p) != 0; }
    PGS_DEV static void sync() { __syncwarp(); }
};

template <>
struct Grp<1> { // one thread = one group: every "collective" is the identity, nothing synchronises
    uint32_t gl, shift;
    PGS_DEV Grp() : gl(0), shift(threadIdx.x & 31) {}
    PGS_DEV uint32_t ballot(bool p) const { return p ? 1u : 0u; }
    template <class T> PGS_DEV T shfl(T v, uint32_t) const { return v; }
    template <class T> PGS_DEV T shfl_down(T v, uint32_t) const { return v; }
    template <class T> PGS_DEV T shfl_up(T v, uint32_t) const { return v; }
    PGS_DEV static bool any(bool p) { return p; }
    PGS_DEV static void sync() {}
};

// Compare two byte strings held in key rows (4-byte aligned shared memory, readable up to the next multiple of 4).
// Returns <0, 0, >0; dpos = index of the first differing byte, or min(la, lb) when one is a prefix of the other.
// `from` = a number of leading bytes already known to be equal (the compare starts at the word that holds byte `from`).
// Executed by the whole warp; groups with en = false take part in the collectives and get 0.
template <uint32_t G>
PGS_DEV int row_cmp(const Grp<G> &g, bool en, const uint32_t *a, uint32_t la, const uint32_t *b, uint32_t lb, uint32_t &dpos, uint32_t from = 0)
{
    const uint32_t m = en ? (la < lb ? la : lb) : 0u;
    int res = 2; // undecided
#pragma unroll 1
    for (uint32_t base = from & ~3u; g.any(res == 2 && base < m); base += 4 * G) {
        const uint32_t off = base + 4 * g.gl;
        uint32_t x = 0;
        if (res == 2 && off < m) {
            x = a[off >> 2] ^ b[off >> 2];
            if (m - off < 4) x &= (1u << (8 * (m - off))) - 1u;
        }
        const uint32_t bal = g.ballot(x != 0);
        const uint32_t first = (uint32_t)__ffs((int)bal) - 1;
        const uint32_t xx = g.shfl(x, first);
        if (res == 2 && bal) {
            const uint32_t at = base + 4 * first + (((uint32_t)__ffs((int)xx) - 1) >> 3);
            dpos = at;
            const uint32_t ba = (a[at >> 2] >> (8 * (at & 3))) & 0xffu, bb = (b[at >> 2] >> (8 * (at & 3))) & 0xffu;
            res = ba < bb ? -1 : 1;
        }
    }
    if (!en) return 0;
    if (res == 2) {
        dpos = m;
        res = la < lb ? -1 : (la > lb ? 1 : 0);
    }
    return res;
}

// ---- sequential cursor over the blocks of one HBM-resident run ------------------------------------------------------------
// Group-uniform state of one cursor, in shared memory.  The cursor reads entries straight from global memory: one
// dependent round trip per entry (the header), everything else of the entry's head lies in the same or the next cache line.
// Latency is hidden by the number of groups in flight, not by staging.
struct CurState { // 32-bit fields only: any 4-byte-aligned stride between the states of neighbouring groups works
    uint32_t base_lo, base_hi; // blk_off[b]
    uint32_t nb_lo, nb_hi;     // blk_off[b + 1], fetched asynchronously when block b was entered
    uint32_t nb_r0, nb_r1;     // blk_rec[b + 1], blk_rec[b + 2] (same)
    uint32_t bsize, nb_size;   // blk_size[b], blk_size[b + 1] (same)
    uint32_t b, b_end;         // current block; first block that does not belong to the cursor's range
    uint32_t p, elen;          // offset of the current entry inside its block, its encoded length
    uint32_t rem;              // entries left in the block, the current one included
    uint32_t klen;             // internal-key length of the current entry (user key + 8)
    uint32_t vlen, voff;       // value length, value offset inside the block
    uint32_t shared;           // the entry's `shared` field (prefix shared with the previous key of the run)
    uint32_t ets_le;           // first four value bytes as loaded (BE32 expire_ts, byte-swapped when used)
    uint32_t tr_lo, tr_hi;     // trailer: seq << 8 | type
    uint32_t chk_from;         // blocks >= chk_from may hold keys above the range's upper bound
    uint32_t live;             // 0 once the cursor is exhausted
    uint32_t kp_hi, kp_lo;     // the first eight key bytes as a big-endian number (zero padded): most order decisions need no more
    uint32_t hi_lcp;           // compaction walker: bytes the key shares with the range's upper bound (0x80000000: not known)
    uint32_t hw0, hw1, hw2;    // the aligned words that hold the NEXT entry's first eight bytes (its header), fetched
    uint32_t hvalid;           // asynchronously when this entry was decoded; hvalid = there is such an entry and it was fetched
};
PGS_DEV unsigned long long cur_trailer(const CurState *c) { return ((unsigned long long)c->tr_hi << 32) | c->tr_lo; }
PGS_DEV unsigned long long cur_base(const CurState *c) { return ((unsigned long long)c->base_hi << 32) | c->base_lo; }

// start fetching the metadata of block b + 1 (asynchronous copies into the state; consumed when the block is entered)
template <uint32_t G>
PGS_DEV void cur_prefetch_next(const Grp<G> &g, bool en, const RunDev &r, CurState *c, uint32_t b)
{
    if (en && b + 1 < r.nb) { // blk_off and blk_rec have nb + 1 entries
#pragma unroll
        for (uint32_t i = g.gl; i < 5; i += G) {
            if (i == 0) async_copy4(&c->nb_lo, (const uint32_t *)(r.blk_off + b + 1));
            if (i == 1) async_copy4(&c->nb_hi, (const uint32_t *)(r.blk_off + b + 1) + 1);
            if (i == 2) async_copy4(&c->nb_r0, r.blk_rec + b + 1);
            if (i == 3) async_copy4(&c->nb_r1, r.blk_rec + b + 2);
            if (i == 4) async_copy4(&c->nb_size, r.blk_size + b + 1);
        }
    }
    async_copy_commit();
}

// three varint32 (shared, non_shared, value_len) at A, any shape; returns the header length or 0 (malformed).  Rare path.
static __device__ __noinline__ uint32_t parse_header_slow(const uint8_t *A, uint32_t &sh, uint32_t &ns, uint32_t &vl)
{
    uint32_t c1 = get_varint32(A, 5, sh), c2 = 0, c3 = 0;
    if (c1) c2 = get_varint32(A + c1, 5, ns);
    if (c2) c3 = get_varint32(A + c1 + c2, 5, vl);
    return c3 ? c1 + c2 + c3 : 0u;
}
// 8 bytes at an arbitrary address as two 32-bit halves: three aligned word loads + two funnel shifts (no 64-bit arithmetic)
PGS_DEV void ld_2x32_any(const uint8_t *p, uint32_t &lo, uint32_t &hi)
{
    const uint32_t *w = (const uint32_t *)((uintptr_t)p & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)((uintptr_t)p & 3) * 8;
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    lo = __funnelshift_r(w0, w1, sh);
    hi = __funnelshift_r(w1, w2, sh);
}

// decode the entry at (base, p) of the current block into the state and the key row (groups with en).  prev_klen = internal-
// key length of the previous entry of the block (0 at a block start: the entry must then be a restart point).
// Executed by the whole warp (two warp barriers inside).  Returns 0 or a status.
template <uint32_t G>
PGS_DEV uint32_t cur_decode(const Grp<G> &g, bool en, const RunDev &r, CurState *c, uint32_t *row, uint32_t KS, unsigned long long base,
                            uint32_t p, uint32_t blk_size, uint32_t prev_klen, uint32_t rem_new, bool stashed = false)
{
    uint32_t err = 0, sh = 0, ns = 0, vl = 0, h = 0, klen = 0;
    const uint8_t *src = nullptr;
    const uint8_t *A = nullptr;
    if (en) {
        A = r.data + base + p;
        uint32_t h_lo, h_hi;
        if (stashed) { // the header words arrived while the previous entry was being handled
            const uint32_t s8 = (uint32_t)((uintptr_t)A & 3) * 8, w0 = c->hw0, w1 = c->hw1, w2 = c->hw2;
            h_lo = __funnelshift_r(w0, w1, s8);
            h_hi = __funnelshift_r(w1, w2, s8);
        } else ld_2x32_any(A, h_lo, h_hi);
        h = parse_header8(((unsigned long long)h_hi << 32) | h_lo, sh, ns, vl);
        if (!h) { // uncommon shape (a length of two or more varint bytes): byte-wise decoder
            h = parse_header_slow(A, sh, ns, vl);
            if (!h) err = PGS_CORRUPTION;
        }
        klen = sh + ns;
        if (!err && (sh > prev_klen || klen < 8 || klen - 8 > KS || (unsigned long long)p + h + ns + vl + 8 > blk_size)) err = PGS_CORRUPTION;
        if (!err) {
            // key bytes [sh, sh + ns) <- the entry's delta; lane L owns the words L, L + G, ... of the row
            src = A + h;
            const uint32_t end = sh + ns;
#pragma unroll 1
            for (uint32_t w = (sh >> 2) + g.gl; 4 * w < end; w += G) {
                const uint32_t lo = 4 * w;
                const uint32_t v = ld_u32_any(src + (int32_t)(lo - sh));
                uint32_t keep = 0; // bytes of the word that are not covered by the delta keep their old value
                if (lo < sh) keep = (1u << (8 * (sh - lo))) - 1u;
                if (end - lo < 4) keep |= ~((1u << (8 * (end - lo))) - 1u);
                row[w] = keep ? ((row[w] & keep) | (v & ~keep)) : v;
            }
        }
    }
    g.sync();
    if (en && !err) {
        uint32_t tr_lo, tr_hi;
        if (ns >= 8) ld_2x32_any(src + ns - 8, tr_lo, tr_hi);
        else { const unsigned long long tr = lds_u64_at((const uint8_t *)row, klen - 8); tr_lo = (uint32_t)tr; tr_hi = (uint32_t)(tr >> 32); } // part of the trailer is shared with the previous key
        const uint32_t ets = vl >= 4 ? ld_u32_any(src + ns) : 0u;
        if (g.gl == 0) {
            c->p = p; c->elen = h + ns + vl; c->klen = klen; c->vlen = vl; c->voff = p + h + ns; c->shared = sh; c->ets_le = ets;
            c->rem = rem_new;
            c->hvalid = rem_new >= 2 ? 1u : 0u;
            c->tr_lo = tr_lo; c->tr_hi = tr_hi;
            if (sh < 8) { // the leading bytes changed
                const uint32_t ul = klen - 8;
                uint32_t w0 = row[0], w1 = row[1];
                if (ul < 4) { w0 &= (1u << (8 * ul)) - 1u; w1 = 0; }
                else if (ul < 8) w1 &= (1u << (8 * (ul - 4))) - 1u;
                c->kp_hi = __byte_perm(w0, 0, 0x0123); c->kp_lo = __byte_perm(w1, 0, 0x0123);
            }
        }
        if (rem_new >= 2) { // the next entry of the block: start fetching its header words (consumed by the next cur_next)
            const uint32_t *nw = reinterpret_cast<const uint32_t *>((uintptr_t)(A + h + ns + vl) & ~(uintptr_t)3);
#pragma unroll
            for (uint32_t i = g.gl; i < 3; i += G) async_copy4(i == 0 ? &c->hw0 : i == 1 ? &c->hw1 : &c->hw2, nw + i);
        }
    }
    async_copy_commit();
    g.sync();
    return err;
}

// position the cursor on the first entry of block b (or leave it exhausted when b >= b_end); synchronous metadata loads
template <uint32_t G>
PGS_DEV uint32_t cur_open(const Grp<G> &g, bool en, const RunDev &r, CurState *c, uint32_t *row, uint32_t KS, uint32_t b, uint32_t b_end, uint32_t chk_from)
{
    const bool some = en && b < b_end && b < r.nb;
    unsigned long long base = 0;
    uint32_t r0 = 0, r1 = 0, bsize = 0;
    if (some) { base = r.blk_off[b]; r0 = r.blk_rec[b]; r1 = r.blk_rec[b + 1]; bsize = r.blk_size[b]; }
    if (en && g.gl == 0) {
        c->live = some ? 1u : 0u; c->b = b; c->b_end = b_end; c->chk_from = chk_from;
        if (some) { c->base_lo = (uint32_t)base; c->base_hi = (uint32_t)(base >> 32); c->rem = r1 - r0; c->bsize = bsize; }
    }
    g.sync();
    cur_prefetch_next(g, some, r, c, b);
    const uint32_t err = some && r1 <= r0 ? (uint32_t)PGS_CORRUPTION : 0u; // a block holds at least one entry
    const uint32_t e2 = cur_decode(g, some && !err, r, c, row, KS, base, 0, bsize, 0, r1 - r0);
    return err ? err : e2;
}

// advance to the next entry (groups with en); crossing into the next block uses the metadata fetched when the current block
// was entered.  Leaves live = 0 when the range is exhausted.  Executed by the whole warp.  Returns 0 or a status.
template <uint32_t G>
PGS_DEV uint32_t cur_next(const Grp<G> &g, bool en, const RunDev &r, CurState *c, uint32_t *row, uint32_t KS)
{
    uint32_t rem = 0, b = 0, p = 0, prev_klen = 0, bsize = 0;
    unsigned long long base = 0;
    bool in_block = false, cross = false, done = false, stashed = false;
    if (en) {
        rem = c->rem; b = c->b;
        in_block = rem > 1;
        if (in_block) { base = cur_base(c); p = c->p + c->elen; prev_klen = c->klen; bsize = c->bsize; stashed = c->hvalid != 0; }
        else if (b + 1 >= c->b_end || b + 1 >= r.nb) done = true;
        else cross = true;
    }
    async_copy_wait_all(); // the header words fetched when the current entry was decoded (and, long ago, the next block's metadata)
    g.sync(); // every lane is done with the old key row and state, and sees the fetched words
    uint32_t r0 = 0, r1 = 0;
    if (g.any(cross || done)) { // a block boundary (about one step in thirteen)
        if (cross) { base = ((unsigned long long)c->nb_hi << 32) | c->nb_lo; r0 = c->nb_r0; r1 = c->nb_r1; bsize = c->nb_size; }
        g.sync();
        if (en && g.gl == 0) {
            if (done) { c->live = 0; c->b = b + 1; }
            else if (cross) { c->b = b + 1; c->base_lo = (uint32_t)base; c->base_hi = (uint32_t)(base >> 32); c->bsize = bsize; }
        }
        g.sync();
        cur_prefetch_next(g, cross, r, c, b + 1);
    }
    const uint32_t err = cross && r1 <= r0 ? (uint32_t)PGS_CORRUPTION : 0u;
    const uint32_t e2 = cur_decode(g, (in_block || cross) && !err, r, c, row, KS, base, p, bsize, prev_klen, in_block ? rem - 1 : r1 - r0, stashed);
    return err ? err : e2;
}

// order of two cursor heads as internal keys: user key ascending, then trailer (seq, type) descending, then run index.
// Whole warp; by_byte = decided by a differing key byte at dpos (the LCP shortcut of the merge loop relies on that).
template <uint32_t G>
PGS_DEV bool head_before(const Grp<G> &g, bool en, const CurState *cs, const uint32_t *rows, uint32_t KSW, uint32_t a, uint32_t b, uint32_t &dpos, bool &by_byte,
                         uint32_t from = 0) // from: leading bytes known to be equal
{
    uint32_t la = 0, lb = 0;
    bool full = en; // the first eight bytes decide most of the time: two scalar compares, no collective
    if (en) {
        la = cs[a].klen - 8; lb = cs[b].klen - 8;
        const uint32_t ah = cs[a].kp_hi, al = cs[a].kp_lo, bh = cs[b].kp_hi, bl = cs[b].kp_lo;
        if ((ah != bh || al != bl) && la >= 8 && lb >= 8) {
            dpos = ah != bh ? (uint32_t)__clz((int)(ah ^ bh)) >> 3 : 4 + ((uint32_t)__clz((int)(al ^ bl)) >> 3);
            by_byte = true;
            full = false;
        }
    }
    if (!g.any(full)) {
        if (!en) { by_byte = false; return false; }
        const uint32_t ah = cs[a].kp_hi, bh = cs[b].kp_hi;
        return ah != bh ? ah < bh : cs[a].kp_lo < cs[b].kp_lo;
    }
    uint32_t dfull = 0;
    const int c = row_cmp(g, full, rows + a * KSW, la, rows + b * KSW, lb, dfull, from);
    if (!en) { by_byte = false; return false; }
    if (!full) {
        const uint32_t ah = cs[a].kp_hi, bh = cs[b].kp_hi;
        return ah != bh ? ah < bh : cs[a].kp_lo < cs[b].kp_lo;
    }
    dpos = dfull;
    by_byte = c != 0 && dpos < (la < lb ? la : lb);
    if (c) return c < 0;
    const unsigned long long ta = cur_trailer(&cs[a]), tb = cur_trailer(&cs[b]);
    if (ta != tb) return ta > tb;
    return a < b;
}

// ---- Bloom filter of a run (device-built at upload / compaction time) --------------------------------------------------
// 10 bits per entry, cache-line blocked: an entry hashes to one 64-byte line and sets / tests 6 bits inside it (the shape of
// RocksDB's cache-local full filter, v8.5.3 util/bloom_impl.h, not in tree).  Entries are whole user keys and hash-key
// prefixes (HashkeyTransform: the first 2 + BE16 bytes), as the reference configures its filter
// (src/server/pegasus_server_impl_init.cpp:817-843).  The hash is a position-salted XOR of per-word mixes, so the lanes of
// a group hash their own words of a key row and combine with shuffles.
PGS_DEV void bloom_word(uint32_t w, uint32_t idx, uint32_t &ha, uint32_t &hb)
{
    uint32_t a = (w + 0x9E3779B9u * (idx + 1)) * 0x85EBCA6Bu;
    a ^= a >> 15; a *= 0xC2B2AE35u; a ^= a >> 13;
    uint32_t b = a * 0x27D4EB2Fu; // the second half rides on the first mix
    b ^= b >> 16;
    ha ^= a; hb ^= b;
}
PGS_DEV unsigned long long bloom_finish(uint32_t ha, uint32_t hb, uint32_t len)
{
    unsigned long long h = ((unsigned long long)(ha ^ (len * 0x9E3779B1u)) << 32) | hb;
    h ^= h >> 29; h *= 0xD6E8FEB86659FD93ull; h ^= h >> 32;
    return h;
}
// hash of the first len bytes of a key row (4-byte aligned, any address space); every lane of the group gets the result (whole warp)
template <uint32_t G>
PGS_DEV unsigned long long bloom_hash_row(const Grp<G> &g, const uint32_t *row, uint32_t len)
{
    uint32_t ha = 0, hb = 0;
#pragma unroll 1
    for (uint32_t w = g.gl; 4 * w < len; w += G) {
        uint32_t x = row[w];
        if (len - 4 * w < 4) x &= (1u << (8 * (len - 4 * w))) - 1u;
        bloom_word(x, w, ha, hb);
    }
#pragma unroll
    for (uint32_t d = G / 2; d; d >>= 1) { ha ^= __shfl_xor_sync(kFull, ha, (int)d); hb ^= __shfl_xor_sync(kFull, hb, (int)d); }
    return bloom_finish(ha, hb, len);
}
// the same hash by one thread over bytes anywhere
PGS_DEV unsigned long long bloom_hash_bytes(const uint8_t *key, uint32_t len)
{
    uint32_t ha = 0, hb = 0;
    for (uint32_t w = 0; 4 * w < len; w++) {
        uint32_t x = 0;
        for (uint32_t b = 0; b < 4 && 4 * w + b < len; b++) x |= (uint32_t)key[4 * w + b] << (8 * b);
        bloom_word(x, w, ha, hb);
    }
    return bloom_finish(ha, hb, len);
}
PGS_DEV uint32_t bloom_bit(unsigned long long h, uint32_t i) // i-th of the 6 bit positions (0..511) inside the line
{
    uint32_t x = (uint32_t)h + i * 0x9E3779B1u;
    x ^= x >> 15; x *= 0x2C1B3C6Du; x ^= x >> 12;
    return x & 511u;
}
PGS_DEV bool bloom_may_contain(const uint32_t *bits, uint32_t n_lines, unsigned long long h)
{
    if (n_lines == 0) return true; // no filter built
    const uint32_t *line = bits + 16 * (size_t)(((h >> 32) * (unsigned long long)n_lines) >> 32);
#pragma unroll
    for (uint32_t i = 0; i < 6; i++) {
        const uint32_t bit = bloom_bit(h, i);
        if (!((line[bit >> 5] >> (bit & 31)) & 1u)) return false;
    }
    return true;
}
// lanes 0..5 of a group set one bit each (sub < 6); a single thread passes sub = 0..5 in a loop
PGS_DEV void bloom_add_bit(uint32_t *bits, uint32_t n_lines, unsigned long long h, uint32_t sub)
{
    uint32_t *line = bits + 16 * (size_t)(((h >> 32) * (unsigned long long)n_lines) >> 32);
    const uint32_t bit = bloom_bit(h, sub);
    atomicOr(&line[bit >> 5], 1u << (bit & 31));
}
PGS_HD uint32_t bloom_lines_for(unsigned long long n_entries) { return (uint32_t)((n_entries * 10 + 511) / 512 + 1); }
// length of the HashkeyTransform prefix of a raw key (hashkey_transform.h:40-60); 0 = not in domain
PGS_DEV uint32_t hashkey_prefix_len(const uint8_t *key, uint32_t len)
{
    if (len < 2) return 0;
    const uint32_t p = 2 + (((uint32_t)key[0] << 8) | key[1]);
    return p <= len ? p : 0;
}

} // namespace pgs
