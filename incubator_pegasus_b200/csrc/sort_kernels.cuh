// sort_kernels.cuh — flat records in any order sorted into internal-key order on the GPU (host side: pgs_run_build_unsorted in
// engine.cu), then gathered into sorted copies that the run build (build_kernels.cuh) takes unchanged.
//
// Order: user keys bytewise as unsigned bytes, a proper prefix first; equal user keys by seq << 8 | type descending.
// Method: groups of records tied so far are refined one 8-byte window of the user key per round.  Round w sorts the records
// still tied by the key (group, window w big-endian and zero-padded, bytes of the key inside the window 0..8) with stable LSD
// radix passes, 8 bits per pass.  The byte count makes "ab" sort before "ab\0" and marks where a key ends.  A record whose key
// ended before window w (all records of its group did: they share the key so far) is keyed by ~(seq << 8 | type) with the count
// kSortTrailer instead, so the round after a key's end orders its versions.  After each round a record alone in its group is
// final; the others, still tied, go on.  Two records tied after their trailer round are a duplicate internal key.  Rounds are at
// most kMaxUkeyLen / 8 + 2; each costs the records still tied, so the work is the records' distinguishing prefixes / 8.
//   k_sort_check     one thread per record: offsets ascending inside [0, off[n]], user key <= kMaxUkeyLen; identity order
//   (host)           reads the summary: bad offsets or a long key refuse the call before any key byte is read
//   per round w:
//   k_sort_keys      one thread per tied record: its round key into buffer 0, which key bytes differ across the records, and
//                    whether it differs from the record before it in its group
//   (host)           reads the summary: the tied records m, the bytes that vary (only those get a radix pass).  A round in
//                    which no group splits moves nothing and is skipped (a group in its trailer round then holds duplicates).
//   k_sort_hist, k_sort_hist_scan, k_sort_scatter
//                    one stable radix pass over one byte of the key: tile histograms, their scan (digit-major), the scatter
//                    (ranks inside a tile from __match_any_sync, warp by warp, so the pass is stable)
//   k_sort_tile_sums / k_sort_tile_scan / k_sort_place <SortSettle>
//                    each tied slot takes its sorted record; records still tied are compacted with their new group ordinals
//   then k_sort_tile_sums / k_sort_tile_scan / k_sort_place <SortGather> and k_sort_copy write the sorted copy: offsets from a
//   scan of the lengths, seq and type, then one warp per record copies its key and value bytes.
#pragma once
#include "build_kernels.cuh"

namespace pgs {

constexpr uint32_t kSortThreads = 256;                       // 8 warps
constexpr uint32_t kSortWarps = kSortThreads / 32;
constexpr uint32_t kSortItems = 16;                          // per thread of a radix tile
constexpr uint32_t kSortTile = kSortThreads * kSortItems;    // records per CTA of a radix pass and of the scans
constexpr uint32_t kSortScanThreads = 1024;                  // at most, in the one CTA that scans tiles (sort_scan_threads)
constexpr uint32_t kSortDigits = 13;                         // radix digits, least significant first: count, window 0..7, group 0..3
constexpr uint32_t kSortTrailer = 15;                        // count of a round that orders the versions of one user key
constexpr uint32_t kSortMaxRounds = kMaxUkeyLen / 8 + 2;     // windows 0..kMaxUkeyLen / 8, then the trailer

// SortSummary::flags
constexpr uint32_t kSortBadOffsets = 1; // key_off / val_off not ascending inside [0, off[n]]: kInvalidArgument
constexpr uint32_t kSortLongKey = 2;    // a user key over kMaxUkeyLen: kNotSupported
constexpr uint32_t kSortDuplicate = 4;  // two records with the same user key and trailer: kInvalidArgument

struct SortRound {               // what k_sort_keys found in one round
    unsigned long long vary[2];  // the bits of (lo, hi) in which some tied record differs from the first: the radix passes
    uint32_t split, trailer;     // some group has two different keys; some record is in its trailer round
};
struct SortSummary {
    SortRound round[2]; // round w in slot w & 1
    uint32_t m, flags;  // m: the records still tied
};

struct SortParams {
    // input (device copies of the caller's flat arrays)
    const uint8_t *keys, *vals, *type;
    const unsigned long long *key_off, *val_off, *seq;
    uint32_t n, tiles; // tiles: of kSortTile records over n
    // scratch
    uint32_t *perm;                 // [n]: position -> record
    uint32_t *pos[2], *grp[2];      // [n] each: the tied records' positions and group ordinals (current, next)
    unsigned long long *lo[2], *hi[2]; // [n] each: round keys (radix ping-pong)
    uint32_t *rec[2];               // [n] each: the record of each round key
    uint32_t *hist;                 // [256 * tiles]: digit-major tile histograms, then their exclusive scan
    unsigned long long *tile_sum;   // [2 * tiles]
    SortSummary *sum;               // zeroed by the host
    // output: the sorted copy (key_off[n] + 16 and val_off[n] + 16 bytes of keys and values)
    uint8_t *s_keys, *s_vals, *s_type;
    unsigned long long *s_key_off, *s_val_off, *s_seq;
};

__global__ void __launch_bounds__(kSortThreads) k_sort_check(const SortParams P)
{
    const uint32_t n = P.n;
    const unsigned long long kend = P.key_off[n], vend = P.val_off[n];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (i == 0) P.sum->m = n;
        const unsigned long long k0 = P.key_off[i], k1 = P.key_off[i + 1], v0 = P.val_off[i], v1 = P.val_off[i + 1];
        uint32_t flags = 0;
        if (k0 > k1 || k1 > kend || v0 > v1 || v1 > vend) flags = kSortBadOffsets;
        else if (k1 - k0 > kMaxUkeyLen) flags = kSortLongKey;
        if (flags) atomicOr(&P.sum->flags, flags);
        P.perm[i] = i;
        P.pos[0][i] = i;
        P.grp[0][i] = 0;
    }
}

// record r's key in round w: lo = window w of its user key (or ~trailer once the key has ended), c = its byte count
PGS_DEV void sort_window(const SortParams &P, uint32_t r, uint32_t w, unsigned long long &lo, uint32_t &c)
{
    const unsigned long long k0 = P.key_off[r], ulen = P.key_off[r + 1] - k0, at = 8ull * w;
    if (ulen < at) {
        lo = ~((P.seq[r] << 8) | P.type[r]); // the trailer of build_trailer
        c = kSortTrailer;
        return;
    }
    c = ulen - at < 8 ? (uint32_t)(ulen - at) : 8u;
    const uint8_t *p = P.keys + k0 + at;
    unsigned long long x = 0;
    for (uint32_t j = 0; j < 8; j++) x = (x << 8) | (j < c ? p[j] : 0u);
    lo = x;
}
PGS_DEV void sort_key(const SortParams &P, uint32_t cur, uint32_t w, uint32_t k, unsigned long long &lo, unsigned long long &hi, uint32_t &r)
{
    uint32_t c;
    r = P.perm[P.pos[cur][k]];
    sort_window(P, r, w, lo, c);
    hi = ((unsigned long long)P.grp[cur][k] << 4) | c;
}

// m (the tied records) is read from the summary: the grid covers the previous round's count.  Groups are contiguous, so a group
// splits in this round iff some record's key differs from its predecessor's in the same group.
__global__ void __launch_bounds__(kSortThreads) k_sort_keys(const SortParams P, uint32_t cur, uint32_t w)
{
    const uint32_t m = P.sum->m, lane = threadIdx.x & 31;
    unsigned long long lo0 = 0, hi0 = 0, dlo = 0, dhi = 0;
    uint32_t r, split = 0, trailer = 0;
    if (m) sort_key(P, cur, w, 0, lo0, hi0, r);
    SortRound &R = P.sum->round[w & 1];
    if (blockIdx.x == 0 && threadIdx.x == 0) P.sum->round[(w + 1) & 1] = SortRound{}; // the next round's slot
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        unsigned long long lo, hi, lp, hp;
        sort_key(P, cur, w, k, lo, hi, r);
        P.lo[0][k] = lo;
        P.hi[0][k] = hi;
        P.rec[0][k] = r;
        dlo |= lo ^ lo0;
        dhi |= hi ^ hi0;
        trailer |= (hi & 15u) == kSortTrailer;
        if (k > 0) {
            uint32_t rp;
            sort_key(P, cur, w, k - 1, lp, hp, rp);
            split |= (hp >> 4) == (hi >> 4) && (lp != lo || hp != hi);
        }
    }
    const uint32_t a = __reduce_or_sync(kFull, (uint32_t)dlo), b = __reduce_or_sync(kFull, (uint32_t)(dlo >> 32));
    const uint32_t c = __reduce_or_sync(kFull, (uint32_t)dhi), d = __reduce_or_sync(kFull, (uint32_t)(dhi >> 32));
    const uint32_t f = __reduce_or_sync(kFull, split | trailer << 1);
    if (lane == 0 && (a | b | c | d)) {
        atomicOr(&R.vary[0], ((unsigned long long)b << 32) | a);
        atomicOr(&R.vary[1], ((unsigned long long)d << 32) | c);
    }
    if (lane == 0 && (f & 1)) atomicOr(&R.split, 1u);
    if (lane == 0 && (f & 2)) atomicOr(&R.trailer, 1u);
}

// digit d of a round key (hi = group << 4 | count, lo = window), least significant first: the count, the window's 8 bytes, the
// group's 4 bytes
PGS_HD uint32_t sort_digit_of(unsigned long long lo, unsigned long long hi, uint32_t d)
{
    if (d == 0) return (uint32_t)hi & 15u;
    if (d <= 8) return (uint32_t)(lo >> (8 * (d - 1))) & 255u;
    return (uint32_t)(hi >> (4 + 8 * (d - 9))) & 255u;
}
PGS_DEV uint32_t sort_digit(const SortParams &P, uint32_t b, uint32_t k, uint32_t d)
{
    return d >= 1 && d <= 8 ? sort_digit_of(P.lo[b][k], 0, d) : sort_digit_of(0, P.hi[b][k], d);
}

// the histogram of digit d over each tile of buffer b: hist[digit * gridDim.x + tile]
__global__ void __launch_bounds__(kSortThreads) k_sort_hist(const SortParams P, uint32_t b, uint32_t d, uint32_t m)
{
    PGS_SMEM_STATIC(uint32_t s_h[256]);
    const uint32_t base = blockIdx.x * kSortTile, end = min(base + kSortTile, m);
    for (uint32_t x = threadIdx.x; x < 256; x += blockDim.x) s_h[x] = 0;
    __syncthreads();
    for (uint32_t k = base + threadIdx.x; k < end; k += blockDim.x) atomicAdd(&s_h[sort_digit(P, b, k, d)], 1u);
    __syncthreads();
    for (uint32_t x = threadIdx.x; x < 256; x += blockDim.x) P.hist[x * gridDim.x + blockIdx.x] = s_h[x];
}

// one CTA: the 256 * tiles histogram entries become their exclusive prefixes (digit-major: every tile's offset for a digit)
__global__ void __launch_bounds__(kSortScanThreads) k_sort_hist_scan(const SortParams P, uint32_t tiles)
{
    uint32_t q0, q1;
    unsigned long long pre[1], tot[1];
    cta_excl_scan<1>(256 * tiles, [&](uint32_t q, unsigned long long(&v)[1]) { v[0] += P.hist[q]; }, q0, q1, pre, tot);
    __syncthreads(); // every thread has read the counts before any is overwritten
    for (uint32_t q = q0; q < q1; q++) {
        const uint32_t v = P.hist[q];
        P.hist[q] = (uint32_t)pre[0];
        pre[0] += v;
    }
}

// one stable pass: buffer b sorted by digit d into buffer b ^ 1.  Warp w of a tile ranks the tile's records
// [w * 32 * kSortItems, (w + 1) * 32 * kSortItems) 32 at a time, in order, so ranks follow the input order.
__global__ void __launch_bounds__(kSortThreads) k_sort_scatter(const SortParams P, uint32_t b, uint32_t d, uint32_t m)
{
    PGS_SMEM_STATIC(uint32_t s_cnt[kSortWarps][256]);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    const uint32_t base = blockIdx.x * kSortTile + warp * 32 * kSortItems;
    for (uint32_t x = lane; x < 256; x += 32) s_cnt[warp][x] = 0;
    __syncwarp();
    uint32_t slot[kSortItems]; // rank inside the warp << 8 | digit
#pragma unroll
    for (uint32_t c = 0; c < kSortItems; c++) {
        const uint32_t k = base + c * 32 + lane;
        const uint32_t dig = k < m ? sort_digit(P, b, k, d) : 0xFFFFFFFFu;
        const uint32_t peers = __match_any_sync(kFull, dig);
        const uint32_t rank = k < m ? s_cnt[warp][dig] + __popc(peers & lt) : 0u;
        __syncwarp();
        if (k < m && (peers & lt) == 0) s_cnt[warp][dig] += __popc(peers);
        __syncwarp();
        slot[c] = rank << 8 | (dig & 255u);
    }
    __syncthreads();
    // per digit: the tile's global offset, then the warps in order
    for (uint32_t x = threadIdx.x; x < 256; x += blockDim.x) {
        uint32_t run = P.hist[x * gridDim.x + blockIdx.x];
        for (uint32_t v = 0; v < kSortWarps; v++) {
            const uint32_t t = s_cnt[v][x];
            s_cnt[v][x] = run;
            run += t;
        }
    }
    __syncthreads();
    const uint32_t o = b ^ 1;
#pragma unroll
    for (uint32_t c = 0; c < kSortItems; c++) {
        const uint32_t k = base + c * 32 + lane;
        if (k >= m) continue;
        const uint32_t at = s_cnt[warp][slot[c] & 255u] + (slot[c] >> 8);
        P.lo[o][at] = P.lo[b][k];
        P.hi[o][at] = P.hi[b][k];
        P.rec[o][at] = P.rec[b][k];
    }
}

// ---- two-field exclusive scans over items: S gives count, add(i, v), place(i, pre) and total(tot) -------------------------------
template <class S>
__global__ void __launch_bounds__(kSortThreads) k_sort_tile_sums(const S s)
{
    const uint32_t base = blockIdx.x * kSortTile, m = min(kSortTile, s.count - base);
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    cta_excl_scan<2>(m, [&](uint32_t q, unsigned long long(&v)[2]) { s.add(base + q, v); }, q0, q1, pre, tot);
    if (threadIdx.x == 0) { s.P.tile_sum[2 * blockIdx.x] = tot[0]; s.P.tile_sum[2 * blockIdx.x + 1] = tot[1]; }
}
template <class S>
__global__ void __launch_bounds__(kSortScanThreads) k_sort_tile_scan(const S s, uint32_t tiles)
{
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    const unsigned long long *ts = s.P.tile_sum;
    auto add = [&](uint32_t t, unsigned long long(&v)[2]) { v[0] += ts[2 * t]; v[1] += ts[2 * t + 1]; };
    cta_excl_scan<2>(tiles, add, q0, q1, pre, tot);
    __syncthreads(); // every thread has read the sums before any is overwritten
    for (uint32_t t = q0; t < q1; t++) {
        unsigned long long v[2] = {0, 0};
        add(t, v);
        s.P.tile_sum[2 * t] = pre[0];
        s.P.tile_sum[2 * t + 1] = pre[1];
        pre[0] += v[0];
        pre[1] += v[1];
    }
    if (threadIdx.x == 0) s.total(tot);
}
template <class S>
__global__ void __launch_bounds__(kSortThreads) k_sort_place(const S s)
{
    const uint32_t base = blockIdx.x * kSortTile, m = min(kSortTile, s.count - base);
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    cta_excl_scan<2>(m, [&](uint32_t q, unsigned long long(&v)[2]) { s.add(base + q, v); }, q0, q1, pre, tot);
    pre[0] += s.P.tile_sum[2 * blockIdx.x];
    pre[1] += s.P.tile_sum[2 * blockIdx.x + 1];
    for (uint32_t q = q0; q < q1; q++) {
        s.place(base + q, pre);
        s.add(base + q, pre);
    }
}

// After a round's passes (keys in buffer b): slot k of the tied records takes record rec[b][k]; a record alone in its group is
// final, the others stay tied: (kept, kept group heads) are scanned into their compacted slot and group ordinal.
struct SortSettle {
    SortParams P;
    uint32_t count, b, cur;
    PGS_DEV bool differs(uint32_t k) const { return P.lo[b][k] != P.lo[b][k - 1] || P.hi[b][k] != P.hi[b][k - 1]; }
    PGS_DEV void flags(uint32_t k, bool &head, bool &keep) const
    {
        head = k == 0 || differs(k);
        keep = !(head && (k + 1 == count || differs(k + 1)));
    }
    PGS_DEV void add(uint32_t k, unsigned long long (&v)[2]) const
    {
        bool head, keep;
        flags(k, head, keep);
        v[0] += keep;
        v[1] += keep && head;
    }
    PGS_DEV void place(uint32_t k, const unsigned long long (&pre)[2]) const
    {
        bool head, keep;
        flags(k, head, keep);
        const uint32_t p = P.pos[cur][k];
        P.perm[p] = P.rec[b][k];
        if (!keep) return;
        if ((P.hi[b][k] & 15u) == kSortTrailer) atomicOr(&P.sum->flags, kSortDuplicate);
        P.pos[cur ^ 1][pre[0]] = p;
        P.grp[cur ^ 1][pre[0]] = (uint32_t)(pre[1] + head - 1);
    }
    PGS_DEV void total(const unsigned long long (&tot)[2]) const { P.sum->m = (uint32_t)tot[0]; }
};

// The sorted copy: record perm[i] at i, its key and value offsets from a scan of the lengths.
struct SortGather {
    SortParams P;
    uint32_t count;
    PGS_DEV void add(uint32_t i, unsigned long long (&v)[2]) const
    {
        const uint32_t r = P.perm[i];
        v[0] += P.key_off[r + 1] - P.key_off[r];
        v[1] += P.val_off[r + 1] - P.val_off[r];
    }
    PGS_DEV void place(uint32_t i, const unsigned long long (&pre)[2]) const
    {
        const uint32_t r = P.perm[i];
        P.s_key_off[i] = pre[0];
        P.s_val_off[i] = pre[1];
        P.s_seq[i] = P.seq[r];
        P.s_type[i] = P.type[r];
    }
    PGS_DEV void total(const unsigned long long (&tot)[2]) const { P.s_key_off[P.n] = tot[0]; P.s_val_off[P.n] = tot[1]; }
};

// one warp per record: its key and value bytes to their sorted place
__global__ void __launch_bounds__(kSortThreads) k_sort_copy(const SortParams P)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = blockIdx.x * kSortWarps + (threadIdx.x >> 5); i < P.n; i += gridDim.x * kSortWarps) {
        const uint32_t r = P.perm[i];
        warp_copy_bytes(P.s_keys + P.s_key_off[i], P.keys + P.key_off[r], (uint32_t)(P.key_off[r + 1] - P.key_off[r]), lane);
        warp_copy_bytes(P.s_vals + P.s_val_off[i], P.vals + P.val_off[r], (uint32_t)(P.val_off[r + 1] - P.val_off[r]), lane);
    }
}

// ---- plan, buffers, launches: shared by pgs_run_build_unsorted (engine.cu) and the simulator (tools/simt/sim_compact.cpp) ---------
inline void sort_plan(SortParams &P, uint32_t n)
{
    P.n = n;
    P.tiles = (n + kSortTile - 1) / kSortTile;
}
// Sort scratch through alloc(p, count, fill), the sorted copy through alloc_out (it outlives the scratch: the build reads it), with
// fill = a byte value or kNoFill.  kb, vb: key_off[n], val_off[n].
// Scratch: 60 bytes per record (perm 4, positions and groups 2 x 8, round keys 2 x 16, records 2 x 4) plus 1.03 KB of
// histograms and tile sums per 4096 records.  Sorted copy: 25 bytes per record (offsets 2 x 8, seq 8, type 1) plus kb + vb + 32.
template <class Alloc, class AllocOut>
void sort_buffers(SortParams &P, uint64_t kb, uint64_t vb, Alloc &&alloc, AllocOut &&alloc_out)
{
    const uint64_t n = P.n;
    alloc(P.perm, n, kNoFill);
    for (int x = 0; x < 2; x++) {
        alloc(P.pos[x], n, kNoFill);
        alloc(P.grp[x], n, kNoFill);
        alloc(P.lo[x], n, kNoFill);
        alloc(P.hi[x], n, kNoFill);
        alloc(P.rec[x], n, kNoFill);
    }
    alloc(P.hist, 256ull * P.tiles, kNoFill);
    alloc(P.tile_sum, 2ull * P.tiles, kNoFill);
    alloc(P.sum, 1, 0);
    alloc_out(P.s_keys, kb + 16, kNoFill);
    alloc_out(P.s_vals, vb + 16, kNoFill);
    alloc_out(P.s_key_off, n + 1, kNoFill);
    alloc_out(P.s_val_off, n + 1, kNoFill);
    alloc_out(P.s_seq, n, kNoFill);
    alloc_out(P.s_type, n, kNoFill);
}
// the status of a summary's flags, in the documented precedence
inline int32_t sort_status(uint32_t flags)
{
    if (flags & kSortBadOffsets) return PGS_INVALID_ARGUMENT;
    if (flags & kSortLongKey) return PGS_NOT_SUPPORTED;
    if (flags & kSortDuplicate) return PGS_INVALID_ARGUMENT;
    return PGS_OK;
}
// n past kBuildMaxRecords: the offsets are checked on the host (the device passes index records in 32 bits)
inline int32_t sort_status_too_many(uint64_t n, const uint64_t *key_off, const uint64_t *val_off)
{
    for (uint64_t i = 0; i < n; i++)
        if (key_off[i] > key_off[i + 1] || val_off[i] > val_off[i + 1]) return PGS_INVALID_ARGUMENT;
    return PGS_NOT_SUPPORTED;
}
// threads of the one CTA that scans `items`: about 8 items per thread, a whole number of warps, at most kSortScanThreads
inline uint32_t sort_scan_threads(uint64_t items)
{
    const uint64_t t = (items + 8 * 32 - 1) / (8 * 32) * 32;
    return t > kSortScanThreads ? kSortScanThreads : (uint32_t)t;
}
// The whole sort, then the sorted copy.  read(SortSummary &) copies the summary to the host after the work queued so far
// (returns a status); it is called once after the check and once per round.  Returns sort_status, read's error, or kOK.
template <class Read>
int32_t sort_launch(const SortParams &P, uint32_t grid_cap, cudaStream_t st, Read &&read, uint32_t &launches)
{
    auto grid = [&](uint32_t items, uint32_t per_cta) {
        const uint32_t g = (uint32_t)(((uint64_t)items + per_cta - 1) / per_cta);
        return grid_cap && g > grid_cap ? grid_cap : (g ? g : 1u);
    };
    SortSummary s;
    PGS_LAUNCH(k_sort_check, grid(P.n, kSortThreads), kSortThreads, 0, st, P);
    launches++;
    if (const int32_t rc = read(s)) return rc;
    if (const int32_t rc = sort_status(s.flags)) return rc;
    uint32_t cur = 0, m = P.n;
    for (uint32_t w = 0;; w++) {
        if (w > kSortMaxRounds) return PGS_CORRUPTION; // a key over kMaxUkeyLen bytes was refused: unreachable
        PGS_LAUNCH(k_sort_keys, grid(m, kSortThreads), kSortThreads, 0, st, P, cur, w);
        launches++;
        if (const int32_t rc = read(s)) return rc;
        if (const int32_t rc = sort_status(s.flags)) return rc;
        m = s.m;
        if (m < 2) break; // (one record is tied only in round 0, when n is 1)
        const SortRound &R = s.round[w & 1];
        if (!R.split) { // nothing moves; a group that orders versions here holds equal trailers
            if (R.trailer) return sort_status(kSortDuplicate);
            continue;
        }
        const unsigned long long vlo = R.vary[0], vhi = R.vary[1];
        const uint32_t tiles = (m + kSortTile - 1) / kSortTile;
        uint32_t b = 0;
        for (uint32_t d = 0; d < kSortDigits; d++) {
            if (!sort_digit_of(vlo, vhi, d)) continue; // the same digit everywhere: the pass would not move a record
            PGS_LAUNCH(k_sort_hist, tiles, kSortThreads, 0, st, P, b, d, m);
            PGS_LAUNCH(k_sort_hist_scan, 1, sort_scan_threads(256ull * tiles), 0, st, P, tiles);
            PGS_LAUNCH(k_sort_scatter, tiles, kSortThreads, 0, st, P, b, d, m);
            launches += 3;
            b ^= 1;
        }
        const SortSettle settle{P, m, b, cur};
        PGS_LAUNCH(k_sort_tile_sums<SortSettle>, tiles, kSortThreads, 0, st, settle);
        PGS_LAUNCH(k_sort_tile_scan<SortSettle>, 1, sort_scan_threads(tiles), 0, st, settle, tiles);
        PGS_LAUNCH(k_sort_place<SortSettle>, tiles, kSortThreads, 0, st, settle);
        launches += 3;
        cur ^= 1;
    }
    const SortGather gather{P, P.n};
    PGS_LAUNCH(k_sort_tile_sums<SortGather>, P.tiles, kSortThreads, 0, st, gather);
    PGS_LAUNCH(k_sort_tile_scan<SortGather>, 1, sort_scan_threads(P.tiles), 0, st, gather, P.tiles);
    PGS_LAUNCH(k_sort_place<SortGather>, P.tiles, kSortThreads, 0, st, gather);
    PGS_LAUNCH(k_sort_copy, grid(P.n, kSortWarps), kSortThreads, 0, st, P);
    launches += 4;
    return PGS_OK;
}

} // namespace pgs
