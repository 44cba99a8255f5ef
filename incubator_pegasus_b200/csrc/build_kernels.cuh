// build_kernels.cuh — a sorted run built on the GPU from flat records (host side: pgs_run_build in engine.cu).  The blocks are
// byte for byte those of the host RunBuilder (host_util.cpp) at the same block size and restart interval: its
// FlushBlockBySizePolicy cut with the 90 % rule, shared prefixes over the internal key (trailer included), shared = 0 at every
// restart point, the restart array and count, 16-byte block alignment with zero padding.
//
// What makes it parallel: a block's extent and bytes depend only on its first record (fill, restart countdown and shared
// prefixes all restart with a block).
//   k_build_records   one thread per record: offsets in range, order against the previous record (user key ascending, then
//                     seq << 8 | type strictly descending), user key <= kMaxUkeyLen, lcp[i] = the common prefix of the internal
//                     keys i - 1 and i
//   k_build_next      one thread per record i: the builder run from a block that starts at i gives next[i] (the first record of
//                     the following block) and the block's byte size.  Reads lengths and lcp only; the work is the records of a block.
//   k_build_lift      binary lifting over next: level r holds next applied 2^r times (R levels, 2^R >= n)
//   k_build_mark      the block starts 0, next[0], next[next[0]], ... are marked from the top level down: after level r every start
//                     whose block index is below 2^(R - r) is marked.  Marks race only towards nodes of the same chain.
//   k_build_tile_sums, k_build_tile_scan, k_build_place
//                     exclusive scan of (start, padded size) over the records: block index, blk_off and blk_size of every start,
//                     the run's block count, bytes and largest block
//   (host)            reads the BuildSummary, allocates the run
//   k_build_blocks    one warp per block writes the entry heads, the non-shared key bytes and the values (warp-wide copies), the
//                     restart array, the count and the padding
// The upload's two k_index_walk passes then build the index and the Bloom filter over the blocks where they are.
#pragma once
#include "../../include/pegasus_b200.h"
#include "device_util.cuh"

namespace pgs {

constexpr uint32_t kBuildThreads = 256;
constexpr uint32_t kBuildTile = kBuildThreads * 16;    // records per CTA of the scan
constexpr uint32_t kBuildScanThreads = 1024;          // the one CTA that scans the tiles
constexpr uint32_t kBuildWarps = 8;                   // warps (= blocks in flight) per CTA of k_build_blocks
constexpr uint64_t kBuildMaxRecords = 0xFFFFFFF0ull;  // index_buffers' limit on the records of a run
constexpr uint32_t kBuildBlockTooLarge = 0xFFFFFFFFu; // k_build_next: a block past 32 bits

// BuildSummary::flags
constexpr uint32_t kBuildBadOffsets = 1; // key_off / val_off not ascending inside [0, off[n]]: kInvalidArgument
constexpr uint32_t kBuildBadOrder = 2;   // RunBuilder::add's order rule: kInvalidArgument
constexpr uint32_t kBuildLongKey = 4;    // a user key over kMaxUkeyLen (the upload's pass 1 answers the same): kNotSupported
constexpr uint32_t kBuildHugeBlock = 8;  // a block of 4 GB or more: kNotSupported

struct BuildSummary {
    unsigned long long n_blocks, data_bytes; // data_bytes: the 16-aligned end of the last block
    uint32_t max_blk, flags;
};

struct BuildParams {
    // input (device copies of the caller's flat arrays)
    const uint8_t *keys, *vals, *type;
    const unsigned long long *key_off, *val_off, *seq;
    uint32_t n, block_size, restart_interval;
    uint32_t levels; // R: 2^R >= n
    uint32_t tiles;
    // scratch
    uint32_t *lcp;        // [n]
    uint32_t *jump;       // [R * (n + 1)]: level r at r * (n + 1); level 0 = next, next[n] = n
    uint32_t *bsize;      // [n]: the size of the block that starts at i (kBuildBlockTooLarge past 32 bits)
    uint8_t *mark;        // [n + 1]
    unsigned long long *tile_sum; // [2 * tiles]: starts, padded bytes
    uint32_t *first;      // [n + 1]: block b starts at record first[b]; first[n_blocks] = n
    unsigned long long *blk_off; // [n + 1]: blk_off[n_blocks] = data_bytes
    uint32_t *blk_size;   // [n]
    BuildSummary *sum;    // zeroed by the host
    // output (after the summary): the run's block bytes
    uint8_t *data;
};

// byte p of record i's internal key: user key || fixed64_le(seq << 8 | type)
PGS_DEV uint32_t ikey_byte(const uint8_t *uk, uint64_t ulen, unsigned long long tr, uint64_t p)
{
    return p < ulen ? uk[p] : (uint32_t)(tr >> (8 * (p - ulen))) & 0xFFu;
}
PGS_DEV unsigned long long build_trailer(const BuildParams &P, uint32_t i) { return (P.seq[i] << 8) | P.type[i]; }

__global__ void __launch_bounds__(kBuildThreads) k_build_records(const BuildParams P)
{
    const uint32_t n = P.n;
    const unsigned long long kend = P.key_off[n], vend = P.val_off[n];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        P.mark[i] = i == 0;
        if (i == 0) P.mark[n] = 0;
        const unsigned long long k0 = P.key_off[i], k1 = P.key_off[i + 1], v0 = P.val_off[i], v1 = P.val_off[i + 1];
        const unsigned long long kp = i ? P.key_off[i - 1] : k0;
        uint32_t flags = 0, l = 0;
        // every key this thread reads must lie inside the copied bytes, whatever the other threads find
        if (k0 > k1 || k1 > kend || v0 > v1 || v1 > vend || kp > k0) flags = kBuildBadOffsets;
        else {
            const uint64_t ulen = k1 - k0;
            if (ulen > kMaxUkeyLen) flags |= kBuildLongKey;
            if (i > 0) {
                const uint8_t *a = P.keys + kp, *b = P.keys + k0;
                const uint64_t plen = k0 - kp, m = plen < ulen ? plen : ulen;
                uint64_t p = 0;
                while (p < m && a[p] == b[p]) p++;
                const unsigned long long tp = build_trailer(P, i - 1), tr = build_trailer(P, i);
                const int c = p < m ? (a[p] < b[p] ? -1 : 1) : plen < ulen ? -1 : plen > ulen ? 1 : 0;
                if (c > 0 || (c == 0 && tp <= tr)) flags |= kBuildBadOrder;
                if (p == m) { // one user key is a prefix of the other: the internal keys may share trailer bytes too
                    const uint64_t mi = (plen < ulen ? plen : ulen) + 8;
                    while (p < mi && ikey_byte(a, plen, tp, p) == ikey_byte(b, ulen, tr, p)) p++;
                }
                l = p < 0xFFFFFFFFull ? (uint32_t)p : 0xFFFFFFFFu; // (a key that long is refused)
            }
        }
        P.lcp[i] = l;
        if (flags) atomicOr(&P.sum->flags, flags);
    }
}

__global__ void __launch_bounds__(kBuildThreads) k_build_next(const BuildParams P)
{
    const uint32_t n = P.n, ri = P.restart_interval;
    const uint64_t bs = P.block_size, limit = (bs * 90 + 99) / 100;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (i == 0) P.jump[n] = n;
        uint64_t buf = 0, nrst = 1;
        uint32_t j = i;
        for (; j < n; j++) { // RunBuilder::add from a block that starts at i
            const uint32_t pos = j - i;
            const uint64_t klen = P.key_off[j + 1] - P.key_off[j] + 8, vlen = P.val_off[j + 1] - P.val_off[j];
            const bool restart = pos % ri == 0;
            if (pos) { // FlushBlockBySizePolicy::Update
                const uint64_t cur = buf + 4 * nrst + 4;
                bool flush = cur >= bs;
                if (!flush) {
                    const uint64_t after = cur + klen + vlen + (restart ? 4 : 0) + 4 + varint_len((uint32_t)klen) + varint_len((uint32_t)vlen);
                    flush = after > bs && cur > limit;
                }
                if (flush) break;
                nrst += restart;
            }
            const uint32_t shared = restart ? 0u : P.lcp[j];
            buf += varint_len(shared) + varint_len((uint32_t)(klen - shared)) + varint_len((uint32_t)vlen) + klen - shared + vlen;
        }
        const uint64_t size = buf + 4 * nrst + 4;
        P.jump[i] = j;
        P.bsize[i] = size < kBuildBlockTooLarge ? (uint32_t)size : kBuildBlockTooLarge;
    }
}

__global__ void __launch_bounds__(kBuildThreads) k_build_lift(const uint32_t *__restrict__ from, uint32_t *__restrict__ to, uint32_t n)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) to[i] = from[from[i]];
}

__global__ void __launch_bounds__(kBuildThreads) k_build_mark(const uint32_t *__restrict__ jump, uint8_t *mark, uint32_t n)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (mark[i]) mark[jump[i]] = 1;
}

// the (start, padded bytes) of record i, added into v
PGS_DEV void build_start_add(const BuildParams &P, uint32_t i, unsigned long long (&v)[2])
{
    if (P.mark[i]) { v[0] += 1; v[1] += block_pad(P.bsize[i]); }
}

__global__ void __launch_bounds__(kBuildThreads) k_build_tile_sums(const BuildParams P)
{
    const uint32_t base = blockIdx.x * kBuildTile, m = min(kBuildTile, P.n - base);
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    cta_excl_scan<2>(m, [&](uint32_t q, unsigned long long(&v)[2]) { build_start_add(P, base + q, v); }, q0, q1, pre, tot);
    if (threadIdx.x == 0) { P.tile_sum[2 * blockIdx.x] = tot[0]; P.tile_sum[2 * blockIdx.x + 1] = tot[1]; }
}

// one CTA: the tile sums become the tiles' exclusive prefixes, and the totals go to the summary
__global__ void __launch_bounds__(kBuildScanThreads) k_build_tile_scan(const BuildParams P)
{
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    auto add = [&](uint32_t t, unsigned long long(&v)[2]) { v[0] += P.tile_sum[2 * t]; v[1] += P.tile_sum[2 * t + 1]; };
    cta_excl_scan<2>(P.tiles, add, q0, q1, pre, tot);
    __syncthreads(); // every thread has read the sums before any is overwritten
    for (uint32_t t = q0; t < q1; t++) {
        unsigned long long v[2] = {0, 0};
        add(t, v);
        P.tile_sum[2 * t] = pre[0];
        P.tile_sum[2 * t + 1] = pre[1];
        pre[0] += v[0];
        pre[1] += v[1];
    }
    if (threadIdx.x == 0) {
        P.sum->n_blocks = tot[0];
        P.sum->data_bytes = tot[1];
        P.first[tot[0]] = P.n;
        P.blk_off[tot[0]] = tot[1];
    }
}

__global__ void __launch_bounds__(kBuildThreads) k_build_place(const BuildParams P)
{
    const uint32_t base = blockIdx.x * kBuildTile, m = min(kBuildTile, P.n - base);
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    cta_excl_scan<2>(m, [&](uint32_t q, unsigned long long(&v)[2]) { build_start_add(P, base + q, v); }, q0, q1, pre, tot);
    pre[0] += P.tile_sum[2 * blockIdx.x];
    pre[1] += P.tile_sum[2 * blockIdx.x + 1];
    uint32_t max_blk = 0, flags = 0;
    for (uint32_t q = q0; q < q1; q++) {
        const uint32_t i = base + q;
        if (!P.mark[i]) continue;
        const uint32_t size = P.bsize[i];
        P.first[pre[0]] = i;
        P.blk_off[pre[0]] = pre[1];
        P.blk_size[pre[0]] = size;
        if (size == kBuildBlockTooLarge) flags = kBuildHugeBlock;
        max_blk = max(max_blk, size);
        pre[0] += 1;
        pre[1] += block_pad(size);
    }
    if (max_blk) atomicMax(&P.sum->max_blk, max_blk);
    if (flags) atomicOr(&P.sum->flags, flags);
}

// one warp per block: 32 entries at a time, each lane sizes one entry head; a warp scan places them, then the warp copies
// each entry's key suffix and value in turn
__global__ void __launch_bounds__(kBuildWarps * 32) k_build_blocks(const BuildParams P, uint32_t nb)
{
    const uint32_t lane = threadIdx.x & 31, ri = P.restart_interval;
    for (uint32_t b = blockIdx.x * kBuildWarps + (threadIdx.x >> 5); b < nb; b += gridDim.x * kBuildWarps) {
        const uint32_t s = P.first[b], e = P.first[b + 1], size = P.blk_size[b];
        uint8_t *base = P.data + P.blk_off[b];
        const uint32_t nrst = (e - s + ri - 1) / ri, rst_at = size - 4 * nrst - 4;
        uint32_t carry = 0;
        for (uint32_t c = s; c < e; c += 32) {
            const uint32_t j = c + lane, pos = j - s;
            const bool valid = j < e, restart = pos % ri == 0;
            uint32_t klen = 0, vlen = 0, shared = 0, head = 0;
            if (valid) {
                klen = (uint32_t)(P.key_off[j + 1] - P.key_off[j]) + 8;
                vlen = (uint32_t)(P.val_off[j + 1] - P.val_off[j]);
                shared = restart ? 0u : P.lcp[j];
                head = varint_len(shared) + varint_len(klen - shared) + varint_len(vlen);
            }
            const uint32_t esz = valid ? head + klen - shared + vlen : 0u;
            const uint32_t incl = warp_incl_scan(esz, lane), off = carry + incl - esz;
            if (valid) {
                uint32_t h = put_varint32_s(base + off, shared);
                h += put_varint32_s(base + off + h, klen - shared);
                put_varint32_s(base + off + h, vlen);
                if (restart) {
                    uint8_t *r = base + rst_at + 4 * (pos / ri);
                    r[0] = (uint8_t)off; r[1] = (uint8_t)(off >> 8); r[2] = (uint8_t)(off >> 16); r[3] = (uint8_t)(off >> 24);
                }
            }
            const uint32_t cnt = min(32u, e - c);
            for (uint32_t t = 0; t < cnt; t++) {
                const uint32_t jt = c + t;
                const uint32_t at = __shfl_sync(kFull, off + head, t), sh = __shfl_sync(kFull, shared, t);
                const uint32_t kl = __shfl_sync(kFull, klen, t), vl = __shfl_sync(kFull, vlen, t);
                const uint8_t *uk = P.keys + P.key_off[jt];
                const unsigned long long tr = build_trailer(P, jt);
                uint8_t *dst = base + at - sh;
                for (uint32_t p = sh + lane; p < kl; p += 32) dst[p] = (uint8_t)ikey_byte(uk, kl - 8, tr, p);
                warp_copy_bytes(base + at + kl - sh, P.vals + P.val_off[jt], vl, lane);
            }
            carry += __shfl_sync(kFull, incl, 31);
        }
        if (lane == 0) { uint8_t *r = base + size - 4; r[0] = (uint8_t)nrst; r[1] = (uint8_t)(nrst >> 8); r[2] = (uint8_t)(nrst >> 16); r[3] = (uint8_t)(nrst >> 24); }
        for (uint32_t p = size + lane; p < block_pad(size); p += 32) base[p] = 0;
    }
}

// ---- plan, buffers, launches: shared by pgs_run_build (engine.cu) and the simulator (tools/simt/sim_compact.cpp) ----------------
// The plan of n records: the lifting levels and the scan tiles.
inline void build_plan(BuildParams &P, uint32_t n, uint32_t block_size, uint32_t restart_interval)
{
    P.n = n;
    P.block_size = block_size;
    P.restart_interval = restart_interval;
    P.levels = 1;
    while ((1ull << P.levels) < n) P.levels++;
    P.tiles = (n + kBuildTile - 1) / kBuildTile;
}
// The caller's n flat records as the inputs of P (BuildParams or SortParams), through buf(pointer, bytes, init) as get_buffers
// uses it.  The keys and the values keep 16 bytes of slack behind them.
template <class Params, class F>
void stage_records(Params &P, uint64_t n, const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals, const uint64_t *val_off,
                   const uint64_t *seq, const uint8_t *type, F &&buf)
{
    buf(P.keys, key_off[n] + 16, ReadInit{keys, key_off[n]});
    buf(P.vals, val_off[n] + 16, ReadInit{vals, val_off[n]});
    buf(P.key_off, 8 * (n + 1), ReadInit{key_off, 8 * (n + 1)});
    buf(P.val_off, 8 * (n + 1), ReadInit{val_off, 8 * (n + 1)});
    buf(P.seq, 8 * n, ReadInit{seq, 8 * n});
    buf(P.type, n, ReadInit{type, n});
}
// The scratch of the first phase: alloc(p, count, fill) with fill = a byte value or kNoFill.  4·R + 25 bytes per record
// (R = ceil(log2 n) levels of next), plus the tiles.
template <class Alloc>
void build_buffers(BuildParams &P, Alloc &&alloc)
{
    const uint64_t n = P.n;
    alloc(P.lcp, n, kNoFill);
    alloc(P.jump, (uint64_t)P.levels * (n + 1), kNoFill);
    alloc(P.bsize, n, kNoFill);
    alloc(P.mark, n + 1, kNoFill);
    alloc(P.tile_sum, 2ull * P.tiles, kNoFill);
    alloc(P.first, n + 1, kNoFill);
    alloc(P.blk_off, n + 1, kNoFill);
    alloc(P.blk_size, n, kNoFill);
    alloc(P.sum, 1, 0);
}
// grid of the per-record kernels: at most grid_cap CTAs (0: one thread per record)
inline uint32_t build_grid(uint32_t n, uint32_t grid_cap)
{
    const uint32_t g = (n + kBuildThreads - 1) / kBuildThreads;
    return grid_cap && g > grid_cap ? grid_cap : g;
}
// First phase, up to the summary: block starts, sizes, offsets.  phase(i) is called after the record and next passes (0), the
// chain (1) and the scan (2).  Returns the launches.
template <class Phase>
uint32_t build_launch_plan(const BuildParams &P, uint32_t grid_cap, cudaStream_t st, Phase &&phase)
{
    const uint32_t g = build_grid(P.n, grid_cap), g1 = build_grid(P.n + 1, grid_cap), n = P.n;
    uint32_t launches = 0;
    PGS_LAUNCH(k_build_records, g, kBuildThreads, 0, st, P);
    PGS_LAUNCH(k_build_next, g, kBuildThreads, 0, st, P);
    launches += 2;
    phase(0);
    const uint64_t lv = (uint64_t)n + 1;
    for (uint32_t r = 1; r < P.levels; r++, launches++)
        PGS_LAUNCH(k_build_lift, g1, kBuildThreads, 0, st, (const uint32_t *)(P.jump + (r - 1) * lv), P.jump + r * lv, n);
    for (uint32_t r = P.levels; r-- > 0; launches++) PGS_LAUNCH(k_build_mark, g, kBuildThreads, 0, st, (const uint32_t *)(P.jump + r * lv), P.mark, n);
    phase(1);
    PGS_LAUNCH(k_build_tile_sums, P.tiles, kBuildThreads, 0, st, P);
    PGS_LAUNCH(k_build_tile_scan, 1, kBuildScanThreads, 0, st, P);
    PGS_LAUNCH(k_build_place, P.tiles, kBuildThreads, 0, st, P);
    phase(2);
    return launches + 3;
}
// Second phase: P.data holds the summary's data_bytes; every block's bytes and padding are written.
inline uint32_t build_launch_blocks(const BuildParams &P, uint32_t nb, uint32_t grid_cap, cudaStream_t st)
{
    uint32_t g = (nb + kBuildWarps - 1) / kBuildWarps;
    if (grid_cap && g > grid_cap) g = grid_cap;
    if (nb) PGS_LAUNCH(k_build_blocks, g, kBuildWarps * 32, 0, st, P, nb);
    return nb ? 1 : 0;
}
// the status of a summary's flags: RunBuilder::add refuses the order first; the upload refuses a long key
inline int32_t build_status(uint32_t flags)
{
    if (flags & (kBuildBadOffsets | kBuildBadOrder)) return PGS_INVALID_ARGUMENT;
    if (flags & (kBuildLongKey | kBuildHugeBlock)) return PGS_NOT_SUPPORTED;
    return PGS_OK;
}

} // namespace pgs
