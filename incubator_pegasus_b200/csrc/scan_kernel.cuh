// scan_kernel.cuh — k_scan, the block-staging range-scan kernel: every REVERSE scan (SeekForPrev + Prev loops of on_multi_get
// reverse mode, src/server/pegasus_server_impl.cpp:689-756), and every forward request of a batch that holds a reverse one.
// One CTA per request; chunks of blocks of every run are staged with TMA, decoded, merged by rank, newest version / tombstone
// visibility applied, then the reference's loop (stop key, first-exclusive, range_read_limiter counts and sizes, TTL / sort-key
// filters) is evaluated with block-wide scans walking chunk by chunk.  Each phase of a chunk is one function below, in the
// order k_scan calls them; the barriers between phases are in k_scan.  Included by lookup.cu (nvcc, sm_90a) and by the host
// SIMT interpreter (tools/simt/sim_compact.cpp), which runs the same source on the CPU, bulk copies and mbarriers included
// (device_util.cuh's PGS_SIM stand-ins complete a copy at once).
#pragma once
#include "read_kernels.cuh"

namespace pgs {

// ------------------------------------------------------------------------------------------------
// k_scan (reverse and mixed-direction batches)
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kScanThreads = 256;
constexpr uint32_t kScanWarps = kScanThreads / 32;
constexpr uint32_t kScanMaxBlocks = 128;
constexpr uint32_t kScanRecExtra = 48;
// scan_carve's own overhead beyond the chunk weights: a 16-byte gap after the blocks and up to 8 padding record slots
__host__ __device__ inline uint32_t scan_carve_slack(uint32_t KS) { return 16 + 8 * (KS + kScanRecExtra); }

struct ScanShared {
    unsigned long long mbar;
    uint32_t error, done;
    uint32_t in_bytes, n_rec, n_blk, n_valid, n_vis;
    uint32_t lo_len, hi_len, has_lo, has_hi, lo_incl, hi_incl; // chunk validity bounds
    uint32_t cur[kMaxReadRuns], nblk[kMaxReadRuns], nrec[kMaxReadRuns], in_off[kMaxReadRuns], rec_base[kMaxReadRuns], blk_base[kMaxReadRuns];
    uint32_t vlo[kMaxReadRuns], vhi[kMaxReadRuns], more[kMaxReadRuns], want_end[kMaxReadRuns];
    uint32_t tb_off[kScanMaxBlocks], tb_size[kScanMaxBlocks], tb_rec[kScanMaxBlocks], tb_nrec[kScanMaxBlocks];
    uint32_t scan[33];
    // carried loop state
    uint32_t count, iter_count, expire_count, filter_count, n_out;
    unsigned long long size, arena_used;
    uint32_t complete, iter_valid, lookahead, resume_len;
    uint32_t P, F; // per chunk
    uint32_t cand_len[kMaxReadRuns];
    uint32_t grec0[kMaxReadRuns]; // index of the slice's first record inside its run
    unsigned long long crc[256];
};

struct ScanArrays {
    uint8_t *in, *arena;
    unsigned long long *trailer;
    uint32_t *voff, *vlen, *A1, *A2, *A3;
    uint16_t *klen, *rank, *order, *vis;
    uint8_t *flags, *state;
    uint32_t total;
};
PGS_DEV ScanArrays scan_carve(uint8_t *pool, uint32_t in_bytes, uint32_t n, uint32_t KS)
{
    ScanArrays a;
    uint32_t n8 = (n + 8) & ~7u;
    uint32_t off = ((in_bytes + 15) & ~15u) + 16;
    a.in = pool;
    a.arena = pool + off; off += n8 * KS;
    a.trailer = (unsigned long long *)(pool + off); off += n8 * 8;
    a.voff = (uint32_t *)(pool + off); off += n8 * 4;
    a.vlen = (uint32_t *)(pool + off); off += n8 * 4;
    a.A1 = (uint32_t *)(pool + off); off += n8 * 4;
    a.A2 = (uint32_t *)(pool + off); off += n8 * 4;
    a.A3 = (uint32_t *)(pool + off); off += n8 * 4;
    a.klen = (uint16_t *)(pool + off); off += n8 * 2;
    a.rank = (uint16_t *)(pool + off); off += n8 * 2;
    a.order = (uint16_t *)(pool + off); off += n8 * 2;
    a.vis = (uint16_t *)(pool + off); off += n8 * 2;
    a.flags = pool + off; off += n8;
    a.state = pool + off; off += n8;
    a.total = off;
    return a;
}

template <class F>
PGS_DEV uint32_t scan_chunked(uint32_t n, uint32_t *out, uint32_t *scratch, F f)
{
    uint32_t ipt = (n + blockDim.x - 1) / blockDim.x;
    uint32_t begin = min(threadIdx.x * ipt, n), end = min(begin + ipt, n);
    uint32_t local = 0;
    for (uint32_t i = begin; i < end; i++) local += f(i);
    uint32_t total;
    uint32_t pre = block_excl_scan(local, scratch, &total);
    for (uint32_t i = begin; i < end; i++) { uint32_t v = f(i); out[i] = pre; pre += v; }
    if (threadIdx.x == 0) out[n] = total;
    __syncthreads();
    return total;
}

enum : uint8_t { SF_VALID = 1, SF_SHADOW = 2 };

// k_scan's dynamic shared memory: key slots of KS + 8 zero-padded bytes (no stored key is longer than KS), then the staging pool.
// lo / hi = the chunk's validity bounds (lower exclusive or inclusive, upper), pre = the seek key's hash-key prefix, end = the
// range end, cand = one slot per run: its candidate for the chunk's far bound.  `slot` keeps the pool (the TMA destination)
// 16-byte aligned.
struct ScanSlots {
    uint32_t slot;
    uint8_t *lo, *hi, *pre, *end, *cand, *pool;
    PGS_DEV ScanSlots(uint8_t *dyn, uint32_t KS, uint32_t NR)
        : slot((KS + 8 + 15) & ~15u), lo(dyn), hi(dyn + slot), pre(dyn + 2 * slot), end(dyn + 3 * slot), cand(dyn + 4 * slot),
          pool(dyn + (4 + NR) * slot) {}
};

// a request in its iteration direction: where the iterator starts (seek: "start" forward, "stop" reverse), the range end and
// whether it is inclusive, pre_len (prefix_same_as_start: the iterator only lives inside the seek key's hash-key prefix) and
// the request's output slices
struct ScanDir {
    bool rev, end_incl;
    const uint8_t *seek, *end;
    uint32_t seek_len, end_len, pre_len;
    pgs_kv *kvs; uint8_t *arena;
};
PGS_DEV ScanDir scan_dir(const ScanParams &P, const ScanReqDev &Q, uint32_t rq)
{
    ScanDir R;
    const uint8_t *start = P.blob + Q.start_off, *stop = P.blob + Q.stop_off;
    R.rev = Q.reverse != 0;
    R.seek = R.rev ? stop : start; R.seek_len = R.rev ? Q.stop_len : Q.start_len;
    R.end = R.rev ? start : stop; R.end_len = R.rev ? Q.start_len : Q.stop_len; R.end_incl = R.rev ? Q.start_inclusive : Q.stop_inclusive;
    R.pre_len = 0;
    if (Q.prefix_same_as_start && !R.rev && Q.start_len >= 2) {
        const uint32_t hl = be16(start);
        if (2 + hl <= Q.start_len) R.pre_len = 2 + hl;
    }
    R.kvs = P.kvs + (size_t)rq * P.kv_stride;
    R.arena = P.arena + (size_t)rq * P.arena_stride;
    return R;
}
// the run whose slice of the chunk holds item i, given the first item of every run's slice (slices follow in run order)
PGS_DEV uint32_t run_of(const uint32_t *base, uint32_t NR, uint32_t i) { uint32_t j = 0; while (j + 1 < NR && i >= base[j + 1]) j++; return j; }
// the first (lowest) of the m blocks a run loads from its cursor c: forward c is that block, reverse the last one
PGS_DEV uint32_t first_block(bool rev, uint32_t c, uint32_t m) { return rev ? c + 1 - m : c; }
// bytes staged for blocks [lo_b, lo_b + m): up to the 16-aligned end of the last of them, so that a gap behind it (an upload
// takes any offsets) is not loaded -- a gap of 4 GiB would otherwise wrap the 32-bit size or overflow the pool
PGS_DEV uint32_t stage_bytes(const RunDev &r, uint32_t lo_b, uint32_t m)
{
    const uint32_t last = lo_b + m - 1;
    return (uint32_t)(((r.blk_off[last] + r.blk_size[last] + 15) & ~15ull) - r.blk_off[lo_b]);
}

// ---- request setup -----------------------------------------------------------------------------------------------------------
// initial cursors (one warp per run, 33-ary index search): first block whose last key >= the seek key (reverse: the last block
// when there is none).  want_end: first block whose last key >= the range end.  The two searches of a run are independent
// chains of global round trips: different warps take them.
PGS_DEV void seek_cursors(ScanShared &S, const ScanParams &P, const ScanDir &R)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, NR = P.rr.n;
    const Grp<32> wg;
    for (uint32_t task = warp; task < 2 * NR; task += kScanWarps) {
        const uint32_t j = task >> 1;
        const RunDev &r = P.rr.runs[j];
        if (task & 1) {
            const uint32_t we = grp_index_bound(wg, true, r, R.end, R.end_len, false);
            if (lane == 0) S.want_end[j] = we;
        } else {
            uint32_t b = grp_index_bound(wg, true, r, R.seek, R.seek_len, false);
            if (R.rev && b >= r.nb) b = r.nb ? r.nb - 1 : 0;
            if (lane == 0) S.cur[j] = b;
        }
    }
}
// the loop state and the crc table; the first chunk's bound in iteration direction is the seek key; the prefix and the range end
// are staged once per request
PGS_DEV void begin_request(ScanShared &S, const ScanSlots &K, const ScanParams &P, const ScanReqDev &Q, const ScanDir &R, uint32_t KS)
{
    if (threadIdx.x == 0) {
        S.count = S.iter_count = S.expire_count = S.filter_count = S.n_out = 0;
        S.size = 0; S.arena_used = 0;
        S.complete = 0; S.iter_valid = 0; S.lookahead = 0; S.resume_len = 0; S.done = 0; S.error = 0;
    }
    if (P.crc_table && Q.validate_hash)
        for (uint32_t i = threadIdx.x; i < 256; i += kScanThreads) S.crc[i] = P.crc_table[i];
    for (uint32_t i = threadIdx.x; i < KS + 8; i += kScanThreads) {
        const uint8_t v = i < R.seek_len && i < KS ? R.seek[i] : 0;
        if (R.rev) K.hi[i] = v; else K.lo[i] = v;
        K.pre[i] = i < R.pre_len ? R.seek[i] : 0;
        K.end[i] = i < R.end_len ? R.end[i] : 0;
    }
    if (threadIdx.x == 0) {
        // keys longer than KS cannot exist in the runs; a seek key longer than KS that shares its first KS bytes with a stored
        // key sorts after it: the truncated bound is inclusive (reverse) / exclusive (forward)
        const bool long_seek = R.seek_len > KS;
        const uint32_t sl = long_seek ? KS : R.seek_len;
        // a seek key beyond the range end: the reference meets a record equal to it at its range-end check, before the
        // first-exclusive skip, and completes there -- so the first chunk keeps that record even when the seek is exclusive
        const int se = cmp_bytes(P.blob + Q.start_off, Q.start_len, P.blob + Q.stop_off, Q.stop_len);
        const bool seek_past_end = se > 0 || (se == 0 && !R.end_incl);
        if (R.rev) { S.hi_len = sl; S.has_hi = 1; S.hi_incl = long_seek || Q.stop_inclusive || seek_past_end; S.has_lo = 0; S.lo_len = 0; S.lo_incl = 0; }
        else { S.lo_len = sl; S.has_lo = 1; S.lo_incl = !long_seek && (Q.start_inclusive || seek_past_end); S.has_hi = 0; S.hi_len = 0; S.hi_incl = 1; }
    }
}

// ---- chunk loop ---------------------------------------------------------------------------------------------------------------
// choose blocks (warp 0; lane j = run j, a couple of independent global loads per run): how many blocks every run stages,
// where they go in the pool and where their records start.  Sets S.done when every run is exhausted (the iterator is invalid).
PGS_DEV void choose_blocks(ScanShared &S, const ScanParams &P, bool rev, uint32_t KS, uint8_t *pool)
{
    const uint32_t j = threadIdx.x & 31, NR = P.rr.n;
    bool has = false;
    uint32_t c = 0, m = 0, bytes_j = 0, recs_j = 0, more_j = 0;
    const RunDev *rp = nullptr;
    if (j < NR) {
        rp = &P.rr.runs[j];
        c = S.cur[j];
        has = rev ? (rp->nb > 0 && c != 0xFFFFFFFFu) : (c < rp->nb);
    }
    const uint32_t active = __popc(__ballot_sync(kFull, has));
    if (has) {
        const RunDev &r = *rp;
        // per-run share of the pool, at least one block each (scan_dyn_bytes)
        const uint32_t budget = (P.pool_bytes - 64 - scan_carve_slack(KS)) / active;
        uint32_t maxm = 1;
        if (!S.lookahead) { // the wanted range end limits the first fetches
            uint32_t want_end = S.want_end[j];
            maxm = rev ? (c >= want_end ? c - want_end + 1 : 1) : (want_end >= c ? want_end - c + 1 : 1);
            if (!rev && maxm > r.nb - c) maxm = r.nb - c;
            if (rev && maxm > c + 1) maxm = c + 1;
        }
        if (maxm > kScanMaxBlocks / active) maxm = kScanMaxBlocks / active; // the block table holds kScanMaxBlocks
        auto weight = [&](uint32_t mm) -> unsigned long long {
            uint32_t l = first_block(rev, c, mm), h = l + mm;
            return (r.blk_off[h] - r.blk_off[l]) + 32 + (unsigned long long)(r.blk_rec[h] - r.blk_rec[l]) * (KS + kScanRecExtra);
        };
        // largest m in [1, maxm] whose blocks and records fit the budget (cumulative arrays).  The weights of the first eight
        // candidates come from loads issued together (one round trip); only a run that may take more than eight blocks
        // continues with a binary search.
        constexpr uint32_t kProbe = 8;
        const uint32_t np = maxm < kProbe ? maxm : kProbe;
        const uint32_t b0 = rev ? c + 1 : c;
        unsigned long long o[kProbe + 1];
        uint32_t rc[kProbe + 1];
#pragma unroll
        for (uint32_t x = 0; x <= kProbe; x++) {
            const uint32_t idx = x <= np ? (rev ? b0 - x : b0 + x) : b0;
            o[x] = r.blk_off[idx];
            rc[x] = r.blk_rec[idx];
        }
        m = 1;
#pragma unroll
        for (uint32_t x = 2; x <= kProbe; x++) {
            const unsigned long long wb = rev ? o[0] - o[x] : o[x] - o[0];
            const uint32_t wr = rev ? rc[0] - rc[x] : rc[x] - rc[0];
            if (x <= np && wb + 32 + (unsigned long long)wr * (KS + kScanRecExtra) <= budget) m = x; // weights grow with x
        }
        if (m == kProbe && maxm > kProbe) {
            if (weight(maxm) <= budget) m = maxm;
            else {
                uint32_t lo = kProbe, hi = maxm;
                while (lo + 1 < hi) { uint32_t mid = (lo + hi) >> 1; if (weight(mid) <= budget) lo = mid; else hi = mid; }
                m = lo;
            }
        }
        const uint32_t lo_b = first_block(rev, c, m);
        bytes_j = stage_bytes(r, lo_b, m);
        const uint32_t g0 = r.blk_rec[lo_b];
        recs_j = r.blk_rec[lo_b + m] - g0;
        S.grec0[j] = g0;
        more_j = rev ? (lo_b > 0) : (lo_b + m < r.nb);
    }
    const uint32_t ib = warp_incl_scan(bytes_j, j), ir = warp_incl_scan(recs_j, j), im = warp_incl_scan(m, j);
    if (j < NR) {
        S.nblk[j] = m;
        S.in_off[j] = ib - bytes_j;
        S.rec_base[j] = ir - recs_j;
        S.blk_base[j] = im - m;
        S.nrec[j] = recs_j;
        S.more[j] = more_j;
    }
    const uint32_t bytes = __shfl_sync(kFull, ib, 31), recs = __shfl_sync(kFull, ir, 31), blks = __shfl_sync(kFull, im, 31);
    if (j == 0) {
        S.in_bytes = bytes; S.n_rec = recs; S.n_blk = blks;
        ScanArrays a0 = scan_carve(pool, bytes, recs, KS);
        if (a0.total > P.pool_bytes || blks > kScanMaxBlocks || recs > 65000) S.error = PGS_NOT_SUPPORTED;
        if (!active) S.done = 1;
    }
}
// stage the chosen blocks into the pool (thread 0 issues one bulk copy per run), fill the block table and stage every run's
// candidate for the chunk's far bound: the nearest "last loaded block" key of a run that has more blocks.  Candidate keys are
// staged in shared memory (one warp per run, coalesced) before pick_far_bound compares them: a byte-wise compare straight out
// of global memory would pay one round trip per byte.  Returns once the staged blocks have landed.
PGS_DEV void stage_blocks(ScanShared &S, const ScanSlots &K, const ScanArrays &A, const ScanParams &P, bool rev, uint32_t KS, uint32_t &mbar_phase)
{
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NR = P.rr.n;
    if (tid == 0) {
        fence_proxy_async();
        mbar_expect_tx((uint64_t *)&S.mbar, S.in_bytes);
        for (uint32_t j = 0; j < NR; j++) {
            const uint32_t m = S.nblk[j];
            if (!m) continue;
            const RunDev &r = P.rr.runs[j];
            const uint32_t lo_b = first_block(rev, S.cur[j], m);
            tma_load_1d(A.in + S.in_off[j], r.data + r.blk_off[lo_b], stage_bytes(r, lo_b, m), (uint64_t *)&S.mbar);
        }
    }
    for (uint32_t t = tid; t < S.n_blk; t += kScanThreads) {
        const uint32_t j = run_of(S.blk_base, NR, t);
        const RunDev &r = P.rr.runs[j];
        const uint32_t lo_b = first_block(rev, S.cur[j], S.nblk[j]);
        const uint32_t gb = lo_b + (t - S.blk_base[j]);
        S.tb_off[t] = S.in_off[j] + (uint32_t)(r.blk_off[gb] - r.blk_off[lo_b]);
        S.tb_size[t] = r.blk_size[gb];
        S.tb_rec[t] = S.rec_base[j] + (r.blk_rec[gb] - r.blk_rec[lo_b]);
        S.tb_nrec[t] = r.blk_rec[gb + 1] - r.blk_rec[gb];
    }
    for (uint32_t j = warp; j < NR; j += kScanWarps) {
        uint32_t l = 0xFFFFFFFFu;
        if (S.nblk[j] && S.more[j]) {
            const RunDev &r = P.rr.runs[j];
            const uint32_t m = S.nblk[j], lo_b = first_block(rev, S.cur[j], m);
            // forward: last key of the last loaded block; reverse: last key of the block before the first loaded one
            const uint32_t bb = rev ? lo_b - 1 : lo_b + m - 1;
            const uint32_t o = r.ikey_off[bb];
            l = r.ikey_off[bb + 1] - o;
            for (uint32_t i = lane; i < KS + 8; i += 32) K.cand[j * K.slot + i] = i < l ? r.ikeys[o + i] : 0;
        }
        if (lane == 0) S.cand_len[j] = l;
    }
    mbar_wait((uint64_t *)&S.mbar, mbar_phase);
    mbar_phase ^= 1;
}
// thread 0: the run whose candidate is the chunk's far bound (forward the smallest, reverse the largest), -1 for none.
// S.P is free until the loop limits: it holds the answer.
PGS_DEV void pick_far_bound(ScanShared &S, const ScanSlots &K, bool rev, uint32_t NR)
{
    int best = -1;
    for (uint32_t j = 0; j < NR; j++) {
        if (S.cand_len[j] == 0xFFFFFFFFu) continue;
        if (best < 0) { best = (int)j; continue; }
        int c = cmp_bytes(K.cand + j * K.slot, S.cand_len[j], K.cand + best * K.slot, S.cand_len[best]);
        if (rev ? c > 0 : c < 0) best = (int)j;
    }
    S.P = (uint32_t)best;
}
// the far bound becomes the chunk's upper bound (forward, inclusive) or lower bound (reverse, exclusive); without one the
// chunk is open on that side
PGS_DEV void take_far_bound(ScanShared &S, const ScanSlots &K, bool rev, uint32_t KS)
{
    const int best = (int)S.P;
    uint8_t *dst = rev ? K.lo : K.hi;
    if (best >= 0) {
        const uint32_t l = S.cand_len[best];
        for (uint32_t i = threadIdx.x; i < KS + 8; i += kScanThreads) dst[i] = K.cand[best * K.slot + i];
        if (threadIdx.x == 0) { if (rev) { S.lo_len = l; S.has_lo = 1; S.lo_incl = 0; } else { S.hi_len = l; S.has_hi = 1; S.hi_incl = 1; } }
    } else if (threadIdx.x == 0) {
        if (rev) S.has_lo = 0; else S.has_hi = 0;
    }
}
// decode the entry headers: one THREAD per record parses its entry header.  The entry's offset inside its block comes from the
// run's rec_off index, so no thread walks a block's entry chain.  A malformed entry sets S.error.
PGS_DEV void decode_headers(ScanShared &S, const ScanArrays &A, const ScanParams &P, uint32_t KS)
{
    const uint32_t nblk = S.n_blk, NR = P.rr.n;
    for (uint32_t r = threadIdx.x; r < S.n_rec; r += kScanThreads) {
        const uint32_t j = run_of(S.rec_base, NR, r);
        uint32_t lo = 0, hi = nblk; // block of record r: last t with tb_rec[t] <= r
        while (lo + 1 < hi) { uint32_t mid = (lo + hi) >> 1; if (S.tb_rec[mid] <= r) lo = mid; else hi = mid; }
        const uint32_t t = lo;
        const uint8_t *base = A.in + S.tb_off[t];
        const uint32_t size = S.tb_size[t], i = r - S.tb_rec[t], cnt = S.tb_nrec[t];
        uint32_t err = 0, nr = 0;
        if (size < 8) err = PGS_CORRUPTION;
        if (!err) { nr = le32(base + size - 4); if (nr == 0 || (unsigned long long)nr * 4 + 4 > size) err = PGS_CORRUPTION; }
        const uint32_t limit = err ? 0 : size - 4 - 4 * nr;
        const uint32_t p = err ? 0 : P.rr.runs[j].rec_off[S.grec0[j] + (r - S.rec_base[j])];
        if (!err && (p >= limit || (i == 0 && p != 0))) err = PGS_CORRUPTION;
        if (!err) {
            uint32_t sh, ns, vl, h, c;
            h = c = parse_header8(lds_u64_at(A.in, S.tb_off[t] + p), sh, ns, vl); // header bytes from registers
            if (!c) { // uncommon shape: byte-wise decoder
                h = 0;
                c = get_varint32(base + p, limit - p, sh); h += c;
                if (c) { c = get_varint32(base + p + h, limit - p - h, ns); h += c; }
                if (c) { c = get_varint32(base + p + h, limit - p - h, vl); h += c; }
            }
            const uint32_t kl = sh + ns;
            const unsigned long long end = (unsigned long long)p + h + ns + vl;
            if (!c || kl < 8 || kl - 8 > KS || end > limit || (i == 0 && sh != 0) || (i + 1 == cnt && end != limit)) err = PGS_CORRUPTION;
            else {
                A.rank[r] = (uint16_t)sh;  // scratch until the rank phase
                A.order[r] = (uint16_t)ns; // scratch until the scatter phase
                A.A1[r] = S.tb_off[t] + p + h; // the key delta
                A.klen[r] = (uint16_t)(kl - 8);
                A.voff[r] = S.tb_off[t] + p + h + ns;
                A.vlen[r] = vl;
                if (ns >= 8) { A.trailer[r] = lds_u64_at(A.in, S.tb_off[t] + p + h + ns - 8); A.flags[r] = 0; }
                else { A.trailer[r] = 0; A.flags[r] = 1; } // part of the trailer is shared with the previous key: rebuild_keys
            }
        }
        if (err) atomicMax(&S.error, err);
    }
}
// rebuild the keys into the arena: HALF a warp per block, four key bytes per lane.  A shared prefix longer than the previous
// key sets S.error.
PGS_DEV void rebuild_keys(ScanShared &S, const ScanArrays &A, uint32_t KS)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t hl = lane & 15, sub = lane >> 4;
    const uint32_t hmask = sub ? 0xffff0000u : 0x0000ffffu;
    for (uint32_t t = 2 * warp + sub; t < S.n_blk; t += 2 * kScanWarps) {
        const uint32_t rec0 = S.tb_rec[t], nrec = S.tb_nrec[t];
        uint32_t maxk = 0;
        for (uint32_t i = hl; i < nrec; i += 16) maxk = max(maxk, (uint32_t)A.klen[rec0 + i] + 8);
        maxk = __reduce_max_sync(hmask, maxk);
        for (uint32_t pass = 0; pass * 64 < maxk; pass++) {
            const uint32_t p0 = pass * 64 + 4 * hl;
            uint32_t cur = 0, prev_klen = 0; // the four running bytes, little endian
            for (uint32_t i = 0; i < nrec; i++) {
                const uint32_t r = rec0 + i;
                const uint32_t sh = A.rank[r], ns = A.order[r], ulen = A.klen[r], ko = A.A1[r], fl = A.flags[r];
                if (sh > prev_klen) { if (hl == 0) atomicMax(&S.error, (uint32_t)PGS_CORRUPTION); break; }
                prev_klen = ulen + 8;
                const uint32_t a = max(sh, p0), b = min(sh + ns, p0 + 4);
                if (a < b) {
                    const uint32_t so = ko + (a - sh); // delta bytes for positions a..a+3
                    const uint32_t *w = (const uint32_t *)A.in + (so >> 2);
                    const uint32_t x = __funnelshift_r(w[0], w[1], (so & 3) * 8);
                    const uint32_t s0 = 8 * (a - p0), s1 = 8 * (p0 + 4 - b);
                    const uint32_t msk = (0xffffffffu << s0) & (0xffffffffu >> s1);
                    cur = (cur & ~msk) | ((x << s0) & msk);
                }
                const uint32_t pad = (ulen + 7) & ~7u; // slots are zero padded to 8 bytes
                if (p0 < pad) {
                    const uint32_t keep = ulen > p0 ? ulen - p0 : 0;
                    *(uint32_t *)(A.arena + (size_t)r * KS + p0) = keep >= 4 ? cur : (cur & ((1u << (8 * keep)) - 1u));
                }
                if (fl && pass * 64 < ulen + 8 && pass * 64 + 64 > ulen) { // rare: the trailer straddles the shared prefix
                    unsigned long long c = 0;
                    if (p0 >= ulen) { if (p0 < ulen + 8) c = (unsigned long long)cur << (8 * (p0 - ulen)); }
                    else if (ulen - p0 < 4) c = cur >> (8 * (ulen - p0));
                    const uint32_t lo = __reduce_or_sync(hmask, (uint32_t)c), hi = __reduce_or_sync(hmask, (uint32_t)(c >> 32));
                    if (hl == 0) A.trailer[r] |= ((unsigned long long)hi << 32) | lo;
                }
            }
        }
    }
}
// validity window per run: lo (<|<=) key (<=) hi.  Records at or below the lower bound form a prefix of a run's slice and
// records above the upper bound a suffix: counting them in parallel gives the window.  S.vlo and S.vhi start at zero;
// window_count leaves the number of records above the bound in S.vhi, window_close turns it into the window's end.
PGS_DEV void window_count(ScanShared &S, const ScanSlots &K, const ScanArrays &A, uint32_t KS, uint32_t NR)
{
    for (uint32_t r = threadIdx.x; r < S.n_rec; r += kScanThreads) {
        const uint32_t j = run_of(S.rec_base, NR, r);
        const uint8_t *key = A.arena + (size_t)r * KS;
        const uint32_t kl = A.klen[r];
        bool below = false;
        if (S.has_lo) { int c = cmp_slots(key, kl, K.lo, S.lo_len); below = S.lo_incl ? c < 0 : c <= 0; }
        if (below) atomicAdd(&S.vlo[j], 1u);
        else if (S.has_hi) { int c = cmp_slots(key, kl, K.hi, S.hi_len); if (S.hi_incl ? c > 0 : c >= 0) atomicAdd(&S.vhi[j], 1u); }
    }
}
PGS_DEV void window_close(ScanShared &S, uint32_t NR)
{
    const uint32_t j = threadIdx.x;
    if (j < NR) S.vhi[j] = max(S.nrec[j] - S.vhi[j], S.vlo[j]);
}
// merge rank + shadowing, A1 = rank, A2 = shadowed.  rank_own_run: one thread per record: validity, position inside its own
// run, predecessor of the same run.  rank_other_runs: one thread per (record, other run): LCP-aware binary search for the
// number of that run's records that sort before it; ranks accumulate with shared-memory atomics.
PGS_DEV void rank_own_run(const ScanShared &S, const ScanArrays &A, uint32_t KS, uint32_t NR)
{
    for (uint32_t r = threadIdx.x; r < S.n_rec; r += kScanThreads) {
        const uint32_t j = run_of(S.rec_base, NR, r);
        const uint32_t idx = r - S.rec_base[j];
        if (idx < S.vlo[j] || idx >= S.vhi[j]) { A.flags[r] = 0; continue; }
        const uint32_t kl = A.klen[r];
        const bool shadow = idx > 0 && A.klen[r - 1] == kl && cmp_slots(A.arena + (size_t)(r - 1) * KS, kl, A.arena + (size_t)r * KS, kl) == 0;
        A.A1[r] = idx - S.vlo[j];
        A.A2[r] = shadow ? 1u : 0u;
        A.flags[r] = SF_VALID;
    }
}
PGS_DEV void rank_other_runs(const ScanShared &S, const ScanArrays &A, uint32_t KS, uint32_t NR)
{
    const uint32_t km1 = NR - 1, ntask = S.n_rec * km1;
    for (uint32_t id = threadIdx.x; id < ntask; id += kScanThreads) {
        const uint32_t r = id / km1, oi = id - r * km1;
        if (!(A.flags[r] & SF_VALID)) continue;
        const uint32_t j = run_of(S.rec_base, NR, r);
        const uint32_t o = oi < j ? oi : oi + 1;
        if (S.vhi[o] == S.vlo[o]) continue;
        const uint8_t *key = A.arena + (size_t)r * KS;
        const uint32_t kl = A.klen[r];
        const unsigned long long tr = A.trailer[r];
        uint32_t base = S.rec_base[o], lo = S.vlo[o], hi = S.vhi[o];
        uint32_t lcp_lo = 0, lcp_hi = 0; // words shared with the keys just outside [lo, hi)
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1, q = base + mid, d;
            int c = cmp_slots_from(A.arena + (size_t)q * KS, A.klen[q], key, kl, min(lcp_lo, lcp_hi), &d);
            bool before;
            if (c != 0) before = c < 0;
            else {
                unsigned long long tq = A.trailer[q];
                before = tq > tr || (tq == tr && o < j);
            }
            if (before) { lo = mid + 1; lcp_lo = d; } else { hi = mid; lcp_hi = d; }
        }
        if (lo > S.vlo[o]) {
            atomicAdd(&A.A1[r], lo - S.vlo[o]);
            uint32_t q = base + lo - 1;
            if (A.klen[q] == kl && cmp_slots(A.arena + (size_t)q * KS, kl, key, kl) == 0) atomicOr(&A.A2[r], 1u);
        }
    }
}
// order = the valid records in merge order; shadowed ones are flagged
PGS_DEV void merge_order(const ScanShared &S, const ScanArrays &A)
{
    for (uint32_t r = threadIdx.x; r < S.n_rec; r += kScanThreads)
        if (A.flags[r] & SF_VALID) {
            A.order[A.A1[r]] = (uint16_t)r;
            if (A.A2[r]) A.flags[r] = SF_VALID | SF_SHADOW;
        }
}
// vis = the visible records (newest version of a key, not a tombstone) in iteration order; returns their number
PGS_DEV uint32_t visible_list(ScanShared &S, const ScanArrays &A, bool rev)
{
    const uint32_t nv = S.n_valid;
    auto at = [&](uint32_t p) -> uint32_t { return A.order[rev ? nv - 1 - p : p]; };
    const uint32_t nvis = scan_chunked(nv, A.A1, S.scan, [&](uint32_t p) -> uint32_t {
        uint32_t r = at(p);
        return (!(A.flags[r] & SF_SHADOW) && (uint8_t)A.trailer[r] == PGS_TYPE_VALUE) ? 1u : 0u;
    });
    for (uint32_t p = threadIdx.x; p < nv; p += kScanThreads) {
        uint32_t r = at(p);
        if (!(A.flags[r] & SF_SHADOW) && (uint8_t)A.trailer[r] == PGS_TYPE_VALUE) A.vis[A.A1[p]] = (uint16_t)r;
    }
    return nvis;
}
// per visible record: state | 0x10 in the seek prefix | 0x20 in the range; A2 <- 1 if the state is normal (count), A3 <- its
// output bytes if normal (size), rank (free once the visible list stands) <- the output key's offset in the user key (the
// output key runs to the key's end).  Records outside the seek prefix end the iterator.
PGS_DEV void record_states(const ScanShared &S, const ScanSlots &K, const ScanArrays &A, const ScanParams &P, const ScanReqDev &Q,
                           const ScanDir &R, uint32_t KS, uint32_t nvis)
{
    const uint32_t hdr = user_data_offset(P.data_version);
    for (uint32_t v = threadIdx.x; v < nvis; v += kScanThreads) {
        uint32_t r = A.vis[v];
        const uint8_t *key = A.arena + (size_t)r * KS;
        uint32_t kl = A.klen[r];
        bool in_prefix = true;
        if (R.pre_len) {
            in_prefix = kl >= R.pre_len;
            for (uint32_t i = 0; in_prefix && i < R.pre_len; i++) in_prefix = key[i] == K.pre[i];
        }
        int c = cmp_bytes(key, kl, K.end, R.end_len); // reads at most min(kl, end_len) <= KS bytes of the staged range end
        bool in_range = R.rev ? (c > 0 || (c == 0 && R.end_incl)) : (c < 0 || (c == 0 && R.end_incl));
        if (Q.has_upper && !R.rev) in_prefix = in_prefix && c < 0; // iterate_upper_bound (sortkey_count)
        const uint32_t vl = A.vlen[r];
        const ScanRecord o = scan_record(Q, P.blob, S.crc, P.now, hdr, key, kl, vl, vl >= 4 ? be32(A.in + A.voff[r]) : 0u);
        A.state[v] = o.st | (in_prefix ? 0x10 : 0) | (in_range ? 0x20 : 0);
        A.A2[v] = o.st == RS_NORMAL ? 1u : 0u;
        A.A3[v] = o.st == RS_NORMAL ? o.klen + o.vlen : 0u;
        A.rank[v] = (uint16_t)o.koff;
    }
}
// the reference loop, evaluated for all positions at once.  F: first position where the iterator is out of its prefix or
// beyond the range end.  P: first position where `count < max_count && limiter.valid()` fails.  A1 = size prefix, A2 = count
// prefix.
PGS_DEV void loop_limits(ScanShared &S, const ScanArrays &A, const ScanReqDev &Q, uint32_t nvis)
{
    for (uint32_t v = threadIdx.x; v < nvis; v += kScanThreads) {
        uint8_t s = A.state[v];
        if (!(s & 0x10) || !(s & 0x20)) atomicMin(&S.F, v);
        bool ok = !S.lookahead && (S.count + A.A2[v] < Q.max_count) && (S.iter_count + v < Q.max_iter_count) &&
                  (Q.max_iter_size == 0 || S.size + A.A1[v] < Q.max_iter_size);
        if (!ok) atomicMin(&S.P, v);
    }
}
// emit the normal records of the processed positions [0, nproc): one warp per record.  An output that does not fit the
// request's slices sets S.error = PGS_ABORTED.
PGS_DEV void emit(ScanShared &S, const ScanArrays &A, const ScanParams &P, const ScanReqDev &Q, const ScanDir &R, uint32_t KS, uint32_t nproc)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const Grp<32> wg;
    const uint32_t hdr = user_data_offset(P.data_version);
    for (uint32_t v = warp; v < nproc; v += kScanWarps) {
        if ((A.state[v] & 0xF) != RS_NORMAL) continue;
        uint32_t r = A.vis[v], kl = A.klen[r], vl = A.vlen[r];
        const uint8_t *key = A.arena + (size_t)r * KS;
        const uint32_t koff = A.rank[v], klen_out = kl > koff ? kl - koff : 0u, vlen_out = A.A3[v] - klen_out;
        uint32_t slot = S.n_out + (A.A2[v]);
        unsigned long long aoff = S.arena_used + A.A1[v];
        if (slot >= P.kv_stride || aoff + klen_out + vlen_out > P.arena_stride) { if (lane == 0) atomicMax(&S.error, (uint32_t)PGS_ABORTED); continue; }
        warp_copy_bytes(R.arena + aoff, key + koff, klen_out, lane);
        if (vlen_out) grp_copy(wg, R.arena + aoff + klen_out, A.in + A.voff[r] + hdr, vlen_out);
        if (lane == 0) {
            pgs_kv kv;
            kv.key_off = (uint32_t)aoff; kv.key_len = klen_out;
            kv.value_off = (uint32_t)aoff + klen_out; kv.value_len = vlen_out;
            kv.expire_ts = Q.return_expire_ts && vl >= 4 ? be32(A.in + A.voff[r]) : 0;
            R.kvs[slot] = kv;
        }
    }
}
// thread 0: advance the loop state past the processed positions and decide whether the scan is done (and how)
PGS_DEV void advance(ScanShared &S, const ScanSlots &K, const ScanArrays &A, const ScanParams &P, const ScanReqDev &Q, const ScanDir &R,
                     uint32_t KS, uint32_t rq, uint32_t Pp, uint32_t Ff)
{
    const uint32_t nproc = min(Pp, Ff), nvis = S.n_vis;
    uint32_t stand = 0xFFFFFFFFu; // the loop ended by its limits with the iterator on visible record `stand`
    if (!S.lookahead) {
        uint32_t exp = 0, fil = 0;
        for (uint32_t v = 0; v < nproc; v++) { uint8_t s = A.state[v] & 0xF; exp += s == RS_EXPIRED; fil += s == RS_FILTERED; }
        uint32_t normals = A.A2[nproc];
        S.expire_count += exp; S.filter_count += fil;
        S.iter_count += nproc;
        S.count += normals;
        if (!Q.count_only) { S.n_out += normals; S.arena_used += A.A1[nproc]; }
        S.size += A.A1[nproc];
        // a processed record equal to the range end completes the scan (`if (c == 0) complete`)
        bool hit_end = false;
        if (nproc > 0 && R.end_incl) {
            uint32_t r = A.vis[nproc - 1];
            hit_end = cmp_bytes(A.arena + (size_t)r * KS, A.klen[r], K.end, R.end_len) == 0;
        }
        if (hit_end) { S.complete = 1; S.iter_valid = 1; S.done = 1; }
        else if (Pp <= Ff && Pp < nvis) stand = Pp; // limits ended the loop while the iterator stands on vis[Pp]
        else if (Ff < nvis) { // reached a record outside the prefix (iterator invalid) or past the end (complete)
            uint8_t s = A.state[Ff];
            if (!(s & 0x10)) { S.iter_valid = 0; S.done = 1; }
            else { S.complete = 1; S.iter_valid = 1; S.done = 1; }
        } else {
            // chunk fully consumed.  Did the limits run out exactly here?
            bool ok = (S.count < Q.max_count) && (S.iter_count < Q.max_iter_count) && (Q.max_iter_size == 0 || S.size < Q.max_iter_size);
            if (!ok) S.lookahead = 1; // need to know whether the iterator is still valid
        }
    } else if (nvis > 0) stand = 0; // look-ahead: the iterator stands on the first visible record
    if (stand != 0xFFFFFFFFu) {
        const uint32_t r = A.vis[stand];
        const bool valid = (A.state[stand] & 0x10) != 0;
        S.iter_valid = valid; S.done = 1;
        if (valid) { S.resume_len = A.klen[r]; put_resume_key(P, rq, A.arena + (size_t)r * KS, A.klen[r], 0, 1); }
    }
    if (!S.done) {
        bool any_more = false;
        for (uint32_t j = 0; j < P.rr.n; j++) any_more |= S.more[j] != 0;
        if (!any_more) { S.done = 1; S.iter_valid = 0; }
    }
}
// the next chunk starts at this chunk's far bound: forward it becomes the lower bound (exclusive), reverse the upper bound
// (inclusive)
PGS_DEV void next_bounds(ScanShared &S, const ScanSlots &K, bool rev, uint32_t KS)
{
    for (uint32_t i = threadIdx.x; i < KS + 8; i += kScanThreads) { if (rev) K.hi[i] = K.lo[i]; else K.lo[i] = K.hi[i]; }
    if (threadIdx.x == 0) {
        if (rev) { S.hi_len = S.lo_len; S.has_hi = 1; S.hi_incl = 1; }
        else { S.lo_len = S.hi_len; S.has_lo = 1; S.lo_incl = 0; }
    }
}
// move every run's cursor past the consumed key range (one warp per run).  Forward: first block whose last key > bound;
// reverse: first block whose last key >= bound.
PGS_DEV void next_cursors(ScanShared &S, const ScanSlots &K, const ScanArrays &A, const ScanParams &P, bool rev, uint32_t KS)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, NR = P.rr.n;
    const Grp<32> wg;
    for (uint32_t j = warp; j < NR; j += kScanWarps) {
        const RunDev &r = P.rr.runs[j];
        uint32_t b;
        if (rev) { // blocks after b hold only keys > bound; b itself may hold keys <= bound
            b = grp_index_bound(wg, true, r, K.hi, S.hi_len, false);
            if (b >= r.nb) b = r.nb ? r.nb - 1 : 0xFFFFFFFFu;
            if (!r.nb) b = 0xFFFFFFFFu;
        } else {
            // forward: the bound is the smallest "last key of the last loaded block" over the runs, so the first block whose
            // last key is > bound lies at or right behind this chunk's loaded blocks; their last keys are decoded in the
            // arena -- no index search in global memory
            const uint32_t m = S.nblk[j];
            uint32_t cnt = 0;
            for (uint32_t t0 = 0; t0 < m; t0 += 32) {
                const uint32_t t = t0 + lane;
                bool le = false;
                if (t < m) {
                    const uint32_t tt = S.blk_base[j] + t, nrec = S.tb_nrec[tt];
                    const uint32_t rl = S.tb_rec[tt] + nrec - 1;
                    le = nrec == 0 || cmp_slots(A.arena + (size_t)rl * KS, A.klen[rl], K.lo, S.lo_len) <= 0;
                }
                cnt += __popc(__ballot_sync(kFull, le));
            }
            b = S.cur[j] + cnt; // a run without loaded blocks keeps its (exhausted) cursor
        }
        if (lane == 0) S.cur[j] = b;
    }
}

__global__ void __launch_bounds__(kScanThreads, 4) k_scan(const __grid_constant__ ScanParams P)
{
    PGS_SMEM_DYN(dyn);
    PGS_SMEM_STATIC(ScanShared S);
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    const uint32_t KS = P.KS, NR = P.rr.n;
    const ScanSlots K(dyn, KS, NR);
    if (tid == 0) { mbar_init((uint64_t *)&S.mbar, 1); mbar_fence_init(); }
    __syncthreads();
    uint32_t mbar_phase = 0;
    for (uint32_t rq = blockIdx.x; rq < P.n; rq += gridDim.x) {
        const ScanReqDev &Q = P.reqs[rq];
        const ScanDir R = scan_dir(P, Q, rq);
        seek_cursors(S, P, R);
        begin_request(S, K, P, Q, R, KS);
        __syncthreads();

        for (;;) {
            __syncthreads();
            const bool stop_now = S.done || S.error;
            __syncthreads();
            if (stop_now) break;
            if (warp == 0) choose_blocks(S, P, R.rev, KS, K.pool);
            __syncthreads();
            if (S.done || S.error) break;
            const ScanArrays A = scan_carve(K.pool, S.in_bytes, S.n_rec, KS);
            stage_blocks(S, K, A, P, R.rev, KS, mbar_phase);
            __syncthreads();
            if (tid == 0) pick_far_bound(S, K, R.rev, NR);
            __syncthreads();
            take_far_bound(S, K, R.rev, KS);
            __syncthreads();
            decode_headers(S, A, P, KS);
            __syncthreads();
            if (S.error) break;
            rebuild_keys(S, A, KS);
            __syncthreads();
            if (S.error) break;
            if (tid < NR) { S.vlo[tid] = 0; S.vhi[tid] = 0; }
            __syncthreads();
            window_count(S, K, A, KS, NR);
            __syncthreads();
            window_close(S, NR);
            __syncthreads();
            if (tid == 0) { uint32_t nv = 0; for (uint32_t j = 0; j < NR; j++) nv += S.vhi[j] - S.vlo[j]; S.n_valid = nv; }
            rank_own_run(S, A, KS, NR);
            __syncthreads();
            if (NR > 1) rank_other_runs(S, A, KS, NR);
            __syncthreads();
            merge_order(S, A);
            __syncthreads();
            const uint32_t nvis = visible_list(S, A, R.rev);
            __syncthreads();
            record_states(S, K, A, P, Q, R, KS, nvis);
            __syncthreads();
            // count / size prefixes over the visible list: A2 becomes the exclusive count prefix in place, A1 the size prefix
            scan_chunked(nvis, A.A1, S.scan, [&](uint32_t v) -> uint32_t { return A.A2[v]; });
            for (uint32_t v = tid; v <= nvis; v += kScanThreads) A.A2[v] = A.A1[v];
            __syncthreads();
            scan_chunked(nvis, A.A1, S.scan, [&](uint32_t v) -> uint32_t { return A.A3[v]; });
            if (tid == 0) { S.P = nvis; S.F = nvis; S.n_vis = nvis; }
            __syncthreads();
            loop_limits(S, A, Q, nvis);
            __syncthreads();
            const uint32_t Pp = S.P, Ff = S.F;
            const uint32_t nproc = min(Pp, Ff); // processed positions [0, nproc)
            if (!S.lookahead && nproc > 0 && !Q.count_only) emit(S, A, P, Q, R, KS, nproc);
            __syncthreads();
            if (tid == 0) advance(S, K, A, P, Q, R, KS, rq, Pp, Ff);
            __syncthreads();
            if (!S.done) {
                next_bounds(S, K, R.rev, KS);
                __syncthreads();
                next_cursors(S, K, A, P, R.rev, KS);
                __syncthreads();
            }
        }
        if (tid == 0)
            put_scan_result(P, rq, S.error, S.n_out, S.count, S.iter_count, S.expire_count, S.filter_count, S.size, S.complete != 0,
                            S.iter_valid != 0, S.resume_len, S.arena_used);
        __syncthreads();
    }
}

// Host side (shared with the CPU simulation driver under tools/simt).
// what the device leaves k_scan for dynamic shared memory, given its opt-in limit and the kernel's static shared memory
inline uint64_t scan_max_dyn(uint64_t max_smem_optin, uint64_t static_smem) { return max_smem_optin - static_smem - 256; }

// the smallest staging pool a launch accepts: every chunk stages at least one block of every run that still has blocks, so
// the pool holds one largest block of each run, plus scan_carve's padding
inline uint64_t scan_min_pool(uint32_t n_runs, uint32_t KS, uint32_t max_blk, uint32_t max_rec)
{
    const uint64_t one = (((uint64_t)max_blk + 15) & ~15ull) + 32 + (uint64_t)max_rec * (KS + kScanRecExtra);
    return one * (n_runs ? n_runs : 1) + 64 + scan_carve_slack(KS);
}

// the dynamic shared memory of a k_scan launch over n_runs runs (largest block: max_blk bytes, max_rec records) for a batch
// of n_req requests; max_dyn is what the device leaves for dynamic shared memory.  Returns the launch's dynamic size and sets
// *pool to the staging pool inside it, or returns 0 when the smallest pool (scan_min_pool) does not fit.
inline uint64_t scan_dyn_bytes(uint32_t n_runs, uint32_t KS, uint32_t max_blk, uint32_t max_rec, uint32_t n_req, uint64_t max_dyn,
                               uint32_t *pool)
{
    const uint64_t fixed_dyn = (4 + (uint64_t)n_runs) * ((KS + 8 + 15) & ~15u);
    const uint64_t min_pool = scan_min_pool(n_runs, KS, max_blk, max_rec);
    uint64_t want = min_pool - 64 + 4096;
    if (want < 48 * 1024) want = 48 * 1024;
    if (n_req == 1 && want < 160 * 1024) want = 160 * 1024;
    uint64_t dyn = fixed_dyn + want < max_dyn ? fixed_dyn + want : max_dyn;
    if (dyn < fixed_dyn + min_pool) return 0;
    dyn &= ~127ull;
    *pool = (uint32_t)(dyn - fixed_dyn);
    return dyn;
}

// The kernel of a scan launch over the runs R (P.n set).  Forward batches: k_scan_fwd<G, multi>, the lane-group iterators of
// read_kernels.cuh, unless the groups' key rows do not fit shared memory (user keys of a few KB).  A batch with a reverse
// request, and a single-partition forward batch whose key rows do not fit: k_scan, which stages records instead of keeping
// a key row per run and group.  max_smem_optin = the device's opt-in shared memory per CTA, scan_static = k_scan's static
// shared memory.  Test knobs: force_G = k_scan_fwd's lanes per group (at least the run count), pool_cap = an upper bound on
// k_scan's staging pool, never below scan_min_pool.
inline int32_t scan_plan(ScanParams &P, const ReadRunSet &R, bool any_reverse, uint32_t max_smem_optin, uint64_t scan_static,
                         ReadLaunch<ScanParams> &L, uint32_t force_G = 0, uint32_t pool_cap = 0)
{
    P.rr = R.rr;
    P.KS = R.KS;
    const ReadGeometry fwd = scan_fwd_geometry(R.rr.n, R.KS, force_G);
    const bool fwd_fits = fwd.dyn <= max_smem_optin;
    if (!fwd_fits && R.multi) {
        set_error("scan: %u runs with keys of %u bytes do not fit shared memory", R.rr.n, R.KS);
        return PGS_NOT_SUPPORTED;
    }
    if (!any_reverse && fwd_fits) {
        if (fwd.G < R.rr.n) return PGS_INVALID_ARGUMENT;
        fwd.apply(P);
        L = {scan_fwd_kernel(fwd.G, R.multi), kReadThreads, fwd.dyn, kReadThreads / fwd.G};
        return PGS_OK;
    }
    uint64_t dyn = scan_dyn_bytes(R.rr.n, R.KS, R.bb.max_blk, R.bb.max_rec, P.n, scan_max_dyn(max_smem_optin, scan_static), &P.pool_bytes);
    if (!dyn) {
        set_error("scan: blocks too large for shared memory");
        return PGS_NOT_SUPPORTED;
    }
    if (pool_cap) {
        const uint64_t fixed_dyn = dyn - P.pool_bytes;
        P.pool_bytes = std::max(std::min(P.pool_bytes, pool_cap), (uint32_t)scan_min_pool(R.rr.n, R.KS, R.bb.max_blk, R.bb.max_rec));
        dyn = fixed_dyn + P.pool_bytes;
    }
    L = {k_scan, kScanThreads, (uint32_t)dyn, 1};
    return PGS_OK;
}

} // namespace pgs
