// read_kernels.cuh — the read path on the GPU, built on the lane-group iterators of group.cuh.
//
//   k_get       batched point lookup (DB::Get / DB::MultiGet as used by on_get / on_multi_get(sort_keys) / on_batch_get /
//               on_ttl, src/server/pegasus_server_impl.cpp:441,804,948,1106): one GROUP of lanes per key (four keys per warp
//               at 8 lanes); per run, newest -> oldest: a per-run Bloom filter of whole keys (HashkeyTransform prefix +
//               sort key, src/server/pegasus_server_impl_init.cpp:817-843) skips runs that cannot hold the key, then
//               block-index search (last user key per block, (G+1)-ary over the lanes), restart-interval decode from the
//               block start, user-key compare; newest version wins, a tombstone ends the search; TTL check and header strip
//               fused.
//   k_scan_fwd  forward range scans (NewIterator + Seek + Next loops of on_multi_get range mode, on_get_scanner, on_scan,
//               on_sortkey_count, :617-756,1243-1320,1444-1490,1042-1062): one group per request runs RocksDB's merging
//               iterator over the runs -- seek every run, smallest head first, newest version / tombstone visibility -- and the
//               reference's loop around it (stop key, first-exclusive, range_read_limiter counts and sizes, TTL / hash /
//               sort-key filters) record by record, exactly in the reference's order.  The 32/G groups of a warp run in lock
//               step on different requests; entries are read straight from HBM, records are copied to the output arena.
//   (reverse scans keep the block-staging kernel k_scan of lookup.cu.)
//   k_pack_offsets / k_pack_copy  the packed read-back of a scan batch of either kernel: one CTA places every request's
//               output, then one CTA per request copies it to its place.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "group.cuh"

namespace pgs {

constexpr uint32_t kMaxReadRuns = 32;
constexpr uint32_t kReadThreads = 128;

struct ReadRuns {
    RunDev runs[kMaxReadRuns];
    uint32_t n;
};

struct ScanReqDev {
    uint32_t start_off, start_len, stop_off, stop_len, hf_off, hf_len, sf_off, sf_len;
    uint8_t start_inclusive, stop_inclusive, reverse, no_value, key_mode, return_expire_ts, count_only, validate_hash;
    uint8_t prefix_same_as_start, has_upper, pad[2];
    int32_t hash_filter_type, sort_filter_type;
    uint32_t max_count, max_iter_count;
    unsigned long long max_iter_size;
    int32_t pidx, partition_version;
};

// validate_filter of the read path: pegasus_server_impl.cpp:2350-2380 (an empty pattern matches, an unknown type fails).
// PGS_FT_MATCH_ANYWHERE / _PREFIX / _POSTFIX (1..3) are the MATCH_* types (0..2) plus one.
PGS_DEV bool dev_validate_filter(int32_t type, const uint8_t *pat, uint32_t pl, const uint8_t *v, uint32_t vl)
{
    if (type == PGS_FT_NO_FILTER) return true;
    if (type < PGS_FT_NO_FILTER || type > PGS_FT_MATCH_POSTFIX) return false;
    return pl == 0 || pattern_match((uint32_t)(type - PGS_FT_MATCH_ANYWHERE), pat, pl, v, vl);
}

// ---- block-index search ------------------------------------------------------------------------------------------------------
// (G+1)-ary search over a run's block index (last user key of every block): every round the G lanes of a group probe G
// pivots, so the chain of dependent global loads is ~log_{G+1}(nb) long.  upper = false: first block whose last key >= key;
// upper = true: first block whose last key > key.  Whole warp; groups with en = false get 0.  `key` may live in any space.
template <uint32_t G>
PGS_DEV uint32_t grp_index_bound(const Grp<G> &g, bool en, const RunDev &r, const uint8_t *key, uint32_t klen, bool upper)
{
    uint32_t lo = 0, hi = en ? r.nb : 0u;
    while (g.any(hi - lo > G)) {
        const bool wide = hi - lo > G;
        const uint32_t span = hi - lo;
        const uint32_t piv = lo + (uint32_t)(((unsigned long long)span * (g.gl + 1)) / (G + 1));
        bool before = false; // the pivot block lies strictly before the answer
        if (wide) {
            const uint32_t o = r.ikey_off[piv], l = r.ikey_off[piv + 1] - o;
            const int c = cmp_bytes4(r.ikeys + o, l, key, klen);
            before = upper ? c <= 0 : c < 0;
        }
        const uint32_t cnt = (uint32_t)__popc(g.ballot(before)); // monotone: lanes 0..cnt-1 are true
        const uint32_t p_lo = g.shfl(piv, cnt ? cnt - 1 : 0u), p_hi = g.shfl(piv, cnt);
        if (wide) {
            if (cnt) lo = p_lo + 1;
            if (cnt < G) hi = p_hi;
        }
    }
    bool before = false;
    if (lo + g.gl < hi) {
        const uint32_t o = r.ikey_off[lo + g.gl], l = r.ikey_off[lo + g.gl + 1] - o;
        const int c = cmp_bytes4(r.ikeys + o, l, key, klen);
        before = upper ? c <= 0 : c < 0;
    }
    return lo + (uint32_t)__popc(g.ballot(before));
}

// position cursor C on the first entry of run r whose user key is >= key (the newest version of that key comes first).
// `keyrow` = the key in a key row (shared memory), klen its length.  Whole warp.  Returns 0 or a status.
template <uint32_t G>
PGS_DEV uint32_t cur_seek(const Grp<G> &g, bool en, const RunDev &r, CurState *C, uint32_t *row, uint32_t KS, const uint32_t *keyrow, uint32_t klen)
{
    const uint32_t b = grp_index_bound(g, en, r, (const uint8_t *)keyrow, klen, false);
    uint32_t err = cur_open(g, en, r, C, row, KS, b, en ? r.nb : 0u, 0xFFFFFFFFu);
    for (;;) { // entries of the block that sort before the key
        const bool lv = en && !err && C->live;
        uint32_t dpos;
        const int c = row_cmp(g, lv, row, lv ? C->klen - 8 : 0u, keyrow, klen, dpos);
        const bool more = lv && c < 0;
        if (!g.any(more)) break;
        const uint32_t e2 = cur_next(g, more, r, C, row, KS);
        if (more) err = e2;
    }
    return err;
}

// group copy global -> global, any alignment: destination-aligned 16-byte stores, the source re-aligned with funnel shifts
template <uint32_t G>
PGS_DEV void grp_copy(const Grp<G> &g, uint8_t *dst, const uint8_t *src, uint32_t n)
{
    uint32_t lead = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (lead > n) lead = n;
    for (uint32_t i = g.gl; i < lead; i += G) dst[i] = src[i];
    dst += lead; src += lead; n -= lead;
    const uint32_t nch = n >> 4;
    const uint32_t *sw = (const uint32_t *)((uintptr_t)src & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)((uintptr_t)src & 3) * 8;
    for (uint32_t c = g.gl; c < nch; c += G) {
        const uint32_t *w = sw + 4 * c;
        const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3];
        uint4 o;
        if (sh == 0) o = make_uint4(w0, w1, w2, w3);
        else {
            const uint32_t w4 = w[4];
            o.x = __funnelshift_r(w0, w1, sh); o.y = __funnelshift_r(w1, w2, sh); o.z = __funnelshift_r(w2, w3, sh); o.w = __funnelshift_r(w3, w4, sh);
        }
        *reinterpret_cast<uint4 *>(dst + 16 * c) = o;
    }
    for (uint32_t i = 16 * nch + g.gl; i < n; i += G) dst[i] = src[i];
}

// ---- k_get ----------------------------------------------------------------------------------------------------------------
struct GetParams {
    ReadRuns rr;
    const uint8_t *keys;
    const uint32_t *key_off;
    uint32_t n, now, data_version;
    uint32_t KS, KSW, group_smem;
    pgs_get_result *results;
    uint8_t *arena;
    unsigned long long arena_cap;
    unsigned long long *arena_cursor; // [0] = arena bytes, [1] = data blocks probed, [2] = runs skipped by the Bloom filter
    uint32_t *error;
    uint32_t *ticket;
    // several partitions in one launch (pgs_get_batch_multi): key q belongs to partition slot key_part[q], whose runs are
    // multi_runs[multi_begin[slot] .. multi_begin[slot + 1]); null for a single-partition batch (rr)
    const RunDev *multi_runs;
    const uint32_t *multi_begin;
    const uint32_t *key_part;
};

template <uint32_t G, bool MULTI>
__global__ void __launch_bounds__(kReadThreads) k_get(const __grid_constant__ GetParams P)
{
    PGS_SMEM_DYN(dyn);
    const Grp<G> g;
    constexpr uint32_t NGW = 32 / G;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    RunDev *runs = (RunDev *)dyn;
    for (uint32_t i = threadIdx.x; i < kMaxReadRuns; i += blockDim.x) runs[i] = P.rr.runs[i < P.rr.n ? i : 0];
    __syncthreads();
    uint8_t *gs = dyn + kMaxReadRuns * sizeof(RunDev) + (size_t)(warp * NGW + g.shift / G) * P.group_smem;
    CurState *C = (CurState *)gs;
    uint32_t *row = (uint32_t *)(gs + sizeof(CurState)), *keyrow = row + P.KSW;
    const uint32_t KS = P.KS, NR = P.rr.n;
    unsigned long long probes = 0, skipped = 0;
    for (;;) {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(P.ticket, NGW);
        t0 = __shfl_sync(kFull, t0, 0);
        if (t0 >= P.n) break;
        const uint32_t q = t0 + g.shift / G;
        const bool en = q < P.n;
        uint32_t klen = 0, err = 0;
        const uint8_t *key = P.keys;
        if (en) { key = P.keys + P.key_off[q]; klen = P.key_off[q + 1] - P.key_off[q]; }
        const uint32_t klen_row = klen > KS ? KS + 1 : klen; // longer than any stored key: its first KS+1 bytes order it the same way
        for (uint32_t i = g.gl; i < klen_row; i += G) ((uint8_t *)keyrow)[i] = key[i];
        g.sync();
        const unsigned long long bh = bloom_hash_row(g, keyrow, klen_row);
        pgs_get_result res;
        res.status = PGS_NOT_FOUND;
        res.expire_ts = 0; res.value_off = 0; res.value_len = 0; res.expired = 0;
        res.reserved[0] = res.reserved[1] = res.reserved[2] = 0;
        bool pending = en && klen <= KS; // a key longer than every stored key cannot be found
        const RunDev *rbase = runs;      // the runs of the key's partition, newest -> oldest (MULTI: in global memory)
        uint32_t nr = NR;
        if constexpr (MULTI) {
            if (en) {
                const uint32_t slot = P.key_part[q];
                rbase = P.multi_runs + P.multi_begin[slot];
                nr = P.multi_begin[slot + 1] - P.multi_begin[slot];
            }
        }
        for (uint32_t ri = 0; MULTI ? g.any(pending && ri < nr) : ri < NR; ri++) {
            if (!MULTI && !g.any(pending)) break;
            const bool act = pending && ri < nr;
            const RunDev &r = MULTI ? (act ? rbase[ri] : runs[0]) : runs[ri];
            bool probe = act;
            if (probe && !bloom_may_contain(r.bloom, r.bloom_lines, bh)) { probe = false; if (g.gl == 0) skipped++; }
            if (!g.any(probe)) continue;
            const uint32_t e1 = cur_seek(g, probe, r, C, row, KS, keyrow, klen_row);
            if (probe) {
                if (g.gl == 0 && C->b < r.nb) probes++;
                if (e1) { err = e1; pending = false; }
            }
            uint32_t dpos;
            const bool cand = probe && !e1 && C->live; // cur_seek stopped at the first entry >= key: a hit iff equal
            const int c = row_cmp(g, cand, row, cand ? C->klen - 8 : 0u, keyrow, klen_row, dpos);
            const bool hit = cand && c == 0; // newest version of the key in this run
            bool copy = false;
            uint32_t ulen = 0;
            const uint32_t hdr = user_data_offset(P.data_version);
            if (hit) {
                pending = false;
                if ((C->tr_lo & 0xffu) == PGS_TYPE_VALUE) {
                    const uint32_t vl = C->vlen;
                    const uint32_t ets = vl >= 4 ? __byte_perm(C->ets_le, 0, 0x0123) : 0u;
                    res.expire_ts = ets;
                    if (ts_expired(P.now, ets)) res.expired = 1; // check_if_record_expired -> NotFound (pegasus_server_impl.cpp:443-448)
                    else { copy = true; ulen = vl >= hdr ? vl - hdr : 0; }
                }
            }
            unsigned long long off = 0;
            if (copy && g.gl == 0) off = atomicAdd(P.arena_cursor, (unsigned long long)((ulen + 3) & ~3u));
            off = g.shfl(off, 0);
            if (copy) {
                if (off + ulen > P.arena_cap) res.status = PGS_INCOMPLETE;
                else {
                    res.status = PGS_OK;
                    res.value_off = (uint32_t)off;
                    res.value_len = ulen;
                    grp_copy(g, P.arena + off, r.data + cur_base(C) + C->voff + hdr, ulen);
                }
            }
        }
        if (en && g.gl == 0) {
            P.results[q] = res;
            if (err) atomicMax(P.error, err);
        }
        g.sync();
    }
    if (g.gl == 0) {
        if (probes) atomicAdd(P.arena_cursor + 1, probes);
        if (skipped) atomicAdd(P.arena_cursor + 2, skipped);
    }
}

// ---- k_scan_fwd ---------------------------------------------------------------------------------------------------------------
struct ScanParams {
    ReadRuns rr;
    const ScanReqDev *reqs;
    const uint8_t *blob; // request byte strings
    uint32_t n, now, data_version;
    uint32_t KS, KSW, group_smem, pool_bytes;
    pgs_scan_result *results;
    pgs_kv *kvs;
    uint32_t kv_stride;
    uint8_t *arena;
    unsigned long long arena_stride;
    uint8_t *resume;
    uint32_t resume_stride;
    const unsigned long long *crc_table;
    uint32_t *error;
    uint32_t *ticket;
    // requests of several partitions in one launch (pgs_range_scan_many_multi, forward only): request i reads the runs
    // multi_runs[multi_begin[req_part[i]] .. multi_begin[req_part[i] + 1]); rr.n = the largest run count; null otherwise
    const RunDev *multi_runs;
    const uint32_t *multi_begin;
    const uint32_t *req_part;
};

enum : uint8_t { RS_NORMAL = 0, RS_EXPIRED = 1, RS_FILTERED = 2, RS_HASH_INVALID = 3 };

// validate_key_value_for_scan (pegasus_server_impl.cpp:2382-2431) of a visible record inside the range, for both scan kernels:
// its state, and what an RS_NORMAL record puts out -- key bytes [koff, koff + klen) of the user key (key_mode 1: the sort key)
// and vlen value bytes behind the hdr-byte value header (none with no_value).  crc = the crc64 table (read when validate_hash).
struct ScanRecord {
    uint8_t st;
    uint32_t koff, klen, vlen;
};
PGS_DEV ScanRecord scan_record(const ScanReqDev &Q, const uint8_t *blob, const unsigned long long *crc, uint32_t now, uint32_t hdr,
                               const uint8_t *key, uint32_t ulen, uint32_t vlen, uint32_t expire_ts)
{
    const KeyParts k = split_key(key, ulen);
    ScanRecord o;
    o.st = RS_NORMAL;
    if (ts_expired(now, expire_ts)) o.st = RS_EXPIRED;
    else if (Q.validate_hash && (Q.partition_version < 0 || Q.pidx > Q.partition_version || // :2397-2404
                                 (ulen >= 2 && (long long)(pegasus_key_hash(crc, key, ulen) & (unsigned long long)(long long)Q.partition_version) !=
                                                   (long long)Q.pidx)))
        o.st = RS_HASH_INVALID;
    else if (!dev_validate_filter(Q.hash_filter_type, blob + Q.hf_off, Q.hf_len, k.hk, k.hkl) ||
             !dev_validate_filter(Q.sort_filter_type, blob + Q.sf_off, Q.sf_len, k.sk, k.skl))
        o.st = RS_FILTERED;
    o.koff = Q.key_mode == 1 ? 2 + k.hkl : 0u;
    o.klen = Q.key_mode == 1 ? k.skl : ulen;
    o.vlen = Q.no_value ? 0u : (vlen >= hdr ? vlen - hdr : 0u);
    return o;
}

// the key request rq's scan context resumes at; lanes [lane, lane + step, ...] copy it, at most resume_stride bytes
PGS_DEV void put_resume_key(const ScanParams &P, uint32_t rq, const uint8_t *key, uint32_t len, uint32_t lane, uint32_t step)
{
    uint8_t *rk = P.resume + (size_t)rq * P.resume_stride;
    for (uint32_t i = lane; i < len && i < P.resume_stride; i += step) rk[i] = key[i];
}

// the result of request rq once its loop has ended (one thread)
PGS_DEV void put_scan_result(const ScanParams &P, uint32_t rq, uint32_t err, uint32_t n_out, uint32_t count, uint32_t iter_count,
                             uint32_t expire_count, uint32_t filter_count, unsigned long long size, bool complete, bool iter_valid,
                             uint32_t resume_len, unsigned long long arena_used)
{
    pgs_scan_result res;
    res.status = err ? (int32_t)err : PGS_OK;
    res.n_kvs = n_out; res.count = count; res.iter_count = iter_count; res.expire_count = expire_count; res.filter_count = filter_count;
    res.size = size;
    res.complete = complete ? 1 : 0; res.iter_valid = iter_valid ? 1 : 0; res.reserved[0] = res.reserved[1] = 0;
    res.resume_len = iter_valid ? resume_len : 0;
    res.arena_used = arena_used;
    P.results[rq] = res;
    if (err) atomicMax(P.error, err);
}

// the merge order of two cursor heads of k_scan_fwd: user key ascending, trailer (seq, type) descending, run index.  Whole
// warp; false for groups without en.  (head_before of the compaction walker states the same order with a shortcut over the
// first eight key bytes, which measured slower here.)
template <uint32_t G>
PGS_DEV bool run_before(const Grp<G> &g, bool en, const CurState *cs, const uint32_t *rows, uint32_t KSW, uint32_t a, uint32_t b, uint32_t &dpos)
{
    uint32_t la = 0, lb = 0;
    if (en) { la = cs[a].klen - 8; lb = cs[b].klen - 8; }
    const int c = row_cmp(g, en, rows + a * KSW, la, rows + b * KSW, lb, dpos);
    if (!en) return false;
    if (c) return c < 0;
    const unsigned long long ta = cur_trailer(&cs[a]), tb = cur_trailer(&cs[b]);
    return ta != tb ? ta > tb : a < b;
}

template <uint32_t G, bool MULTI>
__global__ void __launch_bounds__(kReadThreads) k_scan_fwd(const __grid_constant__ ScanParams P)
{
    PGS_SMEM_DYN(dyn);
    const Grp<G> g;
    constexpr uint32_t NGW = 32 / G;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long *crc = (unsigned long long *)dyn; // 2 KB, filled when a request validates partition hashes
    RunDev *runs = (RunDev *)(dyn + 2048);
    if (P.crc_table)
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) crc[i] = P.crc_table[i];
    for (uint32_t i = threadIdx.x; i < kMaxReadRuns; i += blockDim.x) runs[i] = P.rr.runs[i < P.rr.n ? i : 0];
    __syncthreads();
    const uint32_t KS = P.KS, KSW = P.KSW, NR = P.rr.n;
    uint8_t *gs = dyn + 2048 + kMaxReadRuns * sizeof(RunDev) + (size_t)(warp * NGW + g.shift / G) * P.group_smem;
    CurState *cs = (CurState *)gs;
    uint32_t *rows = (uint32_t *)(gs + (size_t)NR * sizeof(CurState));
    uint32_t *rowSTART = rows + NR * KSW, *rowSTOP = rowSTART + KSW, *rowLAST = rowSTOP + KSW;
    const uint32_t hdr = user_data_offset(P.data_version);

    for (;;) {
        uint32_t t0 = 0;
        if (lane == 0) t0 = atomicAdd(P.ticket, NGW);
        t0 = __shfl_sync(kFull, t0, 0);
        if (t0 >= P.n) break;
        const uint32_t rq = t0 + g.shift / G;
        const bool en = rq < P.n;
        const ScanReqDev &Q = P.reqs[en ? rq : 0];
        // ---- the request's bounds into key rows (a bound longer than any stored key: its first KS+1 bytes order it the same way)
        const uint8_t *start = P.blob + Q.start_off, *stop = P.blob + Q.stop_off;
        const uint32_t start_len = Q.start_len > KS ? KS + 1 : Q.start_len, stop_len = Q.stop_len > KS ? KS + 1 : Q.stop_len;
        if (en) {
            for (uint32_t i = g.gl; i < start_len; i += G) ((uint8_t *)rowSTART)[i] = start[i];
            for (uint32_t i = g.gl; i < stop_len; i += G) ((uint8_t *)rowSTOP)[i] = stop[i];
        }
        g.sync();
        // prefix_same_as_start: the iterator only lives inside the seek key's hash-key prefix (HashkeyTransform::InDomain)
        uint32_t pre_len = 0;
        if (en && Q.prefix_same_as_start && Q.start_len >= 2) {
            const uint32_t hl = ((uint32_t)start[0] << 8) | start[1];
            if (2 + hl <= Q.start_len && 2 + hl <= KS) pre_len = 2 + hl;
            else if (2 + hl <= Q.start_len) pre_len = 0xFFFFFFFFu; // a prefix longer than any stored key: nothing is in the domain
        }
        const unsigned long long pre_hash = bloom_hash_row(g, rowSTART, pre_len != 0xFFFFFFFFu ? pre_len : 0u);
        pgs_kv *kvs = P.kvs + (size_t)rq * P.kv_stride;
        uint8_t *arena = P.arena + (size_t)rq * P.arena_stride;
        uint32_t err = 0;

        // the runs of the request's partition (MULTI: in global memory, per request)
        const RunDev *rbase = runs;
        uint32_t nr = NR;
        if constexpr (MULTI) {
            if (en) {
                const uint32_t slot = P.req_part[rq];
                rbase = P.multi_runs + P.multi_begin[slot];
                nr = P.multi_begin[slot + 1] - P.multi_begin[slot];
            }
        }
        // ---- Seek: every run's cursor to its first entry >= start; runs whose Bloom filter excludes the prefix stay closed ----
        uint32_t live = 0, my_run = 0, dpos = 0;
        for (uint32_t j = 0; j < NR; j++) {
            bool use = en && !err && pre_len != 0xFFFFFFFFu && j < nr;
            const RunDev &rj = MULTI ? (use ? rbase[j] : runs[0]) : runs[j];
            if (use && pre_len && !bloom_may_contain(rj.bloom, rj.bloom_lines, pre_hash)) use = false;
            CurState *C = &cs[j];
            if (en && !use && g.gl == 0) C->live = 0;
            const uint32_t e1 = cur_seek(g, use, rj, C, rows + j * KSW, KS, rowSTART, start_len);
            if (use) err = e1;
            g.sync();
            const bool ins = use && !err && C->live;
            uint32_t pos = live;
            bool searching = ins;
            for (uint32_t i = 0; g.any(searching && i < live); i++) {
                const uint32_t r = g.shfl(my_run, i) & 31u;
                if (run_before(g, searching && i < live, cs, rows, KSW, j, r, dpos)) { pos = i; searching = false; }
            }
            const uint32_t up = g.shfl_up(my_run, 1);
            if (ins) {
                if (g.gl > pos && g.gl <= live) my_run = up;
                if (g.gl == pos) my_run = j;
                live++;
            }
        }

        // ---- the iterator loop (pegasus_server_impl.cpp:617-756 / 1266-1320 / 1444-1490), one merged record per step ----------
        uint32_t count = 0, iter_count = 0, expire_count = 0, filter_count = 0, n_out = 0, resume_len = 0;
        unsigned long long size = 0, arena_used = 0;
        bool complete = false, iter_valid = false, done = !en || err != 0, have_last = false, first_excl = en && !Q.start_inclusive;
        uint32_t last_len = 0;
        for (;;) {
            const bool act = !done;
            if (!g.any(act)) break;
            const bool exhausted = act && live == 0; // Valid() == false
            if (exhausted) { done = true; iter_valid = false; }
            const bool rec = act && !exhausted;
            const uint32_t c = g.shfl(my_run, 0) & 31u;
            CurState *C = &cs[c];
            uint32_t *row = rows + c * KSW;
            uint32_t ulen = 0, vlen = 0, type = 0;
            if (rec) { ulen = C->klen - 8; vlen = C->vlen; type = C->tr_lo & 0xffu; }
            // newest version of each user key only; a tombstone hides the key
            const bool cmpl = rec && have_last;
            const int cl = row_cmp(g, cmpl, row, ulen, rowLAST, last_len, dpos);
            const bool shadow = cmpl && cl == 0;
            const bool visible = rec && !shadow && type == PGS_TYPE_VALUE;
            // the loop's view of a visible record
            uint32_t d_stop = 0, d_start = 0;
            const int c2 = row_cmp(g, visible, row, ulen, rowSTOP, stop_len, d_stop);
            const bool need_first = visible && first_excl;
            int c_first = 1;
            if (g.any(need_first)) c_first = row_cmp(g, need_first, row, ulen, rowSTART, start_len, d_start);
            bool advance = rec; // hidden records are stepped over
            if (visible) {
                const uint8_t *key = (const uint8_t *)row;
                bool valid = true; // Iterator::Valid(): inside the seek prefix, below iterate_upper_bound
                if (pre_len) { // the key starts with the seek prefix: word by word (the rows are 4-byte aligned)
                    valid = ulen >= pre_len;
                    const uint32_t nw = pre_len >> 2;
                    for (uint32_t w = 0; valid && w < nw; w++) valid = row[w] == rowSTART[w];
                    if (valid && (pre_len & 3)) valid = ((row[nw] ^ rowSTART[nw]) & ((1u << (8 * (pre_len & 3))) - 1u)) == 0;
                }
                if (Q.has_upper && c2 >= 0) valid = false;
                const bool guards = count < Q.max_count && iter_count < Q.max_iter_count && !(Q.max_iter_size > 0 && size >= Q.max_iter_size);
                if (!guards || !valid) { // the while condition fails: the loop ends with the iterator standing here
                    done = true; iter_valid = valid; advance = false;
                } else if (c2 > 0 || (c2 == 0 && !Q.stop_inclusive)) {
                    done = true; iter_valid = true; complete = true; advance = false;
                } else if (first_excl && c_first == 0) {
                    first_excl = false; // the start key itself, excluded: it.Next(); continue
                } else {
                    first_excl = false;
                    iter_count++;
                    const uint32_t ets = vlen >= 4 ? __byte_perm(C->ets_le, 0, 0x0123) : 0u;
                    const ScanRecord o = scan_record(Q, P.blob, crc, P.now, hdr, key, ulen, vlen, ets);
                    if (o.st == RS_EXPIRED) expire_count++;
                    else if (o.st == RS_FILTERED) filter_count++;
                    else if (o.st == RS_NORMAL) {
                        const uint32_t koff = o.koff, klen_out = o.klen, vlen_out = o.vlen;
                        count++;
                        size += klen_out + vlen_out;
                        if (!Q.count_only) {
                            if (n_out >= P.kv_stride || arena_used + klen_out + vlen_out > P.arena_stride) { err = PGS_ABORTED; done = true; }
                            else {
                                uint8_t *dst = arena + arena_used;
                                for (uint32_t i = g.gl; i < klen_out; i += G) dst[i] = key[koff + i];
                                if (vlen_out) grp_copy(g, dst + klen_out, (MULTI ? rbase[c] : runs[c]).data + cur_base(C) + C->voff + hdr, vlen_out);
                                if (g.gl == 0) {
                                    pgs_kv kv;
                                    kv.key_off = (uint32_t)arena_used; kv.key_len = klen_out;
                                    kv.value_off = (uint32_t)arena_used + klen_out; kv.value_len = vlen_out;
                                    kv.expire_ts = Q.return_expire_ts && vlen >= 4 ? ets : 0u;
                                    kvs[n_out] = kv;
                                }
                                n_out++;
                                arena_used += klen_out + vlen_out;
                            }
                        }
                    }
                    if (c2 == 0) { done = true; iter_valid = true; complete = true; advance = false; } // `if (c == 0) complete`
                }
                if (done && iter_valid && !complete) { // the scan context resumes here
                    resume_len = ulen;
                    put_resume_key(P, rq, key, ulen, g.gl, G);
                }
            }
            g.sync(); // every lane has read rowLAST
            if (rec && !shadow && advance) {
                for (uint32_t w = g.gl; 4 * w < ulen; w += G) rowLAST[w] = row[w];
                have_last = true;
                last_len = ulen;
            }
            g.sync();
            // step the cursor, restore the merge order
            const bool adv = rec && advance && !err;
            const uint32_t e3 = cur_next(g, adv, MULTI ? (adv ? rbase[c] : runs[0]) : runs[c], C, row, KS);
            if (adv && e3) { err = e3; done = true; }
            const bool alive = adv && !e3 && C->live != 0;
            bool searching = alive && live > 1;
            uint32_t pos = 0;
            const bool reorder = searching;
            for (uint32_t i = 1; g.any(searching && i < live); i++) {
                const uint32_t r = g.shfl(my_run, i) & 31u;
                const bool e = searching && i < live;
                const bool bf = run_before(g, e, cs, rows, KSW, c, r, dpos);
                if (e) { if (bf) searching = false; else pos = i; }
            }
            const uint32_t dn = g.shfl_down(my_run, 1);
            if (adv && !e3 && !alive) { if (g.gl + 1 < live) my_run = dn; live--; }
            else if (reorder && pos > 0) { if (g.gl < pos) my_run = dn; if (g.gl == pos) my_run = c; }
        }
        if (en && g.gl == 0)
            put_scan_result(P, rq, err, n_out, count, iter_count, expire_count, filter_count, size, complete, iter_valid, resume_len, arena_used);
        g.sync();
    }
}

// ---- launch planning (host side; shared with the CPU simulation driver under tools/simt) -------------------------------------
// user-key capacity of a read launch's key rows: the longest user key of its runs, at least 8 bytes, a multiple of 8
inline uint32_t read_key_slot(uint32_t max_ukey) { return std::max(8u, (max_ukey + 7) & ~7u); }

// the requests of a scan batch as the kernels read them: fixed-size records + their byte strings back to back in one blob
struct ScanBatch {
    std::vector<ScanReqDev> reqs;
    std::string blob;          // + 16 bytes of slack
    bool need_crc = false;     // a request validates partition hashes
    bool any_reverse = false;  // a request iterates backwards (k_scan)
};
inline ScanBatch flatten_scan_requests(const pgs_scan_request *reqs, uint32_t n)
{
    ScanBatch b;
    b.reqs.resize(n);
    auto put = [&](const pgs_blob &x, uint32_t &off, uint32_t &len) {
        off = (uint32_t)b.blob.size();
        len = x.len;
        if (x.len) b.blob.append((const char *)x.data, x.len);
    };
    for (uint32_t i = 0; i < n; i++) {
        const pgs_scan_request &q = reqs[i];
        ScanReqDev &d = b.reqs[i];
        memset(&d, 0, sizeof d);
        put(q.start, d.start_off, d.start_len);
        put(q.stop, d.stop_off, d.stop_len);
        put(q.hash_filter, d.hf_off, d.hf_len);
        put(q.sort_filter, d.sf_off, d.sf_len);
        d.start_inclusive = q.start_inclusive; d.stop_inclusive = q.stop_inclusive; d.reverse = q.reverse;
        d.no_value = q.no_value; d.key_mode = q.key_mode; d.return_expire_ts = q.return_expire_ts;
        d.count_only = q.count_only; d.validate_hash = q.validate_hash; d.prefix_same_as_start = q.prefix_same_as_start;
        d.has_upper = q.reserved[0]; // iterate_upper_bound (internal flag used by sortkey_count)
        d.hash_filter_type = q.hash_filter_type; d.sort_filter_type = q.sort_filter_type;
        d.max_count = q.max_count; d.max_iter_count = q.max_iter_count; d.max_iter_size = q.max_iter_size;
        d.pidx = q.pidx; d.partition_version = q.partition_version;
        b.need_crc |= q.validate_hash != 0;
        b.any_reverse |= q.reverse != 0;
    }
    b.blob.append(16, '\0');
    return b;
}

// the per-request output slices of a scan launch (P.KS set): kv_stride records, an arena slice of arena_stride bytes rounded
// up to 16, and a resume-key slot of resume_stride bytes.  pgs_kv's offsets are 32-bit, so a slice holds at most 4 GiB - 16
// bytes: an output that passes that ends as any output that passes its slice, with PGS_ABORTED.  A slot shorter than the
// launch's key slot cannot hold every resume key: then the kernels write them to slots of KS bytes and none is reported
// (returns false).
constexpr unsigned long long kMaxScanSlice = (1ull << 32) - 16;
inline bool scan_output_strides(ScanParams &P, unsigned long long arena_stride, uint32_t kv_stride, uint32_t resume_stride)
{
    const bool report_resume = resume_stride >= P.KS;
    P.kv_stride = kv_stride;
    P.arena_stride = std::min((arena_stride + 15) & ~15ull, kMaxScanSlice);
    P.resume_stride = report_resume ? resume_stride : P.KS;
    return report_resume;
}

// a multi-partition launch: rr.n = the most runs of one partition slot, and every entry of rr.runs is a valid dummy run for
// the groups that have no request (packed[begin[s] .. begin[s + 1]) are the runs of slot s)
inline void multi_read_runs(const std::vector<RunDev> &packed, const std::vector<uint32_t> &begin, ReadRuns &rr)
{
    rr.n = 0;
    for (size_t s = 0; s + 1 < begin.size(); s++) rr.n = std::max(rr.n, begin[s + 1] - begin[s]);
    for (uint32_t i = 0; i < kMaxReadRuns; i++) rr.runs[i] = packed.empty() ? RunDev{} : packed[0];
}

// shared memory of a k_get / k_scan_fwd launch: G lanes per group, KS / KSW the key row's bytes / 32-bit words, group_smem
// one group's cursor states and key rows, dyn the launch's dynamic shared memory
struct ReadGeometry {
    uint32_t G, KS, KSW, group_smem, dyn;
    template <class Params> void apply(Params &P) const { P.KS = KS; P.KSW = KSW; P.group_smem = group_smem; }
};
inline ReadGeometry get_geometry(uint32_t KS)
{
    ReadGeometry g;
    g.G = 8;
    g.KS = KS;
    g.KSW = (KS + 8) / 4 + 1;
    g.group_smem = (uint32_t)((sizeof(CurState) + 2 * g.KSW * 4 + 15) & ~(size_t)15);
    g.dyn = kMaxReadRuns * (uint32_t)sizeof(RunDev) + (kReadThreads / g.G) * g.group_smem;
    return g;
}
// n_runs = the most runs one request reads; force_G overrides the lanes per group (tests)
inline ReadGeometry scan_fwd_geometry(uint32_t n_runs, uint32_t KS, uint32_t force_G = 0)
{
    ReadGeometry g;
    g.G = force_G ? force_G : n_runs <= 8 ? 8 : n_runs <= 16 ? 16 : 32;
    g.KS = KS;
    g.KSW = (KS + 8) / 4 + 1;
    g.group_smem = (uint32_t)((n_runs * (sizeof(CurState) + g.KSW * 4) + 3 * g.KSW * 4 + 15) & ~(size_t)15);
    g.dyn = 2048 + kMaxReadRuns * (uint32_t)sizeof(RunDev) + (kReadThreads / g.G) * g.group_smem;
    return g;
}

typedef void (*scan_fwd_kernel_t)(const ScanParams);
constexpr uint32_t kScanFwdGs[] = {8, 16, 32};
// a template only so that the kernels are instantiated where it is first called, which keeps their order in the binary
template <class = void>
inline scan_fwd_kernel_t scan_fwd_kernel(uint32_t G, bool multi)
{
    const scan_fwd_kernel_t k[3][2] = {{k_scan_fwd<8, false>, k_scan_fwd<8, true>},
                                       {k_scan_fwd<16, false>, k_scan_fwd<16, true>},
                                       {k_scan_fwd<32, false>, k_scan_fwd<32, true>}};
    return k[G == 8 ? 0 : G == 16 ? 1 : 2][multi ? 1 : 0];
}

// ---- the read launch plan: what the library (lookup.cu) and the simulator (tools/simt) both launch ------------------------------
void set_error(const char *fmt, ...); // the message of a refused call (engine.cu; the simulator prints it)

// the largest block of a launch's runs, in bytes and in records (k_scan's staging pool, scan_kernel.cuh)
struct ScanBlockBound {
    uint32_t max_blk = 0, max_rec = 0;
    void add(const pgs_run_info &i) { max_blk = std::max(max_blk, i.max_block_size); max_rec = std::max(max_rec, i.max_block_records); }
};

// The runs of one read launch.  A call with a key / request slot index (multi) uses the MULTI instantiations, even with one
// slot: slot s reads packed[begin[s] .. begin[s + 1]) and rr holds dummies (multi_read_runs).  Any other call reads its one
// slot's runs from the kernels' shared-memory table rr.  KS = the launch's key slot, bb = the largest block of its runs.
struct ReadRunSet {
    bool multi = false;
    ReadRuns rr{};
    uint32_t KS = 8;
    ScanBlockBound bb;
    std::vector<RunDev> packed;
    std::vector<uint32_t> begin{0};
    bool empty() const { return packed.empty(); } // every iterator is invalid from the start: no launch
};
// slots = one run list (newest first) per partition slot, of runs with dev() and info (the library's Run, the simulator's
// HostRun).  PGS_NOT_SUPPORTED when a slot has more than kMaxReadRuns runs or a user key longer than kMaxUkeyLen.
template <class Slots>
inline int32_t read_run_set(const Slots &slots, bool multi, ReadRunSet &R)
{
    R.multi = multi;
    uint32_t mk = 0;
    for (const auto &runs : slots) {
        if (runs.size() > kMaxReadRuns) {
            set_error("read: %zu runs > %u (compact first)", runs.size(), kMaxReadRuns);
            return PGS_NOT_SUPPORTED;
        }
        uint32_t slot_mk = 0;
        for (const auto &r : runs) {
            R.packed.push_back(r->dev());
            R.bb.add(r->info);
            slot_mk = std::max(slot_mk, r->info.max_ukey_len);
        }
        if (slot_mk > kMaxUkeyLen) return PGS_NOT_SUPPORTED;
        mk = std::max(mk, slot_mk);
        R.begin.push_back((uint32_t)R.packed.size());
    }
    R.KS = read_key_slot(mk);
    if (multi) multi_read_runs(R.packed, R.begin, R.rr);
    else { R.rr.n = (uint32_t)R.packed.size(); std::copy(R.packed.begin(), R.packed.end(), R.rr.runs); }
    return PGS_OK;
}

// the kernel of a read launch, its block size and dynamic shared memory, and how many requests one CTA takes
template <class Params>
struct ReadLaunch {
    void (*kernel)(const Params);
    uint32_t threads, dyn, per_cta;
};
// launches L over P.n requests on at most max_ctas CTAs (the library: as many as the device holds at once)
template <class Params>
inline void read_launch(const ReadLaunch<Params> &L, const Params &P, uint64_t max_ctas, cudaStream_t st)
{
    const uint32_t grid = (uint32_t)std::min<uint64_t>((P.n + L.per_cta - 1) / L.per_cta, max_ctas);
    PGS_LAUNCH(L.kernel, grid, L.threads, L.dyn, st, P);
}

// k_get over the runs R: P's runs and key rows; PGS_NOT_SUPPORTED when the key rows do not fit the device's shared memory
inline int32_t get_plan(GetParams &P, const ReadRunSet &R, uint32_t max_smem_optin, ReadLaunch<GetParams> &L)
{
    const ReadGeometry geo = get_geometry(R.KS);
    if (geo.dyn > max_smem_optin) return PGS_NOT_SUPPORTED;
    P.rr = R.rr;
    geo.apply(P);
    L = {R.multi ? k_get<8, true> : k_get<8, false>, kReadThreads, geo.dyn, kReadThreads / geo.G};
    return PGS_OK;
}

// the initial content of a launch buffer: src_bytes copied from the host, or every byte set to fill, or none
struct ReadInit {
    const void *src = nullptr;
    uint64_t src_bytes = 0;
    int fill = kNoFill;
};
constexpr ReadInit kZero{nullptr, 0, 0};

// the buffers of a multi-partition launch: its packed runs, their slot bounds, and the slot of each of its n requests
template <class F>
inline void multi_buffers(const ReadRunSet &R, const RunDev *&runs, const uint32_t *&begin, const uint32_t *&part, const uint32_t *req_part,
                          uint64_t n, F &&buf)
{
    if (!R.multi) return;
    buf(runs, sizeof(RunDev) * R.packed.size(), ReadInit{R.packed.data(), sizeof(RunDev) * R.packed.size()});
    buf(begin, 4 * R.begin.size(), ReadInit{R.begin.data(), 4 * R.begin.size()});
    buf(part, 4 * n, ReadInit{req_part, 4 * n});
}

// Every device buffer of a k_get launch (P.n set): buf(pointer, bytes, init) allocates the bytes and gives them their content.
// The keys and the arena carry 16 bytes of slack; error[0] is the launch's status and error[1] its ticket counter.
// pgs_get_result::value_off is 32-bit: a call uses at most the first 4 GiB - 1 of the arena.  A value that would end beyond
// that gets PGS_INCOMPLETE like any value that does not fit, and arena_cursor[0] still reports the whole need.
template <class F>
inline void get_buffers(GetParams &P, const ReadRunSet &R, const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part,
                        uint64_t arena_cap, F &&buf)
{
    const uint64_t n = P.n;
    P.arena_cap = std::min<uint64_t>(arena_cap, UINT32_MAX);
    buf(P.keys, key_off[n] + 16, ReadInit{keys, key_off[n]});
    buf(P.key_off, 4 * (n + 1), ReadInit{key_off, 4 * (n + 1)});
    buf(P.results, sizeof(pgs_get_result) * n, ReadInit{});
    buf(P.arena, P.arena_cap + 16, ReadInit{});
    buf(P.arena_cursor, 32, kZero);
    buf(P.error, 16, kZero);
    P.ticket = P.error + 1;
    multi_buffers(R, P.multi_runs, P.multi_begin, P.key_part, key_part, n, buf);
}

// Every device buffer of a scan launch of the batch B (P.n and P.KS set), as get_buffers: the requests, and per request an
// output slice of arena_stride bytes, kv_stride records and a resume slot (scan_output_strides), each array with 16 bytes of
// slack.  Returns false when the resume slots are too short to report resume keys.
template <class F>
inline bool scan_buffers(ScanParams &P, const ReadRunSet &R, const ScanBatch &B, const uint32_t *req_part, unsigned long long arena_stride,
                         uint32_t kv_stride, uint32_t resume_stride, F &&buf)
{
    const uint64_t n = P.n;
    const bool report_resume = scan_output_strides(P, arena_stride, kv_stride, resume_stride);
    buf(P.reqs, sizeof(ScanReqDev) * n, ReadInit{B.reqs.data(), sizeof(ScanReqDev) * n});
    buf(P.blob, B.blob.size(), ReadInit{B.blob.data(), B.blob.size()});
    buf(P.arena, P.arena_stride * n + 16, ReadInit{});
    buf(P.kvs, sizeof(pgs_kv) * P.kv_stride * n + 16, ReadInit{});
    buf(P.resume, (uint64_t)P.resume_stride * n + 16, ReadInit{});
    buf(P.results, sizeof(pgs_scan_result) * n, ReadInit{});
    buf(P.error, 16, kZero);
    P.ticket = P.error + 1;
    multi_buffers(R, P.multi_runs, P.multi_begin, P.req_part, req_part, n, buf);
    return report_resume;
}

// ---- the packed read-back of a scan batch of n > 1 requests (the library and the simulator) -------------------------------------
// k_pack_offsets places request i's output at arena_base[i] of one packed arena, with arena_base[i + 1] - arena_base[i] = its
// arena_used rounded up to 16, and its kvs at kv_base[i], the exclusive prefix of n_kvs.  The caller reads the totals
// arena_base[n] and kv_base[n]; when they fit its arena and kv array, k_pack_copy copies every slice to its place, so that one copy
// each brings the whole batch back.  The bytes between a request's output and the next 16-byte boundary are left unspecified.
__global__ void __launch_bounds__(1024) k_pack_offsets(const pgs_scan_result *__restrict__ res, uint32_t n, unsigned long long *__restrict__ abase,
                                                      uint32_t *__restrict__ kbase)
{
    auto add = [&](uint32_t i, unsigned long long (&v)[2]) { v[0] += (res[i].arena_used + 15) & ~15ull; v[1] += res[i].n_kvs; };
    uint32_t q0, q1;
    unsigned long long pre[2], tot[2];
    cta_excl_scan<2>(n, add, q0, q1, pre, tot);
    for (uint32_t i = q0; i < q1; i++) {
        abase[i] = pre[0];
        kbase[i] = (uint32_t)pre[1];
        add(i, pre);
    }
    if (threadIdx.x == 0) { abase[n] = tot[0]; kbase[n] = (uint32_t)tot[1]; }
}
__global__ void k_pack_copy(const pgs_scan_result *__restrict__ res, uint32_t n, const uint8_t *__restrict__ arena,
                            unsigned long long arena_stride, const pgs_kv *__restrict__ kvs, uint32_t kv_stride,
                            const unsigned long long *__restrict__ abase, const uint32_t *__restrict__ kbase,
                            uint8_t *__restrict__ parena, pgs_kv *__restrict__ pkvs)
{
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        uint32_t chunks = (uint32_t)((res[i].arena_used + 15) >> 4);
        const uint4 *src = (const uint4 *)(arena + (size_t)i * arena_stride);
        uint4 *dst = (uint4 *)(parena + abase[i]);
        for (uint32_t c = threadIdx.x; c < chunks; c += blockDim.x) dst[c] = src[c];
        for (uint32_t k = threadIdx.x; k < res[i].n_kvs; k += blockDim.x) pkvs[kbase[i] + k] = kvs[(size_t)i * kv_stride + k];
    }
}

// the buffers of a packed read-back, each allocated by the launch that writes it
struct ScanPack {
    unsigned long long *arena_base = nullptr; // n + 1 entries
    uint32_t *kv_base = nullptr;              // n + 1 entries
    uint8_t *arena = nullptr;                 // arena_base[n] bytes + 16 of slack
    pgs_kv *kvs = nullptr;                    // kv_base[n] + 1 records
};
// the offsets of the launched batch P, on one CTA; buf as for scan_buffers
template <class F>
inline void pack_offsets_launch(const ScanParams &P, ScanPack &K, cudaStream_t st, F &&buf)
{
    buf(K.arena_base, sizeof(unsigned long long) * (P.n + 1ull), ReadInit{});
    buf(K.kv_base, sizeof(uint32_t) * (P.n + 1ull), ReadInit{});
    if (!K.arena_base || !K.kv_base) return; // an allocation failed: the caller reports its allocator's status
    PGS_LAUNCH(k_pack_offsets, 1, 1024, 0, st, (const pgs_scan_result *)P.results, P.n, K.arena_base, K.kv_base);
}
// the packed arena and kvs of P (arena_bytes = arena_base[n], n_kvs = kv_base[n]), one request per CTA on at most max_ctas CTAs
template <class F>
inline void pack_copy_launch(const ScanParams &P, ScanPack &K, uint64_t arena_bytes, uint64_t n_kvs, uint32_t max_ctas, cudaStream_t st, F &&buf)
{
    buf(K.arena, arena_bytes + 16, ReadInit{});
    buf(K.kvs, sizeof(pgs_kv) * (n_kvs + 1), ReadInit{});
    if (!K.arena || !K.kvs) return;
    PGS_LAUNCH(k_pack_copy, std::min(P.n, max_ctas), 128, 0, st, (const pgs_scan_result *)P.results, P.n,
               (const uint8_t *)P.arena, P.arena_stride, (const pgs_kv *)P.kvs, P.kv_stride, (const unsigned long long *)K.arena_base,
               (const uint32_t *)K.kv_base, K.arena, K.kvs);
}

} // namespace pgs
