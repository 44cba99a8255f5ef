// index_kernel.cuh — the block index and Bloom filter of a run, built on the device when the run is uploaded or built
// (engine.cu).  Also compiled by the host SIMT interpreter (tools/simt/sim_compact.cpp), so that the CPU suite reads runs through
// the index and filter this kernel builds, planned and launched as the library does.
//
// index build: one warp walks one block (entries are sequential inside a restart interval and the last key needs every
// delta before it), the running internal key lives in a per-warp shared-memory scratch.  Two passes:
//   k_index_walk<false>  records and last-user-key length per block, run statistics, number of Bloom prefix entries
//   (host)               index_buffers: prefix sums over the blocks -> blk_rec, ikey_off
//   k_index_walk<true>   index keys, entry offsets, Bloom filter (sized bloom_lines_for(n_records + n_prefix))
#pragma once
#include "group.cuh"

namespace pgs {

struct IndexStats {
    unsigned long long n_records, n_tomb, raw_key, raw_val, min_seq, max_seq, n_prefix;
    uint32_t max_ukey, max_vlen, max_blk_rec, error;
};
constexpr uint32_t kIdxWarps = 8;
constexpr uint32_t kIdxScratch = kMaxUkeyLen + 16;

template <bool kEmitKey>
__global__ void __launch_bounds__(kIdxWarps * 32)
k_index_walk(const uint8_t *__restrict__ data, const uint64_t *__restrict__ blk_off,
             const uint32_t *__restrict__ blk_size, uint32_t nb, uint32_t *__restrict__ nrec_out,
             uint32_t *__restrict__ lastlen_out, const uint32_t *__restrict__ ikey_off,
             uint8_t *__restrict__ ikeys, const uint32_t *__restrict__ blk_rec, uint32_t *__restrict__ rec_off,
             uint32_t *__restrict__ bloom, uint32_t bloom_lines, IndexStats *__restrict__ stats, uint32_t b_begin)
{
    const Grp<32> g;
    PGS_SMEM_DYN(smem);
    uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t b = b_begin + blockIdx.x * kIdxWarps + warp; // blocks [b_begin, nb)
    if (b >= nb) return;
    uint8_t *scr = smem + warp * kIdxScratch;
    const uint8_t *base = data + blk_off[b];
    uint32_t size = blk_size[b];
    uint32_t err = 0;
    uint32_t nr = 0;
    if (size < 8) err = PGS_CORRUPTION;
    if (!err) {
        const uint8_t *t = base + size - 4;
        nr = t[0] | (t[1] << 8) | (t[2] << 16) | ((uint32_t)t[3] << 24);
        if (nr == 0 || (uint64_t)nr * 4 + 4 > size) err = PGS_CORRUPTION;
    }
    uint32_t limit = err ? 0 : size - 4 - 4 * nr;
    uint32_t p = 0, prev_klen = 0, nrec = 0;
    unsigned long long raw_key = 0, raw_val = 0, n_tomb = 0, min_seq = ~0ull, max_seq = 0;
    uint32_t max_ukey = 0, max_vlen = 0, n_prefix = 0, prev_pl = 0xFFFFFFFFu;
    while (!err && p < limit) {
        uint32_t shared, non_shared, vlen, h = 0, c;
        c = get_varint32(base + p, limit - p, shared);
        h += c;
        if (c) { c = get_varint32(base + p + h, limit - p - h, non_shared); h += c; }
        if (c) { c = get_varint32(base + p + h, limit - p - h, vlen); h += c; }
        if (!c) { err = PGS_CORRUPTION; break; }
        uint32_t klen = shared + non_shared;
        if (shared > prev_klen || klen < 8 || (uint64_t)p + h + non_shared + vlen > limit) { err = PGS_CORRUPTION; break; }
        if (klen > kMaxUkeyLen + 8) { err = PGS_NOT_SUPPORTED; break; }
        for (uint32_t i = lane; i < non_shared; i += 32) scr[shared + i] = base[p + h + i];
        if (kEmitKey && lane == 0) rec_off[blk_rec[b] + nrec] = p;
        __syncwarp();
        { // Bloom entries: the whole user key, and its hash-key prefix whenever that differs from the previous entry's
            const uint32_t ulen = klen - 8;
            const uint32_t pl = hashkey_prefix_len(scr, ulen);
            const bool new_prefix = pl != 0 && (pl != prev_pl || shared < pl);
            prev_pl = pl;
            if (kEmitKey) {
                if (bloom_lines) {
                    const unsigned long long hk = bloom_hash_row(g, (const uint32_t *)scr, ulen);
                    if (lane < 6) bloom_add_bit(bloom, bloom_lines, hk, lane);
                    if (new_prefix) {
                        const unsigned long long hp = bloom_hash_row(g, (const uint32_t *)scr, pl);
                        if (lane < 6) bloom_add_bit(bloom, bloom_lines, hp, lane);
                    }
                }
            } else if (new_prefix) n_prefix++;
        }
        if (!kEmitKey && lane == 0) {
            unsigned long long tr = 0;
            for (int i = 7; i >= 0; i--) tr = (tr << 8) | scr[klen - 8 + i];
            unsigned long long seq = tr >> 8;
            n_tomb += ((uint8_t)tr == PGS_TYPE_DELETION);
            min_seq = seq < min_seq ? seq : min_seq;
            max_seq = seq > max_seq ? seq : max_seq;
            raw_key += klen - 8;
            raw_val += vlen;
            max_ukey = max(max_ukey, klen - 8);
            max_vlen = max(max_vlen, vlen);
        }
        __syncwarp();
        nrec++;
        prev_klen = klen;
        p += h + non_shared + vlen;
    }
    if (!err && nrec == 0) err = PGS_CORRUPTION;
    if (kEmitKey) {
        if (!err) {
            uint32_t ulen = prev_klen - 8;
            uint8_t *dst = ikeys + ikey_off[b];
            for (uint32_t i = lane; i < ulen; i += 32) dst[i] = scr[i];
        }
    } else if (lane == 0) {
        nrec_out[b] = nrec;
        lastlen_out[b] = err ? 0 : prev_klen - 8;
        atomicAdd(&stats->n_records, (unsigned long long)nrec);
        atomicAdd(&stats->n_tomb, n_tomb);
        atomicAdd(&stats->raw_key, raw_key);
        atomicAdd(&stats->raw_val, raw_val);
        atomicAdd(&stats->n_prefix, (unsigned long long)n_prefix);
        atomicMin(&stats->min_seq, min_seq);
        atomicMax(&stats->max_seq, max_seq);
        atomicMax(&stats->max_ukey, max_ukey);
        atomicMax(&stats->max_vlen, max_vlen);
        atomicMax(&stats->max_blk_rec, nrec);
    }
    if (err && lane == 0) atomicMax(&stats->error, err);
}

// host, before anything is copied: the handle rule of pgs_run_upload.  Every block starts on a multiple of kBlockAlign, at or
// behind the end of the block before it, and ends inside the caller's data_bytes; gaps between blocks and bytes behind the last
// one are allowed.  Returns nb, or the index of the first handle that breaks the rule; end = the end of the last block and
// max_blk = the largest block size (of the handles in front of a bad one).
inline uint32_t run_handles_check(const uint64_t *blk_off, const uint32_t *blk_size, uint32_t nb, uint64_t data_bytes, uint64_t &end,
                                  uint32_t &max_blk)
{
    end = 0;
    max_blk = 0;
    for (uint32_t b = 0; b < nb; b++) {
        // (no sum of offset and size on the left: an offset near 2^64 must not wrap into range)
        if (blk_off[b] % kBlockAlign || blk_off[b] < end || blk_off[b] > data_bytes || blk_size[b] > data_bytes - blk_off[b]) return b;
        end = blk_off[b] + blk_size[b];
        max_blk = blk_size[b] > max_blk ? blk_size[b] : max_blk;
    }
    return nb;
}

// ---- plan, buffers, launches: shared by the upload and the run build (engine.cu) and the simulator (tools/simt/sim_compact.cpp)
// index_scratch, pass 1 (once, or once per chunk of blocks), its results on the host, index_buffers, pass 2.
struct IndexParams {
    // the run's blocks: blk_off[nb + 1] (the last one the 16-aligned end of the blocks), blk_size[nb]
    const uint8_t *data;
    const uint64_t *blk_off;
    const uint32_t *blk_size;
    uint32_t nb;
    // pass-1 scratch (index_scratch): records and last-user-key length per block, the run's statistics (index_stats_init)
    uint32_t *nrec, *lastlen;
    IndexStats *stats;
    // the index (index_buffers): blk_rec / ikey_off [nb + 1], the index keys, the entry offsets, the Bloom filter
    uint32_t *blk_rec, *ikey_off;
    uint8_t *ikeys;
    uint32_t *rec_off, *bloom;
    uint32_t bloom_lines;
};

inline IndexStats index_stats_init() { return IndexStats{0, 0, 0, 0, ~0ull, 0, 0, 0, 0, 0, 0}; } // min_seq = ~0

// pass 1's scratch through alloc(p, count, fill) (fill = a byte value or kNoFill); the caller sets *X.stats = index_stats_init()
template <class Alloc>
void index_scratch(IndexParams &X, Alloc &&alloc)
{
    alloc(X.nrec, X.nb, kNoFill);
    alloc(X.lastlen, X.nb, kNoFill);
    alloc(X.stats, 1, kNoFill);
}

// pass 1 over the blocks [b0, b1); returns the launches
inline uint32_t index_launch_pass1(const IndexParams &X, uint32_t b0, uint32_t b1, cudaStream_t st)
{
    if (b1 <= b0) return 0;
    PGS_LAUNCH(k_index_walk<false>, (b1 - b0 + kIdxWarps - 1) / kIdxWarps, kIdxWarps * 32, kIdxWarps * kIdxScratch, st, X.data, X.blk_off,
               X.blk_size, b1, X.nrec, X.lastlen, nullptr, nullptr, nullptr, nullptr, nullptr, 0u, X.stats, b0);
    return 1;
}

// Between the passes, with pass 1's nrec / lastlen [nb] and stats st on the host: the index layout into the host arrays rec_cum /
// key_cum [nb + 1], the exclusive prefix sums of the records and of the last-user-key lengths (the first record and the index
// key of every block; the caller copies them to X.blk_rec / X.ikey_off), and the run r's index buffers through alloc(p, count,
// fill), X pointed at them.  Returns the walks' verdict, or kNotSupported beyond the index's 32-bit offsets.
template <class RunT, class Alloc>
int32_t index_buffers(IndexParams &X, RunT &r, const uint32_t *nrec, const uint32_t *lastlen, const IndexStats &st, uint32_t *rec_cum,
                      uint32_t *key_cum, Alloc &&alloc)
{
    const uint32_t nb = X.nb;
    if (st.error) {
        set_error("run upload: block scan failed with status %u", st.error);
        return (int32_t)st.error;
    }
    uint64_t rc = 0, kc = 0;
    for (uint32_t b = 0; b < nb; b++) {
        rec_cum[b] = (uint32_t)rc;
        key_cum[b] = (uint32_t)kc;
        rc += nrec[b];
        kc += lastlen[b];
    }
    if (rc > 0xFFFFFFF0ull || kc > 0xFFFFFFF0ull) {
        set_error("run too large for 32-bit record / index-key offsets");
        return PGS_NOT_SUPPORTED;
    }
    rec_cum[nb] = (uint32_t)rc;
    key_cum[nb] = (uint32_t)kc;
    alloc(r.d_blk_rec, nb + 1ull, kNoFill);
    alloc(r.d_ikey_off, nb + 1ull, kNoFill);
    alloc(r.d_ikeys, key_cum[nb] + 16ull, kNoFill);
    alloc(r.d_rec_off, rec_cum[nb] + 1ull, kNoFill);
    r.n_bloom_entries = st.n_records + st.n_prefix;
    r.bloom_lines = bloom_lines_for(r.n_bloom_entries);
    alloc(r.d_bloom, r.bloom_lines * 16ull, 0);
    X.blk_rec = r.d_blk_rec, X.ikey_off = r.d_ikey_off, X.ikeys = r.d_ikeys;
    X.rec_off = r.d_rec_off, X.bloom = r.d_bloom, X.bloom_lines = r.bloom_lines;
    return PGS_OK;
}

// pass 2 over every block; returns the launches
inline uint32_t index_launch_pass2(const IndexParams &X, cudaStream_t st)
{
    if (!X.nb) return 0;
    PGS_LAUNCH(k_index_walk<true>, (X.nb + kIdxWarps - 1) / kIdxWarps, kIdxWarps * 32, kIdxWarps * kIdxScratch, st, X.data, X.blk_off,
               X.blk_size, X.nb, nullptr, nullptr, X.ikey_off, X.ikeys, X.blk_rec, X.rec_off, X.bloom, X.bloom_lines, X.stats, 0u);
    return 1;
}

// host, after the second pass: the run's pgs_run_info from the index statistics, the block count, the 16-aligned end of its
// blocks and its largest block (level and run id are the caller's)
inline void run_info_from_index(const IndexStats &st, uint32_t n_blocks, uint64_t data_bytes, uint32_t max_blk, pgs_run_info &info)
{
    info.n_blocks = n_blocks;
    info.data_bytes = data_bytes;
    info.n_records = st.n_records;
    info.n_tombstones = st.n_tomb;
    info.raw_key_bytes = st.raw_key;
    info.raw_value_bytes = st.raw_val;
    info.max_ukey_len = st.max_ukey;
    info.max_value_len = st.max_vlen;
    info.max_block_size = max_blk;
    info.max_block_records = st.max_blk_rec;
    info.smallest_seq = st.min_seq;
    info.largest_seq = st.max_seq;
}

} // namespace pgs
