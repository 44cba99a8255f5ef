// device_util.cuh — device-side primitives shared by the sm_90a kernels: TMA bulk copies and
// mbarriers (inline PTX), varint decode, byte-string compares, warp/block scans, misaligned
// warp copies.
#pragma once
#ifndef PGS_SIM
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "format.h"

// PGS_SIM: the same sources compiled by g++ against tools/simt/simt.h (a host-side SIMT interpreter used by the CPU tests
// of the kernels' logic); inline PTX is replaced by synchronous equivalents there.
#ifndef PGS_SIM
#define PGS_SMEM_DYN(name) extern __shared__ __align__(128) uint8_t name[]
#define PGS_SMEM_STATIC(decl) __shared__ decl
#define PGS_LAUNCH(kernel, grid, block, dyn, stream, ...) kernel<<<(grid), (block), (dyn), (stream)>>>(__VA_ARGS__)
#endif

namespace pgs {

#define PGS_DEV __device__ __forceinline__

constexpr uint32_t kWarp = 32;
constexpr uint32_t kFull = 0xffffffffu;
constexpr int kNoFill = -1; // a launch buffer the host leaves unset (compact_buffers, get_buffers, scan_buffers)
// the initial content of a launch buffer: src_bytes copied from the host, or every byte set to fill, or none
struct ReadInit {
    const void *src = nullptr;
    uint64_t src_bytes = 0;
    int fill = kNoFill;
};
constexpr ReadInit kZero{nullptr, 0, 0};
void set_error(const char *fmt, ...); // the message of a refused call (engine.cu; the simulator prints it)

// the job whose range [base[j], base[j + 1]) holds x (base[0] = 0 <= x < base[n]; empty ranges are skipped)
PGS_HD uint32_t job_of(const uint32_t *base, uint32_t n, uint32_t x)
{
    uint32_t lo = 0, hi = n; // base[lo] <= x < base[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (base[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// ---- shared-memory addressing / mbarrier / TMA bulk (cp.async.bulk) ----------------------------
#ifdef PGS_SIM
// The stand-ins check what the device would fault on or hang at: a bulk copy's addresses and size, and an mbarrier whose
// expected bytes differ from the bytes its copies completed.  The barrier word holds the bytes expected and not yet arrived.
#define PGS_SIM_CHECK(cond, ...) do { if (!(cond)) { fprintf(stderr, "sim: " __VA_ARGS__); fputc('\n', stderr); abort(); } } while (0)
PGS_DEV void sim_check_bulk(const void *smem, const void *gmem, uint32_t bytes)
{
    PGS_SIM_CHECK(!((uintptr_t)smem & 15) && !((uintptr_t)gmem & 15) && !(bytes & 15) && bytes,
                  "bulk copy of %u bytes between %p (shared) and %p (global): addresses must be 16-aligned, the size a multiple of 16",
                  bytes, smem, gmem);
}
PGS_DEV void mbar_init(uint64_t *bar, uint32_t) { *bar = 0; }
PGS_DEV void mbar_fence_init() {}
PGS_DEV void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { *bar += bytes; }
PGS_DEV void mbar_wait(uint64_t *bar, uint32_t)
{
    PGS_SIM_CHECK(*bar == 0, "mbarrier wait with %lld expected bytes that no copy delivers", (long long)*bar);
}
PGS_DEV bool mbar_try_wait(uint64_t *bar, uint32_t parity) { mbar_wait(bar, parity); return true; }
PGS_DEV void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    sim_check_bulk(smem_dst, gmem_src, bytes);
    PGS_SIM_CHECK((int64_t)(*bar - bytes) >= 0, "bulk copy of %u bytes completes on an mbarrier that expects %lld: expect_tx comes first",
                  bytes, (long long)*bar);
    memcpy(smem_dst, gmem_src, bytes);
    *bar -= bytes;
}
PGS_DEV void tma_store_1d(void *gmem_dst, const void *smem_src, uint32_t bytes)
{
    sim_check_bulk(smem_src, gmem_dst, bytes);
    memcpy(gmem_dst, smem_src, bytes);
}
PGS_DEV void tma_store_commit() {}
PGS_DEV void tma_store_wait_read0() {}
PGS_DEV void tma_store_wait_all() {}
PGS_DEV void fence_proxy_async() {}
PGS_DEV void async_copy4(void *smem_dst, const void *gmem_src) { memcpy(smem_dst, gmem_src, 4); }
PGS_DEV void async_copy16(void *smem_dst, const void *gmem_src) { memcpy(smem_dst, gmem_src, 16); }
PGS_DEV void async_copy_wait_upto(uint32_t) {}
PGS_DEV void async_copy_commit() {}
PGS_DEV void async_copy_wait_all() {}
#else
PGS_DEV uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

PGS_DEV void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
PGS_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
PGS_DEV void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
PGS_DEV bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
PGS_DEV void mbar_wait(uint64_t *bar, uint32_t parity)
{
    while (!mbar_try_wait(bar, parity)) {
    }
}
// global -> shared bulk copy through the TMA unit; bytes % 16 == 0, both addresses 16-aligned
PGS_DEV void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// shared -> global bulk copy through the TMA unit (bulk async-group completion); bytes % 16 == 0, both addresses 16-aligned
PGS_DEV void tma_store_1d(void *gmem_dst, const void *smem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
PGS_DEV void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the source bytes of all but the newest N committed bulk groups have been read (their shared memory may be rewritten)
PGS_DEV void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
PGS_DEV void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy writes to shared memory become visible to the async proxy (TMA) that reads them next
PGS_DEV void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// small asynchronous global -> shared copies (LDGSTS): the issuing thread does not wait for the data
PGS_DEV void async_copy4(void *smem_dst, const void *gmem_src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// 16 bytes, both addresses 16-aligned, past L1 (streamed data)
PGS_DEV void async_copy16(void *smem_dst, const void *gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
PGS_DEV void async_copy_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most n (0..3) of this thread's newest committed groups are still in flight
PGS_DEV void async_copy_wait_upto(uint32_t n)
{
    if (n == 0) asm volatile("cp.async.wait_group 0;" ::: "memory");
    else if (n == 1) asm volatile("cp.async.wait_group 1;" ::: "memory");
    else if (n == 2) asm volatile("cp.async.wait_group 2;" ::: "memory");
    else asm volatile("cp.async.wait_group 3;" ::: "memory");
}
PGS_DEV void async_copy_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
#endif

// ---- varint (RocksDB util/coding.h encoding) ---------------------------------------------------
// returns bytes consumed, 0 on malformed / out of range
PGS_DEV uint32_t get_varint32(const uint8_t *p, uint32_t avail, uint32_t &v)
{
    uint32_t r = 0;
#pragma unroll
    for (uint32_t i = 0; i < 5; i++) {
        if (i >= avail) return 0;
        uint32_t b = p[i];
        r |= (b & 127u) << (7 * i);
        if (!(b & 128u)) { v = r; return i + 1; }
    }
    return 0;
}
PGS_DEV uint32_t put_varint32_s(uint8_t *p, uint32_t v) // shared-memory / generic byte stores; returns bytes written
{
    uint32_t n = 0;
    while (v >= 128u) { p[n++] = (uint8_t)(v | 128u); v >>= 7; }
    p[n++] = (uint8_t)v;
    return n;
}

// ---- byte-string compare -------------------------------------------------------------------------
// generic pointers, any alignment; returns <0, 0, >0 like memcmp-then-length
PGS_DEV int cmp_bytes(const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb)
{
    uint32_t m = la < lb ? la : lb;
    for (uint32_t i = 0; i < m; i++) {
        int d = (int)a[i] - (int)b[i];
        if (d) return d;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}
// 4 bytes at an arbitrary address of any address space: two aligned 32-bit loads + funnel shift.  Touches at most 3
// bytes before p and 3 bytes past p+3 inside the same aligned words (buffers carry >= 16 bytes of slack).
PGS_DEV uint32_t ld_u32_any(const uint8_t *p)
{
    const uint32_t *w = (const uint32_t *)((uintptr_t)p & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)((uintptr_t)p & 3) * 8;
    return sh ? __funnelshift_r(w[0], w[1], sh) : w[0];
}
// cmp_bytes, four bytes per step (the byte loop pays one dependent load per byte when the strings live in global memory)
PGS_DEV int cmp_bytes4(const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb)
{
    const uint32_t m = la < lb ? la : lb;
    for (uint32_t i = 0; i < m; i += 4) {
        uint32_t x = ld_u32_any(a + i), y = ld_u32_any(b + i);
        const uint32_t left = m - i;
        if (left < 4) { const uint32_t msk = (1u << (8 * left)) - 1u; x &= msk; y &= msk; }
        if (x != y) {
            x = __byte_perm(x, 0, 0x0123); // first byte most significant
            y = __byte_perm(y, 0, 0x0123);
            return x < y ? -1 : 1;
        }
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}
// does v match a NON-EMPTY pattern: anywhere in it, as its prefix or as its postfix (match_type: MATCH_* of format.h; any other
// type never matches).  What an empty pattern means is the caller's rule.
PGS_DEV bool pattern_match(uint32_t match_type, const uint8_t *pat, uint32_t pl, const uint8_t *v, uint32_t vl)
{
    if (vl < pl) return false;
    if (match_type == MATCH_PREFIX) {
        for (uint32_t i = 0; i < pl; i++) if (v[i] != pat[i]) return false;
        return true;
    }
    if (match_type == MATCH_POSTFIX) {
        const uint8_t *s = v + vl - pl;
        for (uint32_t i = 0; i < pl; i++) if (s[i] != pat[i]) return false;
        return true;
    }
    if (match_type == MATCH_ANYWHERE) {
        for (uint32_t s = 0; s + pl <= vl; s++) {
            uint32_t i = 0;
            while (i < pl && v[s + i] == pat[i]) i++;
            if (i == pl) return true;
        }
    }
    return false;
}
PGS_DEV uint64_t bswap64(uint64_t x)
{
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}
// both keys live in 8-byte aligned slots that are zero padded up to a multiple of 8:
// word-wise big-endian compare + length tie-break == bytewise lexicographic compare
PGS_DEV int cmp_slots(const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb)
{
    uint32_t m = la < lb ? la : lb;
    uint32_t words = (m + 7) >> 3;
    const uint64_t *wa = (const uint64_t *)a, *wb = (const uint64_t *)b;
    for (uint32_t i = 0; i < words; i++) {
        uint64_t x = wa[i], y = wb[i];
        if (x != y) {
            x = bswap64(x);
            y = bswap64(y);
            return x < y ? -1 : 1;
        }
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}
// same compare, skipping the first `start` 8-byte words (known equal); *diff = index of the first differing word
// (or the number of compared words when one key is a prefix of the other).  Lets a binary search over sorted
// keys skip the prefix shared with both bounds (LCP-aware search).
PGS_DEV int cmp_slots_from(const uint8_t *a, uint32_t la, const uint8_t *b, uint32_t lb, uint32_t start, uint32_t *diff)
{
    uint32_t m = la < lb ? la : lb;
    uint32_t words = (m + 7) >> 3;
    const uint64_t *wa = (const uint64_t *)a, *wb = (const uint64_t *)b;
    for (uint32_t i = start; i < words; i++) {
        uint64_t x = wa[i], y = wb[i];
        if (x != y) {
            *diff = i;
            x = bswap64(x);
            y = bswap64(y);
            return x < y ? -1 : 1;
        }
    }
    *diff = words;
    return la < lb ? -1 : (la > lb ? 1 : 0);
}
// 8 bytes at an arbitrary shared-memory address, addressed as (4-byte aligned base, byte offset): three aligned 32-bit loads +
// funnel shifts.  Plain pointer arithmetic, so the compiler keeps the loads in the shared address space (a uintptr_t round trip
// turns them into generic loads)
PGS_DEV uint64_t lds_u64_at(const uint8_t *base4, uint32_t off)
{
    const uint32_t *w = (const uint32_t *)base4 + (off >> 2);
    uint32_t sh = (off & 3) * 8;
    uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
    return ((uint64_t)hi << 32) | lo;
}
// three varint32 (shared, non_shared, value_len) out of the 8 header bytes in x; returns the header length, or 0
// when the common shape (shared < 128, non_shared < 128, value_len < 2^21) does not apply and the caller must use
// the byte-wise decoder
PGS_DEV uint32_t parse_header8(uint64_t x, uint32_t &a, uint32_t &b, uint32_t &c)
{
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    if (lo & 0x00008080u) return 0; // a multi-byte shared / non_shared length
    a = lo & 0x7fu;
    b = (lo >> 8) & 0x7fu;
    uint32_t b2 = (lo >> 16) & 0xffu, b3 = lo >> 24, b4 = hi & 0xffu;
    if (!(b2 & 0x80u)) { c = b2; return 3; }
    if (!(b3 & 0x80u)) { c = (b2 & 0x7fu) | (b3 << 7); return 4; }
    if (!(b4 & 0x80u)) { c = (b2 & 0x7fu) | ((b3 & 0x7fu) << 7) | (b4 << 14); return 5; }
    return 0;
}

// ---- scans -----------------------------------------------------------------------------------------
PGS_DEV uint32_t warp_incl_scan(uint32_t v, uint32_t lane)
{
#pragma unroll
    for (uint32_t d = 1; d < 32; d <<= 1) {
        uint32_t n = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += n;
    }
    return v;
}
// exclusive scan of one value per thread over the whole CTA (blockDim.x <= 1024, multiple of 32).
// `scratch` = 33 uint32 in shared memory.  Returns the exclusive prefix, *total = sum.
PGS_DEV uint32_t block_excl_scan(uint32_t v, uint32_t *scratch, uint32_t *total)
{
    uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t inc = warp_incl_scan(v, lane);
    __syncthreads(); // scratch may still be read from a previous call
    if (lane == 31) scratch[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nw ? scratch[lane] : 0;
        uint32_t ws = warp_incl_scan(w, lane);
        scratch[lane] = ws - w;
        if (lane == 31) scratch[32] = ws;
    }
    __syncthreads();
    *total = scratch[32];
    return scratch[warp] + inc - v;
}
// exclusive scan of N u64 fields over n items in ONE CTA (blockDim.x <= 1024, a multiple of 32).  Thread t owns the contiguous
// items [q0, q1) (returned); add(q, v) adds the fields of item q to v.  pre = the sums over the items before q0, tot = the sums
// over all n items.
template <uint32_t N, class Add>
PGS_DEV void cta_excl_scan(uint32_t n, Add add, uint32_t &q0, uint32_t &q1, unsigned long long (&pre)[N], unsigned long long (&tot)[N])
{
    PGS_SMEM_STATIC(unsigned long long s_w[N][33]);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x;
    q0 = min(tid * per, n);
    q1 = min(q0 + per, n);
    unsigned long long loc[N], inc[N];
#pragma unroll
    for (uint32_t x = 0; x < N; x++) loc[x] = 0;
    for (uint32_t q = q0; q < q1; q++) add(q, loc);
#pragma unroll
    for (uint32_t x = 0; x < N; x++) {
        inc[x] = loc[x];
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const unsigned long long o = __shfl_up_sync(kFull, inc[x], d);
            if (lane >= d) inc[x] += o;
        }
        if (lane == 31) s_w[x][warp] = inc[x];
    }
    __syncthreads();
#pragma unroll
    for (uint32_t x = 0; x < N; x++) {
        const unsigned long long w = lane < nw ? s_w[x][lane] : 0;
        unsigned long long ws = w;
#pragma unroll
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const unsigned long long o = __shfl_up_sync(kFull, ws, d);
            if (lane >= d) ws += o;
        }
        tot[x] = __shfl_sync(kFull, ws, 31);
        pre[x] = __shfl_sync(kFull, ws - w, (int)warp) + inc[x] - loc[x];
    }
}

// ---- warp copies ------------------------------------------------------------------------------------
// byte-granular copy (any address space), all 32 lanes participate
PGS_DEV void warp_copy_bytes(uint8_t *dst, const uint8_t *src, uint32_t n, uint32_t lane)
{
    for (uint32_t i = lane; i < n; i += 32) dst[i] = src[i];
}

} // namespace pgs
