// simt.h — a small host-side SIMT interpreter for the kernels of this repo (development / CPU test tool, NOT product code).
//
// The CUDA sources under incubator_pegasus_b200/csrc are warp-synchronous code: lanes of a group exchange values
// with shuffles and ballots and never rely on hardware scheduling.  Compiled with g++ -DPGS_SIM, every CUDA thread
// becomes a ucontext fiber on ONE OS thread; a fiber runs until it reaches a collective (shuffle, ballot, __syncwarp,
// __syncthreads), where it yields until every lane named in the mask has arrived.  Global and shared memory are plain
// host memory, atomics are plain read-modify-writes (one OS thread), TMA bulk copies complete synchronously.
// That is enough to execute the kernels' control flow, address arithmetic and byte shuffling bit for bit on a machine
// without a GPU; it says nothing about timing, memory ordering or anything the hardware decides.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <functional>
#include <map>
#include <vector>

namespace simt {

struct dim3v { uint32_t x, y, z; };

struct Barrier { uint32_t count = 0, gen = 0; };

struct Fiber {
    ucontext_t ctx;
    uint8_t *stack = nullptr;
    bool done = false;
    uint32_t tid = 0;
};

struct Cta {
    uint32_t nthreads = 0, live = 0, bid = 0, grid = 0;
    std::vector<Fiber> fibers;
    std::vector<uint64_t> xchg;                       // one exchange slot per thread
    std::vector<uint32_t> site;                       // source line of the collective each thread is in (divergence check)
    std::map<uint64_t, Barrier> warp_bars;            // (warp << 32 | mask) -> barrier
    std::map<uint32_t, Barrier> named_bars;           // bar.sync id
    Barrier cta_bar;
    uint8_t *dyn = nullptr;
    size_t dyn_bytes = 0;
    ucontext_t sched;
    int cur = -1;
    uint64_t progress = 0;
};

inline Cta *&cta() { static Cta *c = nullptr; return c; }
inline std::function<void()> *&body() { static std::function<void()> *b = nullptr; return b; }

inline void yield_()
{
    Cta *c = cta();
    swapcontext(&c->fibers[c->cur].ctx, &c->sched);
}

inline void fiber_main()
{
    Cta *c = cta();
    (*body())();
    c->fibers[c->cur].done = true;
    c->live--;
    c->progress++;
    swapcontext(&c->fibers[c->cur].ctx, &c->sched);
}

inline void wait_barrier(Barrier &b, uint32_t expected)
{
    Cta *c = cta();
    const uint32_t mygen = b.gen;
    if (++b.count >= expected) { b.count = 0; b.gen++; c->progress++; return; }
    while (b.gen == mygen) yield_();
}

inline uint32_t tid_() { return cta()->fibers[cta()->cur].tid; }
inline uint32_t lane_() { return tid_() & 31; }
inline Barrier &warp_bar(uint32_t mask) { return cta()->warp_bars[((uint64_t)(tid_() >> 5) << 32) | mask]; }
inline void sync_mask(uint32_t mask)
{
    if (!(mask >> lane_() & 1)) { fprintf(stderr, "simt: lane %u calls a collective with mask %08x that does not name it\n", lane_(), mask); abort(); }
    wait_barrier(warp_bar(mask), (uint32_t)__builtin_popcount(mask));
}

// deposit a value, wait for the group, read any lane's value, wait again (nobody overwrites a slot that is still being read)
inline uint32_t &cur_site() { static uint32_t s = 0; return s; } // set by the collective macros right before the call
template <class F>
inline uint64_t exchange(uint32_t mask, uint64_t mine, F pick)
{
    Cta *c = cta();
    const uint32_t base = tid_() & ~31u, line = cur_site();
    c->xchg[tid_()] = mine;
    c->site[tid_()] = line;
    sync_mask(mask);
    // every lane named by the mask must be inside the SAME collective: a mismatch is a control-flow divergence around a
    // full-mask collective, which on the GPU is undefined behaviour (hang or garbage)
    for (uint32_t l = 0; l < 32; l++)
        if ((mask >> l & 1) && c->site[base + l] != line) {
            fprintf(stderr, "simt: divergent collective: lane %u is at source line %u, lane %u at line %u (mask %08x)\n", lane_(), line, l, c->site[base + l], mask);
            abort();
        }
    uint64_t r = pick(&c->xchg[base]);
    sync_mask(mask);
    return r;
}

inline void run_cta(Cta &c, std::function<void()> &fn, size_t stack_bytes)
{
    cta() = &c;
    body() = &fn;
    c.fibers.resize(c.nthreads);
    c.xchg.assign(c.nthreads, 0);
    c.site.assign(c.nthreads, 0);
    c.live = c.nthreads;
    for (uint32_t t = 0; t < c.nthreads; t++) {
        Fiber &f = c.fibers[t];
        f.tid = t;
        f.done = false;
        f.stack = (uint8_t *)malloc(stack_bytes);
        getcontext(&f.ctx);
        f.ctx.uc_stack.ss_sp = f.stack;
        f.ctx.uc_stack.ss_size = stack_bytes;
        f.ctx.uc_link = nullptr;
        makecontext(&f.ctx, (void (*)())fiber_main, 0);
    }
    uint64_t last_progress = ~0ull;
    uint32_t idle_rounds = 0;
    while (c.live > 0) {
        const uint64_t before = c.progress;
        for (uint32_t t = 0; t < c.nthreads; t++) {
            if (c.fibers[t].done) continue;
            c.cur = (int)t;
            swapcontext(&c.sched, &c.fibers[t].ctx);
        }
        if (c.progress == before && before == last_progress) {
            if (++idle_rounds > 1000) { fprintf(stderr, "simt: deadlock in CTA %u (%u live threads wait for lanes that never arrive)\n", c.bid, c.live); abort(); }
        } else idle_rounds = 0;
        last_progress = before;
    }
    for (auto &f : c.fibers) free(f.stack);
    c.fibers.clear();
    c.warp_bars.clear();
    c.named_bars.clear();
}

template <class K, class... A>
inline void launch(K kernel, uint32_t grid, uint32_t block, size_t dyn_bytes, A... args)
{
    std::function<void()> fn = [&]() { kernel(args...); };
    for (uint32_t b = 0; b < grid; b++) {
        Cta c;
        c.nthreads = block;
        c.bid = b;
        c.grid = grid;
        c.dyn_bytes = dyn_bytes;
        c.dyn = (uint8_t *)aligned_alloc(128, (dyn_bytes + 255) & ~(size_t)127);
        memset(c.dyn, 0xCD, dyn_bytes);
        run_cta(c, fn, 256 * 1024);
        free(c.dyn);
    }
    cta() = nullptr;
}

} // namespace simt

// ---- CUDA surface ------------------------------------------------------------------------------------------------------
#define __device__
#define __global__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __maxnreg__(...)
#define __grid_constant__
#define __restrict__
#define __align__(n) __attribute__((aligned(n)))

struct simt_idx_ { uint32_t x, y = 0, z = 0; };
#define threadIdx (simt_idx_{simt::tid_()})
#define blockIdx (simt_idx_{simt::cta()->bid})
#define blockDim (simt_idx_{simt::cta()->nthreads})
#define gridDim (simt_idx_{simt::cta()->grid})

inline void __syncthreads() { simt::wait_barrier(simt::cta()->cta_bar, simt::cta()->live); }
inline int __syncthreads_or(int pred) // every thread deposits, all meet, all read, all meet again before a slot is reused
{
    simt::Cta *c = simt::cta();
    c->xchg[simt::tid_()] = pred != 0;
    __syncthreads();
    int any = 0;
    for (uint32_t t = 0; t < c->nthreads; t++) any |= c->fibers[t].done ? 0 : (int)c->xchg[t];
    __syncthreads();
    return any;
}
inline void __syncwarp(uint32_t mask = 0xffffffffu) { simt::sync_mask(mask); }
inline void simt_named_bar(uint32_t id, uint32_t n) { simt::wait_barrier(simt::cta()->named_bars[id], n); }

template <class T>
inline T __shfl_sync(uint32_t mask, T v, int src, int width = 32)
{
    static_assert(sizeof(T) <= 8, "shfl");
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint32_t lane = simt::lane_();
    const uint32_t s = (lane & ~(uint32_t)(width - 1)) | ((uint32_t)src & (uint32_t)(width - 1));
    uint64_t r = simt::exchange(mask, raw, [&](uint64_t *w) { return w[s]; });
    T o;
    memcpy(&o, &r, sizeof(T));
    return o;
}
template <class T>
inline T __shfl_up_sync(uint32_t mask, T v, unsigned d, int width = 32)
{
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint32_t lane = simt::lane_(), seg = lane & ~(uint32_t)(width - 1);
    uint64_t r = simt::exchange(mask, raw, [&](uint64_t *w) { return (lane - seg) >= d ? w[lane - d] : w[lane]; });
    T o;
    memcpy(&o, &r, sizeof(T));
    return o;
}
template <class T>
inline T __shfl_down_sync(uint32_t mask, T v, unsigned d, int width = 32)
{
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint32_t lane = simt::lane_(), seg = lane & ~(uint32_t)(width - 1);
    uint64_t r = simt::exchange(mask, raw, [&](uint64_t *w) { return (lane - seg) + d < (uint32_t)width ? w[lane + d] : w[lane]; });
    T o;
    memcpy(&o, &r, sizeof(T));
    return o;
}
template <class T>
inline T __shfl_xor_sync(uint32_t mask, T v, int m, int width = 32)
{
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    const uint32_t lane = simt::lane_();
    (void)width;
    uint64_t r = simt::exchange(mask, raw, [&](uint64_t *w) { return w[lane ^ (uint32_t)m]; });
    T o;
    memcpy(&o, &r, sizeof(T));
    return o;
}
inline uint32_t __ballot_sync(uint32_t mask, int pred)
{
    return (uint32_t)simt::exchange(mask, pred ? 1u : 0u, [&](uint64_t *w) {
        uint32_t b = 0;
        for (uint32_t l = 0; l < 32; l++) if ((mask >> l & 1) && w[l]) b |= 1u << l;
        return (uint64_t)b;
    });
}
template <class T>
inline uint32_t __match_any_sync(uint32_t mask, T v)
{
    static_assert(sizeof(T) <= 8, "match");
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    return (uint32_t)simt::exchange(mask, raw, [&](uint64_t *w) {
        uint32_t b = 0;
        for (uint32_t l = 0; l < 32; l++) if ((mask >> l & 1) && w[l] == raw) b |= 1u << l;
        return (uint64_t)b;
    });
}
inline int __any_sync(uint32_t mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(uint32_t mask, int pred) { return __ballot_sync(mask, pred) == mask; }
inline uint32_t __activemask() { return 0xffffffffu; }
template <class F>
inline uint32_t simt_reduce(uint32_t mask, uint32_t v, F f)
{
    return (uint32_t)simt::exchange(mask, v, [&](uint64_t *w) {
        bool first = true;
        uint32_t acc = 0;
        for (uint32_t l = 0; l < 32; l++) if (mask >> l & 1) { acc = first ? (uint32_t)w[l] : f(acc, (uint32_t)w[l]); first = false; }
        return (uint64_t)acc;
    });
}
inline uint32_t __reduce_add_sync(uint32_t m, uint32_t v) { return simt_reduce(m, v, [](uint32_t a, uint32_t b) { return a + b; }); }
inline uint32_t __reduce_max_sync(uint32_t m, uint32_t v) { return simt_reduce(m, v, [](uint32_t a, uint32_t b) { return a > b ? a : b; }); }
inline uint32_t __reduce_min_sync(uint32_t m, uint32_t v) { return simt_reduce(m, v, [](uint32_t a, uint32_t b) { return a < b ? a : b; }); }
inline uint32_t __reduce_or_sync(uint32_t m, uint32_t v) { return simt_reduce(m, v, [](uint32_t a, uint32_t b) { return a | b; }); }
inline uint32_t __reduce_and_sync(uint32_t m, uint32_t v) { return simt_reduce(m, v, [](uint32_t a, uint32_t b) { return a & b; }); }

// bit tricks
inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) { s &= 31; return s ? (lo >> s) | (hi << (32 - s)) : lo; }
inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t s) { s &= 31; return s ? (hi << s) | (lo >> (32 - s)) : hi; }
inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel)
{
    uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }
inline int __popc(uint32_t x) { return __builtin_popcount(x); }
inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
inline int __clz(int x) { return x ? __builtin_clz((uint32_t)x) : 32; }
inline uint32_t __brev(uint32_t x) { uint32_t r = 0; for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i); return r; }
inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
template <class T> inline T min(T a, T b) { return a < b ? a : b; }
template <class T> inline T max(T a, T b) { return a > b ? a : b; }
inline uint32_t min(uint32_t a, int b) { return a < (uint32_t)b ? a : (uint32_t)b; }

// atomics (single OS thread: plain read-modify-write)
template <class T, class U> inline T atomicAdd(T *p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> inline T atomicMax(T *p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> inline T atomicMin(T *p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> inline T atomicOr(T *p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> inline T atomicExch(T *p, U v) { T o = *p; *p = (T)v; return o; }
template <class T> inline T atomicCAS(T *p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }

struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; } __attribute__((aligned(16)));
inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

typedef struct simt_stream_ *cudaStream_t; // launches run synchronously, in order
#define PGS_SMEM_DYN(name) uint8_t *name = simt::cta()->dyn
#define PGS_SMEM_STATIC(decl) static decl
#define PGS_LAUNCH(kernel, grid, block, dyn, stream, ...) simt::launch(kernel, (uint32_t)(grid), (uint32_t)(block), (size_t)(dyn), __VA_ARGS__)

// the collectives record their source line (see simt::exchange)
#define __shfl_sync(...) (simt::cur_site() = __LINE__, __shfl_sync(__VA_ARGS__))
#define __shfl_up_sync(...) (simt::cur_site() = __LINE__, __shfl_up_sync(__VA_ARGS__))
#define __shfl_down_sync(...) (simt::cur_site() = __LINE__, __shfl_down_sync(__VA_ARGS__))
#define __shfl_xor_sync(...) (simt::cur_site() = __LINE__, __shfl_xor_sync(__VA_ARGS__))
#define __ballot_sync(...) (simt::cur_site() = __LINE__, __ballot_sync(__VA_ARGS__))
#define __any_sync(...) (simt::cur_site() = __LINE__, __any_sync(__VA_ARGS__))
#define __match_any_sync(...) (simt::cur_site() = __LINE__, __match_any_sync(__VA_ARGS__))
#define __all_sync(...) (simt::cur_site() = __LINE__, __all_sync(__VA_ARGS__))
