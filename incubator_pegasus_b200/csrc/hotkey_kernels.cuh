// hotkey_kernels.cuh — read-side capture of the hot-key collectors for batched gets (host/hotkey.h holds the state machine).
//
//   k_hotkey_capture  launched next to k_get, only while a partition slot of the call has an active READ collector.  One
//                     lane per key: split the raw key (format.h), hash the hash key with hotkey_hash (the whole warp, as one
//                     group of 32 lanes, hashes keys longer than kHotkeyLaneBytes together), then by the slot's phase:
//                       COARSE  +1 on the key's (slot, bucket) counter, a uint64 array in HBM per partition that accumulates
//                               across launches until an analysis reads and zeroes it;
//                       FINE    a key in the target bucket takes a ticket of its slot; a ticket below the slot's queue room
//                               writes the key's index, and the host copies that many hash keys out of the caller's buffer.
//                     Lanes with the same (slot, bucket) are aggregated with __match_any_sync first, so the hot bucket of a
//                     zipfian batch costs one atomic per warp, not 32; tickets are handed out in lane order within a warp.
#pragma once
#include "device_util.cuh"

namespace pgs {

constexpr uint32_t kHotkeyThreads = 256;
constexpr uint32_t kHotkeyLaneBytes = 64; // hash keys up to this long are hashed by their own lane

// per partition slot of a launch: the phase its READ collector captures in
struct HotkeySlotDev {
    unsigned long long *buckets; // COARSE: n_buckets counters (HBM, per partition)
    uint32_t state;              // HOTKEY_STOPPED / _COARSE / _FINE of host/hotkey.h (0 / 1 / 2)
    uint32_t target;             // FINE: the target bucket
    uint32_t room;               // FINE: free places of the slot's queue
    uint32_t idx_base;           // FINE: the slot's first entry in idx
};

struct HotkeyParams {
    const uint8_t *keys;
    const uint32_t *key_off;
    const uint32_t *key_part; // null: every key belongs to slot 0
    uint32_t n, n_buckets;
    const HotkeySlotDev *slots;
    uint32_t *tickets; // [slot]: fine tickets taken (may exceed the room)
    uint32_t *idx;     // key indices of admitted fine captures, slot s at idx[slots[s].idx_base ...]
};

__global__ void __launch_bounds__(kHotkeyThreads) k_hotkey_capture(const __grid_constant__ HotkeyParams P)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (kHotkeyThreads / 32);
    for (uint32_t base = (blockIdx.x * (kHotkeyThreads / 32) + (threadIdx.x >> 5)) * 32; base < P.n; base += warps * 32) {
        const uint32_t q = base + lane;
        uint32_t slot = 0, state = 0;
        KeyParts k{nullptr, nullptr, 0, 0};
        if (q < P.n) {
            slot = P.key_part ? P.key_part[q] : 0u;
            state = P.slots[slot].state;
            if (state) k = split_key(P.keys + P.key_off[q], P.key_off[q + 1] - P.key_off[q]);
        }
        // short hash keys: one lane each
        const bool is_long = state && k.hkl > kHotkeyLaneBytes;
        unsigned long long h = 0;
        if (state && !is_long) h = hotkey_hash(k.hk, k.hkl);
        // long hash keys: the warp hashes them one after the other, lane L taking the words L, L + 32, ...
        for (uint32_t longs = __ballot_sync(kFull, is_long); longs; longs &= longs - 1) {
            const uint32_t src = (uint32_t)__ffs((int)longs) - 1;
            const uint8_t *hk = (const uint8_t *)__shfl_sync(kFull, (unsigned long long)(uintptr_t)k.hk, (int)src);
            const uint32_t hkl = __shfl_sync(kFull, k.hkl, (int)src);
            unsigned long long s = 0;
            for (uint32_t j = lane; 4 * j < hkl; j += 32) s += hotkey_word_hash(hotkey_word(hk, hkl, j), j);
            for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(kFull, s, m);
            if (lane == src) h = hotkey_finish(s, hkl);
        }
        const uint32_t bucket = state ? (uint32_t)(h % P.n_buckets) : 0u;
        const HotkeySlotDev sd = state ? P.slots[slot] : HotkeySlotDev{nullptr, 0, 0, 0, 0};
        // lanes that count: COARSE keys, and FINE keys of the target bucket; they meet their peers of the same (slot, bucket)
        const bool counts = state == 1 || (state == 2 && bucket == sd.target);
        const unsigned long long id = counts ? ((unsigned long long)slot << 32 | bucket) : ~0ull;
        const uint32_t peers = __match_any_sync(kFull, id);
        const uint32_t leader = (uint32_t)__ffs((int)peers) - 1;
        uint32_t t0 = 0;
        if (counts && lane == leader) {
            if (state == 1) atomicAdd(&sd.buckets[bucket], (unsigned long long)__popc(peers));
            else t0 = atomicAdd(&P.tickets[slot], (uint32_t)__popc(peers));
        }
        t0 = __shfl_sync(kFull, t0, (int)leader);
        if (counts && state == 2) {
            const uint32_t t = t0 + (uint32_t)__popc(peers & ((1u << lane) - 1u));
            if (t < sd.room) P.idx[sd.idx_base + t] = q;
        }
    }
}

} // namespace pgs
