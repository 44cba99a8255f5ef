// lookup.cu — host side of the read path (pgs_get_batch[_multi], pgs_range_scan, pgs_range_scan_many[_multi]).
//
//   k_get / k_scan_fwd (read_kernels.cuh)  point lookups and forward range scans: lane-group iterators straight over HBM.
//   k_scan (scan_kernel.cuh)  REVERSE range scans, every request of a batch that mixes directions, and forward scans
//           whose user keys are too long for k_scan_fwd: one CTA per request stages chunks of blocks of every run in shared memory.
//
// A read is planned and launched by the functions next to its kernels, which the simulator (tools/simt) calls too, as a
// compaction is: read_run_set (the partition slots' runs), get_plan / scan_plan (kernel and shared memory), get_buffers /
// scan_buffers (every device buffer with its size and initial content) and read_launch, and a scan batch's packed read-back by
// pack_offsets_launch / pack_copy_launch.  This file adds what is the library's own: the run snapshot, the occupancy cap, device
// scratch, events, the copies back to the host and the hot-key capture.
#include <algorithm>
#include <cstring>

#include "engine.h"
#include "hotkey_kernels.cuh"
#include "read_kernels.cuh"
#include "scan_kernel.cuh"

namespace pgs {

void set_last_read_stats(float ms, uint64_t probed, uint64_t skipped);

// The runs of a read call's partition slots (parts[0 .. n_slots)), each kept alive in `slots` until the launch is done, as the
// launch plan's run set.  pinned = the runs to read instead of parts[0]'s current ones.  what: the ABI call, for the message.
using SlotRuns = std::vector<std::vector<std::shared_ptr<Run>>>;
static int32_t snapshot_runs(pgs_partition *const *parts, uint32_t n_slots, bool multi, const char *what, SlotRuns &slots, ReadRunSet &R,
                             const std::vector<std::shared_ptr<Run>> *pinned = nullptr)
{
    const Partition &part = parts[0]->p;
    slots.resize(n_slots);
    for (uint32_t s = 0; s < n_slots; s++) {
        Partition &pp = parts[s]->p;
        if (pp.eng != part.eng || pp.data_version != part.data_version) { set_error("%s: partitions of different engines / data versions", what); return PGS_INVALID_ARGUMENT; }
        if (pinned) {
            slots[s] = *pinned;
        } else {
            std::lock_guard<std::mutex> g(pp.mu);
            slots[s] = pp.runs;
        }
    }
    return read_run_set(slots, multi, R);
}

bool scan_stages_every_run(pgs_partition *ph)
{
    SlotRuns slots;
    ReadRunSet R;
    if (snapshot_runs(&ph, 1, false, "", slots, R) != PGS_OK) return false;
    ScanParams P{};
    P.n = 1;
    ReadLaunch<ScanParams> L;
    return scan_plan(P, R, true, ph->p.eng->max_smem_optin, ph->p.eng->scan_static_smem, L) == PGS_OK;
}

// kernels of this file take their dynamic shared-memory size per launch; the opt-in maximum is set once per device here
// (a per-call cudaFuncSetAttribute would race between reader threads)
template <class K>
static cudaError_t allow_max_smem(K kernel, int max_smem)
{
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, kernel);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)a.sharedSizeBytes);
}
int32_t lookup_init_kernels(Engine &e)
{
    const int max_smem = e.max_smem_optin;
    cudaFuncAttributes a;
    PGS_CUDA(cudaFuncGetAttributes(&a, k_scan));
    e.scan_static_smem = (uint32_t)a.sharedSizeBytes;
    PGS_CUDA(allow_max_smem(k_scan, max_smem));
    PGS_CUDA(cudaFuncSetAttribute(k_scan, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    PGS_CUDA(allow_max_smem(k_get<8, false>, max_smem)); PGS_CUDA(allow_max_smem(k_get<8, true>, max_smem));
    for (uint32_t G : kScanFwdGs)
        for (bool multi : {false, true}) PGS_CUDA(allow_max_smem(scan_fwd_kernel(G, multi), max_smem));
    return PGS_OK;
}

// the CTAs of L the device holds at once (resident CTAs per SM for its dynamic shared memory; registers count too)
template <class Params>
static cudaError_t resident_ctas(const Engine &e, const ReadLaunch<Params> &L, uint64_t &ctas)
{
    int occ = 0;
    const cudaError_t rc = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, L.kernel, (int)L.threads, (size_t)L.dyn);
    ctas = (uint64_t)std::max(1, occ) * e.sm_count;
    return rc;
}

int32_t scan_many(pgs_partition *const *parts, uint32_t n_parts, const uint32_t *req_part, const pgs_scan_request *reqs, uint32_t n,
                  uint32_t now, pgs_scan_result *results, const ScanOut &out, const std::vector<std::shared_ptr<Run>> *pinned)
{
    Partition &part = parts[0]->p;
    Engine *e = part.eng;
    SlotRuns slots;
    ReadRunSet R;
    int32_t rc = snapshot_runs(parts, n_parts, req_part != nullptr, "range_scan_many_multi", slots, R, pinned);
    if (rc != PGS_OK) return rc;
    for (uint32_t i = 0; req_part && i < n; i++) {
        if (req_part[i] >= n_parts) { set_error("range_scan_many_multi: request %u names partition slot %u of %u", i, req_part[i], n_parts); return PGS_INVALID_ARGUMENT; }
        if (reqs[i].reverse) { set_error("range_scan_many_multi: reverse scans go through pgs_range_scan_many"); return PGS_NOT_SUPPORTED; }
    }
    if (n == 0) return PGS_OK;
    if (R.empty()) { // empty DB: every iterator is invalid from the start
        memset(results, 0, sizeof(pgs_scan_result) * n);
        if (out.arena_base) for (uint32_t i = 0; i <= n; i++) out.arena_base[i] = 0;
        if (out.kv_base) for (uint32_t i = 0; i <= n; i++) out.kv_base[i] = 0;
        return PGS_OK;
    }
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->read_stream();
    const ScanBatch B = flatten_scan_requests(reqs, n);
    ScanParams P{};
    P.n = n; P.now = now; P.data_version = part.data_version;
    if (B.need_crc) P.crc_table = (const unsigned long long *)e->d_crc;
    ReadLaunch<ScanParams> L;
    rc = scan_plan(P, R, B.any_reverse, e->max_smem_optin, e->scan_static_smem, L);
    if (rc != PGS_OK) return rc;

    LaunchScratch S(st);
    cudaEvent_t ev_a, ev_b;
    PGS_CUDA(S.event(ev_a));
    PGS_CUDA(S.event(ev_b));
    cudaError_t ce = cudaSuccess;
    // resume_stride 0: the caller gave no room for resume keys
    const uint32_t resume_stride = scan_buffers(P, R, B, req_part, out.arena_stride, out.kv_stride, out.resume_stride, device_buffers(S, ce))
                                       ? out.resume_stride : 0;
    PGS_CUDA(ce);
    uint64_t ctas = 0;
    PGS_CUDA(resident_ctas(*e, L, ctas));
    PGS_CUDA(cudaEventRecord(ev_a, st));
    read_launch(L, P, ctas, st);
    PGS_CUDA(cudaEventRecord(ev_b, st));
    e->launches++;
    uint32_t herr = 0;
    if (n == 1) {
        PGS_CUDA(cudaMemcpyAsync(results, P.results, sizeof(pgs_scan_result), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(&herr, P.error, 4, cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaStreamSynchronize(st));
        if (!herr) {
            if (results[0].arena_used > out.arena_cap || results[0].n_kvs > out.kv_cap) return PGS_INCOMPLETE;
            if (results[0].arena_used) PGS_CUDA(cudaMemcpyAsync(out.arena, P.arena, results[0].arena_used, cudaMemcpyDeviceToHost, st));
            if (results[0].n_kvs) PGS_CUDA(cudaMemcpyAsync(out.kvs, P.kvs, sizeof(pgs_kv) * results[0].n_kvs, cudaMemcpyDeviceToHost, st));
            if (results[0].iter_valid && out.resume && resume_stride) PGS_CUDA(cudaMemcpyAsync(out.resume, P.resume, results[0].resume_len, cudaMemcpyDeviceToHost, st));
            PGS_CUDA(cudaStreamSynchronize(st));
        }
        if (out.arena_base) { out.arena_base[0] = 0; out.arena_base[1] = results[0].arena_used; }
        if (out.kv_base) { out.kv_base[0] = 0; out.kv_base[1] = results[0].n_kvs; }
    } else {
        ScanPack K;
        pack_offsets_launch(P, K, st, device_buffers(S, ce));
        PGS_CUDA(ce);
        std::vector<unsigned long long> ab(n + 1);
        std::vector<uint32_t> kb(n + 1);
        PGS_CUDA(cudaMemcpyAsync(ab.data(), K.arena_base, sizeof(unsigned long long) * (n + 1), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(kb.data(), K.kv_base, sizeof(uint32_t) * (n + 1), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(results, P.results, sizeof(pgs_scan_result) * n, cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaMemcpyAsync(&herr, P.error, 4, cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaStreamSynchronize(st));
        e->launches++;
        if (!herr) {
            if (ab[n] > out.arena_cap || kb[n] > out.kv_cap) { set_error("scan_many: output arena too small"); return PGS_INCOMPLETE; }
            pack_copy_launch(P, K, ab[n], kb[n], 8 * e->sm_count, st, device_buffers(S, ce));
            PGS_CUDA(ce);
            e->launches++;
            if (ab[n]) PGS_CUDA(cudaMemcpyAsync(out.arena, K.arena, ab[n], cudaMemcpyDeviceToHost, st));
            if (kb[n]) PGS_CUDA(cudaMemcpyAsync(out.kvs, K.kvs, sizeof(pgs_kv) * kb[n], cudaMemcpyDeviceToHost, st));
            if (out.resume && resume_stride) PGS_CUDA(cudaMemcpyAsync(out.resume, P.resume, (size_t)P.resume_stride * n, cudaMemcpyDeviceToHost, st));
            PGS_CUDA(cudaStreamSynchronize(st));
        }
        if (out.arena_base) for (uint32_t i = 0; i <= n; i++) out.arena_base[i] = ab[i];
        if (out.kv_base) for (uint32_t i = 0; i <= n; i++) out.kv_base[i] = kb[i];
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    set_last_read_stats(ms, 0, 0);
    if (herr) {
        set_error("scan kernel failed with status %u", herr);
        // PGS_ABORTED = a request's output did not fit its arena / kv slice: the caller may retry with more room
        return herr == PGS_CORRUPTION ? PGS_CORRUPTION : (herr == PGS_NOT_SUPPORTED ? PGS_NOT_SUPPORTED : (herr == PGS_ABORTED ? PGS_ABORTED : PGS_IO_ERROR));
    }
    return PGS_OK;
}
// ---- hot-key capture of batched gets (hotkey_kernels.cuh) ------------------------------------------------------------------
Partition::~Partition()
{
    if (hk_dev_buckets) { cudaSetDevice(eng->device); cudaFree(hk_dev_buckets); }
}

int32_t hotkey_control(Partition &p, int32_t type, int32_t action, uint32_t now, std::string &text)
{
    if (action != HOTKEY_START && action != HOTKEY_STOP && action != HOTKEY_QUERY) { text = "invalid detect_action"; return HOTKEY_INVALID_PARAMETERS; }
    if (type != HOTKEY_READ && type != HOTKEY_WRITE) { text = "invalid hotkey_type"; return HOTKEY_INVALID_PARAMETERS; }
    if (type == HOTKEY_WRITE) return p.hk_write.control(action, now, text);
    std::unique_lock<std::shared_mutex> g(p.hk_dev_mu);
    if (action == HOTKEY_START && p.hk_read.state() == HOTKEY_STOPPED) { // the device counters start from zero
        const uint32_t nb = p.hk_read.config().buckets;
        cudaError_t e = cudaSetDevice(p.eng->device);
        if (e == cudaSuccess && p.hk_dev_buckets && p.hk_dev_n != nb) { cudaFree(p.hk_dev_buckets); p.hk_dev_buckets = nullptr; }
        if (e == cudaSuccess && !p.hk_dev_buckets) e = cudaMalloc((void **)&p.hk_dev_buckets, sizeof(unsigned long long) * nb);
        if (e == cudaSuccess) { p.hk_dev_n = nb; e = cudaMemset(p.hk_dev_buckets, 0, sizeof(unsigned long long) * nb); }
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { cuda_fail(e, "hotkey counters"); text = std::string("hotkey counters: ") + cudaGetErrorString(e); return HOTKEY_INVALID_STATE; }
    }
    return p.hk_read.control(action, now, text);
}

int32_t hotkey_analyse(Partition &p, uint32_t now)
{
    p.hk_write.analyse(now);
    std::unique_lock<std::shared_mutex> g(p.hk_dev_mu); // no capturing launch is in flight
    std::vector<uint64_t> dev;
    if (p.hk_dev_buckets && p.hk_read.state() == HOTKEY_COARSE) { // read and zero the counters with one small copy each way
        PGS_CUDA(cudaSetDevice(p.eng->device));
        dev.resize(p.hk_dev_n);
        PGS_CUDA(cudaMemcpy(dev.data(), p.hk_dev_buckets, sizeof(unsigned long long) * p.hk_dev_n, cudaMemcpyDeviceToHost));
        PGS_CUDA(cudaMemset(p.hk_dev_buckets, 0, sizeof(unsigned long long) * p.hk_dev_n));
        PGS_CUDA(cudaDeviceSynchronize());
    }
    p.hk_read.analyse(now, &dev);
    return PGS_OK;
}

// The READ collectors a get launch captures into: the distinct partitions of the call with an active collector, locked
// shared (hk_dev_mu) until the fine captures are handed over, and one slot descriptor per partition slot of the launch.
struct HotkeyCapture {
    std::vector<std::shared_lock<std::shared_mutex>> locks;
    std::vector<HotkeySlotDev> slots;
    std::vector<Partition *> slot_part;
    uint32_t total_room = 0;
    bool any = false;
    uint32_t n_buckets = 0;

    void open(pgs_partition *const *parts, uint32_t n_parts)
    {
        bool active = false;
        for (uint32_t s = 0; s < n_parts; s++) active |= parts[s]->p.hk_read.active();
        if (!active) return; // no detection: nothing is locked, uploaded or launched
        std::vector<Partition *> locked;
        slots.assign(n_parts, HotkeySlotDev{nullptr, 0, 0, 0, 0});
        slot_part.assign(n_parts, nullptr);
        for (uint32_t s = 0; s < n_parts; s++) {
            Partition &pp = parts[s]->p;
            if (!pp.hk_read.active()) continue;
            if (std::find(locked.begin(), locked.end(), &pp) == locked.end()) { locks.emplace_back(pp.hk_dev_mu); locked.push_back(&pp); }
            const HotkeyCollector::Phase ph = pp.hk_read.device_phase();
            // every collector of one engine shares the bucket count of its options; a slot with another count is left out
            if (ph.state == HOTKEY_STOPPED || !pp.hk_dev_buckets || (n_buckets && pp.hk_dev_n != n_buckets)) continue;
            n_buckets = pp.hk_dev_n;
            HotkeySlotDev &d = slots[s];
            d.state = ph.state;
            if (ph.state == HOTKEY_COARSE) d.buckets = pp.hk_dev_buckets;
            else { d.target = ph.target; d.room = ph.room; d.idx_base = total_room; total_room += ph.room; }
            slot_part[s] = &pp;
            any = true;
        }
    }
    // keys the memtable-less shortcut answers without a launch (a partition with no runs): captured on the host
    void capture_on_host(const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part, uint32_t n)
    {
        for (uint32_t i = 0; any && i < n; i++)
            if (Partition *pp = slot_part[key_part ? key_part[i] : 0])
                pp->hk_read.capture_raw_key(std::string_view((const char *)keys + key_off[i], key_off[i + 1] - key_off[i]), 1);
    }
    // the fine captures of a finished launch: the first min(ticket, room) admitted keys of every fine slot
    void hand_over(const uint8_t *keys, const uint32_t *key_off, const std::vector<uint32_t> &tickets, const std::vector<uint32_t> &idx)
    {
        for (uint32_t s = 0; s < slots.size(); s++) {
            if (slots[s].state != HOTKEY_FINE) continue;
            const uint32_t m = std::min(tickets[s], slots[s].room);
            std::vector<std::string> hks;
            for (uint32_t j = 0; j < m; j++) {
                const uint32_t q = idx[slots[s].idx_base + j];
                const KeyParts k = split_key(keys + key_off[q], key_off[q + 1] - key_off[q]);
                hks.emplace_back((const char *)k.hk, k.hkl);
            }
            slot_part[s]->hk_read.add_fine_keys(hks);
        }
    }
};

} // namespace pgs

using namespace pgs;

// one get launch over the keys of one partition (parts[0], key_part null) or of several partitions of one engine
static int32_t get_batch_impl(pgs_partition *const *parts, uint32_t n_parts, const uint8_t *keys, const uint32_t *key_off, const uint32_t *key_part,
                              uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used,
                              bool capture = true)
{
    Partition &part = parts[0]->p;
    Engine *e = part.eng;
    if (arena_used) *arena_used = 0;
    if (n == 0) return PGS_OK;
    SlotRuns slots;
    ReadRunSet R;
    int32_t rc = snapshot_runs(parts, key_part ? n_parts : 1, key_part != nullptr, "get_batch_multi", slots, R);
    if (rc != PGS_OK) return rc;
    for (uint32_t i = 0; key_part && i < n; i++)
        if (key_part[i] >= n_parts) { set_error("get_batch_multi: key %u names partition slot %u of %u", i, key_part[i], n_parts); return PGS_INVALID_ARGUMENT; }
    HotkeyCapture hk;
    if (capture) hk.open(parts, key_part ? n_parts : 1);
    if (R.empty()) {
        for (uint32_t i = 0; i < n; i++) { memset(&results[i], 0, sizeof results[i]); results[i].status = PGS_NOT_FOUND; }
        hk.capture_on_host(keys, key_off, key_part, n);
        return PGS_OK;
    }
    GetParams P{};
    P.n = n; P.now = now; P.data_version = part.data_version;
    ReadLaunch<GetParams> L;
    if ((rc = get_plan(P, R, e->max_smem_optin, L)) != PGS_OK) return rc;
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->read_stream();
    LaunchScratch S(st);
    cudaEvent_t ev_a, ev_b;
    PGS_CUDA(S.event(ev_a));
    PGS_CUDA(S.event(ev_b));
    cudaError_t ce = cudaSuccess;
    get_buffers(P, R, keys, key_off, key_part, arena_cap, device_buffers(S, ce));
    PGS_CUDA(ce);
    uint64_t ctas = 0;
    PGS_CUDA(resident_ctas(*e, L, ctas));
    PGS_CUDA(cudaEventRecord(ev_a, st));
    read_launch(L, P, ctas, st);
    PGS_CUDA(cudaEventRecord(ev_b, st));
    e->launches++;
    // hot-key capture (only while a slot's READ collector is active): its fine tickets and indices come back with the results
    std::vector<uint32_t> hk_tickets, hk_idx;
    if (hk.any) {
        HotkeyParams H{};
        H.keys = P.keys; H.key_off = P.key_off; H.key_part = P.key_part; H.n = n; H.n_buckets = hk.n_buckets;
        const uint32_t n_slots = (uint32_t)hk.slots.size();
        PGS_CUDA(S.upload(H.slots, hk.slots.data(), n_slots));
        PGS_CUDA(S.alloc(H.tickets, sizeof(uint32_t) * (n_slots + (size_t)hk.total_room)));
        PGS_CUDA(cudaMemsetAsync(H.tickets, 0, sizeof(uint32_t) * n_slots, st));
        H.idx = H.tickets + n_slots;
        const uint32_t hgrid = std::min<uint32_t>((n + kHotkeyThreads - 1) / kHotkeyThreads, 8u * e->sm_count);
        k_hotkey_capture<<<hgrid, kHotkeyThreads, 0, st>>>(H);
        e->launches++;
        hk_tickets.resize(n_slots + (size_t)hk.total_room);
        PGS_CUDA(cudaMemcpyAsync(hk_tickets.data(), H.tickets, sizeof(uint32_t) * hk_tickets.size(), cudaMemcpyDeviceToHost, st));
    }
    uint32_t herr = 0;
    unsigned long long cur3[3] = {0, 0, 0};
    PGS_CUDA(cudaMemcpyAsync(results, P.results, sizeof(pgs_get_result) * n, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(cur3, P.arena_cursor, 24, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(&herr, P.error, 4, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaStreamSynchronize(st));
    if (hk.any && hk.total_room) {
        hk_idx.assign(hk_tickets.begin() + hk.slots.size(), hk_tickets.end());
        hk_tickets.resize(hk.slots.size());
        hk.hand_over(keys, key_off, hk_tickets, hk_idx);
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    set_last_read_stats(ms, cur3[1], cur3[2]);
    const unsigned long long used = cur3[0];
    if (arena_used) *arena_used = used;
    if (!herr && used) {
        PGS_CUDA(cudaMemcpyAsync(arena, P.arena, std::min<unsigned long long>(used, P.arena_cap), cudaMemcpyDeviceToHost, st));
        PGS_CUDA(cudaStreamSynchronize(st));
    }
    if (herr) { set_error("get kernel failed with status %u", herr); return herr == PGS_CORRUPTION ? PGS_CORRUPTION : PGS_IO_ERROR; }
    return used > P.arena_cap ? PGS_INCOMPLETE : PGS_OK;
}

// pgs_get_batch, with the READ collector's capture switched on or off (handlers that capture with their own weights)
int32_t pgs::get_batch(pgs_partition *ph, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                       uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used, bool capture)
{
    if (!ph || (n && (!keys || !key_off || !results))) return PGS_INVALID_ARGUMENT;
    return get_batch_impl(&ph, 1, keys, key_off, nullptr, n, now, arena, arena_cap, results, arena_used, capture);
}

extern "C" int32_t pgs_get_batch(pgs_partition *ph,const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now, uint8_t *arena,
                                 uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used)
{
    if (!ph || (n && (!keys || !key_off || !results))) return PGS_INVALID_ARGUMENT;
    return get_batch_impl(&ph, 1, keys, key_off, nullptr, n, now, arena, arena_cap, results, arena_used);
}

extern "C" int32_t pgs_get_batch_multi(pgs_partition *const *parts, uint32_t n_parts, const uint8_t *keys, const uint32_t *key_off,
                                       const uint32_t *key_part, uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap,
                                       pgs_get_result *results, uint64_t *arena_used)
{
    if (!parts || !n_parts || (n && (!keys || !key_off || !key_part || !results))) return PGS_INVALID_ARGUMENT;
    for (uint32_t p = 0; p < n_parts; p++)
        if (!parts[p]) return PGS_INVALID_ARGUMENT;
    return get_batch_impl(parts, n_parts, keys, key_off, key_part, n, now, arena, arena_cap, results, arena_used);
}

extern "C" int32_t pgs_range_scan(pgs_partition *ph, const pgs_scan_request *req, uint32_t now, uint8_t *arena,
                                  uint64_t arena_cap, pgs_kv *kvs, uint32_t kv_cap, uint8_t *resume_key,
                                  uint32_t resume_cap, pgs_scan_result *out)
{
    if (!ph || !req || !out) return PGS_INVALID_ARGUMENT;
    return scan_many(&ph, 1, nullptr, req, 1, now, out, ScanOut{arena, arena_cap, arena_cap, kvs, kv_cap, kv_cap, resume_key, resume_cap, nullptr, nullptr});
}

extern "C" int32_t pgs_range_scan_many(pgs_partition *ph, const pgs_scan_request *reqs, uint32_t n, uint32_t now,
                                       uint64_t arena_stride, uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap,
                                       pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume_keys, uint32_t resume_stride,
                                       pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base)
{
    if (!ph || (n && (!reqs || !results))) return PGS_INVALID_ARGUMENT;
    return scan_many(&ph, 1, nullptr, reqs, n, now, results,
                     ScanOut{arena, arena_stride, arena_cap, kvs, kv_stride, kv_cap, resume_keys, resume_stride, arena_base, kv_base});
}

extern "C" int32_t pgs_range_scan_many_multi(pgs_partition *const *parts, uint32_t n_parts, const pgs_scan_request *reqs, const uint32_t *req_part,
                                             uint32_t n, uint32_t now, uint64_t arena_stride, uint32_t kv_stride, uint8_t *arena,
                                             uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap, uint8_t *resume_keys, uint32_t resume_stride,
                                             pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base)
{
    if (!parts || !n_parts || (n && (!reqs || !req_part || !results))) return PGS_INVALID_ARGUMENT;
    for (uint32_t p = 0; p < n_parts; p++)
        if (!parts[p]) return PGS_INVALID_ARGUMENT;
    return scan_many(parts, n_parts, req_part, reqs, n, now, results,
                     ScanOut{arena, arena_stride, arena_cap, kvs, kv_stride, kv_cap, resume_keys, resume_stride, arena_base, kv_base});
}
