// engine.cu — device engine plumbing: engine / partition handles, run upload (RocksDB-format
// blocks -> HBM) with the device-built block index, run download, run bookkeeping.
// Replaces for this path: DB::Open (pegasus_server_impl.cpp:1551-1860), flush /
// IngestExternalFile (rocksdb_wrapper.cpp:248-270) as far as "a sorted run appears in the DB".
#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <cstring>

#include "engine.h"
#include "index_kernel.cuh"

namespace pgs {

static thread_local std::string g_last_error;
void set_error(const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
}
int32_t cuda_fail(cudaError_t e, const char *what)
{
    set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    return PGS_IO_ERROR; // CUDA faults map to kIOError (SURVEY §8b)
}

// engines that are still open: a run that outlives its engine (caller closed the engine first) must not touch it
static std::mutex g_live_mu;
static std::vector<Engine *> g_live;
static bool engine_alive(Engine *e)
{
    std::lock_guard<std::mutex> g(g_live_mu);
    return std::find(g_live.begin(), g_live.end(), e) != g_live.end();
}

constexpr uint64_t kSpareMin = 64ull << 20; // only buffers this large are worth keeping
constexpr size_t kSpareMax = 8;
constexpr uint64_t kSpareMemDivisor = 8; // spare buffers hold at most 1/8 of the device memory (10 GB on an 80 GB H100)

cudaError_t Engine::alloc_data(Run &r, uint64_t need)
{
    if (need >= kSpareMin) {
        std::lock_guard<std::mutex> g(spare_mu);
        int best = -1;
        for (size_t i = 0; i < spares.size(); i++)
            if (spares[i].cap >= need && spares[i].cap <= 2 * need + kSpareMin && (best < 0 || spares[i].cap < spares[best].cap)) best = (int)i;
        if (best >= 0) {
            r.d_data = spares[best].p;
            r.data_cap = spares[best].cap;
            spares.erase(spares.begin() + best);
            return cudaSuccess;
        }
    }
    r.data_cap = need;
    return cudaMallocAsync(&r.d_data, need, stream);
}
void *Engine::take_pinned(size_t need, size_t *cap)
{
    {
        std::lock_guard<std::mutex> g(pin_mu);
        for (size_t i = 0; i < pins.size(); i++)
            if (pins[i].cap >= need) {
                void *p = pins[i].p;
                *cap = pins[i].cap;
                pins.erase(pins.begin() + i);
                return p;
            }
    }
    void *p = nullptr;
    const size_t want = (need + (1u << 20)) & ~(size_t)((1u << 20) - 1);
    if (cudaMallocHost(&p, want) != cudaSuccess) return nullptr;
    *cap = want;
    return p;
}
void Engine::give_pinned(void *p, size_t cap)
{
    std::lock_guard<std::mutex> g(pin_mu);
    if (pins.size() < 8) pins.push_back(Pin{p, cap});
    else cudaFreeHost(p);
}
void Engine::give_data(uint8_t *p, uint64_t cap)
{
    std::lock_guard<std::mutex> g(spare_mu);
    spares.push_back(Spare{p, cap});
    uint64_t total = 0;
    for (auto &s : spares) total += s.cap;
    while (spares.size() > kSpareMax || total > spare_bytes_max) { // give the smallest ones back to the pool
        size_t m = 0;
        for (size_t i = 1; i < spares.size(); i++) if (spares[i].cap < spares[m].cap) m = i;
        total -= spares[m].cap;
        cudaFreeAsync(spares[m].p, stream);
        spares.erase(spares.begin() + m);
    }
}

// stream-ordered pool: repeated flush / compaction cycles reuse the same HBM without driver calls
Run::Run(Engine *e) : pool_stream(e->stream), eng(e) {}
Run::~Run()
{
    // the bytes go back to the pool without a device sync
    if (d_data && data_cap >= kSpareMin && engine_alive(eng)) eng->give_data(d_data, data_cap);
    else cudaFreeAsync(d_data, pool_stream);
    cudaFreeAsync(d_blk_off, pool_stream);
    cudaFreeAsync(d_blk_size, pool_stream);
    cudaFreeAsync(d_blk_rec, pool_stream);
    cudaFreeAsync(d_ikey_off, pool_stream);
    cudaFreeAsync(d_ikeys, pool_stream);
    cudaFreeAsync(d_rec_off, pool_stream);
    cudaFreeAsync(d_bloom, pool_stream);
}
Engine::~Engine()
{
    {
        std::lock_guard<std::mutex> g(g_live_mu);
        g_live.erase(std::remove(g_live.begin(), g_live.end(), this), g_live.end());
    }
    for (auto &s : spares) cudaFreeAsync(s.p, stream);
    spares.clear();
    if (h_pinned) cudaFreeHost(h_pinned);
    for (auto &s : rd_streams) if (s) cudaStreamDestroy(s);
    if (up_copy) cudaStreamDestroy(up_copy);
    for (auto &pn : pins) cudaFreeHost(pn.p);
    if (d_crc) cudaFree(d_crc);
    if (stream) cudaStreamDestroy(stream);
}
cudaStream_t Engine::read_stream()
{
    static std::atomic<uint32_t> next{0};
    thread_local uint32_t mine = next.fetch_add(1);
    return rd_streams[mine % kReadStreams];
}
// device time of the calling thread's last read call (the getters of the ABI are per thread: readers run concurrently)
static thread_local float t_last_ms = 0.f;
static thread_local uint64_t t_last_probed = 0, t_last_skipped = 0;
void set_last_read_stats(float ms, uint64_t probed, uint64_t skipped) { t_last_ms = ms; t_last_probed = probed; t_last_skipped = skipped; }
int32_t lookup_init_kernels(int max_smem);
int32_t compact_init_kernels(int max_smem);

void *Engine::pinned(size_t bytes)
{
    if (bytes > h_pinned_cap) {
        if (h_pinned) cudaFreeHost(h_pinned);
        h_pinned = nullptr;
        size_t cap = bytes + (bytes >> 2) + 4096;
        if (cudaMallocHost(&h_pinned, cap) != cudaSuccess) { h_pinned_cap = 0; return nullptr; }
        h_pinned_cap = cap;
    }
    return h_pinned;
}
std::shared_ptr<Run> Partition::find(uint64_t id)
{
    for (auto &r : runs)
        if (r->id == id) return r;
    return nullptr;
}
void Partition::insert(std::shared_ptr<Run> r)
{
    size_t pos = 0;
    while (pos < runs.size() && runs[pos]->level < r->level) pos++;
    runs.insert(runs.begin() + pos, std::move(r));
}

int32_t index_init_kernels()
{
    const int smem = (int)(kIdxWarps * kIdxScratch);
    PGS_CUDA(cudaFuncSetAttribute(k_index_walk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    PGS_CUDA(cudaFuncSetAttribute(k_index_walk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    return PGS_OK;
}

// ---- staged upload of one run ---------------------------------------------------------------------------------------------
// stage A (asynchronous): the block bytes travel in chunks on the engine's copy stream; the first index pass (records and
//          last-key length per block, run statistics) runs on each chunk as soon as it has landed, while the next chunk
//          is still on the link
// stage B: waits for the first pass only, lays out the index (host prefix sums over the blocks), starts the second pass
//          (index keys, entry offsets, Bloom filter)
// stage C: waits for the second pass, publishes the run
// pgs_run_upload runs A, B, C back to back; pgs_run_upload_many issues A of the next run before B of the current one, so
// the link never idles between runs.
constexpr uint64_t kUploadChunk = 32ull << 20;

struct UploadJob {
    std::shared_ptr<Run> r;
    Engine *eng = nullptr;
    // pinned staging (one allocation): off[nb+1] u64 | blk_size[nb] u32 | nrec[nb] | lastlen[nb] | rec_cum[nb+1] | key_cum[nb+1] | 2 x IndexStats
    void *pin = nullptr;
    size_t pin_cap = 0;
    uint64_t *off = nullptr;
    uint32_t *h_size = nullptr, *nrec = nullptr, *lastlen = nullptr, *rec_cum = nullptr, *key_cum = nullptr;
    IndexStats *hs_in = nullptr, *hs_out = nullptr;
    uint32_t *d_nrec = nullptr, *d_lastlen = nullptr;
    IndexStats *d_stats = nullptr;
    IndexStats hs{};
    std::vector<cudaEvent_t> events;
    cudaEvent_t pass1 = nullptr;
    uint32_t max_blk = 0;
    ~UploadJob()
    {
        for (cudaEvent_t ev : events) cudaEventDestroy(ev);
        if (pass1) cudaEventDestroy(pass1);
        if (pin && eng) eng->give_pinned(pin, pin_cap);
    }
};

static int32_t upload_stage_a(Engine *e, int32_t level, const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off,
                              const uint32_t *blk_size, uint32_t nb, UploadJob &j)
{
    uint64_t prev_end = 0;
    for (uint32_t b = 0; b < nb; b++) {
        if (blk_off[b] % kBlockAlign || blk_off[b] < prev_end || blk_off[b] + blk_size[b] > data_bytes) {
            set_error("run upload: bad block handle %u", b);
            return PGS_INVALID_ARGUMENT;
        }
        prev_end = blk_off[b] + blk_size[b];
        j.max_blk = std::max(j.max_blk, blk_size[b]);
    }
    auto r = std::make_shared<Run>(e);
    j.r = r;
    j.eng = e;
    {
        const size_t need = 8ull * (nb + 2) + 4ull * (nb + 1) * 5 + 2 * sizeof(IndexStats) + 64;
        j.pin = e->take_pinned(need, &j.pin_cap);
        if (!j.pin) { set_error("run upload: no pinned staging memory"); return PGS_IO_ERROR; }
        uint8_t *q = (uint8_t *)j.pin;
        j.off = (uint64_t *)q; q += 8ull * (nb + 2);
        j.h_size = (uint32_t *)q; q += 4ull * (nb + 1);
        j.nrec = (uint32_t *)q; q += 4ull * (nb + 1);
        j.lastlen = (uint32_t *)q; q += 4ull * (nb + 1);
        j.rec_cum = (uint32_t *)q; q += 4ull * (nb + 1);
        j.key_cum = (uint32_t *)q; q += 4ull * (nb + 1);
        q = (uint8_t *)(((uintptr_t)q + 15) & ~(uintptr_t)15);
        j.hs_in = (IndexStats *)q; j.hs_out = j.hs_in + 1;
    }
    r->level = level;
    r->info.level = level;
    r->info.n_blocks = nb;
    const uint64_t end = (prev_end + kBlockAlign - 1) / kBlockAlign * kBlockAlign;
    const uint64_t nbytes = data_bytes < end ? data_bytes : end;
    r->info.data_bytes = end;
    cudaStream_t st = e->stream, cp = e->up_copy;
    PGS_CUDA(e->alloc_data(*r, end + 256));
    PGS_CUDA(cudaMallocAsync(&r->d_blk_off, sizeof(uint64_t) * (nb + 1), st));
    PGS_CUDA(cudaMallocAsync(&r->d_blk_size, sizeof(uint32_t) * nb, st));
    PGS_CUDA(cudaMallocAsync(&j.d_nrec, sizeof(uint32_t) * nb, st));
    PGS_CUDA(cudaMallocAsync(&j.d_lastlen, sizeof(uint32_t) * nb, st));
    PGS_CUDA(cudaMallocAsync(&j.d_stats, sizeof(IndexStats), st));
    PGS_CUDA(cudaMemsetAsync(r->d_data + nbytes, 0, r->data_cap - nbytes, st));
    memcpy(j.off, blk_off, sizeof(uint64_t) * nb);
    j.off[nb] = end;
    memcpy(j.h_size, blk_size, sizeof(uint32_t) * nb);
    *j.hs_in = IndexStats{};
    j.hs_in->min_seq = ~0ull;
    PGS_CUDA(cudaMemcpyAsync(r->d_blk_off, j.off, sizeof(uint64_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    PGS_CUDA(cudaMemcpyAsync(r->d_blk_size, j.h_size, sizeof(uint32_t) * nb, cudaMemcpyHostToDevice, st));
    PGS_CUDA(cudaMemcpyAsync(j.d_stats, j.hs_in, sizeof(IndexStats), cudaMemcpyHostToDevice, st));
    cudaEvent_t ready;
    PGS_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    j.events.push_back(ready);
    PGS_CUDA(cudaEventRecord(ready, st)); // the copy stream may touch the new buffers from here on
    PGS_CUDA(cudaStreamWaitEvent(cp, ready, 0));
    const size_t smem = kIdxWarps * kIdxScratch;
    uint32_t b0 = 0;
    while (b0 < nb) { // chunks end on block boundaries
        uint32_t b1 = b0 + 1;
        while (b1 < nb && j.off[b1] - j.off[b0] < kUploadChunk) b1++;
        const uint64_t lo = j.off[b0], hi = b1 == nb ? nbytes : std::min<uint64_t>(j.off[b1], nbytes);
        if (hi > lo) PGS_CUDA(cudaMemcpyAsync(r->d_data + lo, data + lo, hi - lo, cudaMemcpyHostToDevice, cp));
        cudaEvent_t ev;
        PGS_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        j.events.push_back(ev);
        PGS_CUDA(cudaEventRecord(ev, cp));
        PGS_CUDA(cudaStreamWaitEvent(st, ev, 0));
        k_index_walk<false><<<(b1 - b0 + kIdxWarps - 1) / kIdxWarps, kIdxWarps * 32, smem, st>>>(
            r->d_data, r->d_blk_off, r->d_blk_size, b1, j.d_nrec, j.d_lastlen, nullptr, nullptr, nullptr, nullptr, nullptr, 0, j.d_stats, b0);
        e->launches++;
        b0 = b1;
    }
    PGS_CUDA(cudaMemcpyAsync(j.nrec, j.d_nrec, sizeof(uint32_t) * nb, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(j.lastlen, j.d_lastlen, sizeof(uint32_t) * nb, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(j.hs_out, j.d_stats, sizeof(IndexStats), cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaEventCreateWithFlags(&j.pass1, cudaEventDisableTiming));
    PGS_CUDA(cudaEventRecord(j.pass1, st));
    return PGS_OK;
}

static int32_t upload_stage_b(Engine *e, UploadJob &j)
{
    Run *r = j.r.get();
    const uint32_t nb = r->info.n_blocks;
    cudaStream_t st = e->stream;
    PGS_CUDA(cudaEventSynchronize(j.pass1));
    j.hs = *j.hs_out;
    cudaFreeAsync(j.d_nrec, st);
    cudaFreeAsync(j.d_lastlen, st);
    j.d_nrec = j.d_lastlen = nullptr;
    if (j.hs.error) {
        set_error("run upload: block scan failed with status %u", j.hs.error);
        return (int32_t)j.hs.error;
    }
    if (!index_layout(j.nrec, j.lastlen, nb, j.rec_cum, j.key_cum)) {
        set_error("run too large for 32-bit record / index-key offsets");
        return PGS_NOT_SUPPORTED;
    }
    const uint32_t rc = j.rec_cum[nb], kc = j.key_cum[nb];
    PGS_CUDA(cudaMallocAsync(&r->d_blk_rec, sizeof(uint32_t) * (nb + 1), st));
    PGS_CUDA(cudaMallocAsync(&r->d_ikey_off, sizeof(uint32_t) * (nb + 1), st));
    PGS_CUDA(cudaMallocAsync(&r->d_ikeys, kc + 16, st));
    PGS_CUDA(cudaMallocAsync(&r->d_rec_off, sizeof(uint32_t) * (rc + 1), st));
    PGS_CUDA(cudaMemcpyAsync(r->d_blk_rec, j.rec_cum, sizeof(uint32_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    PGS_CUDA(cudaMemcpyAsync(r->d_ikey_off, j.key_cum, sizeof(uint32_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    r->n_bloom_entries = j.hs.n_records + j.hs.n_prefix;
    r->bloom_lines = bloom_lines_for(r->n_bloom_entries);
    PGS_CUDA(cudaMallocAsync(&r->d_bloom, (size_t)r->bloom_lines * 64, st));
    PGS_CUDA(cudaMemsetAsync(r->d_bloom, 0, (size_t)r->bloom_lines * 64, st));
    k_index_walk<true><<<(nb + kIdxWarps - 1) / kIdxWarps, kIdxWarps * 32, kIdxWarps * kIdxScratch, st>>>(
        r->d_data, r->d_blk_off, r->d_blk_size, nb, nullptr, nullptr, r->d_ikey_off, r->d_ikeys, r->d_blk_rec, r->d_rec_off, r->d_bloom,
        r->bloom_lines, j.d_stats, 0);
    e->launches++;
    PGS_CUDA(cudaEventRecord(j.pass1, st)); // reused: now marks the end of the second pass
    return PGS_OK;
}

static int32_t upload_stage_c(Engine *e, Partition &p, UploadJob &j, uint64_t *run_id_out)
{
    Run *r = j.r.get();
    PGS_CUDA(cudaEventSynchronize(j.pass1));
    cudaFreeAsync(j.d_stats, e->stream);
    j.d_stats = nullptr;
    run_info_from_index(j.hs, r->info.n_blocks, r->info.data_bytes, j.max_blk, r->info);
    r->id = e->next_run_id++;
    r->info.run_id = r->id;
    {
        std::lock_guard<std::mutex> g(p.mu);
        p.insert(j.r);
    }
    if (run_id_out) *run_id_out = r->id;
    return PGS_OK;
}
// a failed job: nothing of it may still be in flight when its host vectors and device buffers go away
static void upload_abandon(Engine *e, UploadJob &j)
{
    cudaStreamSynchronize(e->up_copy);
    cudaStreamSynchronize(e->stream);
    if (j.d_nrec) cudaFreeAsync(j.d_nrec, e->stream);
    if (j.d_lastlen) cudaFreeAsync(j.d_lastlen, e->stream);
    if (j.d_stats) cudaFreeAsync(j.d_stats, e->stream);
    j.d_nrec = j.d_lastlen = nullptr;
    j.d_stats = nullptr;
}

} // namespace pgs

using namespace pgs;

extern "C" {

const char *pgs_last_error(void) { return g_last_error.c_str(); }

int32_t pgs_engine_open(const pgs_engine_config *cfg, pgs_engine **out)
{
    if (!out) return PGS_INVALID_ARGUMENT;
    *out = nullptr;
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0) {
        // no CPU fallback: the engine exists only on a GPU
        set_error("no CUDA device: %s", cudaGetErrorString(ce));
        return PGS_IO_ERROR;
    }
    auto *h = new pgs_engine;
    Engine &e = h->e;
    if (cfg) e.cfg = *cfg;
    if (!e.cfg.block_size) e.cfg.block_size = kDefaultBlockSize;
    if (!e.cfg.restart_interval) e.cfg.restart_interval = kDefaultRestartInterval;
    int dev = e.cfg.device;
    if (dev < 0) cudaGetDevice(&dev);
    e.device = dev;
    cudaError_t err = cudaSetDevice(dev);
    if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&e.stream, cudaStreamNonBlocking);
    if (err == cudaSuccess) err = cudaDeviceGetAttribute(&e.sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (err == cudaSuccess) err = cudaDeviceGetAttribute(&e.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (err == cudaSuccess) {
        size_t free_b = 0, total_b = 0;
        err = cudaMemGetInfo(&free_b, &total_b);
        e.spare_bytes_max = total_b / kSpareMemDivisor;
    }
    for (auto &s : e.rd_streams) if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&e.up_copy, cudaStreamNonBlocking);
    if (err == cudaSuccess) {
        uint64_t tab[256];
        crc64_make_table(tab);
        err = cudaMalloc(&e.d_crc, sizeof tab);
        if (err == cudaSuccess) err = cudaMemcpy(e.d_crc, tab, sizeof tab, cudaMemcpyHostToDevice);
    }
    if (err == cudaSuccess && (lookup_init_kernels(e.max_smem_optin) != PGS_OK || compact_init_kernels(e.max_smem_optin) != PGS_OK ||
                               index_init_kernels() != PGS_OK)) {
        delete h; // the failing call left its description in pgs_last_error()
        return PGS_IO_ERROR;
    }
    if (err == cudaSuccess) { // keep freed compaction buffers in the stream-ordered pool
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t keep = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    }
    if (err != cudaSuccess) {
        delete h;
        return cuda_fail(err, "engine open");
    }
    {
        std::lock_guard<std::mutex> g(g_live_mu);
        g_live.push_back(&h->e);
    }
    *out = h;
    return PGS_OK;
}
void pgs_engine_close(pgs_engine *e)
{
    if (!e) return;
    cudaSetDevice(e->e.device);
    cudaStreamSynchronize(e->e.stream);
    delete e;
}
void *pgs_engine_stream(pgs_engine *e) { return (void *)e->e.stream; }
int32_t pgs_engine_sync(pgs_engine *e)
{
    PGS_CUDA(cudaSetDevice(e->e.device));
    PGS_CUDA(cudaStreamSynchronize(e->e.stream));
    return PGS_OK;
}
uint64_t pgs_engine_launches(pgs_engine *e) { return e->e.launches.load(); }
float pgs_engine_last_kernel_ms(pgs_engine *) { return t_last_ms; }
uint64_t pgs_engine_last_blocks_probed(pgs_engine *) { return t_last_probed; }
uint64_t pgs_engine_last_runs_skipped(pgs_engine *) { return t_last_skipped; }

int32_t pgs_partition_create(pgs_engine *e, int32_t app_id, int32_t pidx, uint32_t data_version,
                             pgs_partition **out)
{
    if (!e || !out || data_version > 1) return PGS_INVALID_ARGUMENT; // PEGASUS_DATA_VERSION_MAX = 1
    auto *p = new pgs_partition;
    p->p.eng = &e->e;
    p->p.app_id = app_id;
    p->p.pidx = pidx;
    p->p.data_version = data_version;
    *out = p;
    return PGS_OK;
}
void pgs_partition_destroy(pgs_partition *p)
{
    if (!p) return;
    cudaSetDevice(p->p.eng->device);
    cudaStreamSynchronize(p->p.eng->stream);
    delete p;
}

int32_t pgs_run_upload(pgs_partition *ph, int32_t level, const uint8_t *data, uint64_t data_bytes,
                       const uint64_t *blk_off, const uint32_t *blk_size, uint32_t n_blocks,
                       uint64_t *run_id_out)
{
    pgs_run_src src{data, data_bytes, blk_off, blk_size, n_blocks, level};
    return pgs_run_upload_many(ph, &src, 1, run_id_out);
}

int32_t pgs_run_upload_many(pgs_partition *ph, const pgs_run_src *runs, uint32_t n, uint64_t *run_ids_out)
{
    if (!ph || (n && !runs)) return PGS_INVALID_ARGUMENT;
    for (uint32_t i = 0; i < n; i++)
        if (runs[i].level < 0 || (runs[i].n_blocks && (!runs[i].data || !runs[i].blk_off || !runs[i].blk_size))) return PGS_INVALID_ARGUMENT;
    Partition &p = ph->p;
    Engine *e = p.eng;
    PGS_CUDA(cudaSetDevice(e->device));
    std::vector<std::unique_ptr<UploadJob>> jobs(n);
    std::vector<uint64_t> ids(n, 0);
    int32_t rc = PGS_OK;
    auto stage_a = [&](uint32_t i) {
        if (runs[i].n_blocks == 0) return (int32_t)PGS_OK; // an empty run: id 0, nothing resident
        jobs[i] = std::make_unique<UploadJob>();
        return upload_stage_a(e, runs[i].level, runs[i].data, runs[i].data_bytes, runs[i].blk_off, runs[i].blk_size, runs[i].n_blocks, *jobs[i]);
    };
    // the next run's bytes are queued on the link before this run's index is finished
    if (n) rc = stage_a(0);
    uint32_t done = 0;
    for (uint32_t i = 0; i < n && rc == PGS_OK; i++) {
        if (i + 1 < n) rc = stage_a(i + 1);
        if (rc == PGS_OK && jobs[i]) rc = upload_stage_b(e, *jobs[i]);
        if (rc == PGS_OK && i > 0 && jobs[i - 1]) { rc = upload_stage_c(e, p, *jobs[i - 1], &ids[i - 1]); if (rc == PGS_OK) done = i; }
    }
    if (rc == PGS_OK && n && jobs[n - 1]) { rc = upload_stage_c(e, p, *jobs[n - 1], &ids[n - 1]); if (rc == PGS_OK) done = n; }
    if (rc != PGS_OK) { // all or nothing
        for (auto &j : jobs) if (j) upload_abandon(e, *j);
        for (uint32_t i = 0; i < done; i++) if (ids[i]) pgs_run_drop(ph, ids[i]);
        return rc;
    }
    if (run_ids_out) for (uint32_t i = 0; i < n; i++) run_ids_out[i] = ids[i];
    return PGS_OK;
}

int32_t pgs_run_drop(pgs_partition *ph, uint64_t run_id)
{
    Partition &p = ph->p;
    std::lock_guard<std::mutex> g(p.mu);
    for (size_t i = 0; i < p.runs.size(); i++)
        if (p.runs[i]->id == run_id) {
            cudaSetDevice(p.eng->device);
            cudaStreamSynchronize(p.eng->stream);
            p.runs.erase(p.runs.begin() + i);
            return PGS_OK;
        }
    return PGS_NOT_FOUND;
}
int32_t pgs_run_info_get(pgs_partition *ph, uint64_t run_id, pgs_run_info *out)
{
    Partition &p = ph->p;
    std::lock_guard<std::mutex> g(p.mu);
    auto r = p.find(run_id);
    if (!r) return PGS_NOT_FOUND;
    *out = r->info;
    return PGS_OK;
}
int32_t pgs_run_list(pgs_partition *ph, uint64_t *ids, uint32_t cap, uint32_t *n_out)
{
    Partition &p = ph->p;
    std::lock_guard<std::mutex> g(p.mu);
    uint32_t n = (uint32_t)p.runs.size();
    if (n_out) *n_out = n;
    for (uint32_t i = 0; i < n && i < cap; i++) ids[i] = p.runs[i]->id;
    return n <= cap ? PGS_OK : PGS_INCOMPLETE;
}
int32_t pgs_run_download(pgs_partition *ph, uint64_t run_id, uint8_t *data, uint64_t data_cap,
                         uint64_t *blk_off, uint32_t *blk_size, uint32_t blk_cap)
{
    Partition &p = ph->p;
    std::shared_ptr<Run> r;
    {
        std::lock_guard<std::mutex> g(p.mu);
        r = p.find(run_id);
    }
    if (!r) return PGS_NOT_FOUND;
    if (data_cap < r->info.data_bytes || blk_cap < r->info.n_blocks) return PGS_INCOMPLETE;
    Engine *e = p.eng;
    PGS_CUDA(cudaSetDevice(e->device));
    PGS_CUDA(cudaMemcpyAsync(data, r->d_data, r->info.data_bytes, cudaMemcpyDeviceToHost, e->stream));
    PGS_CUDA(cudaMemcpyAsync(blk_off, r->d_blk_off, sizeof(uint64_t) * r->info.n_blocks, cudaMemcpyDeviceToHost, e->stream));
    PGS_CUDA(cudaMemcpyAsync(blk_size, r->d_blk_size, sizeof(uint32_t) * r->info.n_blocks, cudaMemcpyDeviceToHost, e->stream));
    PGS_CUDA(cudaStreamSynchronize(e->stream));
    return PGS_OK;
}

} // extern "C"
