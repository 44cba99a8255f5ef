// engine.cu — device engine plumbing: engine / partition handles, run upload (RocksDB-format
// blocks -> HBM) with the device-built block index, run download, run bookkeeping.
// Replaces for this path: DB::Open (pegasus_server_impl.cpp:1551-1860), flush /
// IngestExternalFile (rocksdb_wrapper.cpp:248-270) as far as "a sorted run appears in the DB".
#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <cstring>

#include "build_kernels.cuh"
#include "engine.h"
#include "index_kernel.cuh"
#include "sort_kernels.cuh"

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
int32_t lookup_init_kernels(Engine &e);
int32_t compact_init_kernels(int max_smem);
int32_t split_init_kernels(int max_smem);

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
    PGS_CUDA(cudaFuncSetAttribute(k_index_walk_many<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    PGS_CUDA(cudaFuncSetAttribute(k_index_walk_many<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
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
    Engine *eng;
    // pinned staging (one allocation): off[nb+1] u64 | blk_size[nb] u32 | nrec[nb] | lastlen[nb] | rec_cum[nb+1] | key_cum[nb+1] | 2 x IndexStats
    void *pin = nullptr;
    size_t pin_cap = 0;
    uint64_t *off = nullptr;
    uint32_t *h_size = nullptr, *nrec = nullptr, *lastlen = nullptr, *rec_cum = nullptr, *key_cum = nullptr;
    IndexStats *hs_in = nullptr, *hs_out = nullptr;
    IndexParams X{};
    LaunchScratch S; // pass 1's device scratch
    std::vector<cudaEvent_t> events;
    cudaEvent_t pass1 = nullptr;
    uint32_t max_blk = 0;
    explicit UploadJob(Engine *e) : eng(e), S(e->stream) {}
    ~UploadJob()
    {
        for (cudaEvent_t ev : events) cudaEventDestroy(ev);
        if (pass1) cudaEventDestroy(pass1);
        if (pin) eng->give_pinned(pin, pin_cap);
    }
};

// the job's pinned staging, its Run and the device buffers of the first pass, for nb blocks that end at `end` (16-aligned)
static int32_t upload_job_init(Engine *e, int32_t level, uint32_t nb, uint64_t end, UploadJob &j)
{
    auto r = std::make_shared<Run>(e);
    j.r = r;
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
    r->info.data_bytes = end;
    cudaStream_t st = e->stream;
    PGS_CUDA(e->alloc_data(*r, end + 256));
    PGS_CUDA(cudaMallocAsync(&r->d_blk_off, sizeof(uint64_t) * (nb + 1), st));
    PGS_CUDA(cudaMallocAsync(&r->d_blk_size, sizeof(uint32_t) * nb, st));
    j.X = IndexParams{r->d_data, r->d_blk_off, r->d_blk_size, nb};
    cudaError_t ce = cudaSuccess;
    index_scratch(j.X, scratch_buffers(j.S, ce));
    PGS_CUDA(ce);
    *j.hs_in = index_stats_init();
    PGS_CUDA(cudaMemcpyAsync(j.X.stats, j.hs_in, sizeof(IndexStats), cudaMemcpyHostToDevice, st));
    return PGS_OK;
}
// after the last first-pass launch: its per-block results come back, j.pass1 marks their arrival
static int32_t upload_pass1_done(Engine *e, UploadJob &j)
{
    const uint32_t nb = j.X.nb;
    cudaStream_t st = e->stream;
    PGS_CUDA(cudaMemcpyAsync(j.nrec, j.X.nrec, sizeof(uint32_t) * nb, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(j.lastlen, j.X.lastlen, sizeof(uint32_t) * nb, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(j.hs_out, j.X.stats, sizeof(IndexStats), cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaEventCreateWithFlags(&j.pass1, cudaEventDisableTiming));
    PGS_CUDA(cudaEventRecord(j.pass1, st));
    return PGS_OK;
}

static int32_t upload_stage_a(Engine *e, int32_t level, const uint8_t *data, uint64_t data_bytes, const uint64_t *blk_off,
                              const uint32_t *blk_size, uint32_t nb, UploadJob &j)
{
    uint64_t prev_end = 0;
    if (const uint32_t b = run_handles_check(blk_off, blk_size, nb, data_bytes, prev_end, j.max_blk); b < nb) {
        set_error("run upload: bad block handle %u", b);
        return PGS_INVALID_ARGUMENT;
    }
    const uint64_t end = block_pad(prev_end);
    const uint64_t nbytes = data_bytes < end ? data_bytes : end;
    if (const int32_t rc = upload_job_init(e, level, nb, end, j)) return rc;
    Run *r = j.r.get();
    cudaStream_t st = e->stream, cp = e->up_copy;
    PGS_CUDA(cudaMemsetAsync(r->d_data + nbytes, 0, r->data_cap - nbytes, st));
    memcpy(j.off, blk_off, sizeof(uint64_t) * nb);
    j.off[nb] = end;
    memcpy(j.h_size, blk_size, sizeof(uint32_t) * nb);
    PGS_CUDA(cudaMemcpyAsync(r->d_blk_off, j.off, sizeof(uint64_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    PGS_CUDA(cudaMemcpyAsync(r->d_blk_size, j.h_size, sizeof(uint32_t) * nb, cudaMemcpyHostToDevice, st));
    cudaEvent_t ready;
    PGS_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    j.events.push_back(ready);
    PGS_CUDA(cudaEventRecord(ready, st)); // the copy stream may touch the new buffers from here on
    PGS_CUDA(cudaStreamWaitEvent(cp, ready, 0));
    uint32_t b0 = 0;
    while (b0 < nb) { // chunks end on block boundaries
        uint32_t b1 = b0 + 1;
        while (b1 < nb && j.off[b1] - j.off[b0] < kUploadChunk) b1++;
        // the first chunk starts at 0: the bytes in front of the first block are the caller's too (pgs_run_download returns them)
        const uint64_t lo = b0 ? j.off[b0] : 0, hi = b1 == nb ? nbytes : std::min<uint64_t>(j.off[b1], nbytes);
        if (hi > lo) PGS_CUDA(cudaMemcpyAsync(r->d_data + lo, data + lo, hi - lo, cudaMemcpyHostToDevice, cp));
        cudaEvent_t ev;
        PGS_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        j.events.push_back(ev);
        PGS_CUDA(cudaEventRecord(ev, cp));
        PGS_CUDA(cudaStreamWaitEvent(st, ev, 0));
        e->launches += index_launch_pass1(j.X, b0, b1, st);
        b0 = b1;
    }
    return upload_pass1_done(e, j);
}

static int32_t upload_stage_b(Engine *e, UploadJob &j)
{
    const uint32_t nb = j.X.nb;
    cudaStream_t st = e->stream;
    PGS_CUDA(cudaEventSynchronize(j.pass1));
    cudaError_t ce = cudaSuccess;
    const int32_t rc = index_buffers(j.X, *j.r, j.nrec, j.lastlen, *j.hs_out, j.rec_cum, j.key_cum, [&](auto *&p, uint64_t n, int fill) {
        const size_t bytes = sizeof(*p) * n;
        if (ce == cudaSuccess) ce = cudaMallocAsync((void **)&p, bytes, st); // ~Run frees the run's buffers
        if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, bytes, st);
    });
    if (rc) return rc;
    PGS_CUDA(ce);
    PGS_CUDA(cudaMemcpyAsync(j.X.blk_rec, j.rec_cum, sizeof(uint32_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    PGS_CUDA(cudaMemcpyAsync(j.X.ikey_off, j.key_cum, sizeof(uint32_t) * (nb + 1), cudaMemcpyHostToDevice, st));
    e->launches += index_launch_pass2(j.X, st);
    PGS_CUDA(cudaEventRecord(j.pass1, st)); // reused: now marks the end of the second pass
    return PGS_OK;
}

static int32_t upload_stage_c(Engine *e, Partition &p, UploadJob &j, uint64_t *run_id_out)
{
    Run *r = j.r.get();
    PGS_CUDA(cudaEventSynchronize(j.pass1));
    run_info_from_index(*j.hs_out, r->info.n_blocks, r->info.data_bytes, j.max_blk, r->info);
    r->id = e->next_run_id++;
    r->info.run_id = r->id;
    {
        std::lock_guard<std::mutex> g(p.mu);
        p.insert(j.r);
    }
    if (run_id_out) *run_id_out = r->id;
    return PGS_OK;
}
// a failed job: nothing of it may still be in flight when its host staging and device buffers go away
static void upload_abandon(Engine *e)
{
    cudaStreamSynchronize(e->up_copy);
    cudaStreamSynchronize(e->stream);
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
    if (err == cudaSuccess && (lookup_init_kernels(e) != PGS_OK || compact_init_kernels(e.max_smem_optin) != PGS_OK ||
                               split_init_kernels(e.max_smem_optin) != PGS_OK || index_init_kernels() != PGS_OK)) {
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
        jobs[i] = std::make_unique<UploadJob>(e);
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
        upload_abandon(e);
        for (uint32_t i = 0; i < done; i++) if (ids[i]) pgs_run_drop(ph, ids[i]);
        return rc;
    }
    if (run_ids_out) for (uint32_t i = 0; i < n; i++) run_ids_out[i] = ids[i];
    return PGS_OK;
}

// device times of the calling thread's last pgs_run_build or pgs_run_build_unsorted: input copy, plan (record, next, chain and
// scan passes), blocks, index; and the sort and gather of the last pgs_run_build_unsorted
static thread_local float t_build_ms[4] = {0, 0, 0, 0};
static thread_local float t_sort_ms = 0;
void pgs_run_build_last_ms(float *ms) { memcpy(ms, t_build_ms, sizeof t_build_ms); }
float pgs_run_build_last_sort_ms(void) { return t_sort_ms; }

// The build from device copies of the records in internal-key order (P's inputs set): its scratch, ev[1], the plan, ev[2], the
// blocks, ev[3], the index, ev[4], and the run installed.  On an error nothing is installed.
static int32_t run_build_sorted(Engine *e, Partition &p, int32_t level, BuildParams &P, LaunchScratch &S, cudaEvent_t *ev,
                                uint64_t *run_id_out)
{
    cudaStream_t st = e->stream;
    cudaError_t ce = cudaSuccess;
    build_buffers(P, scratch_buffers(S, ce));
    PGS_CUDA(ce);
    PGS_CUDA(cudaEventRecord(ev[1], st));
    e->launches += build_launch_plan(P, 0, st, [](int) {});
    size_t pin_cap = 0;
    auto *hsum = (BuildSummary *)e->take_pinned(sizeof(BuildSummary), &pin_cap);
    if (!hsum) { set_error("run build: no pinned staging memory"); return PGS_IO_ERROR; }
    ce = cudaMemcpyAsync(hsum, P.sum, sizeof(BuildSummary), cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaEventRecord(ev[2], st);
    if (ce == cudaSuccess) ce = cudaEventSynchronize(ev[2]);
    const BuildSummary sum = *hsum;
    e->give_pinned(hsum, pin_cap);
    PGS_CUDA(ce);
    if (const int32_t rc = build_status(sum.flags)) {
        set_error(rc == PGS_INVALID_ARGUMENT ? "run build: records out of internal-key order, or offsets out of range"
                                             : "run build: a user key over %u bytes, or a block over 4 GB", kMaxUkeyLen);
        return rc;
    }
    // the blocks are written into the run's buffer, where the upload's passes take them
    const uint32_t nb = (uint32_t)sum.n_blocks;
    UploadJob j(e);
    j.max_blk = sum.max_blk;
    int32_t rc = upload_job_init(e, level, nb, sum.data_bytes, j);
    if (rc == PGS_OK) {
        Run *r = j.r.get();
        P.data = r->d_data;
        ce = cudaMemsetAsync(r->d_data + sum.data_bytes, 0, r->data_cap - sum.data_bytes, st);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->d_blk_off, P.blk_off, sizeof(uint64_t) * (nb + 1), cudaMemcpyDeviceToDevice, st);
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(r->d_blk_size, P.blk_size, sizeof(uint32_t) * nb, cudaMemcpyDeviceToDevice, st);
        if (ce == cudaSuccess) {
            e->launches += build_launch_blocks(P, nb, 0, st);
            ce = cudaEventRecord(ev[3], st);
        }
        rc = ce == cudaSuccess ? PGS_OK : cuda_fail(ce, "run build: blocks");
    }
    if (rc == PGS_OK) {
        e->launches += index_launch_pass1(j.X, 0, nb, st);
        rc = upload_pass1_done(e, j);
    }
    if (rc == PGS_OK) rc = upload_stage_b(e, j);
    if (rc == PGS_OK) {
        ce = cudaEventRecord(ev[4], st);
        rc = ce == cudaSuccess ? upload_stage_c(e, p, j, run_id_out) : cuda_fail(ce, "run build: index");
    }
    if (rc != PGS_OK) upload_abandon(e);
    return rc;
}

int32_t pgs_run_build(pgs_partition *ph, int32_t level, uint64_t n, const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals,
                      const uint64_t *val_off, const uint64_t *seq, const uint8_t *type, uint64_t *run_id_out)
{
    if (!ph || level < 0 || (n && (!key_off || !val_off || !seq || !type))) return PGS_INVALID_ARGUMENT;
    if (n && ((!keys && key_off[n]) || (!vals && val_off[n]))) return PGS_INVALID_ARGUMENT;
    if (run_id_out) *run_id_out = 0;
    memset(t_build_ms, 0, sizeof t_build_ms);
    if (n == 0) return PGS_OK; // an empty run: id 0, nothing resident
    if (n > kBuildMaxRecords) {
        set_error("run build: %llu records exceed the index's 32-bit record offsets", (unsigned long long)n);
        return PGS_NOT_SUPPORTED;
    }
    Partition &p = ph->p;
    Engine *e = p.eng;
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    LaunchScratch S(st);
    cudaEvent_t ev[5];
    for (auto &x : ev) PGS_CUDA(S.event(x));
    PGS_CUDA(cudaEventRecord(ev[0], st));
    // the whole input goes to the device
    BuildParams P{};
    build_plan(P, (uint32_t)n, e->cfg.block_size, e->cfg.restart_interval);
    cudaError_t ce = cudaSuccess;
    stage_records(P, n, keys, key_off, vals, val_off, seq, type, device_buffers(S, ce));
    PGS_CUDA(ce);
    if (const int32_t rc = run_build_sorted(e, p, level, P, S, ev, run_id_out)) return rc;
    if (cudaEventSynchronize(ev[4]) == cudaSuccess)
        for (int i = 0; i < 4; i++) cudaEventElapsedTime(&t_build_ms[i], ev[i], ev[i + 1]);
    return PGS_OK;
}

int32_t pgs_run_build_unsorted(pgs_partition *ph, int32_t level, uint64_t n, const uint8_t *keys, const uint64_t *key_off,
                               const uint8_t *vals, const uint64_t *val_off, const uint64_t *seq, const uint8_t *type,
                               uint64_t *run_id_out)
{
    if (!ph || level < 0 || (n && (!key_off || !val_off || !seq || !type))) return PGS_INVALID_ARGUMENT;
    if (n && ((!keys && key_off[n]) || (!vals && val_off[n]))) return PGS_INVALID_ARGUMENT;
    if (run_id_out) *run_id_out = 0;
    memset(t_build_ms, 0, sizeof t_build_ms);
    t_sort_ms = 0;
    if (n == 0) return PGS_OK; // an empty run: id 0, nothing resident
    if (n > kBuildMaxRecords) {
        const int32_t rc = sort_status_too_many(n, key_off, val_off);
        set_error(rc == PGS_INVALID_ARGUMENT ? "run build: offsets not ascending"
                                             : "run build: %llu records exceed the index's 32-bit record offsets", (unsigned long long)n);
        return rc;
    }
    Partition &p = ph->p;
    Engine *e = p.eng;
    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    LaunchScratch S(st);
    cudaEvent_t ev[5], ev_copied, ev_read;
    for (auto &x : ev) PGS_CUDA(S.event(x));
    PGS_CUDA(S.event(ev_copied));
    PGS_CUDA(S.event(ev_read));
    PGS_CUDA(cudaEventRecord(ev[0], st));
    BuildParams P{};
    build_plan(P, (uint32_t)n, e->cfg.block_size, e->cfg.restart_interval);
    {
        // the input and the sort's scratch are freed (stream-ordered) once the sorted copy is written
        LaunchScratch SS(st);
        SortParams Q{};
        sort_plan(Q, (uint32_t)n);
        cudaError_t ce = cudaSuccess;
        stage_records(Q, n, keys, key_off, vals, val_off, seq, type, device_buffers(SS, ce));
        PGS_CUDA(ce);
        PGS_CUDA(cudaEventRecord(ev_copied, st));
        sort_buffers(Q, key_off[n], val_off[n], scratch_buffers(SS, ce), scratch_buffers(S, ce)); // the sorted copy lives as long as the build's scratch
        PGS_CUDA(ce);
        size_t pin_cap = 0;
        auto *hsum = (SortSummary *)e->take_pinned(sizeof(SortSummary), &pin_cap);
        if (!hsum) { set_error("run build: no pinned staging memory"); return PGS_IO_ERROR; }
        uint32_t launches = 0;
        const int32_t rc = sort_launch(Q, 0, st, [&](SortSummary &s) -> int32_t {
            cudaError_t c = cudaMemcpyAsync(hsum, Q.sum, sizeof(SortSummary), cudaMemcpyDeviceToHost, st);
            if (c == cudaSuccess) c = cudaEventRecord(ev_read, st);
            if (c == cudaSuccess) c = cudaEventSynchronize(ev_read);
            if (c != cudaSuccess) return cuda_fail(c, "run build: sort");
            s = *hsum;
            return PGS_OK;
        }, launches);
        e->give_pinned(hsum, pin_cap);
        e->launches += launches;
        if (rc) {
            if (rc != PGS_IO_ERROR)
                set_error(rc == PGS_INVALID_ARGUMENT ? "run build: offsets out of range, or two records with the same user key, seq and type"
                                                     : "run build: a user key over %u bytes", kMaxUkeyLen);
            return rc;
        }
        build_inputs_sorted(P, Q);
    }
    if (const int32_t rc = run_build_sorted(e, p, level, P, S, ev, run_id_out)) return rc;
    if (cudaEventSynchronize(ev[4]) == cudaSuccess) {
        cudaEventElapsedTime(&t_build_ms[0], ev[0], ev_copied);
        cudaEventElapsedTime(&t_sort_ms, ev_copied, ev[1]);
        for (int i = 1; i < 4; i++) cudaEventElapsedTime(&t_build_ms[i], ev[i], ev[i + 1]);
    }
    return PGS_OK;
}

// The nonempty jobs planned as one record space (build_many_plan) and built in one set of launches: the plan, one wait for the
// summary and every job's status, every job's run allocated, the blocks and index pass 1 over all runs, one wait, index_buffers
// per run, pass 2, one wait, and every run installed under all the partitions' locks.
int32_t pgs_run_build_many(const pgs_run_build_job *jobs, uint32_t n, uint64_t *run_ids_out)
{
    memset(t_build_ms, 0, sizeof t_build_ms);
    if (n == 0) return PGS_OK;
    if (!jobs) { set_error("run build many: %u jobs and no job array", n); return PGS_INVALID_ARGUMENT; }
    if (n > PGS_RUN_BUILD_MANY_MAX_JOBS) { set_error("run build many: %u jobs > %u per call", n, PGS_RUN_BUILD_MANY_MAX_JOBS); return PGS_NOT_SUPPORTED; }
    Engine *e = nullptr;
    std::vector<Partition *> parts(n);
    for (uint32_t i = 0; i < n; i++) {
        const pgs_run_build_job &x = jobs[i];
        if (!x.part || x.level < 0 || (x.n && (!x.key_off || !x.val_off || !x.seq || !x.type)) ||
            (x.n && ((!x.keys && x.key_off[x.n]) || (!x.vals && x.val_off[x.n])))) {
            set_error("run build many: job %u: no partition, a negative level or a missing array", i);
            return PGS_INVALID_ARGUMENT;
        }
        parts[i] = &x.part->p;
        if (!e) e = parts[i]->eng;
        if (parts[i]->eng != e) { set_error("run build many: job %u: its partition is on another engine than job 0's", i); return PGS_INVALID_ARGUMENT; }
    }
    {
        std::vector<Partition *> order = parts;
        std::sort(order.begin(), order.end());
        for (uint32_t i = 1; i < n; i++)
            if (order[i] == order[i - 1]) {
                const uint32_t j = (uint32_t)(std::find(parts.begin(), parts.end(), order[i]) - parts.begin());
                set_error("run build many: job %u: its partition is in another job too", j);
                return PGS_INVALID_ARGUMENT;
            }
    }
    std::vector<const pgs_run_build_job *> J; // the nonempty jobs, and which job each one is
    std::vector<uint32_t> which;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (jobs[i].n > kBuildMaxRecords) {
            set_error("run build many: job %u: %llu records exceed the index's 32-bit record offsets", i, (unsigned long long)jobs[i].n);
            return PGS_NOT_SUPPORTED;
        }
        total += jobs[i].n;
        if (jobs[i].n) { J.push_back(&jobs[i]); which.push_back(i); }
    }
    if (total > kBuildMaxRecords - PGS_RUN_BUILD_MANY_MAX_JOBS) {
        set_error("run build many: %llu records exceed one launch's 32-bit record indices; split the call", (unsigned long long)total);
        return PGS_NOT_SUPPORTED;
    }
    if (run_ids_out) memset(run_ids_out, 0, sizeof(uint64_t) * n);
    const uint32_t jn = (uint32_t)J.size();
    if (jn == 0) return PGS_OK;

    PGS_CUDA(cudaSetDevice(e->device));
    cudaStream_t st = e->stream;
    struct Pinned { // pinned staging of the engine, given back when the call ends
        Engine *e; size_t need; size_t cap = 0; uint8_t *p = (uint8_t *)e->take_pinned(need, &cap);
        ~Pinned() { if (p) e->give_pinned(p, cap); }
    };
    struct Drain { // on an error, nothing of the call may still be in flight when its staging and buffers go
        Engine *e; bool armed = true;
        ~Drain() { if (armed) upload_abandon(e); }
    };
    auto a16 = [](uint64_t x) { return (x + 15) & ~15ull; };
    LaunchScratch S(st);
    std::vector<std::shared_ptr<Run>> runs(jn);
    // the plan's staging: job_rec [jn + 1] | job [jn] | summary | job_out [3 jn] | job_off [jn]
    const uint64_t o_job = a16(4ull * (jn + 1)), o_sum = a16(o_job + sizeof(BuildJob) * jn), o_out = a16(o_sum + sizeof(BuildSummary));
    const uint64_t o_off = a16(o_out + 12ull * jn);
    Pinned pa{e, o_off + 8ull * jn};
    if (!pa.p) { set_error("run build many: no pinned staging memory"); return PGS_IO_ERROR; }
    Drain drain{e};
    uint32_t *job_rec = (uint32_t *)pa.p, *job_out = (uint32_t *)(pa.p + o_out);
    BuildJob *job = (BuildJob *)(pa.p + o_job);
    const BuildSummary &sum = *(const BuildSummary *)(pa.p + o_sum);
    const unsigned long long *job_off = (const unsigned long long *)(pa.p + o_off);
    cudaEvent_t ev[5], ev_read;
    for (auto &x : ev) PGS_CUDA(S.event(x));
    PGS_CUDA(S.event(ev_read));
    PGS_CUDA(cudaEventRecord(ev[0], st));
    BuildManyParams M{};
    build_many_plan(M, J.data(), jn, job_rec, job, e->cfg.block_size, e->cfg.restart_interval);
    cudaError_t ce = cudaSuccess;
    build_many_stage(M, J.data(), job_rec, job, device_buffers(S, ce), [&](const void *dst, const void *src, uint64_t bytes) {
        if (ce == cudaSuccess && bytes) ce = cudaMemcpyAsync((void *)dst, src, bytes, cudaMemcpyHostToDevice, st);
    });
    PGS_CUDA(ce);
    build_many_buffers(M, scratch_buffers(S, ce));
    PGS_CUDA(ce);
    PGS_CUDA(cudaEventRecord(ev[1], st));
    e->launches += build_many_launch_plan(M, 0, st, [](int) {});
    PGS_CUDA(cudaMemcpyAsync(pa.p + o_sum, M.B.sum, sizeof(BuildSummary), cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(job_out, M.job_out, 12ull * jn, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(pa.p + o_off, M.job_off, 8ull * jn, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaEventRecord(ev[2], st));
    PGS_CUDA(cudaEventSynchronize(ev[2]));
    std::vector<uint32_t> nb(jn);
    std::vector<uint64_t> bytes(jn);
    for (uint32_t d = 0; d < jn; d++)
        if (const int32_t rc = build_many_job(M, sum, job_out, job_off, d, nb[d], bytes[d])) {
            if (rc == PGS_INVALID_ARGUMENT) set_error("run build many: job %u: records out of internal-key order, or offsets out of range", which[d]);
            else set_error("run build many: job %u: a user key over %u bytes, or a block over 4 GB", which[d], kMaxUkeyLen);
            return rc;
        }

    // every job's run, and the index staging: nrec [nb] | lastlen [nb] | rec_cum [nb + jn] | key_cum [nb + jn] | then the table
    // the device reads: stats [jn] | out [jn] | X [jn]
    const uint32_t NB = (uint32_t)sum.n_blocks;
    const uint64_t o_rc = 8ull * NB, o_kc = o_rc + 4ull * (NB + jn), o_tab = a16(o_kc + 4ull * (NB + jn));
    const uint64_t t_out = a16(sizeof(IndexStats) * jn), t_x = a16(t_out + sizeof(BuildRunOut) * jn), t_end = t_x + sizeof(IndexParams) * jn;
    Pinned pb{e, o_tab + t_end};
    if (!pb.p) { set_error("run build many: no pinned staging memory"); return PGS_IO_ERROR; }
    Drain drain_b{e};
    uint32_t *h_nrec = (uint32_t *)pb.p, *h_lastlen = h_nrec + NB, *rec_cum = (uint32_t *)(pb.p + o_rc), *key_cum = (uint32_t *)(pb.p + o_kc);
    IndexStats *hs = (IndexStats *)(pb.p + o_tab);
    BuildRunOut *outs = (BuildRunOut *)(pb.p + o_tab + t_out);
    IndexParams *X = (IndexParams *)(pb.p + o_tab + t_x);
    uint32_t *d_nrec = nullptr, *d_lastlen = nullptr;
    uint8_t *d_tab = nullptr;
    PGS_CUDA(S.alloc(d_nrec, 4ull * NB));
    PGS_CUDA(S.alloc(d_lastlen, 4ull * NB));
    PGS_CUDA(S.alloc(d_tab, t_end));
    for (uint32_t d = 0; d < jn; d++) {
        runs[d] = std::make_shared<Run>(e);
        Run &r = *runs[d];
        r.level = r.info.level = J[d]->level;
        PGS_CUDA(e->alloc_data(r, bytes[d] + 256));
        PGS_CUDA(cudaMemsetAsync(r.d_data + bytes[d], 0, r.data_cap - bytes[d], st));
        PGS_CUDA(cudaMallocAsync(&r.d_blk_off, sizeof(uint64_t) * (nb[d] + 1), st));
        PGS_CUDA(cudaMallocAsync(&r.d_blk_size, sizeof(uint32_t) * nb[d], st));
        outs[d] = BuildRunOut{r.d_data, (unsigned long long *)r.d_blk_off, r.d_blk_size};
        X[d] = IndexParams{r.d_data, r.d_blk_off, r.d_blk_size, nb[d]};
        X[d].nrec = d_nrec + job_out[d];
        X[d].lastlen = d_lastlen + job_out[d];
        X[d].stats = (IndexStats *)d_tab + d;
        hs[d] = index_stats_init();
    }
    PGS_CUDA(cudaMemcpyAsync(d_tab, hs, t_end, cudaMemcpyHostToDevice, st));
    M.out = (const BuildRunOut *)(d_tab + t_out);
    const IndexParams *d_X = (const IndexParams *)(d_tab + t_x);
    e->launches += build_many_launch_blocks(M, NB, 0, st);
    PGS_CUDA(cudaEventRecord(ev[3], st));
    e->launches += index_launch_many<false>(d_X, M.job_out, jn, NB, st);
    PGS_CUDA(cudaMemcpyAsync(h_nrec, d_nrec, 4ull * NB, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(h_lastlen, d_lastlen, 4ull * NB, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaMemcpyAsync(hs, d_tab, sizeof(IndexStats) * jn, cudaMemcpyDeviceToHost, st));
    PGS_CUDA(cudaEventRecord(ev_read, st));
    PGS_CUDA(cudaEventSynchronize(ev_read));
    for (uint32_t d = 0; d < jn; d++) {
        const uint32_t b0 = job_out[d];
        const int32_t rc = index_buffers(X[d], *runs[d], h_nrec + b0, h_lastlen + b0, hs[d], rec_cum + b0 + d, key_cum + b0 + d,
                                         [&](auto *&p, uint64_t cnt, int fill) {
                                             const size_t sz = sizeof(*p) * cnt;
                                             if (ce == cudaSuccess) ce = cudaMallocAsync((void **)&p, sz, st); // ~Run frees them
                                             if (ce == cudaSuccess && fill != kNoFill) ce = cudaMemsetAsync(p, fill, sz, st);
                                         });
        if (rc) {
            const std::string m = g_last_error;
            set_error("run build many: job %u: %s", which[d], m.c_str());
            return rc;
        }
        PGS_CUDA(ce);
        PGS_CUDA(cudaMemcpyAsync(X[d].blk_rec, rec_cum + b0 + d, sizeof(uint32_t) * (nb[d] + 1), cudaMemcpyHostToDevice, st));
        PGS_CUDA(cudaMemcpyAsync(X[d].ikey_off, key_cum + b0 + d, sizeof(uint32_t) * (nb[d] + 1), cudaMemcpyHostToDevice, st));
    }
    PGS_CUDA(cudaMemcpyAsync(d_tab + t_x, X, sizeof(IndexParams) * jn, cudaMemcpyHostToDevice, st));
    e->launches += index_launch_many<true>(d_X, M.job_out, jn, NB, st);
    PGS_CUDA(cudaEventRecord(ev[4], st));
    PGS_CUDA(cudaEventSynchronize(ev[4]));
    {
        // all partitions or none: every lock is held, in address order, while the runs go in
        std::vector<Partition *> order;
        for (auto *x : J) order.push_back(&x->part->p);
        std::sort(order.begin(), order.end());
        std::vector<std::unique_lock<std::mutex>> held;
        for (Partition *p : order) held.emplace_back(p->mu);
        for (uint32_t d = 0; d < jn; d++) {
            Run &r = *runs[d];
            run_info_from_index(hs[d], nb[d], bytes[d], job_out[jn + d], r.info);
            r.id = e->next_run_id++;
            r.info.run_id = r.id;
            J[d]->part->p.insert(runs[d]);
            if (run_ids_out) run_ids_out[which[d]] = r.id;
        }
    }
    drain.armed = drain_b.armed = false;
    for (int i = 0; i < 4; i++) cudaEventElapsedTime(&t_build_ms[i], ev[i], ev[i + 1]);
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
