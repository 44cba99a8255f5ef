// server.cpp — the rrdb operator surface of one replica on top of the device engine: the host-side
// mirror of pegasus_server_impl (src/server/pegasus_server_impl.cpp:418-1549 read handlers,
// :2728-3001 app envs, :3373-3456 manual compaction) and of the write path down to the memtable
// (src/server/pegasus_server_write.cpp:92-222, src/server/rocksdb_wrapper.cpp:129-288,
// src/server/pegasus_write_service_impl.h:90-169).  Handlers translate requests into engine calls
// (pgs_get_batch / range scan / pgs_compact); the per-record loops themselves run in CUDA.
//
// Writes land in a host memtable.  Point reads (get / ttl / multi_get with sort keys / batch_get) look there first, like
// DB::Get does (rocksdb_wrapper.cpp:78-127), and send only the misses to the GPU; range reads flush the memtable into an L0
// run first (semantically neutral) so that the iterator loop runs wholly in CUDA.  Scan contexts pin the run set they were
// opened on, like a RocksDB iterator pins its super-version.
// Threading (SURVEY 8b): readers share the replica lock, the single writer / flush / compaction take it exclusively.
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <sys/stat.h>
#include <sstream>
#include <climits>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <random>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../csrc/engine.h"
#include "checkpoint_dir.h"
#include "host_internal.h"

namespace pgs {

constexpr size_t kReadMaxRuns = 12; // a read-triggered flush compacts L0 once the run list grows past this

struct Resp {
    pgs_response view{};
    std::vector<pgs_kv> kvs;
    std::vector<uint32_t> hk_len;
    std::string arena;
    void reset(int32_t app_id, int32_t pidx)
    {
        view = pgs_response{};
        view.app_id = app_id;
        view.partition_index = pidx;
        view.kv_count = -1;
        kvs.clear();
        hk_len.clear();
        arena.clear();
    }
    void add(std::string_view key, std::string_view value, uint32_t expire_ts)
    {
        pgs_kv kv;
        kv.key_off = (uint32_t)arena.size(); kv.key_len = (uint32_t)key.size();
        arena.append(key.data(), key.size());
        kv.value_off = (uint32_t)arena.size(); kv.value_len = (uint32_t)value.size();
        arena.append(value.data(), value.size());
        kv.expire_ts = expire_ts;
        kvs.push_back(kv);
    }
    int32_t seal(int32_t error)
    {
        view.error = error;
        view.n_kvs = (uint32_t)kvs.size();
        view.kvs = kvs.data();
        view.hk_len = hk_len.empty() ? nullptr : hk_len.data();
        view.arena = (const uint8_t *)arena.data();
        view.arena_len = arena.size();
        return error;
    }
};

struct MemRec { uint64_t seq; uint8_t type; std::string value; };

constexpr uint32_t kScanContextTtlSeconds = 300; // pegasus_server_impl.cpp:1377-1385: a parked context expires after 5 minutes

struct ScanContext { // pegasus_scan_context.h:33-95, with the iterator replaced by (pinned runs, resume key)
    std::vector<std::shared_ptr<Run>> runs;
    uint32_t parked_at = 0; // epoch seconds of the call that parked it
    std::string resume, stop;
    bool stop_inclusive, prefix_mode;
    int32_t hash_key_filter_type, sort_key_filter_type;
    std::string hash_key_filter_pattern, sort_key_filter_pattern;
    int32_t batch_size;
    bool no_value, validate_partition_hash, return_expire_ts, only_return_count;
};

struct Server {
    Engine *eng = nullptr;
    pgs_partition *part = nullptr;
    pgs_server_options opt{};
    int32_t app_id = 0, pidx = 0;
    uint32_t data_version = 1;
    uint32_t default_ttl = 0;
    bool validate_partition_hash = false;
    int32_t partition_version = -1;
    std::string ops_bin;
    std::shared_mutex mu; // readers shared; writes, flush, compaction, env updates exclusive
    std::map<std::string, MemRec> mem;
    uint64_t mem_bytes = 0, last_seq = 0;
    int64_t last_committed_decree = 0, last_flushed_decree = 0, last_durable_decree = 0;
    std::mutex ctx_mu; // the scan-context table (touched by readers)
    int64_t ctx_counter = 0;
    uint64_t manual_compact_last_finish_ms = 0; // pegasus_manual_compact_service: _manual_compact_last_finish_time_ms
    bool manual_compact_disabled = false;
    std::unordered_map<int64_t, std::unique_ptr<ScanContext>> ctx;

    uint32_t cfg_scan_count() const { return opt.rocksdb_max_iteration_count ? opt.rocksdb_max_iteration_count : 1000; }
    uint32_t cfg_mget_count() const { return opt.rocksdb_multi_get_max_iteration_count ? opt.rocksdb_multi_get_max_iteration_count : 3000; }
    uint64_t cfg_mget_size() const { return opt.rocksdb_multi_get_max_iteration_size ? opt.rocksdb_multi_get_max_iteration_size : 30ull << 20; }

    pgs_filter_params filter() const
    {
        pgs_filter_params fp{};
        fp.enabled = 1; // enabled once start() knows the data version (pegasus_server_impl.cpp:1780-1784)
        fp.validate_hash = validate_partition_hash;
        fp.data_version = data_version;
        fp.default_ttl = default_ttl;
        fp.pidx = pidx;
        fp.partition_version = partition_version;
        fp.ops = ops_bin.size() > 4 ? (const uint8_t *)ops_bin.data() : nullptr;
        fp.ops_len = (uint32_t)ops_bin.size();
        return fp;
    }
    std::vector<std::shared_ptr<Run>> runs()
    {
        std::lock_guard<std::mutex> g(part->p.mu);
        return part->p.runs;
    }
    int32_t flush_mem()
    {
        if (mem.empty()) return PGS_OK;
        // the memtable (sorted, one version per key) flattened into pinned staging: key_off | val_off | seq | type | keys | values;
        // the device encodes the blocks (pgs_run_build)
        const uint64_t n = mem.size();
        uint64_t kb = 0, vb = 0;
        for (auto &kv : mem) { kb += kv.first.size(); vb += kv.second.value.size(); }
        size_t cap = 0;
        uint8_t *pin = (uint8_t *)eng->take_pinned(8 * (3 * n + 2) + n + kb + vb, &cap);
        if (!pin) { set_error("flush: no pinned staging memory"); return PGS_IO_ERROR; }
        uint64_t *key_off = (uint64_t *)pin, *val_off = key_off + n + 1, *seq = val_off + n + 1;
        uint8_t *type = (uint8_t *)(seq + n), *keys = type + n, *vals = keys + kb;
        uint64_t i = 0, ko = 0, vo = 0;
        for (auto &kv : mem) {
            key_off[i] = ko;
            val_off[i] = vo;
            seq[i] = kv.second.seq;
            type[i] = kv.second.type;
            memcpy(keys + ko, kv.first.data(), kv.first.size());
            memcpy(vals + vo, kv.second.value.data(), kv.second.value.size());
            ko += kv.first.size();
            vo += kv.second.value.size();
            i++;
        }
        key_off[n] = ko;
        val_off[n] = vo;
        uint64_t id = 0;
        int32_t st = pgs_run_build(part, 0, n, keys, key_off, vals, val_off, seq, type, &id);
        eng->give_pinned(pin, cap);
        if (st != PGS_OK) return st;
        mem.clear();
        mem_bytes = 0;
        last_flushed_decree = last_committed_decree; // everything applied so far now lives in an HBM run
        return PGS_OK;
    }
    // L0 (+ the L1 run) -> L1, the engine's stand-in for RocksDB's level0_file_num_compaction_trigger
    int32_t compact_l0(uint32_t now)
    {
        auto rs = runs();
        std::vector<uint64_t> ids;
        for (auto &r : rs)
            if (r->level <= 1) ids.push_back(r->id);
        if (ids.size() < 2) return PGS_OK;
        pgs_filter_params fp = filter();
        return pgs_compact(part, ids.data(), (uint32_t)ids.size(), 1, -1, &fp, now, nullptr);
    }
    int32_t maybe_compact(uint32_t now)
    {
        uint32_t trigger = opt.l0_compaction_trigger ? opt.l0_compaction_trigger : 4;
        uint32_t l0 = 0;
        for (auto &r : runs()) l0 += r->level == 0;
        return l0 >= trigger ? compact_l0(now) : PGS_OK;
    }
    // range reads: the memtable becomes an L0 run, and L0 is folded once the run list grows past kReadMaxRuns, or when the
    // reverse-scan kernel could not stage one block of every run (many L0 runs of small records, such as tombstones)
    bool needs_fold(bool reverse) { return runs().size() > kReadMaxRuns || (reverse && !scan_stages_every_run(part)); }
    bool range_read_needs_prepare(bool reverse) { return !mem.empty() || needs_fold(reverse); }
    int32_t prepare_read(uint32_t now, bool reverse)
    {
        int32_t st = flush_mem();
        if (st != PGS_OK) return st;
        if (needs_fold(reverse)) st = compact_l0(now);
        return st;
    }
    // point reads: newest version in the memtable, if any.  0 = not there, 1 = value, 2 = tombstone
    int mem_get(std::string_view key, std::string_view *value) const
    {
        auto f = mem.find(std::string(key));
        if (f == mem.end()) return 0;
        if (f->second.type != PGS_TYPE_VALUE) return 2;
        *value = f->second.value;
        return 1;
    }
    uint32_t gc_contexts(uint32_t now)
    {
        std::lock_guard<std::mutex> g(ctx_mu);
        uint32_t n = 0;
        for (auto it = ctx.begin(); it != ctx.end();) {
            if (now >= it->second->parked_at && now - it->second->parked_at >= kScanContextTtlSeconds) { it = ctx.erase(it); n++; }
            else ++it;
        }
        return n;
    }
    void mem_write(std::string key, uint8_t type, std::string value, uint32_t now)
    {
        mem_bytes += key.size() + value.size() + 16;
        mem[std::move(key)] = MemRec{++last_seq, type, std::move(value)};
        uint64_t cap = opt.memtable_bytes ? opt.memtable_bytes : 64ull << 20;
        if (mem_bytes >= cap) {
            if (flush_mem() == PGS_OK) maybe_compact(now);
        }
    }
    // write_batch_put_ctx for a local write (rocksdb_wrapper.cpp:129-183): value = header || user data
    void put_one(std::string_view raw_key, std::string_view user, uint32_t expire_ts, uint64_t timestamp_us, uint32_t now)
    {
        if (default_ttl != 0 && expire_ts == 0) expire_ts = now + default_ttl; // db_expire_ts :280-288
        uint64_t timetag = timestamp_us << 8u | (uint64_t)(opt.cluster_id << 1u); // generate_timetag, pegasus_value_schema.h:44-47
        std::string v(user_data_offset(data_version) + user.size(), '\0');
        v[0] = (char)(expire_ts >> 24); v[1] = (char)(expire_ts >> 16); v[2] = (char)(expire_ts >> 8); v[3] = (char)expire_ts;
        if (data_version == 1)
            for (int i = 0; i < 8; i++) v[4 + i] = (char)(timetag >> (56 - 8 * i));
        memcpy(&v[user_data_offset(data_version)], user.data(), user.size());
        mem_write(std::string(raw_key), PGS_TYPE_VALUE, std::move(v), now);
    }

    // one range scan through the engine, growing the output buffers when a result does not fit
    int32_t scan(const pgs_scan_request &rq, uint32_t now, const std::vector<std::shared_ptr<Run>> *pinned, uint64_t size_hint,
                 std::vector<uint8_t> &arena, std::vector<pgs_kv> &kvs, std::string &resume, pgs_scan_result &res)
    {
        uint64_t cap = std::max<uint64_t>(size_hint, 1 << 20);
        uint32_t kv_cap = rq.count_only ? 1 : std::max<uint32_t>(1, std::min<uint32_t>(rq.max_count, 65536));
        for (;;) {
            arena.resize(cap);
            kvs.resize(kv_cap);
            resume.assign(kMaxUkeyLen + 8, '\0');
            const ScanOut out{arena.data(), cap, cap, kvs.data(), kv_cap, kv_cap, (uint8_t *)&resume[0], (uint32_t)resume.size(), nullptr, nullptr};
            int32_t st = scan_many(&part, 1, nullptr, &rq, 1, now, &res, out, pinned);
            if (st == PGS_ABORTED && cap < (4ull << 30)) { // the result did not fit the arena or the record table: grow both
                cap *= 8;
                if (!rq.count_only && kv_cap < rq.max_count) kv_cap = (uint32_t)std::min<uint64_t>((uint64_t)kv_cap * 8, rq.max_count);
                continue;
            }
            if (st != PGS_OK) return st;
            resume.resize(res.iter_valid ? res.resume_len : 0);
            return PGS_OK;
        }
    }
};

// do_manual_compact (pegasus_server_impl.cpp:3373-3456): flush, then CompactRange over the whole column family.
// force=false is BottommostLevelCompaction::kSkip: a DB that already is one bottom run is left alone.
static int32_t do_manual_compact(Server &s, uint32_t now, int32_t target_level, bool force, pgs_compact_result *out)
{
    if (out) memset(out, 0, sizeof *out);
    int32_t st = s.flush_mem(); // flush_all_family_columns(true)
    if (st != PGS_OK) return st;
    auto rs = s.runs();
    if (rs.empty()) return PGS_OK;
    if (!force && rs.size() == 1 && rs[0]->level >= 1) return PGS_OK;
    int32_t level = 1;
    std::vector<uint64_t> ids;
    for (auto &r : rs) { level = std::max(level, r->level); ids.push_back(r->id); }
    if (target_level >= 1) level = target_level;
    while (ids.size() > kMaxRuns) { // deeper than one merge launch: fold the oldest runs first
        std::vector<uint64_t> tail(ids.end() - kMaxRuns, ids.end());
        pgs_filter_params fp = s.filter();
        pgs_compact_result cr{};
        st = pgs_compact(s.part, tail.data(), kMaxRuns, level, 1, &fp, now, &cr);
        if (st != PGS_OK) return st;
        ids.resize(ids.size() - kMaxRuns);
        if (cr.new_run_id) ids.push_back(cr.new_run_id);
    }
    pgs_filter_params fp = s.filter();
    return pgs_compact(s.part, ids.data(), (uint32_t)ids.size(), level, 1, &fp, now, out);
}

static inline std::string_view bsv(const pgs_blob &b) { return std::string_view((const char *)b.data, b.len); }
static inline pgs_blob blob_of(const std::string &s) { return pgs_blob{(const uint8_t *)s.data(), (uint32_t)s.size()}; }
static inline bool filter_type_supported(int32_t t) { return t >= PGS_FT_NO_FILTER && t <= PGS_FT_MATCH_POSTFIX; }

// rocksdb read error -> the replica fails itself on anything but NotFound (replica.cpp:444-459); the
// engine's own failures surface as the same integers.
static int32_t read_fail(Resp &r, int32_t st)
{
    r.kvs.clear();
    r.arena.clear();
    return r.seal(st);
}

using RLock = std::shared_lock<std::shared_mutex>;
// A range read runs on HBM runs only: when the memtable holds anything (or L0 has piled up) the shared lock is traded for
// the exclusive one for the duration of the flush.  Writes that land between the two locks are concurrent with this read.
static int32_t ensure_range_ready(Server &s, RLock &lk, uint32_t now, bool reverse = false)
{
    if (!s.range_read_needs_prepare(reverse)) return PGS_OK;
    lk.unlock();
    int32_t st;
    {
        std::unique_lock<std::shared_mutex> w(s.mu);
        st = s.prepare_read(now, reverse);
    }
    lk.lock();
    return st;
}

// Point lookups of n raw keys: the memtable answers what it holds (newest version wins over every run), the rest goes to
// the GPU in one pgs_get_batch.  res[i].value_off/value_len index `arena` (grown as needed).
// capture: every key is captured once by the READ hot-key collector with weight 1 -- here when the memtable answers it, on
// the device (k_hotkey_capture) when it goes to the GPU; handlers with weights of their own pass false.
static int32_t point_lookup(Server &s, const std::vector<std::string> &keys, uint32_t now, std::vector<pgs_get_result> &res,
                            std::vector<uint8_t> &arena, bool capture = true)
{
    const uint32_t n = (uint32_t)keys.size();
    res.assign(n, pgs_get_result{});
    arena.clear();
    const uint32_t hdr = user_data_offset(s.data_version);
    std::vector<uint32_t> miss;
    for (uint32_t i = 0; i < n; i++) {
        std::string_view v;
        const int m = s.mem_get(keys[i], &v);
        if (m == 0) { miss.push_back(i); continue; }
        if (capture) s.part->p.hk_read.capture_raw_key(keys[i], 1);
        pgs_get_result &r = res[i];
        r.status = PGS_NOT_FOUND;
        if (m == 2) continue; // tombstone
        r.expire_ts = v.size() >= 4 ? be32((const uint8_t *)v.data()) : 0;
        if (ts_expired(now, r.expire_ts)) { r.expired = 1; continue; }
        r.status = PGS_OK;
        r.value_off = (uint32_t)arena.size();
        r.value_len = v.size() >= hdr ? (uint32_t)(v.size() - hdr) : 0;
        arena.insert(arena.end(), v.begin() + (v.size() >= hdr ? hdr : v.size()), v.end());
    }
    if (miss.empty()) return PGS_OK;
    std::string flat;
    std::vector<uint32_t> off(1, 0);
    for (uint32_t i : miss) { flat += keys[i]; off.push_back((uint32_t)flat.size()); }
    std::vector<pgs_get_result> gr(miss.size());
    std::vector<uint8_t> dev(std::max<size_t>(1 << 16, miss.size() * 512));
    uint64_t used = 0;
    int32_t st;
    for (;;) {
        st = get_batch(s.part, (const uint8_t *)flat.data(), off.data(), (uint32_t)miss.size(), now, dev.data(), dev.size(), gr.data(), &used,
                       capture && !used); // a retry with a larger arena captures nothing again
        if (st == PGS_INCOMPLETE && used > dev.size()) { dev.resize(used + 64); continue; }
        break;
    }
    if (st != PGS_OK) return st;
    const uint32_t base = (uint32_t)arena.size();
    arena.insert(arena.end(), dev.begin(), dev.begin() + used);
    for (size_t j = 0; j < miss.size(); j++) {
        res[miss[j]] = gr[j];
        if (gr[j].status == PGS_OK) res[miss[j]].value_off += base;
    }
    return PGS_OK;
}

// ---- on_get / on_ttl (pegasus_server_impl.cpp:418-494, 1088-1149) --------------------------------------
static int32_t do_get(Server &s, std::string_view key, uint32_t now, Resp &r, bool ttl_only)
{
    r.reset(s.app_id, s.pidx);
    std::vector<pgs_get_result> grv;
    std::vector<uint8_t> arena;
    int32_t st = point_lookup(s, {std::string(key)}, now, grv, arena);
    if (st != PGS_OK) return read_fail(r, st);
    const pgs_get_result &gr = grv[0];
    if (gr.expired) r.view.expire_count = 1;
    if (gr.status != PGS_OK) return r.seal(PGS_NOT_FOUND);
    if (ttl_only) {
        r.view.ttl_seconds = gr.expire_ts > 0 ? (int32_t)(gr.expire_ts - now) : -1;
        return r.seal(PGS_OK);
    }
    r.add(std::string_view(), std::string_view((const char *)arena.data() + gr.value_off, gr.value_len), 0);
    return r.seal(PGS_OK);
}

// ---- on_multi_get (:496-904) ----------------------------------------------------------------------------------
static int32_t do_multi_get(Server &s, RLock &lk, const pgs_multi_get_request &q, uint32_t now, Resp &r)
{
    r.reset(s.app_id, s.pidx);
    if (!filter_type_supported(q.sort_key_filter_type)) return r.seal(PGS_INVALID_ARGUMENT);
    int32_t st = q.n_sort_keys == 0 ? ensure_range_ready(s, lk, now, q.reverse != 0) : PGS_OK;
    if (st != PGS_OK) return read_fail(r, st);
    uint32_t max_kv_count = s.cfg_mget_count(), max_iteration_count = s.cfg_mget_count();
    if (q.max_kv_count > 0 && (uint32_t)q.max_kv_count < max_kv_count) max_kv_count = q.max_kv_count;
    int32_t max_kv_size = q.max_kv_size > 0 ? q.max_kv_size : INT_MAX;
    int32_t max_iteration_size_config = s.cfg_mget_size() > 0 ? (int32_t)std::min<uint64_t>(s.cfg_mget_size(), INT_MAX) : INT_MAX;
    int32_t max_iteration_size = std::min(max_kv_size, max_iteration_size_config);
    std::string_view hash_key = bsv(q.hash_key);

    if (q.n_sort_keys == 0) {
        std::string start = make_key(hash_key, bsv(q.start_sortkey));
        bool start_inclusive = q.start_inclusive;
        std::string stop;
        bool stop_inclusive;
        if (q.stop_sortkey.len == 0) { stop = make_next(make_key(hash_key, {})); stop_inclusive = false; }
        else { stop = make_key(hash_key, bsv(q.stop_sortkey)); stop_inclusive = q.stop_inclusive; }
        if (q.sort_key_filter_type == PGS_FT_MATCH_PREFIX && q.sort_key_filter_pattern.len > 0) { // :558-578
            std::string ps = make_key(hash_key, bsv(q.sort_key_filter_pattern));
            std::string pe = make_next(ps);
            if (std::string_view(ps).compare(start) > 0) { start = ps; start_inclusive = true; }
            if (std::string_view(pe).compare(stop) <= 0) { stop = pe; stop_inclusive = false; }
        }
        int c = std::string_view(start).compare(stop);
        if (c > 0 || (c == 0 && (!start_inclusive || !stop_inclusive))) return r.seal(PGS_OK); // :581-607
        pgs_scan_request rq{};
        rq.start = blob_of(start);
        rq.stop = blob_of(stop);
        rq.start_inclusive = start_inclusive;
        rq.stop_inclusive = stop_inclusive;
        rq.reverse = q.reverse;
        rq.no_value = q.no_value;
        rq.key_mode = 1;
        rq.prefix_same_as_start = s.opt.prefix_filter && !q.reverse; // reverse: total_order_seek (:679-688)
        rq.sort_filter_type = q.sort_key_filter_type;
        rq.sort_filter = q.sort_key_filter_pattern;
        rq.max_count = max_kv_count;
        rq.max_iter_count = max_iteration_count;
        rq.max_iter_size = (uint64_t)max_iteration_size;
        rq.pidx = s.pidx;
        rq.partition_version = s.partition_version;
        std::vector<uint8_t> arena;
        std::vector<pgs_kv> kvs;
        std::string resume;
        pgs_scan_result res{};
        st = s.scan(rq, now, nullptr, 0, arena, kvs, resume, res);
        if (st != PGS_OK) return read_fail(r, st);
        if (res.status != PGS_OK) return read_fail(r, res.status);
        for (uint32_t i = 0; i < res.n_kvs; i++) { // reverse mode: re-reverse so that kvs ascend by sort key (:758-764)
            const pgs_kv &kv = kvs[q.reverse ? res.n_kvs - 1 - i : i];
            r.add(std::string_view((const char *)arena.data() + kv.key_off, kv.key_len),
                  std::string_view((const char *)arena.data() + kv.value_off, kv.value_len), 0);
        }
        r.view.iteration_count = res.iter_count;
        r.view.expire_count = res.expire_count;
        r.view.filter_count = res.filter_count;
        return r.seal(res.iter_valid && !res.complete ? PGS_INCOMPLETE : PGS_OK); // :777-787
    }
    // sort_keys given: MultiGet (:789-864)
    std::vector<std::string> keys;
    for (uint32_t i = 0; i < q.n_sort_keys; i++) keys.push_back(make_key(hash_key, bsv(q.sort_keys[i])));
    std::vector<pgs_get_result> gr;
    std::vector<uint8_t> arena;
    st = point_lookup(s, keys, now, gr, arena, false);
    if (st != PGS_OK) return read_fail(r, st);
    int32_t count = 0;
    int64_t size = 0;
    bool exceed_limit = false;
    for (uint32_t i = 0; i < q.n_sort_keys; i++) {
        if (gr[i].expired) { r.view.expire_count++; continue; }
        if (gr[i].status != PGS_OK) continue;
        if (count >= (int32_t)max_kv_count || size >= max_kv_size) { exceed_limit = true; break; }
        std::string_view v = q.no_value ? std::string_view() : std::string_view((const char *)arena.data() + gr[i].value_off, gr[i].value_len);
        r.add(bsv(q.sort_keys[i]), v, 0);
        count++;
        size += q.sort_keys[i].len + v.size();
    }
    return r.seal(exceed_limit ? PGS_INCOMPLETE : PGS_OK);
}

// ---- on_batch_get (:906-1016) ---------------------------------------------------------------------------------
static int32_t do_batch_get(Server &s, const pgs_full_key *fk, uint32_t n, uint32_t now, Resp &r)
{
    r.reset(s.app_id, s.pidx);
    if (n == 0) return r.seal(PGS_INVALID_ARGUMENT);
    std::vector<std::string> keys;
    for (uint32_t i = 0; i < n; i++) keys.push_back(make_key(bsv(fk[i].hash_key), bsv(fk[i].sort_key)));
    std::vector<pgs_get_result> gr;
    std::vector<uint8_t> arena;
    int32_t st = point_lookup(s, keys, now, gr, arena, false);
    if (st != PGS_OK) return read_fail(r, st);
    for (uint32_t i = 0; i < n; i++) {
        if (gr[i].expired) { r.view.expire_count++; continue; }
        if (gr[i].status != PGS_OK) continue;
        std::string hs(bsv(fk[i].hash_key));
        hs += bsv(fk[i].sort_key);
        r.add(hs, std::string_view((const char *)arena.data() + gr[i].value_off, gr[i].value_len), 0);
        r.hk_len.push_back(fk[i].hash_key.len);
    }
    return r.seal(PGS_OK);
}

// ---- on_sortkey_count (:1018-1086) --------------------------------------------------------------------------------
static int32_t do_sortkey_count(Server &s, RLock &lk, std::string_view hash_key, uint32_t now, Resp &r)
{
    r.reset(s.app_id, s.pidx);
    int32_t st = ensure_range_ready(s, lk, now);
    if (st != PGS_OK) return read_fail(r, st);
    std::string start = make_key(hash_key, {}), stop = make_next(start);
    pgs_scan_request rq{};
    rq.start = blob_of(start);
    rq.stop = blob_of(stop);
    rq.start_inclusive = 1;
    rq.stop_inclusive = 0;
    rq.count_only = 1;
    rq.reserved[0] = 1; // iterate_upper_bound = stop
    rq.prefix_same_as_start = s.opt.prefix_filter;
    rq.max_count = UINT32_MAX; // the loop is only time limited (:1052)
    rq.max_iter_count = UINT32_MAX;
    rq.pidx = s.pidx;
    rq.partition_version = s.partition_version;
    std::vector<uint8_t> arena;
    std::vector<pgs_kv> kvs;
    std::string resume;
    pgs_scan_result res{};
    st = s.scan(rq, now, nullptr, 0, arena, kvs, resume, res);
    if (st != PGS_OK) return read_fail(r, st);
    if (res.status != PGS_OK) { r.view.count = 0; return read_fail(r, res.status); }
    r.view.count = res.count;
    r.view.iteration_count = res.iter_count;
    r.view.expire_count = res.expire_count;
    return r.seal(PGS_OK);
}

// ---- on_get_scanner / on_scan (:1151-1547) ----------------------------------------------------------------------------
static int32_t scan_batch(Server &s, std::unique_ptr<ScanContext> ctx, bool start_inclusive, uint32_t limiter_max, uint32_t now, Resp &r)
{
    uint32_t batch_count = s.cfg_scan_count();
    if (ctx->batch_size > 0 && (uint32_t)ctx->batch_size < batch_count) batch_count = ctx->batch_size;
    pgs_scan_request rq{};
    rq.start = blob_of(ctx->resume);
    rq.stop = blob_of(ctx->stop);
    rq.start_inclusive = start_inclusive;
    rq.stop_inclusive = ctx->stop_inclusive;
    rq.no_value = ctx->no_value;
    rq.key_mode = 0;
    rq.return_expire_ts = ctx->return_expire_ts;
    rq.count_only = ctx->only_return_count;
    rq.validate_hash = ctx->validate_partition_hash && s.validate_partition_hash; // request flag && server flag (:2397)
    rq.prefix_same_as_start = ctx->prefix_mode;
    rq.hash_filter_type = ctx->hash_key_filter_type;
    rq.sort_filter_type = ctx->sort_key_filter_type;
    rq.hash_filter = blob_of(ctx->hash_key_filter_pattern);
    rq.sort_filter = blob_of(ctx->sort_key_filter_pattern);
    rq.max_count = batch_count;
    rq.max_iter_count = limiter_max ? limiter_max : batch_count;
    rq.max_iter_size = 0;
    rq.pidx = s.pidx;
    rq.partition_version = s.partition_version;
    std::vector<uint8_t> arena;
    std::vector<pgs_kv> kvs;
    std::string resume;
    pgs_scan_result res{};
    int32_t st = s.scan(rq, now, &ctx->runs, 0, arena, kvs, resume, res);
    if (st != PGS_OK) return read_fail(r, st);
    if (res.status != PGS_OK) return read_fail(r, res.status);
    for (uint32_t i = 0; i < res.n_kvs; i++)
        r.add(std::string_view((const char *)arena.data() + kvs[i].key_off, kvs[i].key_len),
              std::string_view((const char *)arena.data() + kvs[i].value_off, kvs[i].value_len), kvs[i].expire_ts);
    if (ctx->only_return_count) r.view.kv_count = (int32_t)res.count;
    r.view.iteration_count = res.iter_count;
    r.view.expire_count = res.expire_count;
    r.view.filter_count = res.filter_count;
    if (res.iter_valid && !res.complete) { // park the cursor (:1360-1387); it expires after 5 minutes (:1377-1385)
        ctx->resume = resume;
        ctx->parked_at = now;
        std::lock_guard<std::mutex> g(s.ctx_mu);
        int64_t handle = s.ctx_counter++;
        s.ctx[handle] = std::move(ctx);
        r.view.context_id = handle;
    } else {
        r.view.context_id = -1; // SCAN_CONTEXT_ID_COMPLETED
    }
    return r.seal(PGS_OK);
}

static int32_t do_get_scanner(Server &s, RLock &lk, const pgs_get_scanner_request &q, uint32_t now, Resp &r)
{
    r.reset(s.app_id, s.pidx);
    s.gc_contexts(now);
    if (!filter_type_supported(q.hash_key_filter_type) || !filter_type_supported(q.sort_key_filter_type))
        return r.seal(PGS_INVALID_ARGUMENT);
    int32_t st = ensure_range_ready(s, lk, now);
    if (st != PGS_OK) return read_fail(r, st);
    bool prefix_mode = s.opt.prefix_filter;
    if (s.opt.prefix_filter) { // :1188-1198
        uint32_t hl = q.start_key.len >= 2 ? be16(q.start_key.data) : 0;
        if (hl == 0 || q.full_scan) prefix_mode = false; // total_order_seek
    }
    bool start_inclusive = q.start_inclusive;
    std::string start(bsv(q.start_key)), stop(bsv(q.stop_key));
    if (q.hash_key_filter_type == PGS_FT_MATCH_PREFIX && q.hash_key_filter_pattern.len > 0) { // :1207-1223
        std::string ps = make_key(bsv(q.hash_key_filter_pattern), {});
        if (std::string_view(ps).compare(start) > 0) { start = ps; start_inclusive = true; }
    }
    int c = std::string_view(start).compare(stop);
    if (c > 0 || (c == 0 && (!start_inclusive || !q.stop_inclusive))) return r.seal(PGS_OK); // empty range, context_id default
    auto ctx = std::make_unique<ScanContext>();
    ctx->runs = s.runs();
    ctx->resume = start;
    ctx->stop = stop;
    ctx->stop_inclusive = q.stop_inclusive;
    ctx->prefix_mode = prefix_mode;
    ctx->hash_key_filter_type = q.hash_key_filter_type;
    ctx->sort_key_filter_type = q.sort_key_filter_type;
    ctx->hash_key_filter_pattern = std::string(bsv(q.hash_key_filter_pattern));
    ctx->sort_key_filter_pattern = std::string(bsv(q.sort_key_filter_pattern));
    uint32_t batch_count = s.cfg_scan_count();
    if (q.batch_size > 0 && (uint32_t)q.batch_size < batch_count) batch_count = q.batch_size;
    ctx->batch_size = (int32_t)batch_count;
    ctx->no_value = q.no_value;
    ctx->validate_partition_hash = q.validate_partition_hash;
    ctx->return_expire_ts = q.return_expire_ts;
    ctx->only_return_count = q.only_return_count;
    // on_get_scanner's limiter counts up to rocksdb_max_iteration_count, on_scan's up to batch_count (:1252-1266 vs :1434-1442)
    return scan_batch(s, std::move(ctx), start_inclusive, s.cfg_scan_count(), now, r);
}

static int32_t do_scan(Server &s, int64_t context_id, uint32_t now, Resp &r)
{
    r.reset(s.app_id, s.pidx);
    s.gc_contexts(now);
    std::unique_ptr<ScanContext> ctx;
    {
        std::lock_guard<std::mutex> g(s.ctx_mu);
        auto f = s.ctx.find(context_id);
        if (f == s.ctx.end()) return r.seal(PGS_NOT_FOUND); // :1542-1544 (unknown, cleared or expired)
        ctx = std::move(f->second);
        s.ctx.erase(f);
    }
    return scan_batch(s, std::move(ctx), true, 0, now, r);
}

static void parse_envs(const char *envs, uint32_t n, std::vector<std::pair<std::string, std::string>> &out)
{
    const char *p = envs;
    for (uint32_t i = 0; i < n; i++) {
        std::string k(p);
        p += k.size() + 1;
        std::string v(p);
        p += v.size() + 1;
        out.emplace_back(std::move(k), std::move(v));
    }
}

} // namespace pgs

using namespace pgs;
struct pgs_server { Server s; };
struct pgs_response_buf { Resp r; };

extern "C" {

pgs_response_buf *pgs_response_new(void) { return new pgs_response_buf; }
void pgs_response_free(pgs_response_buf *r) { delete r; }
const pgs_response *pgs_response_view(pgs_response_buf *r) { return &r->r.view; }

int32_t pgs_rrdb_update_app_envs(pgs_server *h, const char *envs, uint32_t n_envs, uint32_t now)
{
    Server &s = h->s;
    std::unique_lock<std::shared_mutex> g(s.mu);
    std::vector<std::pair<std::string, std::string>> kv;
    if (envs && n_envs) parse_envs(envs, n_envs, kv);
    // update_app_envs hands over the table's whole env map (pegasus_server_impl.cpp:2728-2741): an absent key means "deleted"
    {
        std::map<std::string, std::string> em(kv.begin(), kv.end());
        auto fd = em.find("default_ttl"); // update_default_ttl :2814-2826: buf2int32 and >= 0, otherwise the old value stays
        if (fd != em.end()) {
            char *endp = nullptr;
            errno = 0;
            const long long v = strtoll(fd->second.c_str(), &endp, 10);
            if (!fd->second.empty() && !*endp && errno == 0 && v >= 0 && v <= INT32_MAX) s.default_ttl = (uint32_t)v;
        }
        auto fv = em.find("replica.split.validate_partition_hash"); // :2966-2983: absent -> false, unparsable -> unchanged (buf2bool)
        if (fv == em.end()) s.validate_partition_hash = false;
        else {
            std::string v = fv->second;
            for (auto &c : v) c = (char)tolower((unsigned char)c);
            if (v == "true") s.validate_partition_hash = true;
            else if (v == "false") s.validate_partition_hash = false;
        }
        auto fo = em.find("user_specified_compaction"); // :2985-3001: absent -> cleared
        if (fo == em.end()) s.ops_bin.clear();
        else { s.ops_bin.clear(); if (!fo->second.empty() && ops_parse(fo->second, s.data_version, s.ops_bin, nullptr) < 0) s.ops_bin.clear(); }
    }
    // start_manual_compact_if_needed (pegasus_manual_compact_service.cpp:83-121): the disabled flag, the running-count limit, then
    // the `once` rule and, when it does not fire, the `periodic` one (times of the local day that holds `now`); the compaction
    // runs inside this call, so check_manual_compact_state's "one is already queued" never applies.  Levels: 0..6.
    pgs_manual_compact_decision dec;
    const uint64_t now_ms = ((uint64_t)now + kEpochBegin) * 1000;
    if (pgs_manual_compact_decide(envs, envs ? n_envs : 0, now_ms, s.manual_compact_last_finish_ms, -1, 6, &dec) != PGS_OK) return PGS_OK;
    s.manual_compact_disabled = dec.disabled != 0;
    if (dec.rule == 0) return PGS_OK;
    if (dec.rule == 2 && now == 0) return PGS_OK; // a call without a clock (pgs_rrdb_start) cannot tell the time of day
    const int32_t target_level = dec.target_level;
    const bool force = dec.bottommost_force != 0;
    int32_t st = do_manual_compact(s, now, target_level, force, nullptr);
    if (st == PGS_OK) s.manual_compact_last_finish_ms = ((uint64_t)now + kEpochBegin) * 1000;
    return st;
}

int32_t pgs_rrdb_start(pgs_engine *e, int32_t app_id, int32_t pidx, const pgs_server_options *opt, const char *envs,
                       uint32_t n_envs, pgs_server **out)
{
    if (!e || !out) return PGS_INVALID_ARGUMENT;
    auto *h = new pgs_server;
    Server &s = h->s;
    s.eng = &e->e;
    s.app_id = app_id;
    s.pidx = pidx;
    if (opt) s.opt = *opt; else s.opt.prefix_filter = 1;
    if (!s.opt.cluster_id) s.opt.cluster_id = 1;
    HotkeyConfig hc;
    if (!hotkey_config(s.opt.hotkey_buckets_num, s.opt.hot_bucket_variance_threshold, s.opt.hot_key_variance_threshold,
                       s.opt.max_seconds_to_detect_hotkey, hc)) {
        set_error("rrdb_start: hotkey_buckets_num %u is not a prime >= 3", s.opt.hotkey_buckets_num);
        delete h;
        return PGS_INVALID_ARGUMENT;
    }
    int32_t st = pgs_partition_create(e, app_id, pidx, s.data_version, &s.part);
    if (st != PGS_OK) { delete h; return st; }
    s.part->p.hk_read.set_config(hc);
    s.part->p.hk_write.set_config(hc);
    std::mt19937_64 rng(std::random_device{}());
    s.ctx_counter = (int64_t)(rng() % (1ull << 31)) << 32; // pegasus_scan_context.h:113-114, kept non-negative
    if (envs && n_envs) pgs_rrdb_update_app_envs(h, envs, n_envs, 0);
    *out = h;
    return PGS_OK;
}
void pgs_rrdb_stop(pgs_server *h)
{
    if (!h) return;
    h->s.ctx.clear();
    pgs_partition_destroy(h->s.part);
    delete h;
}
pgs_partition *pgs_rrdb_partition(pgs_server *h) { return h->s.part; }
void pgs_rrdb_set_partition_version(pgs_server *h, int32_t pv) { h->s.partition_version = pv; }

#define RLOCKED(h) RLock _g((h)->s.mu)
#define WLOCKED(h) std::unique_lock<std::shared_mutex> _g((h)->s.mu)
int32_t pgs_rrdb_get(pgs_server *h, pgs_blob key, uint32_t now, pgs_response_buf *r) { RLOCKED(h); return do_get(h->s, bsv(key), now, r->r, false); }
int32_t pgs_rrdb_ttl(pgs_server *h, pgs_blob key, uint32_t now, pgs_response_buf *r) { RLOCKED(h); return do_get(h->s, bsv(key), now, r->r, true); }
// the READ collector's captures of these handlers (capacity_unit_calculator.cpp:179-269) follow their responses
int32_t pgs_rrdb_multi_get(pgs_server *h, const pgs_multi_get_request *q, uint32_t now, pgs_response_buf *r)
{
    RLOCKED(h);
    const int32_t st = do_multi_get(h->s, _g, *q, now, r->r);
    if (st == PGS_OK || st == PGS_NOT_FOUND || st == PGS_INCOMPLETE || st == PGS_INVALID_ARGUMENT)
        h->s.part->p.hk_read.capture_hash_key(bsv(q->hash_key), r->r.view.n_kvs); // weight = kvs returned
    return st;
}
int32_t pgs_rrdb_batch_get(pgs_server *h, const pgs_full_key *k, uint32_t n, uint32_t now, pgs_response_buf *r)
{
    RLOCKED(h);
    const int32_t st = do_batch_get(h->s, k, n, now, r->r);
    for (uint32_t i = 0; i < r->r.view.n_kvs; i++) // the hash key of every returned record, weight 1
        h->s.part->p.hk_read.capture_hash_key(std::string_view(r->r.arena.data() + r->r.kvs[i].key_off, r->r.hk_len[i]), 1);
    return st;
}
int32_t pgs_rrdb_sortkey_count(pgs_server *h, pgs_blob hk, uint32_t now, pgs_response_buf *r)
{
    RLOCKED(h);
    const int32_t st = do_sortkey_count(h->s, _g, bsv(hk), now, r->r);
    if (st == PGS_OK || st == PGS_NOT_FOUND) h->s.part->p.hk_read.capture_hash_key(bsv(hk), 1);
    return st;
}
int32_t pgs_rrdb_get_scanner(pgs_server *h, const pgs_get_scanner_request *q, uint32_t now, pgs_response_buf *r) { RLOCKED(h); return do_get_scanner(h->s, _g, *q, now, r->r); }
int32_t pgs_rrdb_scan(pgs_server *h, int64_t context_id, uint32_t now, pgs_response_buf *r) { RLOCKED(h); return do_scan(h->s, context_id, now, r->r); }
void pgs_rrdb_clear_scanner(pgs_server *h, int64_t context_id) { std::lock_guard<std::mutex> g(h->s.ctx_mu); h->s.ctx.erase(context_id); }
uint32_t pgs_rrdb_gc(pgs_server *h, uint32_t now) { return h->s.gc_contexts(now); }

int32_t pgs_rrdb_detect_hotkey(pgs_server *h, int32_t type, int32_t action, uint32_t now_s, char *result_buf, uint32_t cap, uint32_t *result_len)
{
    if (!h) return PGS_HOTKEY_INVALID_PARAMETERS;
    std::string text;
    const int32_t out = hotkey_control(h->s.part->p, type, action, now_s, text);
    if (result_buf && cap) memcpy(result_buf, text.data(), std::min<size_t>(cap, text.size()));
    if (result_len) *result_len = (uint32_t)text.size();
    return out;
}
int32_t pgs_rrdb_hotkey_analyse(pgs_server *h, uint32_t now_s) { return h ? hotkey_analyse(h->s.part->p, now_s) : PGS_INVALID_ARGUMENT; }
int32_t pgs_rrdb_hotkey_state(pgs_server *h, int32_t type)
{
    if (!h || (type != PGS_HOTKEY_READ && type != PGS_HOTKEY_WRITE)) return -1;
    return (int32_t)(type == PGS_HOTKEY_READ ? h->s.part->p.hk_read : h->s.part->p.hk_write).state();
}

int32_t pgs_rrdb_get_many(pgs_server *h, const uint8_t *keys, const uint32_t *key_off, uint32_t n, uint32_t now,
                          uint8_t *arena, uint64_t arena_cap, pgs_get_result *results, uint64_t *arena_used)
{
    RLOCKED(h);
    Server &s = h->s;
    if (s.mem.empty()) return pgs_get_batch(s.part, keys, key_off, n, now, arena, arena_cap, results, arena_used);
    // some keys may live in the memtable: answer those on the host, send the rest to the GPU
    std::vector<std::string> ks;
    for (uint32_t i = 0; i < n; i++) ks.emplace_back((const char *)keys + key_off[i], key_off[i + 1] - key_off[i]);
    std::vector<pgs_get_result> gr;
    std::vector<uint8_t> ar;
    int32_t st = point_lookup(s, ks, now, gr, ar);
    if (st != PGS_OK) return st;
    if (arena_used) *arena_used = ar.size();
    memcpy(results, gr.data(), sizeof(pgs_get_result) * n);
    if (ar.size() > arena_cap) return PGS_INCOMPLETE;
    if (!ar.empty()) memcpy(arena, ar.data(), ar.size());
    return PGS_OK;
}

int32_t pgs_rrdb_put(pgs_server *h, pgs_blob key, pgs_blob value, uint32_t expire_ts, int64_t decree,
                     uint64_t timestamp_us, uint32_t now)
{
    WLOCKED(h);
    h->s.last_committed_decree = decree;
    h->s.put_one(bsv(key), bsv(value), expire_ts, timestamp_us, now);
    h->s.part->p.hk_write.capture_raw_key(bsv(key), 1);
    return PGS_OK;
}
int32_t pgs_rrdb_remove(pgs_server *h, pgs_blob key, int64_t decree, uint32_t now)
{
    WLOCKED(h);
    h->s.last_committed_decree = decree;
    h->s.mem_write(std::string(bsv(key)), PGS_TYPE_DELETION, std::string(), now);
    h->s.part->p.hk_write.capture_raw_key(bsv(key), 1);
    return PGS_OK;
}
int32_t pgs_rrdb_on_batched_writes(pgs_server *h, const pgs_write_request *reqs, uint32_t count, int64_t decree, uint64_t timestamp_us,
                                   uint32_t now, int32_t *resp_errors)
{
    if (!h || (count && !reqs)) return PGS_INVALID_ARGUMENT;
    for (uint32_t i = 0; i < count; i++)
        if (reqs[i].op > 1) return PGS_INVALID_ARGUMENT; // not batchable: nothing of the batch is applied
    WLOCKED(h);
    Server &s = h->s;
    s.last_committed_decree = decree;
    if (count == 0) { s.put_one({}, {}, 0, timestamp_us, now); return PGS_OK; } // RPC_REPLICATION_WRITE_EMPTY
    for (uint32_t i = 0; i < count; i++) {
        if (reqs[i].op == 0) s.put_one(bsv(reqs[i].raw_key), bsv(reqs[i].value), reqs[i].expire_ts_seconds, timestamp_us, now);
        else s.mem_write(std::string(bsv(reqs[i].raw_key)), PGS_TYPE_DELETION, std::string(), now);
        s.part->p.hk_write.capture_raw_key(bsv(reqs[i].raw_key), 1);
        if (resp_errors) resp_errors[i] = PGS_OK;
    }
    return PGS_OK;
}
// dsn::buf2int64 (src/utils/string_conv.h:35-62): the whole buffer is one integer for strtoll with base 0 (decimal, 0x.., 0..)
static bool buf2int64(std::string_view buf, int64_t &out)
{
    if (buf.empty()) return false;
    const std::string str(buf);
    errno = 0;
    char *p = nullptr;
    const long long v = std::strtoll(str.c_str(), &p, 0);
    if ((size_t)(p - str.c_str()) != str.size() || errno != 0) return false;
    out = v;
    return true;
}
// incr (pegasus_write_service_impl.h:264-342): read-before-write on the single writer; an absent / expired / empty base counts
// as 0; a base that is not an integer or a sum that leaves int64 answers kInvalidArgument *in the response* (the return value
// stays kOk) and still writes an empty record so that the decree advances; expire_ts_seconds: 0 keeps the record's, < 0
// clears it, > 0 sets it (only > 0 matters for a new record).  *resp_error / *new_value mirror incr_response.
int32_t pgs_rrdb_incr(pgs_server *h, pgs_blob key, int64_t increment, int32_t expire_ts_seconds, int64_t decree, uint64_t timestamp_us,
                      uint32_t now, int32_t *resp_error, int64_t *new_value)
{
    WLOCKED(h);
    Server &s = h->s;
    s.last_committed_decree = decree;
    int32_t dummy_e;
    int64_t dummy_v;
    if (!resp_error) resp_error = &dummy_e;
    if (!new_value) new_value = &dummy_v;
    *new_value = 0;
    std::vector<pgs_get_result> gr;
    std::vector<uint8_t> arena;
    const int32_t st = point_lookup(s, {std::string(bsv(key))}, now, gr, arena);
    if (st != PGS_OK) { *resp_error = st; return st; }
    int64_t nv = increment;
    uint32_t new_ets = expire_ts_seconds > 0 ? (uint32_t)expire_ts_seconds : 0u;
    if (gr[0].status == PGS_OK) { // found and alive
        const std::string_view old((const char *)arena.data() + gr[0].value_off, gr[0].value_len);
        if (!old.empty()) {
            int64_t base;
            if (!buf2int64(old, base)) {
                *resp_error = PGS_INVALID_ARGUMENT;
                s.put_one({}, {}, 0, timestamp_us, now); // empty_put
                return PGS_OK;
            }
            if (__builtin_add_overflow(base, increment, &nv)) {
                *resp_error = PGS_INVALID_ARGUMENT;
                *new_value = base;
                s.put_one({}, {}, 0, timestamp_us, now);
                return PGS_OK;
            }
        }
        new_ets = expire_ts_seconds == 0 ? gr[0].expire_ts : expire_ts_seconds < 0 ? 0u : (uint32_t)expire_ts_seconds;
    }
    s.put_one(bsv(key), std::to_string(nv), new_ets, timestamp_us, now);
    s.part->p.hk_write.capture_raw_key(bsv(key), 1);
    *resp_error = PGS_OK;
    *new_value = nv;
    return PGS_OK;
}

// validate_check (pegasus_write_service_impl.h:1144-1270)
static bool cas_validate(int32_t type, std::string_view operand, bool exist, std::string_view value, bool &invalid)
{
    invalid = false;
    switch (type) {
    case 0: return true;                              // CT_NO_CHECK
    case 1: return !exist;                            // CT_VALUE_NOT_EXIST
    case 2: return !exist || value.empty();           // CT_VALUE_NOT_EXIST_OR_EMPTY
    case 3: return exist;                             // CT_VALUE_EXIST
    case 4: return exist && !value.empty();           // CT_VALUE_NOT_EMPTY
    case 5: case 6: case 7:                           // CT_VALUE_MATCH_ANYWHERE / PREFIX / POSTFIX
        if (!exist) return false;
        if (operand.empty()) return true;
        if (value.size() < operand.size()) return false;
        if (type == 5) return value.find(operand) != std::string_view::npos;
        if (type == 6) return value.substr(0, operand.size()) == operand;
        return value.substr(value.size() - operand.size()) == operand;
    case 8: case 9: case 10: case 11: case 12: {      // CT_VALUE_BYTES_LESS .. GREATER
        if (!exist) return false;
        const int c = value.compare(operand);
        if (c < 0) return type <= 9;
        if (c > 0) return type >= 11;
        return type >= 9 && type <= 11;
    }
    case 13: case 14: case 15: case 16: case 17: {    // CT_VALUE_INT_LESS .. GREATER
        if (!exist) return false;
        int64_t a = 0, b = 0;
        if (!buf2int64(value, a) || !buf2int64(operand, b)) { invalid = true; return false; }
        if (a < b) return type <= 14;
        if (a > b) return type >= 16;
        return type >= 14 && type <= 16;
    }
    }
    return false;
}

// write_weight: the WRITE collector's weight of a successful call (check_and_set 1, check_and_mutate the mutation count)
static int32_t check_and_mutate(Server &s, const pgs_check_and_mutate_request &q, int64_t decree, uint64_t timestamp_us, uint32_t now,
                                pgs_cas_result *res, uint8_t *cv_out, uint32_t cv_cap, int64_t write_weight)
{
    s.last_committed_decree = decree;
    pgs_cas_result dummy;
    if (!res) res = &dummy;
    *res = pgs_cas_result{};
    bool bad = q.n_mutate == 0 || q.check_type < 0 || q.check_type > 17; // empty list / unsupported check type
    for (uint32_t i = 0; i < q.n_mutate && !bad; i++) bad = q.mutate_list[i].operation > 1;
    if (bad) {
        res->error = PGS_INVALID_ARGUMENT;
        s.put_one({}, {}, 0, timestamp_us, now); // empty_put: the decree still advances
        s.part->p.hk_read.capture_hash_key(bsv(q.hash_key), 1);
        return PGS_OK;
    }
    std::vector<pgs_get_result> gr;
    std::vector<uint8_t> arena;
    const int32_t st = point_lookup(s, {make_key(bsv(q.hash_key), bsv(q.check_sort_key))}, now, gr, arena);
    if (st != PGS_OK) { res->error = st; return st; }
    const bool exist = gr[0].status == PGS_OK;
    const std::string_view value = exist ? std::string_view((const char *)arena.data() + gr[0].value_off, gr[0].value_len) : std::string_view();
    if (q.return_check_value) {
        res->check_value_returned = 1;
        if (exist) {
            res->check_value_exist = 1;
            res->check_value_len = (uint32_t)value.size();
            if (cv_out && cv_cap) memcpy(cv_out, value.data(), std::min<size_t>(cv_cap, value.size()));
        }
    }
    bool invalid = false;
    const bool passed = cas_validate(q.check_type, bsv(q.check_operand), exist, value, invalid);
    if (passed) {
        for (uint32_t i = 0; i < q.n_mutate; i++) {
            const pgs_mutate &m = q.mutate_list[i];
            const std::string key = make_key(bsv(q.hash_key), bsv(m.sort_key));
            if (m.operation == 0) s.put_one(key, bsv(m.value), (uint32_t)m.set_expire_ts_seconds, timestamp_us, now);
            else s.mem_write(key, PGS_TYPE_DELETION, std::string(), now);
        }
        res->error = PGS_OK;
        s.part->p.hk_write.capture_hash_key(bsv(q.hash_key), write_weight); // the read was captured by point_lookup
    } else {
        s.put_one({}, {}, 0, timestamp_us, now);
        res->error = invalid ? PGS_INVALID_ARGUMENT : PGS_TRY_AGAIN;
    }
    return PGS_OK;
}
int32_t pgs_rrdb_check_and_mutate(pgs_server *h, const pgs_check_and_mutate_request *q, int64_t decree, uint64_t timestamp_us, uint32_t now,
                                  pgs_cas_result *res, uint8_t *cv_out, uint32_t cv_cap)
{
    if (!h || !q) return PGS_INVALID_ARGUMENT;
    WLOCKED(h);
    return check_and_mutate(h->s, *q, decree, timestamp_us, now, res, cv_out, cv_cap, q->n_mutate);
}
int32_t pgs_rrdb_check_and_set(pgs_server *h, const pgs_check_and_set_request *q, int64_t decree, uint64_t timestamp_us, uint32_t now,
                               pgs_cas_result *res, uint8_t *cv_out, uint32_t cv_cap)
{
    if (!h || !q) return PGS_INVALID_ARGUMENT;
    WLOCKED(h);
    pgs_mutate m{0, q->set_diff_sort_key ? q->set_sort_key : q->check_sort_key, q->set_value, q->set_expire_ts_seconds};
    pgs_check_and_mutate_request r{q->hash_key, q->check_sort_key, q->check_type, q->check_operand, &m, 1, q->return_check_value};
    return check_and_mutate(h->s, r, decree, timestamp_us, now, res, cv_out, cv_cap, 1);
}
int32_t pgs_rrdb_multi_put(pgs_server *h, pgs_blob hash_key, const pgs_blob *sort_keys, const pgs_blob *values,
                           uint32_t n, uint32_t expire_ts, int64_t decree, uint64_t timestamp_us, uint32_t now)
{
    WLOCKED(h);
    Server &s = h->s;
    s.last_committed_decree = decree;
    if (n == 0) { // request.kvs is empty: kInvalidArgument, but an empty record still advances the decree
        s.put_one({}, {}, 0, timestamp_us, now); // empty_put (pegasus_write_service_impl.h:90-99,112-119)
        s.part->p.hk_write.capture_hash_key(bsv(hash_key), 0); // multi_put captures whatever its status (a weight of 0 counts 1)
        return PGS_INVALID_ARGUMENT;
    }
    for (uint32_t i = 0; i < n; i++) s.put_one(make_key(bsv(hash_key), bsv(sort_keys[i])), bsv(values[i]), expire_ts, timestamp_us, now);
    s.part->p.hk_write.capture_hash_key(bsv(hash_key), n);
    return PGS_OK;
}
int32_t pgs_rrdb_multi_remove(pgs_server *h, pgs_blob hash_key, const pgs_blob *sort_keys, uint32_t n, int64_t decree,
                              int64_t *count, uint32_t now)
{
    WLOCKED(h);
    Server &s = h->s;
    s.last_committed_decree = decree;
    if (count) *count = 0;
    if (n == 0) {
        s.put_one({}, {}, 0, 0, now);
        return PGS_INVALID_ARGUMENT;
    }
    for (uint32_t i = 0; i < n; i++) s.mem_write(make_key(bsv(hash_key), bsv(sort_keys[i])), PGS_TYPE_DELETION, std::string(), now);
    s.part->p.hk_write.capture_hash_key(bsv(hash_key), n);
    if (count) *count = n;
    return PGS_OK;
}
int32_t pgs_rrdb_flush(pgs_server *h, uint32_t now)
{
    WLOCKED(h);
    int32_t st = h->s.flush_mem();
    if (st != PGS_OK) return st;
    return h->s.maybe_compact(now);
}
int32_t pgs_rrdb_manual_compact(pgs_server *h, uint32_t now, pgs_compact_result *out)
{
    WLOCKED(h);
    int32_t st = do_manual_compact(h->s, now, -1, true, out); // bottommost_level_compaction = force
    if (st == PGS_OK) h->s.manual_compact_last_finish_ms = ((uint64_t)now + kEpochBegin) * 1000;
    return st;
}
// The same manual-compaction decision on many replicas (the app envs reach every replica of the app at once): each replica is
// prepared as do_manual_compact prepares it, and the merges go to the GPU in one pgs_compact_many.
int32_t pgs_rrdb_manual_compact_many(pgs_server *const *servers, uint32_t n, uint32_t now, pgs_compact_result *out)
{
    if (n == 0) return PGS_OK;
    if (!servers) return PGS_INVALID_ARGUMENT;
    std::vector<Server *> order;
    for (uint32_t i = 0; i < n; i++) {
        if (!servers[i]) return PGS_INVALID_ARGUMENT;
        if (servers[i]->s.part->p.eng != servers[0]->s.part->p.eng) {
            set_error("rrdb_manual_compact_many: replica %u is on another engine than replica 0", i);
            return PGS_INVALID_ARGUMENT;
        }
        order.push_back(&servers[i]->s);
    }
    std::sort(order.begin(), order.end());
    if (std::adjacent_find(order.begin(), order.end()) != order.end()) {
        set_error("rrdb_manual_compact_many: a replica given twice");
        return PGS_INVALID_ARGUMENT;
    }
    std::vector<std::unique_lock<std::shared_mutex>> held;
    for (Server *s : order) held.emplace_back(s->mu);
    if (out) memset(out, 0, sizeof(pgs_compact_result) * (size_t)n);
    // do_manual_compact's preparation per replica: flush, fold a stack deeper than one merge, the level of the merge
    std::vector<std::vector<uint64_t>> ids(n);
    std::vector<pgs_filter_params> fps(n);
    std::vector<pgs_compact_job> jobs;
    std::vector<uint32_t> which; // the replica of each job (a replica without runs has none)
    for (uint32_t i = 0; i < n; i++) {
        Server &s = servers[i]->s;
        if (const int32_t st = s.flush_mem()) return st;
        auto rs = s.runs();
        if (rs.empty()) continue;
        int32_t level = 1;
        for (auto &r : rs) { level = std::max(level, r->level); ids[i].push_back(r->id); }
        while (ids[i].size() > kMaxRuns) {
            std::vector<uint64_t> tail(ids[i].end() - kMaxRuns, ids[i].end());
            pgs_filter_params fp = s.filter();
            pgs_compact_result cr{};
            if (const int32_t st = pgs_compact(s.part, tail.data(), kMaxRuns, level, 1, &fp, now, &cr)) return st;
            ids[i].resize(ids[i].size() - kMaxRuns);
            if (cr.new_run_id) ids[i].push_back(cr.new_run_id);
        }
        fps[i] = s.filter();
        jobs.push_back(pgs_compact_job{s.part, ids[i].data(), (uint32_t)ids[i].size(), level, 1, &fps[i]});
        which.push_back(i);
    }
    std::vector<pgs_compact_result> res(jobs.size());
    if (const int32_t st = pgs_compact_many(jobs.data(), (uint32_t)jobs.size(), now, 0, res.data())) return st;
    for (uint32_t i = 0; i < n; i++) servers[i]->s.manual_compact_last_finish_ms = ((uint64_t)now + kEpochBegin) * 1000;
    if (out)
        for (size_t j = 0; j < jobs.size(); j++) out[which[j]] = res[j];
    return PGS_OK;
}
// ---- checkpoints (pegasus_server_impl.cpp:1951-2336: sync_checkpoint, get_checkpoint, storage_apply_checkpoint) ---------------
// The directory protocol (temporary name, MANIFEST last, rename) lives in checkpoint_dir.h.
int32_t pgs_rrdb_sync_checkpoint(pgs_server *h, const char *dir, uint32_t now, int64_t *decree_out)
{
    (void)now;
    if (!h || !dir) return PGS_INVALID_ARGUMENT;
    WLOCKED(h);
    Server &s = h->s;
    int32_t st = s.flush_mem(); // everything applied so far must be in a run (the reference flushes, then hard-links the SSTs)
    if (st != PGS_OK) return st;
    const int64_t decree = s.last_flushed_decree;
    if (decree_out) *decree_out = decree;
    CheckpointWriter w;
    const int started = w.begin(dir, decree);
    if (started < 0) { set_error("%s", w.error().c_str()); return PGS_IO_ERROR; }
    if (started == 1) { s.last_durable_decree = std::max(s.last_durable_decree, decree); return PGS_OK; } // already there (ERR_WRONG_TIMING upstream)
    auto rs = s.runs(); // level ascending, newest first inside a level
    CheckpointManifest m;
    m.app_id = s.app_id; m.pidx = s.pidx; m.data_version = s.data_version; m.decree = decree; m.last_seq = (long long)s.last_seq;
    std::vector<uint8_t> img;
    uint32_t fileno = 0;
    uint8_t per_level[7]; // rocksdb_compression_type = "lz4" (the reference's default): none for L0 / L1, LZ4 below
    if (pgs_parse_compression_types("lz4", 7, per_level) != PGS_OK) return PGS_INVALID_ARGUMENT;
    for (size_t i = rs.size(); i-- > 0;) { // oldest first: re-ingesting in this order rebuilds the same recency order
        const uint32_t comp = per_level[std::min(std::max(rs[i]->level, 0), 6)];
        uint64_t need = 0;
        st = pgs_sst_export_ex(s.part, rs[i]->id, comp, nullptr, 0, &need);
        if (st != PGS_INCOMPLETE && st != PGS_OK) return st; // the writer's destructor removes the temporary directory
        img.resize(need);
        st = pgs_sst_export_ex(s.part, rs[i]->id, comp, img.data(), img.size(), &need);
        if (st != PGS_OK) return st;
        char name[32];
        snprintf(name, sizeof name, "%06u.sst", ++fileno);
        if (!w.add_file(name, img.data(), need)) { set_error("%s", w.error().c_str()); return PGS_IO_ERROR; }
        m.files.push_back({rs[i]->level, name, (long long)need});
    }
    if (!w.commit(m.str())) { set_error("%s", w.error().c_str()); return PGS_IO_ERROR; }
    s.last_durable_decree = std::max(s.last_durable_decree, decree);
    return PGS_OK;
}
int64_t pgs_rrdb_last_durable_decree(pgs_server *h) { RLOCKED(h); return h->s.last_durable_decree; }
int32_t pgs_rrdb_apply_checkpoint(pgs_server *h, const char *cdir)
{
    if (!h || !cdir) return PGS_INVALID_ARGUMENT;
    std::vector<uint8_t> mf;
    if (!ckpt_read_file(std::string(cdir) + "/MANIFEST", mf)) { set_error("checkpoint: no MANIFEST in %s", cdir); return PGS_NOT_FOUND; }
    CheckpointManifest m;
    if (!m.parse(std::string(mf.begin(), mf.end()))) { set_error("checkpoint: damaged MANIFEST in %s", cdir); return PGS_CORRUPTION; }
    WLOCKED(h);
    Server &s = h->s;
    if (m.data_version != (long long)s.data_version) { set_error("checkpoint: data version %lld, replica has %u", m.data_version, s.data_version); return PGS_NOT_SUPPORTED; }
    std::vector<std::vector<uint8_t>> images(m.files.size());
    for (size_t i = 0; i < m.files.size(); i++)
        if (!ckpt_read_file(std::string(cdir) + "/" + m.files[i].name, images[i]) || (long long)images[i].size() != m.files[i].bytes) {
            set_error("checkpoint: %s/%s is missing or has the wrong size", cdir, m.files[i].name.c_str());
            return PGS_CORRUPTION;
        }
    for (size_t i = 0; i < m.files.size(); i++) { // every image must decode (checksums, block handles) before anything is given up
        uint64_t nbytes = 0;
        uint32_t nblocks = 0;
        const int32_t st = pgs_sst_decode(images[i].data(), images[i].size(), nullptr, 0, nullptr, nullptr, 0, &nbytes, &nblocks);
        if (st != PGS_OK && st != PGS_INCOMPLETE) { set_error("checkpoint: %s/%s does not decode", cdir, m.files[i].name.c_str()); return st; }
    }
    // from here on the old state is gone (storage_apply_checkpoint: the learner's data is replaced)
    for (auto &r : s.runs()) pgs_run_drop(s.part, r->id);
    s.mem.clear();
    s.mem_bytes = 0;
    { std::lock_guard<std::mutex> g(s.ctx_mu); s.ctx.clear(); }
    for (size_t i = 0; i < m.files.size(); i++) {
        uint64_t rid = 0;
        const int32_t st = pgs_sst_ingest(s.part, m.files[i].level, images[i].data(), images[i].size(), &rid);
        if (st != PGS_OK) return st;
    }
    s.last_seq = (uint64_t)m.last_seq;
    s.last_committed_decree = s.last_flushed_decree = s.last_durable_decree = m.decree;
    return PGS_OK;
}
// ---- partition split (local_partition_split.cpp:179-298; replica_split_manager.cpp:278 copy_checkpoint_to_dir(flush = true) +
// storage_apply_checkpoint) ---------------------------------------------------------------------------------------------------
int32_t pgs_rrdb_split(pgs_server *parent, uint32_t src_count, uint32_t dst_count, pgs_server *const *children, uint32_t n,
                       int64_t *decree_out)
{
    if (!parent || !children || src_count == 0 || n == 0 || n > 1024) return PGS_INVALID_ARGUMENT;
    Server &s = parent->s;
    // the children stay locked for the whole call: nothing reaches them until they hold the split state
    std::vector<Server *> kids;
    for (uint32_t i = 0; i < n; i++) {
        if (!children[i]) continue;
        if (children[i] == parent) return PGS_INVALID_ARGUMENT;
        kids.push_back(&children[i]->s);
    }
    std::vector<Server *> order = kids;
    std::sort(order.begin(), order.end());
    if (std::adjacent_find(order.begin(), order.end()) != order.end()) return PGS_INVALID_ARGUMENT;
    std::vector<std::unique_lock<std::shared_mutex>> held;
    for (Server *k : order) held.emplace_back(k->mu);
    for (uint32_t i = 0; i < n; i++) {
        if (!children[i]) continue;
        Server &c = children[i]->s;
        if (!c.mem.empty() || !c.runs().empty() || c.last_committed_decree != 0 || c.last_flushed_decree != 0 ||
            (int64_t)c.pidx != (int64_t)s.pidx + (int64_t)i * src_count) {
            set_error("rrdb_split: child %u is not an empty, new replica of index %lld", i, (long long)s.pidx + (long long)i * src_count);
            return PGS_INVALID_ARGUMENT;
        }
    }
    // the parent's state as copy_checkpoint_to_dir(flush = true) fixes it: memtable flushed, runs snapshotted, under its
    // writer lock; after that the parent takes reads and writes again while the snapshot is split
    std::vector<std::shared_ptr<Run>> snap;
    int64_t decree;
    uint64_t last_seq, mc_finish;
    {
        std::unique_lock<std::shared_mutex> w(s.mu);
        if (const int32_t st = s.flush_mem()) return st;
        snap = s.runs();
        decree = s.last_flushed_decree;
        last_seq = s.last_seq;
        mc_finish = s.manual_compact_last_finish_ms;
    }
    std::vector<pgs_partition *> dst(n, nullptr);
    for (uint32_t i = 0; i < n; i++)
        if (children[i]) dst[i] = children[i]->s.part;
    if (const int32_t st = partition_split(s.part, &snap, src_count, dst_count, dst.data(), n, nullptr)) return st;
    for (Server *k : kids) {
        k->last_seq = last_seq; // new writes on the child win over every copied version
        k->last_committed_decree = k->last_flushed_decree = decree;
        k->last_durable_decree = 0;
        k->manual_compact_last_finish_ms = mc_finish;
    }
    if (decree_out) *decree_out = decree;
    return PGS_OK;
}
int64_t pgs_rrdb_last_flushed_decree(pgs_server *h) { RLOCKED(h); return h->s.last_flushed_decree; }
int64_t pgs_rrdb_last_committed_decree(pgs_server *h) { RLOCKED(h); return h->s.last_committed_decree; }

} // extern "C"
