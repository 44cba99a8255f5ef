// host_util.cpp — host-side pieces of the product that do no device work:
//   * key schema + crc64 (pegasus_key_schema.h:41-183, utils/crc.cpp:45-86,289-295)
//   * the sorted-run builder used by flush (RocksDB BlockBuilder + FlushBlockBySizePolicy)
//   * raw block decode (egress)
//   * `user_specified_compaction` JSON -> binary ops table (compaction_operation.cpp:162-186)
//   * the manual-compaction rules (pegasus_manual_compact_service.cpp:83-313)
#include <algorithm>
#include <cerrno>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <map>
#include <string>
#include <string_view>
#include <vector>

#include "../../include/pegasus_b200.h"
#include "../csrc/format.h"
#include "host_internal.h"

namespace pgs {

// ---- crc64 (crc64_make_table, format.h) -----------------------------------------------------
const uint64_t *crc64_table()
{
    static uint64_t tab[256];
    static bool ready = [] {
        crc64_make_table(tab);
        return true;
    }();
    (void)ready;
    return tab;
}
uint64_t crc64(const uint8_t *p, uint64_t n, uint64_t init)
{
    const uint64_t *t = crc64_table();
    uint64_t c = ~init;
    while (n--) c = t[(uint8_t)(c ^ *p++)] ^ (c >> 8);
    return ~c;
}

std::string make_key(std::string_view hk, std::string_view sk)
{
    std::string k(2 + hk.size() + sk.size(), '\0');
    k[0] = (char)(hk.size() >> 8);
    k[1] = (char)hk.size();
    memcpy(&k[2], hk.data(), hk.size());
    memcpy(&k[2 + hk.size()], sk.data(), sk.size());
    return k;
}
std::string make_next(std::string k) // pegasus_key_schema.h:65-98
{
    size_t p = k.size() - 1;
    while ((uint8_t)k[p] == 0xFF) p--;
    k[p] = (char)((uint8_t)k[p] + 1);
    k.resize(p + 1);
    return k;
}
uint64_t key_hash(std::string_view key) // pegasus_key_schema.h:150-165
{
    if (key.size() < 2) return 0;
    return pegasus_key_hash(crc64_table(), (const uint8_t *)key.data(), (uint32_t)key.size());
}

// ---- run builder ----------------------------------------------------------------------------
static inline void put_varint(std::string &d, uint32_t v)
{
    while (v >= 128) { d.push_back((char)(v | 128)); v >>= 7; }
    d.push_back((char)v);
}
static inline void put_u32(std::string &d, uint32_t v) { d.append((const char *)&v, 4); }

void RunBuilder::flush_block()
{
    if (entries_ == 0) return;
    for (uint32_t r : restarts_) put_u32(buf_, r);
    put_u32(buf_, (uint32_t)restarts_.size());
    while (data_.size() % kBlockAlign) data_.push_back(0);
    blk_off_.push_back(data_.size());
    blk_size_.push_back((uint32_t)buf_.size());
    data_ += buf_;
    buf_.clear();
    restarts_.assign(1, 0);
    counter_ = 0;
    entries_ = 0;
    last_key_.clear();
}

int32_t RunBuilder::add(std::string_view ukey, uint64_t seq, uint8_t type, std::string_view value)
{
    // order check: user key ascending, then seq descending
    if (have_prev_) {
        int c = std::string_view(prev_ukey_).compare(ukey);
        if (c > 0 || (c == 0 && prev_trailer_ <= ((seq << 8) | type))) return PGS_INVALID_ARGUMENT;
    }
    size_t klen = ukey.size() + 8;
    if (entries_ > 0) { // FlushBlockBySizePolicy::Update
        size_t cur = buf_.size() + restarts_.size() * 4 + 4;
        bool flush = cur >= block_size_;
        if (!flush) {
            size_t after = cur + klen + value.size() + (counter_ >= restart_interval_ ? 4 : 0) + 4 +
                           varint_len((uint32_t)klen) + varint_len((uint32_t)value.size());
            size_t limit = ((size_t)block_size_ * 90 + 99) / 100;
            flush = after > block_size_ && cur > limit;
        }
        if (flush) flush_block();
    }
    uint64_t trailer = (seq << 8) | type;
    std::string ik(ukey);
    ik.append((const char *)&trailer, 8);
    uint32_t shared = 0;
    if (counter_ >= restart_interval_) {
        restarts_.push_back((uint32_t)buf_.size());
        counter_ = 0;
    } else {
        size_t m = std::min(last_key_.size(), ik.size());
        while (shared < m && last_key_[shared] == ik[shared]) shared++;
    }
    put_varint(buf_, shared);
    put_varint(buf_, (uint32_t)ik.size() - shared);
    put_varint(buf_, (uint32_t)value.size());
    buf_.append(ik.data() + shared, ik.size() - shared);
    buf_.append(value.data(), value.size());
    last_key_ = std::move(ik);
    counter_++;
    entries_++;
    n_records_++;
    prev_ukey_.assign(ukey.data(), ukey.size());
    prev_trailer_ = trailer;
    have_prev_ = true;
    return PGS_OK;
}

void RunBuilder::finish()
{
    flush_block();
    while (data_.size() % kBlockAlign) data_.push_back(0);
}

// ---- block decode -----------------------------------------------------------------------------
static const uint8_t *get_varint(const uint8_t *p, const uint8_t *limit, uint32_t *v)
{
    uint32_t r = 0;
    for (uint32_t shift = 0; shift <= 28 && p < limit; shift += 7) {
        uint32_t b = *p++;
        if (b & 128) r |= (b & 127) << shift;
        else { *v = r | (b << shift); return p; }
    }
    return nullptr;
}

int32_t decode_blocks(const uint8_t *data, const uint64_t *blk_off, const uint32_t *blk_size,
                      uint32_t n_blocks, const std::function<void(std::string_view, uint64_t, uint8_t, std::string_view)> &fn)
{
    std::string key;
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint8_t *base = data + blk_off[b];
        uint32_t size = blk_size[b];
        if (size < 8) return PGS_CORRUPTION;
        uint32_t nr;
        memcpy(&nr, base + size - 4, 4);
        if (nr == 0 || (uint64_t)nr * 4 + 4 > size) return PGS_CORRUPTION;
        const uint8_t *p = base, *limit = base + size - 4 - 4 * nr;
        key.clear();
        while (p < limit) {
            uint32_t shared, non_shared, vlen;
            p = get_varint(p, limit, &shared);
            if (p) p = get_varint(p, limit, &non_shared);
            if (p) p = get_varint(p, limit, &vlen);
            if (!p || shared > key.size() || (uint64_t)(limit - p) < (uint64_t)non_shared + vlen) return PGS_CORRUPTION;
            key.resize(shared);
            key.append((const char *)p, non_shared);
            if (key.size() < 8) return PGS_CORRUPTION;
            uint64_t trailer;
            memcpy(&trailer, key.data() + key.size() - 8, 8);
            fn(std::string_view(key.data(), key.size() - 8), trailer >> 8, (uint8_t)trailer,
               std::string_view((const char *)p + non_shared, vlen));
            p += non_shared + vlen;
        }
    }
    return PGS_OK;
}

// ---- JSON (subset) + ops table ----------------------------------------------------------------
namespace {
struct J {
    enum K { Null, Bool, Num, Str, Arr, Obj } k = Null;
    bool b = false, integral = false, negative = false;
    uint64_t mag = 0;
    std::string s;
    std::vector<J> arr;
    std::vector<std::pair<std::string, J>> obj;
    const J *find(const char *name) const
    {
        for (auto &m : obj)
            if (m.first == name) return &m.second;
        return nullptr;
    }
};
struct Parser {
    const char *p, *end;
    void skip() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p; }
    bool lit(const char *w)
    {
        size_t n = strlen(w);
        if ((size_t)(end - p) < n || memcmp(p, w, n)) return false;
        p += n;
        return true;
    }
    bool string(std::string &o)
    {
        if (p >= end || *p != '"') return false;
        ++p;
        while (p < end && *p != '"') {
            char c = *p++;
            if (c != '\\') { o.push_back(c); continue; }
            if (p >= end) return false;
            c = *p++;
            switch (c) {
            case 'n': o.push_back('\n'); break;
            case 't': o.push_back('\t'); break;
            case 'r': o.push_back('\r'); break;
            case 'b': o.push_back('\b'); break;
            case 'f': o.push_back('\f'); break;
            case '"': case '\\': case '/': o.push_back(c); break;
            case 'u': {
                if (end - p < 4) return false;
                unsigned cp = 0;
                for (int i = 0; i < 4; i++) {
                    char h = *p++;
                    cp = cp * 16 + (h >= '0' && h <= '9' ? h - '0' : h >= 'a' && h <= 'f' ? h - 'a' + 10 : h >= 'A' && h <= 'F' ? h - 'A' + 10 : 0xFFFF);
                    if (cp > 0xFFFFF) return false;
                }
                if (cp < 0x80) o.push_back((char)cp);
                else if (cp < 0x800) { o.push_back((char)(0xC0 | cp >> 6)); o.push_back((char)(0x80 | (cp & 63))); }
                else { o.push_back((char)(0xE0 | cp >> 12)); o.push_back((char)(0x80 | ((cp >> 6) & 63))); o.push_back((char)(0x80 | (cp & 63))); }
                break;
            }
            default: return false;
            }
        }
        if (p >= end) return false;
        ++p;
        return true;
    }
    bool value(J &v, int depth = 0)
    {
        if (depth > 32) return false;
        skip();
        if (p >= end) return false;
        if (*p == '"') { v.k = J::Str; return string(v.s); }
        if (*p == '{') {
            v.k = J::Obj;
            ++p;
            skip();
            if (p < end && *p == '}') { ++p; return true; }
            while (true) {
                skip();
                std::string name;
                if (!string(name)) return false;
                skip();
                if (p >= end || *p++ != ':') return false;
                J child;
                if (!value(child, depth + 1)) return false;
                v.obj.emplace_back(std::move(name), std::move(child));
                skip();
                if (p >= end) return false;
                if (*p == ',') { ++p; continue; }
                if (*p == '}') { ++p; return true; }
                return false;
            }
        }
        if (*p == '[') {
            v.k = J::Arr;
            ++p;
            skip();
            if (p < end && *p == ']') { ++p; return true; }
            while (true) {
                J child;
                if (!value(child, depth + 1)) return false;
                v.arr.push_back(std::move(child));
                skip();
                if (p >= end) return false;
                if (*p == ',') { ++p; continue; }
                if (*p == ']') { ++p; return true; }
                return false;
            }
        }
        if (lit("true")) { v.k = J::Bool; v.b = true; return true; }
        if (lit("false")) { v.k = J::Bool; return true; }
        if (lit("null")) return true;
        v.k = J::Num;
        if (*p == '-') { v.negative = true; ++p; }
        if (p >= end || *p < '0' || *p > '9') return false;
        v.integral = true;
        while (p < end && *p >= '0' && *p <= '9') {
            uint64_t d = *p++ - '0';
            if (v.mag > (UINT64_MAX - d) / 10) v.integral = false;
            v.mag = v.mag * 10 + d;
        }
        if (p < end && (*p == '.' || *p == 'e' || *p == 'E')) {
            v.integral = false;
            while (p < end && (strchr("+-.eE", *p) || (*p >= '0' && *p <= '9'))) ++p;
        }
        return true;
    }
};
bool parse_json(std::string_view text, J &out)
{
    Parser ps{text.data(), text.data() + text.size()};
    if (!ps.value(out)) return false;
    ps.skip();
    return ps.p == ps.end;
}
// dsn::json decode rule for DEFINE_JSON_SERIALIZATION structs (json_helper.h:254-278)
struct Fields {
    const J &o;
    int listed = 0, got = 0;
    bool bad = false;
    explicit Fields(const J &j) : o(j) { bad = j.k != J::Obj; }
    const J *take(const char *name, J::K kind)
    {
        listed++;
        if (bad) return nullptr;
        const J *m = o.find(name);
        if (!m) return nullptr;
        if (m->k != kind) { bad = true; return nullptr; }
        got++;
        return m;
    }
    bool ok() const { return !bad && (got == listed || got == (int)o.obj.size()); }
};
int name_index(const std::string &s, std::initializer_list<const char *> names)
{
    int i = 0;
    for (const char *n : names) {
        if (s == n) return i;
        i++;
    }
    return i;
}
struct RuleBin { uint8_t type, match; uint32_t start_ttl = 0, stop_ttl = 0; std::string pattern; };
bool rule_decode(int type, const std::string &params, RuleBin &r)
{
    J j;
    if (!parse_json(params, j)) return false;
    Fields f(j);
    r.type = (uint8_t)type;
    r.match = MATCH_INVALID;
    if (type == RULE_TTL_RANGE) {
        for (auto pr : {std::make_pair("start_ttl", &r.start_ttl), std::make_pair("stop_ttl", &r.stop_ttl)}) {
            if (const J *m = f.take(pr.first, J::Num)) {
                if (!m->integral || m->negative || m->mag > UINT32_MAX) return false;
                *pr.second = (uint32_t)m->mag;
            }
        }
    } else {
        if (const J *m = f.take("pattern", J::Str)) r.pattern = m->s;
        if (const J *m = f.take("match_type", J::Str))
            r.match = (uint8_t)name_index(m->s, {"SMT_MATCH_ANYWHERE", "SMT_MATCH_PREFIX", "SMT_MATCH_POSTFIX"});
    }
    return f.ok();
}
} // namespace

int64_t ops_parse(std::string_view json, uint32_t /*data_version*/, std::string &out, uint32_t *n_ops_out)
{
    out.clear();
    uint32_t n_ops = 0;
    out.append((const char *)&n_ops, 4);
    if (n_ops_out) *n_ops_out = 0;
    J root;
    if (!parse_json(json, root) || root.k != J::Obj) return (int64_t)out.size();
    const J *ops = root.find("ops");
    if (!ops || ops->k != J::Arr) return (int64_t)out.size();
    struct RawOp { int type; std::string params; std::vector<std::pair<int, std::string>> rules; };
    std::vector<RawOp> raw;
    for (const J &jo : ops->arr) { // a malformed element fails the whole vector decode
        Fields f(jo);
        RawOp ro;
        ro.type = 2;
        if (const J *m = f.take("type", J::Str)) ro.type = name_index(m->s, {"COT_UPDATE_TTL", "COT_DELETE"});
        if (const J *m = f.take("params", J::Str)) ro.params = m->s;
        if (const J *m = f.take("rules", J::Arr)) {
            for (const J &jr : m->arr) {
                Fields fr(jr);
                int rt = 3;
                std::string rp;
                if (const J *t = fr.take("type", J::Str))
                    rt = name_index(t->s, {"FRT_HASHKEY_PATTERN", "FRT_SORTKEY_PATTERN", "FRT_TTL_RANGE"});
                if (const J *t = fr.take("params", J::Str)) rp = t->s;
                if (!fr.ok()) return (int64_t)out.size();
                ro.rules.emplace_back(rt, std::move(rp));
            }
        }
        if (!f.ok()) return (int64_t)out.size();
        raw.push_back(std::move(ro));
    }
    for (const RawOp &ro : raw) {
        std::vector<RuleBin> rules;
        for (auto &rr : ro.rules) {
            RuleBin rb;
            if (rr.first > RULE_TTL_RANGE) continue; // unknown rule type: factory returns nullptr
            if (rule_decode(rr.first, rr.second, rb)) rules.push_back(std::move(rb));
        }
        if (rules.empty()) continue;
        uint8_t op_type, ttl_type = TTL_INVALID;
        uint32_t ttl_value = 0;
        if (ro.type == 1) {
            op_type = OP_DELETE;
        } else if (ro.type == 0) {
            op_type = OP_UPDATE_TTL;
            J j;
            if (!parse_json(ro.params, j)) continue;
            Fields f(j);
            if (const J *m = f.take("type", J::Str))
                ttl_type = (uint8_t)name_index(m->s, {"UTOT_FROM_NOW", "UTOT_FROM_CURRENT", "UTOT_TIMESTAMP"});
            bool bad = false;
            if (const J *m = f.take("value", J::Num)) {
                if (!m->integral || m->negative || m->mag > UINT32_MAX) bad = true;
                else ttl_value = (uint32_t)m->mag;
            }
            if (bad || !f.ok()) continue;
        } else {
            continue;
        }
        uint16_t nr = (uint16_t)rules.size();
        out.push_back((char)op_type);
        out.push_back((char)ttl_type);
        out.append((const char *)&nr, 2);
        out.append((const char *)&ttl_value, 4);
        for (auto &r : rules) {
            uint16_t pl = (uint16_t)r.pattern.size();
            out.push_back((char)r.type);
            out.push_back((char)r.match);
            out.append((const char *)&pl, 2);
            out.append((const char *)&r.start_ttl, 4);
            out.append((const char *)&r.stop_ttl, 4);
            out += r.pattern;
            while (out.size() % 4) out.push_back(0);
        }
        n_ops++;
    }
    memcpy(&out[0], &n_ops, 4);
    if (n_ops_out) *n_ops_out = n_ops;
    return (int64_t)out.size();
}

} // namespace pgs

// ================================================================================================
using namespace pgs;
struct pgs_run_builder { RunBuilder rb; pgs_run_builder(uint32_t b, uint32_t r) : rb(b, r) {} };

extern "C" {

int32_t pgs_generate_key(const uint8_t *hk, uint32_t hk_len, const uint8_t *sk, uint32_t sk_len,
                         uint8_t *out, uint32_t cap)
{
    if (hk_len >= 0xFFFF) return -PGS_INVALID_ARGUMENT; // CHECK_LT(hash_key.length(), UINT16_MAX)
    uint32_t n = 2 + hk_len + sk_len;
    if (n > cap) return -PGS_INCOMPLETE;
    out[0] = (uint8_t)(hk_len >> 8);
    out[1] = (uint8_t)hk_len;
    memcpy(out + 2, hk, hk_len);
    memcpy(out + 2 + hk_len, sk, sk_len);
    return (int32_t)n;
}
int32_t pgs_generate_next_blob(const uint8_t *hk, uint32_t hk_len, const uint8_t *sk,
                               uint32_t sk_len, int32_t with_sort_key, uint8_t *out, uint32_t cap)
{
    if (hk_len >= 0xFFFF) return -PGS_INVALID_ARGUMENT;
    std::string k = make_next(make_key(std::string_view((const char *)hk, hk_len),
                                       with_sort_key ? std::string_view((const char *)sk, sk_len) : std::string_view()));
    if (k.size() > cap) return -PGS_INCOMPLETE;
    memcpy(out, k.data(), k.size());
    return (int32_t)k.size();
}
uint64_t pgs_key_hash(const uint8_t *raw_key, uint32_t len)
{
    if (len < 2) return 0;
    return key_hash(std::string_view((const char *)raw_key, len));
}
uint64_t pgs_crc64(const uint8_t *data, uint64_t len, uint64_t init) { return crc64(data, len, init); }

pgs_run_builder *pgs_run_builder_new(uint32_t block_size, uint32_t restart_interval)
{
    return new pgs_run_builder(block_size ? block_size : kDefaultBlockSize,
                               restart_interval ? restart_interval : kDefaultRestartInterval);
}
int32_t pgs_run_builder_add(pgs_run_builder *b, const uint8_t *ukey, uint32_t ukey_len, uint64_t seq,
                            uint8_t type, const uint8_t *value, uint32_t value_len)
{
    return b->rb.add(std::string_view((const char *)ukey, ukey_len), seq, type,
                     std::string_view((const char *)value, value_len));
}
int32_t pgs_run_builder_add_many(pgs_run_builder *b, uint64_t n, const uint8_t *keys,
                                 const uint64_t *key_off, const uint8_t *vals, const uint64_t *val_off,
                                 const uint64_t *seq, const uint8_t *type)
{
    for (uint64_t i = 0; i < n; i++) {
        int32_t st = b->rb.add(std::string_view((const char *)keys + key_off[i], key_off[i + 1] - key_off[i]), seq[i],
                               type[i], std::string_view((const char *)vals + val_off[i], val_off[i + 1] - val_off[i]));
        if (st != PGS_OK) return st;
    }
    return PGS_OK;
}
int32_t pgs_run_builder_finish(pgs_run_builder *b, const uint8_t **data, uint64_t *data_bytes,
                               const uint64_t **blk_off, const uint32_t **blk_size, uint32_t *n_blocks)
{
    b->rb.finish();
    *data = (const uint8_t *)b->rb.data().data();
    *data_bytes = b->rb.data().size();
    *blk_off = b->rb.blk_off().data();
    *blk_size = b->rb.blk_size().data();
    *n_blocks = (uint32_t)b->rb.blk_off().size();
    return PGS_OK;
}
void pgs_run_builder_free(pgs_run_builder *b) { delete b; }

int32_t pgs_blocks_decode(const uint8_t *data, const uint64_t *blk_off, const uint32_t *blk_size,
                          uint32_t n_blocks, pgs_decode_sizes *sizes, uint8_t *keys, uint64_t *key_off,
                          uint8_t *vals, uint64_t *val_off, uint64_t *seq, uint8_t *type)
{
    uint64_t n = 0, kb = 0, vb = 0;
    bool write = keys != nullptr;
    int32_t st = decode_blocks(data, blk_off, blk_size, n_blocks,
                               [&](std::string_view k, uint64_t s, uint8_t t, std::string_view v) {
                                   if (write) {
                                       key_off[n] = kb;
                                       val_off[n] = vb;
                                       memcpy(keys + kb, k.data(), k.size());
                                       memcpy(vals + vb, v.data(), v.size());
                                       seq[n] = s;
                                       type[n] = t;
                                   }
                                   n++;
                                   kb += k.size();
                                   vb += v.size();
                               });
    if (write) { key_off[n] = kb; val_off[n] = vb; }
    if (sizes) { sizes->n_records = n; sizes->key_bytes = kb; sizes->value_bytes = vb; }
    return st;
}

int64_t pgs_compaction_ops_parse(const char *json, uint32_t json_len, uint32_t data_version, uint8_t *out,
                                 uint32_t cap, uint32_t *n_ops_out)
{
    std::string bin;
    int64_t n = ops_parse(std::string_view(json, json_len), data_version, bin, n_ops_out);
    if ((uint64_t)n > cap) return -PGS_INCOMPLETE;
    memcpy(out, bin.data(), bin.size());
    return n;
}

// ---- manual-compaction rules -------------------------------------------------------------------------------------------------
// dsn::buf2int32 / buf2int64 (utils/string_conv.h:35-62): the whole buffer is one strtoll(base 0) integer inside the type's range
static bool whole_int(const std::string &str, long long lo, long long hi, long long &out)
{
    if (str.empty()) return false;
    errno = 0;
    char *p = nullptr;
    const long long v = std::strtoll(str.c_str(), &p, 0);
    if ((size_t)(p - str.c_str()) != str.size() || errno != 0 || v < lo || v > hi) return false;
    out = v;
    return true;
}
// utils/time_utils.h:118-129: "H:M" with 0 <= H <= 23, 0 <= M <= 59 (sscanf: trailing text is ignored) -> seconds of the day, or -1
static int hh_mm_seconds(const std::string &s)
{
    int hour = 0, min = 0;
    if (sscanf(s.c_str(), "%d:%d", &hour, &min) == 2 && hour >= 0 && hour <= 23 && min >= 0 && min <= 59) return 3600 * hour + 60 * min;
    return -1;
}

int32_t pgs_manual_compact_decide(const char *envs, uint32_t n_envs, uint64_t now_ms, uint64_t last_finish_ms, int64_t today_midnight_s,
                                  int32_t num_levels, pgs_manual_compact_decision *out)
{
    if (!out || (n_envs && !envs)) return PGS_INVALID_ARGUMENT;
    std::map<std::string, std::string> m;
    const char *p = envs;
    for (uint32_t i = 0; i < n_envs; i++) {
        std::string k(p);
        p += k.size() + 1;
        std::string v(p);
        p += v.size() + 1;
        m[k] = v;
    }
    memset(out, 0, sizeof *out);
    out->target_level = -1;
    auto f = m.find("manual_compact.disabled");
    out->disabled = f != m.end() && f->second == "true";
    out->max_concurrent_running_count = INT_MAX;
    long long v = 0;
    f = m.find("manual_compact.max_concurrent_running_count");
    if (f != m.end() && whole_int(f->second, INT_MIN, INT_MAX, v)) out->max_concurrent_running_count = (int32_t)v;
    if (out->disabled || out->max_concurrent_running_count <= 0) return PGS_OK;

    std::string prefix;
    f = m.find("manual_compact.once.trigger_time");
    if (f != m.end() && whole_int(f->second, LLONG_MIN, LLONG_MAX, v) && v > 0 && (uint64_t)v > last_finish_ms / 1000) {
        out->rule = 1;
        prefix = "manual_compact.once.";
    }
    if (!out->rule) {
        f = m.find("manual_compact.periodic.trigger_time");
        if (f != m.end()) {
            if (today_midnight_s < 0) { // the local day that holds now_ms
                time_t t = (time_t)(now_ms / 1000);
                struct tm tmv;
                localtime_r(&t, &tmv);
                tmv.tm_hour = tmv.tm_min = tmv.tm_sec = 0;
                today_midnight_s = (int64_t)mktime(&tmv);
            }
            size_t b = 0;
            const std::string &list = f->second;
            while (b <= list.size() && !out->rule) {
                size_t e = list.find(',', b);
                if (e == std::string::npos) e = list.size();
                const int sec = e > b ? hh_mm_seconds(list.substr(b, e - b)) : -1;
                if (sec >= 0) {
                    const uint64_t t_ms = (uint64_t)(today_midnight_s + sec) * 1000;
                    if (last_finish_ms < t_ms && t_ms < now_ms) out->rule = 2;
                }
                b = e + 1;
            }
            if (out->rule) prefix = "manual_compact.periodic.";
        }
    }
    if (!out->rule) return PGS_OK;
    f = m.find(prefix + "target_level");
    if (f != m.end() && whole_int(f->second, INT_MIN, INT_MAX, v) && (v == -1 || (v >= 1 && v <= num_levels))) out->target_level = (int32_t)v;
    f = m.find(prefix + "bottommost_level_compaction");
    out->bottommost_force = f != m.end() && f->second == "force";
    return PGS_OK;
}

// compression_str_to_type (pegasus_server_impl.cpp:3062-3080): exact names only
static bool compression_of(const std::string &s, uint8_t &t)
{
    if (s == "none") t = 0;
    else if (s == "snappy") t = 1;
    else if (s == "lz4") t = 4;
    else if (s == "zstd") t = 7;
    else return false;
    return true;
}
int32_t pgs_parse_compression_types(const char *config, uint32_t num_levels, uint8_t *per_level)
{
    if (!config || !per_level || num_levels == 0 || num_levels > 64) return PGS_INVALID_ARGUMENT;
    static const std::string header = "per_level:";
    const std::string cfg(config);
    std::vector<uint8_t> tmp(num_levels, 0);
    if (cfg.find(header) != std::string::npos) { // one type per level; split_args drops empty items, the last type repeats
        std::vector<std::string> types;
        const std::string list = cfg.size() >= header.size() ? cfg.substr(header.size()) : std::string();
        size_t b = 0;
        while (b <= list.size()) {
            size_t e = list.find(',', b);
            if (e == std::string::npos) e = list.size();
            if (e > b) types.push_back(list.substr(b, e - b));
            b = e + 1;
        }
        uint8_t last = 0;
        for (uint32_t i = 0; i < num_levels; i++) {
            if (i < types.size() && !compression_of(types[i], last)) return PGS_INVALID_ARGUMENT;
            tmp[i] = last;
        }
    } else { // one type for the levels >= 2 (ColumnFamilyOptions::OptimizeLevelStyleCompaction)
        uint8_t t = 0;
        if (!compression_of(cfg, t)) return PGS_INVALID_ARGUMENT;
        for (uint32_t i = 2; i < num_levels; i++) tmp[i] = t;
    }
    memcpy(per_level, tmp.data(), num_levels);
    return PGS_OK;
}

int32_t pgs_manual_compact_state_check(uint64_t now_ms, uint64_t last_finish_ms, int32_t min_interval_s, uint64_t *enqueue_ms)
{
    if (!enqueue_ms) return 0;
    if (min_interval_s <= 0 || last_finish_ms == 0 || now_ms - last_finish_ms > (uint64_t)min_interval_s * 1000) {
        if (*enqueue_ms != 0) return 0;
        *enqueue_ms = now_ms;
        return 1;
    }
    return 0;
}

} // extern "C"
