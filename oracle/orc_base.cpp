// orc_base.cpp — CPU ORACLE (test infrastructure only): crc64, key/value schema, JSON,
// compaction rules / operations and KeyWithTTLCompactionFilter::Filter, restated from the
// reference.  Each function cites the reference file:line it follows.
#include "orc_internal.h"

#include <algorithm>

namespace orc {

// -------------------------------------------------------------------------------------------
// crc64: src/utils/crc.cpp:45-86 (compute loop), :289-295 (polynomial bit list).  The table is
// generated from the polynomial instead of being copied; oracle/_ref (the reference's own
// crc.cpp compiled as-is) pins it in tests/test_oracle_golden.py.
// -------------------------------------------------------------------------------------------
static const uint64_t *crc64_table()
{
    static uint64_t tab[256];
    static bool init = false;
    if (!init) {
        static const int bits[] = {63, 61, 59, 58, 56, 55, 52, 49, 48, 47, 46, 44, 41, 37, 36, 34,
                                   32, 31, 28, 26, 23, 22, 19, 16, 13, 12, 10, 9,  6,  4,  3,  0};
        uint64_t poly = 0;
        for (int n : bits) poly += 1ull << (63 - n); // BIT64(n)
        for (uint32_t i = 0; i < 256; i++) {
            uint64_t c = i;
            for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ poly : (c >> 1);
            tab[i] = c;
        }
        init = true;
    }
    return tab;
}

uint64_t crc64(const void *p, size_t n, uint64_t init)
{
    const uint64_t *tab = crc64_table();
    const uint8_t *d = (const uint8_t *)p;
    uint64_t c = ~init;
    for (size_t i = 0; i < n; i++) c = tab[(uint8_t)(c ^ d[i])] ^ (c >> 8);
    return ~c;
}

// -------------------------------------------------------------------------------------------
// key schema: src/base/pegasus_key_schema.h
// -------------------------------------------------------------------------------------------
std::string generate_key(sv hk, sv sk) // :41-59
{
    std::string k;
    k.resize(2 + hk.size() + sk.size());
    put_be16((uint8_t *)&k[0], (uint16_t)hk.size());
    memcpy(&k[2], hk.data(), hk.size());
    if (!sk.empty()) memcpy(&k[2 + hk.size()], sk.data(), sk.size());
    return k;
}

static std::string bump(std::string k) // strip trailing 0xFF, increment, truncate
{
    size_t p = k.size() - 1;
    while ((uint8_t)k[p] == 0xFF) p--;
    k[p] = (char)((uint8_t)k[p] + 1);
    k.resize(p + 1);
    return k;
}
std::string next_blob(sv hk) { return bump(generate_key(hk, sv())); }        // :65-82
std::string next_blob(sv hk, sv sk) { return bump(generate_key(hk, sk)); } // :87-98

void restore_key(sv key, sv &hk, sv &sk) // :102-146
{
    uint16_t l = be16((const uint8_t *)key.data());
    hk = l > 0 ? key.substr(2, l) : sv();
    sk = key.size() > 2u + l ? key.substr(2 + l) : sv();
}

uint64_t key_hash(sv key) // :150-165
{
    uint16_t l = be16((const uint8_t *)key.data());
    if (l > 0) return crc64(key.data() + 2, l, 0);
    return crc64(key.data() + 2, key.size() - 2, 0);
}

bool check_key_hash(sv key, int32_t pidx, int32_t pv) // :174-183
{
    return (int64_t)(key_hash(key) & (uint64_t)(int64_t)pv) == (int64_t)pidx;
}

// -------------------------------------------------------------------------------------------
// value schema: src/base/pegasus_value_schema.h:133-226
// -------------------------------------------------------------------------------------------
std::string generate_value(uint32_t version, uint32_t expire_ts, uint64_t timetag, sv data)
{
    std::string v;
    size_t h = user_data_offset(version);
    v.resize(h + data.size());
    put_be32((uint8_t *)&v[0], expire_ts);
    if (version == 1) put_be64((uint8_t *)&v[4], timetag);
    if (!data.empty()) memcpy(&v[h], data.data(), data.size());
    return v;
}

// -------------------------------------------------------------------------------------------
// JSON (the subset dsn::json / rapidjson is used for on this path)
// -------------------------------------------------------------------------------------------
namespace {
struct JP {
    const char *p, *e;
    void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) p++; }
    bool str(std::string &out)
    {
        if (p >= e || *p != '"') return false;
        p++;
        out.clear();
        while (p < e && *p != '"') {
            if (*p == '\\') {
                p++;
                if (p >= e) return false;
                switch (*p) {
                case '"': out += '"'; break;
                case '\\': out += '\\'; break;
                case '/': out += '/'; break;
                case 'b': out += '\b'; break;
                case 'f': out += '\f'; break;
                case 'n': out += '\n'; break;
                case 'r': out += '\r'; break;
                case 't': out += '\t'; break;
                case 'u': {
                    // p points at the 'u' of an escape; reads its four hex digits and leaves p on the last one
                    auto hex4 = [&](unsigned &cp) {
                        if (e - p < 5) return false;
                        cp = 0;
                        for (int i = 1; i <= 4; i++) {
                            char c = p[i];
                            cp <<= 4;
                            if (c >= '0' && c <= '9') cp |= c - '0';
                            else if (c >= 'a' && c <= 'f') cp |= c - 'a' + 10;
                            else if (c >= 'A' && c <= 'F') cp |= c - 'A' + 10;
                            else return false;
                        }
                        p += 4;
                        return true;
                    };
                    unsigned cp;
                    if (!hex4(cp)) return false;
                    if (cp >= 0xD800 && cp <= 0xDFFF) { // RapidJSON's surrogate rule: a high surrogate and a low one make one code point
                        unsigned lo;
                        if (cp > 0xDBFF || e - p < 3 || p[1] != '\\' || p[2] != 'u') return false;
                        p += 2;
                        if (!hex4(lo) || lo < 0xDC00 || lo > 0xDFFF) return false;
                        cp = (((cp - 0xD800) << 10) | (lo - 0xDC00)) + 0x10000;
                    }
                    if (cp < 0x80) out += (char)cp;
                    else if (cp < 0x800) { out += (char)(0xC0 | (cp >> 6)); out += (char)(0x80 | (cp & 0x3F)); }
                    else if (cp < 0x10000) { out += (char)(0xE0 | (cp >> 12)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
                    else { out += (char)(0xF0 | (cp >> 18)); out += (char)(0x80 | ((cp >> 12) & 0x3F)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
                    break;
                }
                default: return false;
                }
                p++;
            } else {
                out += *p++;
            }
        }
        if (p >= e) return false;
        p++;
        return true;
    }
    bool val(JVal &v, int depth)
    {
        if (depth > 64) return false;
        ws();
        if (p >= e) return false;
        if (*p == '{') {
            p++;
            v.t = JVal::Obj;
            ws();
            if (p < e && *p == '}') { p++; return true; }
            for (;;) {
                ws();
                std::string k;
                if (!str(k)) return false;
                ws();
                if (p >= e || *p != ':') return false;
                p++;
                JVal c;
                if (!val(c, depth + 1)) return false;
                v.o.emplace_back(std::move(k), std::move(c));
                ws();
                if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == '}') { p++; return true; }
                return false;
            }
        }
        if (*p == '[') {
            p++;
            v.t = JVal::Arr;
            ws();
            if (p < e && *p == ']') { p++; return true; }
            for (;;) {
                JVal c;
                if (!val(c, depth + 1)) return false;
                v.a.push_back(std::move(c));
                ws();
                if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == ']') { p++; return true; }
                return false;
            }
        }
        if (*p == '"') { v.t = JVal::Str; return str(v.s); }
        if (e - p >= 4 && !memcmp(p, "true", 4)) { v.t = JVal::Bool; v.b = true; p += 4; return true; }
        if (e - p >= 5 && !memcmp(p, "false", 5)) { v.t = JVal::Bool; v.b = false; p += 5; return true; }
        if (e - p >= 4 && !memcmp(p, "null", 4)) { v.t = JVal::Null; p += 4; return true; }
        // number
        const char *s = p;
        bool neg = false;
        if (*p == '-') { neg = true; p++; }
        if (p >= e || *p < '0' || *p > '9') return false;
        uint64_t u = 0;
        bool overflow = false;
        while (p < e && *p >= '0' && *p <= '9') {
            uint64_t d = *p - '0';
            if (u > (UINT64_MAX - d) / 10) overflow = true;
            u = u * 10 + d;
            p++;
        }
        bool is_int = !overflow;
        if (p < e && (*p == '.' || *p == 'e' || *p == 'E')) {
            is_int = false;
            while (p < e && (*p == '.' || *p == 'e' || *p == 'E' || *p == '+' || *p == '-' || (*p >= '0' && *p <= '9'))) p++;
        }
        (void)s;
        v.t = JVal::Num;
        v.is_int = is_int;
        v.neg = neg;
        v.u = u;
        return true;
    }
};
} // namespace

bool json_parse(sv text, JVal &out)
{
    JP jp{text.data(), text.data() + text.size()};
    if (!jp.val(out, 0)) return false;
    jp.ws();
    return jp.p == jp.e;
}

// -------------------------------------------------------------------------------------------
// rules: src/server/compaction_filter_rule.cpp:31-90
// -------------------------------------------------------------------------------------------
bool string_pattern_match(sv value, int match_type, sv pattern) // :31-54
{
    if (pattern.empty()) return false;
    if (value.size() < pattern.size()) return false;
    switch (match_type) {
    case SMT_MATCH_ANYWHERE: return value.find(pattern) != sv::npos;
    case SMT_MATCH_PREFIX: return memcmp(value.data(), pattern.data(), pattern.size()) == 0;
    case SMT_MATCH_POSTFIX:
        return memcmp(value.data() + value.size() - pattern.size(), pattern.data(), pattern.size()) == 0;
    default: return false;
    }
}

// server read path filter: src/server/pegasus_server_impl.cpp:2350-2380 (empty pattern => true)
bool validate_filter(int filter_type, sv pattern, sv value)
{
    switch (filter_type) {
    case PGS_FT_NO_FILTER: return true;
    case PGS_FT_MATCH_ANYWHERE:
    case PGS_FT_MATCH_PREFIX:
    case PGS_FT_MATCH_POSTFIX:
        if (pattern.empty()) return true;
        if (value.size() < pattern.size()) return false;
        if (filter_type == PGS_FT_MATCH_ANYWHERE) return value.find(pattern) != sv::npos;
        if (filter_type == PGS_FT_MATCH_PREFIX) return memcmp(value.data(), pattern.data(), pattern.size()) == 0;
        return memcmp(value.data() + value.size() - pattern.size(), pattern.data(), pattern.size()) == 0;
    default: return false;
    }
}

bool Rule::match(sv hk, sv sk, sv value, uint32_t now) const
{
    switch (type) {
    case FRT_HASHKEY_PATTERN: return string_pattern_match(hk, match_type, pattern); // :58-63
    case FRT_SORTKEY_PATTERN: return string_pattern_match(sk, match_type, pattern); // :67-72
    case FRT_TTL_RANGE: {                                                           // :76-90
        uint32_t expire_ts = extract_expire_ts(data_version, value);
        if (expire_ts == 0 && start_ttl == 0 && stop_ttl == 0) return true;
        // u32 wrap-around arithmetic exactly like the reference
        return (uint32_t)(start_ttl + now) <= expire_ts && (uint32_t)(stop_ttl + now) >= expire_ts;
    }
    default: return false;
    }
}

// -------------------------------------------------------------------------------------------
// operations: src/server/compaction_operation.cpp:33-113
// -------------------------------------------------------------------------------------------
bool Op::all_rules_match(sv hk, sv sk, sv value, uint32_t now) const // :33-47
{
    if (rules.empty()) return false;
    for (auto &r : rules)
        if (!r.match(hk, sk, value, now)) return false;
    return true;
}

bool Op::filter(sv hk, sv sk, sv value, uint32_t now, std::string *new_value, bool *changed) const
{
    if (!all_rules_match(hk, sk, value, now)) return false;
    if (type == COT_DELETE) return true; // :58-68
    if (type != COT_UPDATE_TTL) return false;
    uint32_t new_ts = 0; // :77-113
    switch (ttl_type) {
    case UTOT_FROM_NOW: new_ts = now + ttl_value; break;
    case UTOT_FROM_CURRENT: {
        uint32_t ttl = extract_expire_ts(data_version, value);
        if (ttl == 0) return false;
        new_ts = ttl_value + ttl;
        break;
    }
    case UTOT_TIMESTAMP: new_ts = ttl_value - kEpochBegin; break;
    default: return false;
    }
    std::string nv(value);
    put_be32((uint8_t *)&nv[0], new_ts);
    *new_value = std::move(nv);
    *changed = true;
    return false;
}

// JSON decode rule of DEFINE_JSON_SERIALIZATION (src/common/json_helper.h:254-278): every listed
// member that is present must decode; success iff all listed members were present or the object
// has no member besides the parsed ones.
namespace {
struct Dec {
    const JVal &in;
    int args = 0, parsed = 0;
    bool ok = true;
    explicit Dec(const JVal &j) : in(j) { if (in.t != JVal::Obj) ok = false; }
    bool str(const char *k, std::string &out)
    {
        if (!ok) return false;
        args++;
        if (const JVal *v = in.get(k)) {
            if (v->t != JVal::Str) return ok = false;
            out = v->s;
            parsed++;
        }
        return true;
    }
    bool u32(const char *k, uint32_t &out)
    {
        if (!ok) return false;
        args++;
        if (const JVal *v = in.get(k)) {
            // UINT_TYPE_SERIALIZATION: IsUint64 and within range (json_helper.h:431-445)
            if (v->t != JVal::Num || !v->is_int || v->neg || v->u > UINT32_MAX) return ok = false;
            out = (uint32_t)v->u;
            parsed++;
        }
        return true;
    }
    bool done() const { return ok && (parsed == args || parsed == (int)in.o.size()); }
};
int enum_of(const std::string &s, const char *const *names, int n)
{
    for (int i = 0; i < n; i++)
        if (s == names[i]) return i;
    return n; // INVALID
}
const char *kSmt[] = {"SMT_MATCH_ANYWHERE", "SMT_MATCH_PREFIX", "SMT_MATCH_POSTFIX"};
const char *kFrt[] = {"FRT_HASHKEY_PATTERN", "FRT_SORTKEY_PATTERN", "FRT_TTL_RANGE"};
const char *kCot[] = {"COT_UPDATE_TTL", "COT_DELETE"};
const char *kUtot[] = {"UTOT_FROM_NOW", "UTOT_FROM_CURRENT", "UTOT_TIMESTAMP"};
} // namespace

bool rule_from_json(int type, sv params, uint32_t data_version, Rule &out)
{
    JVal j;
    if (!json_parse(params, j)) return false;
    out = Rule();
    out.type = type;
    out.data_version = data_version;
    Dec d(j);
    if (type == FRT_TTL_RANGE) { // DEFINE_JSON_SERIALIZATION(start_ttl, stop_ttl)
        d.u32("start_ttl", out.start_ttl);
        d.u32("stop_ttl", out.stop_ttl);
    } else if (type == FRT_HASHKEY_PATTERN || type == FRT_SORTKEY_PATTERN) {
        std::string mt; // DEFINE_JSON_SERIALIZATION(pattern, match_type)
        bool had = j.t == JVal::Obj && j.get("match_type");
        d.str("pattern", out.pattern);
        d.str("match_type", mt);
        if (had) out.match_type = enum_of(mt, kSmt, 3);
    } else {
        return false;
    }
    return d.done();
}

bool update_ttl_from_json(sv params, Op &out) // compaction_operation.h:142-151
{
    JVal j;
    if (!json_parse(params, j)) return false;
    Dec d(j);
    std::string ty;
    bool had = j.t == JVal::Obj && j.get("type");
    d.str("type", ty);
    d.u32("value", out.ttl_value);
    if (had) out.ttl_type = enum_of(ty, kUtot, 3);
    return d.done();
}

std::vector<Op> ops_from_json(sv json, uint32_t data_version) // compaction_operation.cpp:162-186
{
    std::vector<Op> res;
    JVal j;
    if (!json_parse(json, j) || j.t != JVal::Obj) return res;
    // json_helper {ops}: the one listed member must decode when present
    const JVal *ops = j.get("ops");
    if (!ops) return res; // parsed 0 == MemberCount only if object is empty; nothing to do either way
    if (ops->t != JVal::Arr) return res;
    // decode all ops first: any malformed op makes the whole decode fail (vector decode)
    struct RawRule { int type; std::string params; };
    struct RawOp { int type; std::string params; std::vector<RawRule> rules; };
    std::vector<RawOp> raw;
    for (auto &jo : ops->a) {
        RawOp ro;
        Dec d(jo);
        std::string ty;
        bool had_type = jo.t == JVal::Obj && jo.get("type");
        d.str("type", ty);
        d.str("params", ro.params);
        ro.type = had_type ? enum_of(ty, kCot, 2) : COT_INVALID;
        if (!d.ok) return res;
        d.args++;
        if (const JVal *jr = jo.get("rules")) {
            if (jr->t != JVal::Arr) return res;
            for (auto &r : jr->a) {
                RawRule rr;
                Dec dr(r);
                std::string rty;
                bool had_rt = r.t == JVal::Obj && r.get("type");
                dr.str("type", rty);
                dr.str("params", rr.params);
                if (!dr.done()) return res;
                rr.type = had_rt ? enum_of(rty, kFrt, 3) : FRT_INVALID;
                ro.rules.push_back(std::move(rr));
            }
            d.parsed++;
        }
        if (!d.done()) return res;
        raw.push_back(std::move(ro));
    }
    for (auto &ro : raw) {
        Op op;
        op.data_version = data_version;
        for (auto &rr : ro.rules) { // create_compaction_filter_rules :139-151
            Rule r;
            if (rr.type == FRT_INVALID) continue; // factory has no such name -> nullptr
            if (rule_from_json(rr.type, rr.params, data_version, r)) op.rules.push_back(std::move(r));
        }
        if (op.rules.empty()) continue;
        if (ro.type == COT_DELETE) {
            op.type = COT_DELETE;
        } else if (ro.type == COT_UPDATE_TTL) {
            op.type = COT_UPDATE_TTL;
            if (!update_ttl_from_json(ro.params, op)) continue;
        } else {
            continue;
        }
        res.push_back(std::move(op));
    }
    return res;
}

// -------------------------------------------------------------------------------------------
// KeyWithTTLCompactionFilter::Filter — src/server/key_ttl_compaction_filter.h:55-121
// -------------------------------------------------------------------------------------------
DropReason compaction_filter(const FilterParams &fp, sv key, sv value, uint32_t now,
                             std::string *new_value, bool *changed)
{
    if (!fp.enabled) return kKeep;     // :61-63
    if (key.size() < 2) return kKeep;  // :67-69 (empty write)
    // a value too short for its expire_ts header: pegasus_extract_expire_ts reads past it (an assert of data_input that
    // release builds compile out); such a value is kept as it stands (DESIGN §8)
    if (value.size() < 4) return kKeep;
    uint32_t expire_ts = extract_expire_ts(fp.data_version, value);
    sv entry = value;
    if (fp.default_ttl != 0 && expire_ts == 0) { // :73-79
        expire_ts = now + fp.default_ttl;
        *new_value = std::string(value);
        put_be32((uint8_t *)&(*new_value)[0], expire_ts);
        *changed = true;
    }
    if (fp.ops && !fp.ops->empty()) { // :81-89,94-108
        // every op sees the value as of entry to user_specified_operation_filter (SURVEY §3.5
        // step 4: the reference aliases *new_value here; the defined behaviour is kept)
        std::string entry_copy(*changed ? sv(*new_value) : entry);
        sv hk, sk;
        restore_key(key, hk, sk);
        for (auto &op : *fp.ops)
            if (op.filter(hk, sk, entry_copy, now, new_value, changed)) return kDropUser;
    }
    if (ts_expired(now, expire_ts)) return kDropExpired; // :91
    // check_if_stale_split_data :114-121
    if (fp.validate_hash && fp.partition_version >= 0 && fp.pidx <= fp.partition_version &&
        !check_key_hash(key, fp.pidx, fp.partition_version))
        return kDropStale;
    return kKeep;
}

} // namespace orc

// ===========================================================================================
// C API
// ===========================================================================================
using namespace orc;
static inline sv mk(const uint8_t *p, uint32_t n) { return sv((const char *)p, n); }

extern "C" {

uint64_t orc_crc64(const uint8_t *p, uint64_t n, uint64_t init) { return crc64(p, n, init); }

static int32_t out_str(const std::string &s, uint8_t *out, uint32_t cap)
{
    if (s.size() > cap) return -(int32_t)s.size();
    memcpy(out, s.data(), s.size());
    return (int32_t)s.size();
}
int32_t orc_generate_key(const uint8_t *hk, uint32_t hk_len, const uint8_t *sk, uint32_t sk_len,
                         uint8_t *out, uint32_t cap)
{
    return out_str(generate_key(mk(hk, hk_len), mk(sk, sk_len)), out, cap);
}
int32_t orc_generate_next_blob(const uint8_t *hk, uint32_t hk_len, const uint8_t *sk,
                               uint32_t sk_len, int32_t with_sk, uint8_t *out, uint32_t cap)
{
    return out_str(with_sk ? next_blob(mk(hk, hk_len), mk(sk, sk_len)) : next_blob(mk(hk, hk_len)), out, cap);
}
int32_t orc_restore_key(const uint8_t *key, uint32_t len, uint32_t *hk_len, uint32_t *sk_len)
{
    if (len < 2) return -1;
    sv hk, sk;
    restore_key(mk(key, len), hk, sk);
    *hk_len = (uint32_t)hk.size();
    *sk_len = (uint32_t)sk.size();
    return 0;
}
uint64_t orc_key_hash(const uint8_t *key, uint32_t len) { return key_hash(mk(key, len)); }
int32_t orc_check_key_hash(const uint8_t *key, uint32_t len, int32_t pidx, int32_t pv)
{
    return check_key_hash(mk(key, len), pidx, pv);
}
int32_t orc_hashkey_transform(const uint8_t *key, uint32_t len)
{
    if (len < 2) return -1; // InDomain (hashkey_transform.h:56-60)
    return (int32_t)hashkey_prefix(mk(key, len)).size();
}
uint64_t orc_generate_timetag(uint64_t ts, uint8_t cluster_id, int32_t deleted)
{
    return ts << 8u | (uint64_t)(cluster_id << 1u) | (deleted ? 1u : 0u); // pegasus_value_schema.h:44-47
}
int32_t orc_generate_value(uint32_t version, uint32_t expire_ts, uint64_t timetag,
                           const uint8_t *data, uint32_t len, uint8_t *out, uint32_t cap)
{
    return out_str(generate_value(version, expire_ts, timetag, mk(data, len)), out, cap);
}
uint32_t orc_extract_expire_ts(uint32_t version, const uint8_t *v, uint32_t len)
{
    return extract_expire_ts(version, mk(v, len));
}
uint64_t orc_extract_timetag(uint32_t, const uint8_t *v, uint32_t) { return be64(v + 4); } // :87-95
int32_t orc_user_data_offset(uint32_t version) { return (int32_t)user_data_offset(version); }
void orc_update_expire_ts(uint32_t, uint8_t *v, uint32_t, uint32_t ts) { put_be32(v, ts); } // :99-110
int32_t orc_check_if_ts_expired(uint32_t now, uint32_t ts) { return ts_expired(now, ts); }

int32_t orc_string_pattern_match(const uint8_t *v, uint32_t vlen, int32_t mt, const uint8_t *pat,
                                 uint32_t plen)
{
    return string_pattern_match(mk(v, vlen), mt, mk(pat, plen));
}
int32_t orc_validate_filter(int32_t ft, const uint8_t *pat, uint32_t plen, const uint8_t *v,
                            uint32_t vlen)
{
    return validate_filter(ft, mk(pat, plen), mk(v, vlen));
}
int32_t orc_ttl_range_rule_match(uint32_t start_ttl, uint32_t stop_ttl, uint32_t expire_ts,
                                 uint32_t now)
{
    Rule r;
    r.type = FRT_TTL_RANGE;
    r.start_ttl = start_ttl;
    r.stop_ttl = stop_ttl;
    std::string v = generate_value(1, expire_ts, 0, sv());
    return r.match(sv(), sv(), v, now);
}
int32_t orc_rule_create(int32_t rule_type, const char *params, uint32_t len, char *pattern_out,
                        uint32_t cap, int32_t *match_type, uint32_t *start_ttl, uint32_t *stop_ttl)
{
    Rule r;
    if (!rule_from_json(rule_type, sv(params, len), 1, r)) return 0;
    if (pattern_out && cap) {
        size_t n = std::min<size_t>(cap - 1, r.pattern.size());
        memcpy(pattern_out, r.pattern.data(), n);
        pattern_out[n] = 0;
    }
    if (match_type) *match_type = r.match_type;
    if (start_ttl) *start_ttl = r.start_ttl;
    if (stop_ttl) *stop_ttl = r.stop_ttl;
    return 1;
}
int32_t orc_update_ttl_create(const char *params, uint32_t len, int32_t *type, uint32_t *value)
{
    Op op;
    if (!update_ttl_from_json(sv(params, len), op)) return 0;
    *type = op.ttl_type;
    *value = op.ttl_value;
    return 1;
}

orc_ops *orc_ops_create(const char *json, uint32_t len, uint32_t data_version)
{
    auto *o = new orc_ops;
    o->ops = ops_from_json(sv(json, len), data_version);
    return o;
}
void orc_ops_free(orc_ops *o) { delete o; }
uint32_t orc_ops_count(const orc_ops *o) { return (uint32_t)o->ops.size(); }
int32_t orc_ops_describe(const orc_ops *o, uint32_t i, int32_t *op_type, int32_t *ttl_type,
                         uint32_t *ttl_value, uint32_t *n_rules)
{
    if (i >= o->ops.size()) return -1;
    const Op &op = o->ops[i];
    *op_type = op.type;
    *ttl_type = op.ttl_type;
    *ttl_value = op.ttl_value;
    *n_rules = (uint32_t)op.rules.size();
    return 0;
}
int32_t orc_ops_describe_rule(const orc_ops *o, uint32_t i, uint32_t r, int32_t *rule_type,
                              int32_t *match_type, char *pattern, uint32_t cap, uint32_t *start_ttl,
                              uint32_t *stop_ttl)
{
    if (i >= o->ops.size() || r >= o->ops[i].rules.size()) return -1;
    const Rule &ru = o->ops[i].rules[r];
    *rule_type = ru.type;
    *match_type = ru.match_type;
    size_t n = std::min<size_t>(cap ? cap - 1 : 0, ru.pattern.size());
    if (cap) { memcpy(pattern, ru.pattern.data(), n); pattern[n] = 0; }
    *start_ttl = ru.start_ttl;
    *stop_ttl = ru.stop_ttl;
    return 0;
}
orc_ops *orc_ops_build(int32_t op_type, int32_t ttl_type, uint32_t ttl_value, uint32_t n_rules,
                       const int32_t *rule_type, const int32_t *match_type,
                       const char *const *pattern, const uint32_t *start_ttl,
                       const uint32_t *stop_ttl, uint32_t data_version)
{
    auto *o = new orc_ops;
    Op op;
    op.type = op_type;
    op.ttl_type = ttl_type;
    op.ttl_value = ttl_value;
    op.data_version = data_version;
    for (uint32_t i = 0; i < n_rules; i++) {
        Rule r;
        r.type = rule_type[i];
        r.match_type = match_type[i];
        r.pattern = pattern[i] ? pattern[i] : "";
        r.start_ttl = start_ttl[i];
        r.stop_ttl = stop_ttl[i];
        r.data_version = data_version;
        op.rules.push_back(r);
    }
    o->ops.push_back(op);
    return o;
}
int32_t orc_op_all_rules_match(const orc_ops *o, uint32_t i, const uint8_t *hk, uint32_t hk_len,
                               const uint8_t *sk, uint32_t sk_len, const uint8_t *v, uint32_t vlen,
                               uint32_t now)
{
    return o->ops[i].all_rules_match(mk(hk, hk_len), mk(sk, sk_len), mk(v, vlen), now);
}
int32_t orc_op_filter(const orc_ops *o, uint32_t i, const uint8_t *hk, uint32_t hk_len,
                      const uint8_t *sk, uint32_t sk_len, const uint8_t *v, uint32_t vlen,
                      uint32_t now, uint8_t *new_value, int32_t *value_changed)
{
    std::string nv;
    bool ch = false;
    bool del = o->ops[i].filter(mk(hk, hk_len), mk(sk, sk_len), mk(v, vlen), now, &nv, &ch);
    *value_changed = ch;
    if (ch) memcpy(new_value, nv.data(), nv.size());
    return del;
}
int32_t orc_filter(const orc_filter_params *p, const uint8_t *key, uint32_t klen, const uint8_t *v,
                   uint32_t vlen, uint32_t now, uint8_t *new_value, int32_t *value_changed)
{
    FilterParams fp;
    fp.enabled = p->enabled;
    fp.validate_hash = p->validate_hash;
    fp.data_version = p->data_version;
    fp.default_ttl = p->default_ttl;
    fp.pidx = p->pidx;
    fp.partition_version = p->partition_version;
    fp.ops = p->ops ? &p->ops->ops : nullptr;
    std::string nv;
    bool ch = false;
    DropReason r = compaction_filter(fp, mk(key, klen), mk(v, vlen), now, &nv, &ch);
    *value_changed = ch;
    if (ch) memcpy(new_value, nv.data(), nv.size());
    return r != kKeep;
}

} // extern "C"
