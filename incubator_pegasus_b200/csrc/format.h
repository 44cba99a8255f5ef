// format.h — byte formats shared by the host code and the CUDA kernels of the product.
//
// Pegasus side (kept bit-exact, they are what clients and replicas exchange):
//   raw key   = BE16(len(hashkey)) || hashkey || sortkey      src/base/pegasus_key_schema.h:35-59
//   raw value = BE32(expire_ts) [|| BE64(timetag)] || user     src/base/pegasus_value_schema.h:158,205
// LSM side (RocksDB v8.5.3's data-block encoding, restated; the engine keeps it so that the
// decode work is the honest one and real SST blocks can be ingested later):
//   internal key = user_key || fixed64_le((seq << 8) | type)
//   entry        = varint32 shared | varint32 non_shared | varint32 value_len | key_delta | value
//   block        = entries | fixed32_le restart_offset[n] | fixed32_le n
// HBM-resident run = blocks (each start 16-byte aligned so cp.async.bulk can move them) plus a
// device-built index: per block its offset, size, cumulative record count and last user key.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PGS_HD __host__ __device__ __forceinline__
#else
#define PGS_HD inline
#endif

namespace pgs {

constexpr uint32_t kDefaultBlockSize = 4096;
constexpr uint32_t kDefaultRestartInterval = 16;
constexpr uint32_t kBlockAlign = 16;
constexpr uint32_t kMaxRuns = 16;        // k of one merge launch
constexpr uint32_t kMaxUkeyLen = 4096;   // compaction / lookup fast path limit
constexpr uint32_t kEpochBegin = 1451606400u; // src/base/pegasus_utils.h:39

PGS_HD uint32_t be32(const uint8_t *p)
{
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
PGS_HD uint16_t be16(const uint8_t *p) { return (uint16_t)((p[0] << 8) | p[1]); }
PGS_HD uint32_t le32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
PGS_HD uint32_t le16(const uint8_t *p) { return p[0] | (p[1] << 8); }
PGS_HD uint32_t varint_len(uint32_t v) { return v < 128 ? 1 : v < 16384 ? 2 : v < 2097152 ? 3 : v < 268435456 ? 4 : 5; }
PGS_HD uint32_t user_data_offset(uint32_t version) { return version == 1 ? 12u : 4u; }
PGS_HD bool ts_expired(uint32_t now, uint32_t ts) { return ts > 0 && ts <= now; }

// the hash key and sort key of a raw key.  A hash-key length that runs past the key is clamped to it (the reference CHECKs),
// so a malformed key is never read outside its buffer; a key shorter than two bytes has neither.
struct KeyParts {
    const uint8_t *hk, *sk;
    uint32_t hkl, skl;
};
PGS_HD KeyParts split_key(const uint8_t *key, uint32_t len)
{
    uint32_t hkl = len >= 2 ? be16(key) : 0u;
    if (hkl + 2 > len) hkl = len >= 2 ? len - 2 : 0u;
    return {key + 2, key + 2 + hkl, hkl, len >= 2 ? len - 2 - hkl : 0u};
}

// pegasus_key_hash (pegasus_key_schema.h:150-165): crc64 of the hash key, or of the sort key when the hash key is empty.
// `table` = the crc64 table of crc64_make_table (uint64_t on the host, unsigned long long copies on the device).
template <class T>
PGS_HD uint64_t pegasus_key_hash(const T *table, const uint8_t *key, uint32_t len)
{
    const KeyParts k = split_key(key, len);
    const uint8_t *p = k.hkl ? k.hk : k.sk;
    const uint32_t n = k.hkl ? k.hkl : k.skl;
    uint64_t c = ~0ull;
    for (uint32_t i = 0; i < n; i++) c = table[(uint8_t)(c ^ p[i])] ^ (c >> 8);
    return ~c;
}

// Bucket hash of the hot-key collectors (host/hotkey.h, hotkey_kernels.cuh): it only decides which hash keys share a coarse
// bucket, never which key is reported.  Not crc64: every key of a partition has the same crc64 % partition_count, so crc64
// buckets would be correlated with the partition.  The hash is a sum of independently mixed 32-bit words (word j = bytes
// 4j..4j+3 little endian, zero padded past the end, mixed with its index), so that the lanes of a group can each hash some
// words of a long key and add their partial sums.
PGS_HD uint32_t hotkey_word(const uint8_t *p, uint32_t len, uint32_t j)
{
    uint32_t w = 0;
    for (uint32_t b = 0; b < 4 && 4 * j + b < len; b++) w |= (uint32_t)p[4 * j + b] << (8 * b);
    return w;
}
PGS_HD uint64_t hotkey_mix(uint64_t x)
{
    x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27; x *= 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
PGS_HD uint64_t hotkey_word_hash(uint32_t w, uint32_t j) { return hotkey_mix(((uint64_t)j << 32 | w) + 0x9E3779B97F4A7C15ull); }
PGS_HD uint64_t hotkey_finish(uint64_t sum, uint32_t len) { return hotkey_mix(sum ^ ((uint64_t)len * 0xD6E8FEB86659FD93ull)); }
PGS_HD uint64_t hotkey_hash(const uint8_t *p, uint32_t len)
{
    uint64_t s = 0;
    for (uint32_t j = 0; 4 * j < len; j++) s += hotkey_word_hash(hotkey_word(p, len, j), j);
    return hotkey_finish(s, len);
}
PGS_HD uint32_t hotkey_bucket(const uint8_t *hash_key, uint32_t len, uint32_t n_buckets) { return (uint32_t)(hotkey_hash(hash_key, len) % n_buckets); }

// crc64 table (host): reflected CRC-64, table driven; polynomial bits from utils/crc.cpp:289-295
inline void crc64_make_table(uint64_t tab[256])
{
    const int bits[] = {63, 61, 59, 58, 56, 55, 52, 49, 48, 47, 46, 44, 41, 37, 36, 34,
                        32, 31, 28, 26, 23, 22, 19, 16, 13, 12, 10, 9,  6,  4,  3,  0};
    uint64_t poly = 0;
    for (int b : bits) poly |= 1ull << (63 - b);
    for (uint32_t i = 0; i < 256; i++) {
        uint64_t c = i;
        for (int r = 0; r < 8; r++) c = (c >> 1) ^ ((c & 1) ? poly : 0);
        tab[i] = c;
    }
}

// binary ops table handed to the compaction kernel (pgs_compaction_ops_parse):
//   u32 n_ops
//   per op : u8 op_type(0 update_ttl,1 delete) u8 ttl_type u16 n_rules u32 ttl_value
//   per rule: u8 rule_type u8 match_type u16 pattern_len u32 start_ttl u32 stop_ttl
//             pattern bytes, zero padded to a multiple of 4
enum { OP_UPDATE_TTL = 0, OP_DELETE = 1 };
enum { RULE_HASHKEY = 0, RULE_SORTKEY = 1, RULE_TTL_RANGE = 2 };
enum { MATCH_ANYWHERE = 0, MATCH_PREFIX = 1, MATCH_POSTFIX = 2, MATCH_INVALID = 3 };
enum { TTL_FROM_NOW = 0, TTL_FROM_CURRENT = 1, TTL_TIMESTAMP = 2, TTL_INVALID = 3 };

// true when t[0..len) is a table of the form above that the compaction kernel may walk: every op and rule type is known and
// the walk ends exactly at len.  A caller of the C ABI may hand in any bytes; the kernel trusts the framing.
inline bool ops_table_valid(const uint8_t *t, uint64_t len)
{
    if (len < 4) return false;
    const uint32_t n_ops = t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24;
    uint64_t p = 4;
    for (uint32_t o = 0; o < n_ops; o++) {
        if (len - p < 8) return false;
        const uint32_t op_type = t[p], ttl_type = t[p + 1], n_rules = t[p + 2] | (uint32_t)t[p + 3] << 8;
        if (op_type > OP_DELETE || ttl_type > TTL_INVALID) return false;
        p += 8;
        for (uint32_t r = 0; r < n_rules; r++) {
            if (len - p < 12) return false;
            const uint32_t rule_type = t[p], match_type = t[p + 1], pl = t[p + 2] | (uint32_t)t[p + 3] << 8;
            if (rule_type > RULE_TTL_RANGE || match_type > MATCH_INVALID) return false;
            const uint64_t step = 12 + ((pl + 3) & ~3u);
            if (len - p < step) return false;
            p += step;
        }
    }
    return p == len;
}

// what kernels see of one HBM-resident sorted run
struct RunDev {
    const uint8_t *data;      // blocks, each start 16-aligned; readable up to blk_off[nb] (+slack)
    const uint64_t *blk_off;  // [nb+1] byte offset of block b; blk_off[nb] = 16-aligned end
    const uint32_t *blk_size; // [nb]   exact encoded size
    const uint32_t *blk_rec;  // [nb+1] cumulative record count
    const uint32_t *ikey_off; // [nb+1] offsets into ikeys
    const uint8_t *ikeys;     // last user key of every block, back to back
    const uint32_t *rec_off;  // [n_records] byte offset of every entry inside its block (reverse-scan kernel)
    const uint32_t *bloom;    // Bloom filter over whole user keys and hash-key prefixes: bloom_lines lines of 64 bytes (0 = none)
    uint32_t bloom_lines;
    uint32_t nb;
    uint32_t max_ukey_len;
    uint32_t pad;
};

} // namespace pgs
