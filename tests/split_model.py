"""The partition split restated in plain Python (the tests' reference): the reference's per-record loop of
local_partition_split (src/shell/commands/local_partition_split.cpp:238-283) routes every record of a parent partition
pidx of src_count to writer (pegasus_key_hash(key) % dst_count) / src_count, in the run's order.  Here a record with an empty
user key (the empty write) is dropped; every version, tombstone and value is kept as it is."""

_M = (1 << 64) - 1
# crc64 polynomial bits of the reference (utils/crc.cpp:289-295), reflected table
_BITS = (63, 61, 59, 58, 56, 55, 52, 49, 48, 47, 46, 44, 41, 37, 36, 34, 32, 31, 28, 26, 23, 22, 19, 16, 13, 12, 10, 9, 6, 4, 3, 0)
_POLY = sum(1 << (63 - b) for b in _BITS)


def _table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ (_POLY if c & 1 else 0)
        t.append(c)
    return t


_TAB = _table()


def crc64(data: bytes) -> int:
    c = _M
    for b in data:
        c = _TAB[(c ^ b) & 0xFF] ^ (c >> 8)
    return ~c & _M


def key_hash(key: bytes) -> int:
    """pegasus_key_hash (pegasus_key_schema.h:150-165): crc64 of the hash key, or of the sort key when the hash key is
    empty; a hash-key length that runs past the key is clamped to it"""
    hkl = int.from_bytes(key[:2], "big") if len(key) >= 2 else 0
    if hkl + 2 > len(key):
        hkl = len(key) - 2 if len(key) >= 2 else 0
    return crc64(key[2:2 + hkl] if hkl else key[2:])


def child_of(key: bytes, src_count: int, dst_count: int) -> int:
    return (key_hash(key) % dst_count) // src_count


def split_items(items, src_count: int, dst_count: int):
    """items (ukey, seq, type, value) of one run in order -> (list of the children's items, empty writes dropped)"""
    out = [[] for _ in range(dst_count // src_count)]
    dropped = 0
    for it in items:
        if not it[0]:
            dropped += 1
            continue
        out[child_of(it[0], src_count, dst_count)].append(it)
    return out, dropped
