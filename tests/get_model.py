"""A plain Python model of the point lookup (k_get) and of the runs' Bloom filters, shared by the get tests (simulator, device,
oracle pin).

model_get() answers one key the way on_get does (src/server/pegasus_server_impl.cpp:441-490): the newest run holding the user
key decides, its newest version is the answer, a tombstone means NotFound, an expired value means NotFound with `expired`, and
the user data is the value without its header.  model_stats() predicts the two counters a get launch reports
(pgs_engine_last_blocks_probed / pgs_engine_last_runs_skipped) exactly; for that the model rebuilds every run's filter bit
for bit: the hash and the bit layout restate group.cuh, the sizing rules restate engine.cu (upload) and compact.cu
(compaction).  Runs are given NEWEST FIRST, as Partition.runs() lists them."""
import numpy as np

M32 = 0xFFFFFFFF
M64 = (1 << 64) - 1
NOT_FOUND, OK, INCOMPLETE = 1, 0, 7


# ---- the filter (group.cuh: bloom_word, bloom_finish, bloom_bit, bloom_may_contain) ---------------------------------------
def bloom_word(w, idx, ha, hb):
    a = ((w + 0x9E3779B9 * (idx + 1)) * 0x85EBCA6B) & M32
    a ^= a >> 15
    a = (a * 0xC2B2AE35) & M32
    a ^= a >> 13
    b = (a * 0x27D4EB2F) & M32
    b ^= b >> 16
    return ha ^ a, hb ^ b


def bloom_finish(ha, hb, n):
    h = ((ha ^ ((n * 0x9E3779B1) & M32)) << 32) | hb
    h ^= h >> 29
    h = (h * 0xD6E8FEB86659FD93) & M64
    h ^= h >> 32
    return h


def bloom_hash(key):
    """the hash of a byte string: little-endian 32-bit words, the last one zero padded, salted by position and length"""
    ha = hb = 0
    padded = key + b"\0" * (-len(key) % 4)
    for i, w in enumerate(np.frombuffer(padded, "<u4").tolist()):
        ha, hb = bloom_word(w, i, ha, hb)
    return bloom_finish(ha, hb, len(key))


def bloom_bit(h, i):
    x = ((h & M32) + i * 0x9E3779B1) & M32
    x ^= x >> 15
    x = (x * 0x2C1B3C6D) & M32
    x ^= x >> 12
    return x & 511


def bloom_lines_for(n):
    """10 bits per entry in 512-bit lines, one line extra"""
    return (10 * n + 511) // 512 + 1


def prefix_len(key):
    """HashkeyTransform: the first 2 + BE16 bytes of a key; 0 when the key is shorter than that"""
    if len(key) < 2:
        return 0
    p = 2 + int.from_bytes(key[:2], "big")
    return p if p <= len(key) else 0


class Bloom:
    """n_lines lines of 512 bits; an entry hashes to one line and sets 6 bits in it"""

    def __init__(self, n_lines):
        self.n_lines = n_lines
        self.lines = [0] * n_lines

    def _line(self, h):
        return ((h >> 32) * self.n_lines) >> 32

    def add(self, key):
        h = bloom_hash(key)
        li = self._line(h)
        for i in range(6):
            self.lines[li] |= 1 << bloom_bit(h, i)

    def may_contain(self, key):
        if self.n_lines == 0:
            return True
        h = bloom_hash(key)
        line = self.lines[self._line(h)]
        return all(line >> bloom_bit(h, i) & 1 for i in range(6))

    def words(self):
        """the filter as the device holds it: n_lines x 16 little-endian uint32"""
        return np.array([(line >> (32 * w)) & M32 for line in self.lines for w in range(16)], np.uint32)


# ---- runs -------------------------------------------------------------------------------------------------------------
def _varint(buf, p):
    v = sh = 0
    while True:
        c = buf[p]
        p += 1
        v |= (c & 127) << sh
        sh += 7
        if c < 128:
            return v, p


def parse_blocks(br):
    """a BlockRun -> per block, its entries as (user key, seq, type, value, shared)"""
    data = br.data.tobytes()
    blocks = []
    for off, size in zip(br.blk_off.tolist(), br.blk_size.tolist()):
        blk = data[off:off + size]
        nr = int.from_bytes(blk[-4:], "little")
        limit, p, key, ents = size - 4 - 4 * nr, 0, b"", []
        while p < limit:
            sh, p = _varint(blk, p)
            ns, p = _varint(blk, p)
            vl, p = _varint(blk, p)
            key = key[:sh] + blk[p:p + ns]
            p += ns
            tr = int.from_bytes(key[-8:], "little")
            ents.append((key[:-8], tr >> 8, tr & 0xFF, blk[p:p + vl], sh))
            p += vl
        blocks.append(ents)
    return blocks


class ModelRun:
    """one run as the lookup sees it: the newest version of every user key, the last user key, the filter"""

    def __init__(self, blocks, bloom, n_bloom_entries):
        self.blocks = blocks
        self.newest = {}
        for ents in blocks:
            for k, _s, t, v, _sh in ents:
                self.newest.setdefault(k, (t, v))   # entries are ordered by (key, seq descending)
        self.last_key = blocks[-1][-1][0] if blocks else None
        self.bloom = bloom
        self.n_bloom_entries = n_bloom_entries


def uploaded_run(br):
    """the filter k_index_walk builds at upload (engine.cu): every user key, plus the hash-key prefix of every entry whose
    prefix length is non-zero and differs from the previous entry's in the same block, or whose `shared` is shorter than
    the prefix; sized for n_records + that count"""
    blocks = parse_blocks(br)
    entries = []
    for ents in blocks:
        prev_pl = None
        for k, _s, _t, _v, sh in ents:
            entries.append(k)
            pl = prefix_len(k)
            if pl and (pl != prev_pl or sh < pl):
                entries.append(k[:pl])
            prev_pl = pl
    bloom = Bloom(bloom_lines_for(len(entries)))
    for e in entries:
        bloom.add(e)
    return ModelRun(blocks, bloom, len(entries))


def compacted_run(br, inputs):
    """the filter k_emit builds for a compaction output whose inputs were all uploaded (compact.cu): sized for the inputs'
    entries together; its bits are every surviving user key and every distinct surviving hash-key prefix"""
    blocks = parse_blocks(br)
    bloom = Bloom(bloom_lines_for(sum(r.n_bloom_entries for r in inputs)))
    prefixes = set()
    for ents in blocks:
        for k, *_ in ents:
            bloom.add(k)
            pl = prefix_len(k)
            if pl:
                prefixes.add(k[:pl])
    for p in prefixes:
        bloom.add(p)
    return ModelRun(blocks, bloom, None)


def unknown_filter_run(br):
    """a run whose filter the model does not rebuild (deeper compaction generations): values only, no stats"""
    return ModelRun(parse_blocks(br), None, None)


def key_slot(run_lists):
    """KS of a launch (lookup.cu snapshot_runs): the longest user key of the runs rounded up to 8, at least 8; for a
    multi-partition launch the maximum over the partitions"""
    mk = max([len(k) for runs in run_lists for r in runs for k in r.newest] + [0])
    return max(8, (mk + 7) & ~7)


# ---- the lookup ---------------------------------------------------------------------------------------------------------
def model_get(runs, key, now, data_version=1, ks=None):
    """-> dict(status, expired, expire_ts, value) as pgs_get_result + the value bytes (None unless OK)"""
    ks = key_slot([runs]) if ks is None else ks
    miss = dict(status=NOT_FOUND, expired=0, expire_ts=0, value=None)
    if len(key) > ks:
        return miss
    for r in runs:
        if key not in r.newest:
            continue
        t, v = r.newest[key]
        if t == 0:
            return miss
        ets = int.from_bytes(v[:4], "big") if len(v) >= 4 else 0
        if 0 < ets <= now:
            return dict(status=NOT_FOUND, expired=1, expire_ts=ets, value=None)
        hdr = 12 if data_version == 1 else 4
        return dict(status=OK, expired=0, expire_ts=ets, value=v[hdr:] if len(v) >= hdr else b"")
    return miss


def model_stats(runs, keys, ks=None):
    """-> (blocks probed, runs skipped): per key, newest run first until a hit: a run whose filter excludes the key counts a
    skip; otherwise a key <= the run's last user key counts a probe.  A key longer than KS touches no run."""
    ks = key_slot([runs]) if ks is None else ks
    probes = skipped = 0
    for key in keys:
        if len(key) > ks:
            continue
        for r in runs:
            if r.bloom is not None and not r.bloom.may_contain(key):
                skipped += 1
                continue
            if r.last_key is not None and key <= r.last_key:
                probes += 1
            if key in r.newest:
                break
    return probes, skipped


def query_keys(runs, rng=None):
    """the query set of the get tests: every stored key, the first and last key of every block, every stored key with a byte
    added or removed, the bare hash key of every stored key (it hashes like the prefix entry), short keys, absent keys"""
    stored = sorted({k for r in runs for k in r.newest})
    q = list(stored)
    for r in runs:
        for ents in r.blocks:
            q += [ents[0][0], ents[-1][0]]
    for k in stored:
        q += [k + b"\x00", k + b"\xff", k[:-1]]
        pl = prefix_len(k)
        if pl:
            q.append(k[:pl])
    q += [b"", b"\x00", b"\xff", b"\x00\x00", b"\x00\x01", b"\x00\x01z", b"\xff\xff", b"zz-absent", b"\x00\x03abc-absent"]
    if stored:
        ks = key_slot([runs])
        q += [stored[-1][:1] * ks, b"\x00" * ks, b"\x00" * (ks + 1), b"\x7f" * (ks + 1), b"\x00\x01" + b"a" * 4095]
    return q


def flat_keys(keys):
    """keys -> (uint8 array, uint32 offsets) as pgs_get_batch takes them"""
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    flat = np.frombuffer(b"".join(keys), np.uint8).copy() if off[-1] else np.zeros(1, np.uint8)
    return flat, off


def check_results(results, arena, keys, want, cap=None):
    """compare pgs_get_result records + arena with model_get answers, field by field; values must be 4-aligned, inside the
    arena cap and disjoint.  -> the number of OK results"""
    spans, n_ok = [], 0
    for i, (k, w) in enumerate(zip(keys, want)):
        r = results[i]
        got = dict(status=r.status, expired=r.expired, expire_ts=r.expire_ts)
        assert got == {f: w[f] for f in got}, (i, k[:40], len(k), got, {f: w[f] for f in got})
        if w["status"] == OK:
            n_ok += 1
            assert r.value_len == len(w["value"]), (i, k[:40], r.value_len, len(w["value"]))
            assert arena[r.value_off:r.value_off + r.value_len].tobytes() == w["value"], (i, k[:40])
            assert r.value_off % 4 == 0 and (cap is None or r.value_off + r.value_len <= cap), (i, r.value_off)
            if r.value_len:
                spans.append((r.value_off, r.value_off + r.value_len))
        else:
            assert r.value_len == 0 and r.value_off == 0, (i, k[:40])
    spans.sort()
    for a, b in zip(spans, spans[1:]):
        assert a[1] <= b[0], ("overlapping values", a, b)
    return n_ok


# ---- data -----------------------------------------------------------------------------------------------------------------
def _raw_key(hk, sk):
    return len(hk).to_bytes(2, "big") + hk + sk


HOT = _raw_key(b"hot", b"key")


def sweep_keys(rng, long_keys=True):
    """user keys of every length 0..300 (random bytes), hash keys of every length 0..140 (with two sort keys and the bare hash
    key), pairs of hash keys that differ only in their last byte, and user keys of 4085..4096 bytes"""
    keys = {bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in range(301)}
    for n in range(141):
        hk = bytes((97 + (n + i) % 26) for i in range(n))
        keys |= {_raw_key(hk, b""), _raw_key(hk, b"s1"), _raw_key(hk, b"s2" * (n % 7))}
    for n in (1, 2, 3, 4, 5, 7, 8, 9, 31, 32, 33, 63, 64, 65, 127, 128, 140):
        keys |= {_raw_key(b"p" * (n - 1) + c, b"x") for c in (b"a", b"b")}
    if long_keys:
        keys |= {_raw_key(b"L", b"q" * (n - 3)) for n in (4085, 4088, 4090, 4093, 4094, 4096)}
    return sorted(keys)


def sweep_items(rng, n_runs, keys, now, hot=0):
    """n_runs runs, NEWEST FIRST, each a random half of `keys` with one or two versions; 15 % tombstones; values of 0, 3, 4,
    11, 12 and more bytes (shorter than or equal to the header among them), half of those >= 4 bytes with an expire_ts
    around `now` (`now` itself among them) or none; `hot` versions of HOT (tombstones among them) in the oldest run"""
    seq = 0
    runs_items = []
    for r in range(n_runs):
        items = {}
        for k in keys:
            if rng.random() < 0.5:
                continue
            for _ in range(int(rng.integers(1, 3))):
                seq += 1
                if rng.random() < 0.15:
                    items[(k, -seq)] = (k, seq, 0, b"")
                    continue
                vl = int(rng.choice([0, 3, 4, 11, 12, 13, 20, 40, 100]))
                v = bytes(rng.integers(0, 256, vl, dtype=np.uint8))
                if vl >= 4:
                    u = rng.random()
                    ets = 0 if u < 0.5 else int(rng.choice([now - 100, now - 1, now, now + 1, now + 100]))
                    v = ets.to_bytes(4, "big") + v[4:]
                items[(k, -seq)] = (k, seq, 1, v)
        if r == 0:
            for _ in range(hot):
                seq += 1
                t = 0 if rng.random() < 0.3 else 1
                items[(HOT, -seq)] = (HOT, seq, t, (0).to_bytes(4, "big") + bytes(8) + b"v%d" % seq if t else b"")
        runs_items.append([items[k] for k in sorted(items)])
    return runs_items[::-1]
