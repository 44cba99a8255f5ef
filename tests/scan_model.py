"""A plain Python model of the range-scan loop, shared by the scan tests (simulator, device, oracle pin).

model_scan() is the reference's iterator loop (src/server/pegasus_server_impl.cpp:617-756 multi_get, :1243-1320 scanners) over
the VISIBLE records of a database (newest version of each user key; tombstones hide the key), evaluated record by record:
forward = Seek(start) + Next, reverse = SeekForPrev(stop) + Prev.  It returns what a pgs_scan_result holds plus the kvs in
iteration order (the kernels emit them so; the server re-reverses a reverse multi_get).  The helpers below marshal request
dicts into pgs_scan_request arrays and read the answers of pgs_range_scan / pgs_range_scan_many back."""
import bisect
import ctypes as C

import numpy as np

from incubator_pegasus_b200 import synth

NOW = synth.NOW


def be(n, w):
    return int(n).to_bytes(w, "big")


def raw_key(hk, sk):
    return be(len(hk), 2) + hk + sk


def value(ets, data):
    return be(ets, 4) + be((1 << 8) | 2, 8) + data


def next_key(b):
    """the smallest key greater than every key that starts with b (b must not be all 0xff)"""
    b = bytearray(b)
    while b and b[-1] == 0xFF:
        b.pop()
    b[-1] += 1
    return bytes(b)


def make_db(pgs, rng, n_runs, hashkeys, sort_per_hk, big=False):
    """n_runs runs, NEWEST FIRST (as Partition.runs): each write gets a global seq; a run holds a random subset of keys."""
    seq = 0
    runs_items = []
    for r in range(n_runs):  # oldest run first while generating
        items = {}
        for hk in hashkeys:
            for s in range(sort_per_hk):
                if rng.random() < 0.45:
                    continue
                sk = b"s%04d" % s
                for _ in range(int(rng.integers(1, 3))):
                    seq += 1
                    u = rng.random()
                    if u < 0.12:
                        items[(raw_key(hk, sk), -seq)] = (raw_key(hk, sk), seq, 0, b"")
                    else:
                        ets = 0 if u < 0.6 else (NOW + int(rng.integers(1, 1000)) if u < 0.85 else NOW - int(rng.integers(0, 1000)))
                        dl = int(rng.integers(0, 30)) if not big or rng.random() < 0.9 else int(rng.integers(600, 1500))
                        items[(raw_key(hk, sk), -seq)] = (raw_key(hk, sk), seq, 1, value(ets, bytes(rng.integers(0, 256, dl, dtype=np.uint8))))
        runs_items.append([items[k] for k in sorted(items)])
    runs_items.reverse()  # newest first
    return [pgs.Records.from_list(it) for it in runs_items if it], runs_items


def visible(runs_items):
    """newest version of every user key; tombstones hide the key.  -> sorted [(key, value)]"""
    best = {}
    for items in runs_items:
        for k, s, t, v in items:
            if k not in best or s > best[k][0]:
                best[k] = (s, t, v)
    return [(k, v) for k, (s, t, v) in sorted(best.items()) if t == 1], best


def crc64(data):
    """crc64 of src/utils/crc.cpp (reflected, polynomial 0x9a6c9329ac4bc9b5), as check_pegasus_key_hash uses it"""
    from test_kernel_sim import crc_table
    tab = crc64.tab = getattr(crc64, "tab", None) or crc_table()
    c = (1 << 64) - 1
    for b in data:
        c = tab[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ ((1 << 64) - 1)


def expire_ts(v):
    """BE32 of the value's first four bytes; a value shorter than that (which the reference never writes) has none, as
    the kernels read it"""
    return int.from_bytes(v[:4], "big") if len(v) >= 4 else 0


def _match(ft, pat, s):
    """validate_filter of the read path (pegasus_server_impl.cpp:2350-2380): an empty pattern matches"""
    if ft == 0 or not pat:
        return True
    return {1: pat in s, 2: s.startswith(pat), 3: s.endswith(pat)}[ft]


def _state(k, v, q, now):
    """validate_key_value_for_scan (:2382-2430): 'normal', 'expired', 'hash' (kHashInvalid) or 'filtered'"""
    ets = expire_ts(v)
    if 0 < ets <= now:
        return "expired"
    hl = int.from_bytes(k[:2], "big") if len(k) >= 2 else 0
    if 2 + hl > len(k):
        hl = max(0, len(k) - 2)
    hk, sk = k[2:2 + hl], k[2 + hl:]
    if q.get("validate_hash"):
        pv, pidx = q.get("partition_version", -1), q.get("pidx", 0)
        bad = pv < 0 or pidx > pv
        if not bad and len(k) >= 2:
            bad = (crc64(hk if hk else sk) & pv) != pidx
        if bad:
            return "hash"
    if not _match(q.get("hft", 0), q.get("hpat", b""), hk) or not _match(q.get("sft", 0), q.get("spat", b""), sk):
        return "filtered"
    return "normal"


def model_scan(vis, q, now=NOW):
    """the reference loop over the visible records; returns dict like pgs_scan_result + kvs (in iteration order).
    q: start, stop, start_inclusive, stop_inclusive, max_count, max_iter_count, max_iter_size, key_mode, and optionally
    reverse, prefix (prefix_same_as_start), has_upper, no_value, count_only, return_expire_ts, hft/hpat, sft/spat,
    validate_hash/pidx/partition_version."""
    start, stop, rev = q["start"], q["stop"], bool(q.get("reverse"))
    keys = [k for k, _ in vis]
    if rev:
        pos, step = bisect.bisect_right(keys, stop) - 1, -1    # SeekForPrev(stop)
        first_excl, skip_key = not q["stop_inclusive"], stop
    else:
        pos, step = bisect.bisect_left(keys, start), 1         # Seek(start)
        first_excl, skip_key = not q["start_inclusive"], start
    prefix = None  # prefix_same_as_start / iterate_upper_bound: forward iterators only (reverse seeks in total order)
    if not rev and q.get("prefix") and len(start) >= 2:
        hl = int.from_bytes(start[:2], "big")
        if 2 + hl <= len(start):
            prefix = start[:2 + hl]

    def valid(p):
        if p < 0 or p >= len(vis):
            return False
        k = vis[p][0]
        if prefix is not None and k[:len(prefix)] != prefix:
            return False
        if not rev and q.get("has_upper") and k >= stop:
            return False
        return True

    def beyond_end(k):  # the range end in iteration direction
        if rev:
            return k < start or (k == start and not q["start_inclusive"])
        return k > stop or (k == stop and not q["stop_inclusive"])
    end_key = start if rev else stop
    count = it = exp = fil = size = 0
    kvs = []
    complete = False
    while count < q["max_count"] and it < q["max_iter_count"] and not (q["max_iter_size"] > 0 and size >= q["max_iter_size"]) and valid(pos):
        k, v = vis[pos]
        if beyond_end(k):
            complete = True
            break
        if first_excl:
            first_excl = False
            if k == skip_key:
                pos += step
                continue
        it += 1
        st = _state(k, v, q, now)
        if st == "expired":
            exp += 1
        elif st == "filtered":
            fil += 1
        elif st == "normal":
            hl = int.from_bytes(k[:2], "big")
            ko = k[2 + hl:] if q["key_mode"] == 1 else k
            vo = b"" if q.get("no_value") else v[12:]
            count += 1
            size += len(ko) + len(vo)
            if not q.get("count_only"):
                kvs.append((ko, vo, expire_ts(v) if q.get("return_expire_ts") else 0))
        if k == end_key:
            complete = True
            break
        pos += step
    iv = valid(pos)
    return dict(count=count, iter_count=it, expire_count=exp, filter_count=fil, size=size, complete=complete, iter_valid=iv,
                resume=vis[pos][0] if iv and not complete else None, kvs=kvs)


def scan_list(hks):
    """the request list of the scan tests: multi_get shapes over every hash key with each limit, bounds, filters"""
    reqs = []
    for hk in hks + [b"nope"]:
        lo, hi = raw_key(hk, b""), raw_key(hk, b"\xff" * 8)
        nxt = next_key(raw_key(hk, b""))
        base = dict(start=lo, stop=nxt, start_inclusive=True, stop_inclusive=False, key_mode=1, prefix=1,
                    max_count=3000, max_iter_count=3000, max_iter_size=0)
        reqs.append(base)                                                               # multi_get: whole hash key
        reqs.append(dict(base, max_count=7))                                            # count limit
        reqs.append(dict(base, max_iter_count=9))                                       # iteration limit
        reqs.append(dict(base, max_iter_size=100))                                      # size limit
        reqs.append(dict(base, start=raw_key(hk, b"s0010"), stop=raw_key(hk, b"s0020"), stop_inclusive=True))
        reqs.append(dict(base, start=raw_key(hk, b"s0010"), start_inclusive=False, stop=raw_key(hk, b"s0010"), stop_inclusive=True))
        reqs.append(dict(base, start=raw_key(hk, b"s0005"), start_inclusive=False, no_value=1))
        reqs.append(dict(base, sft=3, spat=b"7"))                                       # sort-key postfix filter
        reqs.append(dict(base, sft=1, spat=b"01", count_only=1))
        reqs.append(dict(base, has_upper=1, count_only=1, max_count=2**32 - 1, max_iter_count=2**32 - 1))  # sortkey_count
        reqs.append(dict(base, key_mode=0, prefix=0, stop=hi, hft=2, hpat=hk[:1], return_expire_ts=1, max_count=11))  # scanner batch
        reqs.append(dict(base, key_mode=0, prefix=0, validate_hash=1, pidx=1, partition_version=3, max_count=20))  # partition hash
    reqs.append(dict(start=b"", stop=b"\xff\xff\xff", start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0,
                     max_count=100000, max_iter_count=100000, max_iter_size=0))         # full table
    reqs.append(dict(start=b"\x00\x02h", stop=b"\x00\x02h5", start_inclusive=True, stop_inclusive=False, key_mode=0, prefix=0,
                     max_count=40, max_iter_count=1000, max_iter_size=0))
    return reqs


def filter_list(full):
    """the record rules over a whole-range request `full`: every hash- and sort-key filter type, an empty pattern, and
    validate_hash with a stale partition index, an invalid partition version and a valid one"""
    reqs = []
    for ft in (1, 2, 3):
        reqs += [dict(full, hft=ft, hpat=b"h1"), dict(full, sft=ft, spat=b"1", max_count=50), dict(full, hft=ft, hpat=b"", sft=ft, spat=b"00")]
    reqs += [dict(full, validate_hash=1, pidx=5, partition_version=3),          # stale partition index: every record kHashInvalid
             dict(full, validate_hash=1, pidx=0, partition_version=-1),
             dict(full, validate_hash=1, pidx=2, partition_version=7, max_count=40),
             dict(full, key_mode=1, no_value=1, return_expire_ts=1), dict(full, count_only=1), dict(full, return_expire_ts=1, max_count=60)]
    return reqs


def mirror(q):
    """the same request iterated the other way (prefix_same_as_start and has_upper then have no effect)"""
    return dict(q, reverse=not q.get("reverse"))


def scan_requests(pgs, reqs, keep):
    """request dicts -> a pgs_scan_request array (the byte strings stay alive in `keep`)"""
    def blob(b):
        buf = (C.c_uint8 * max(1, len(b))).from_buffer_copy(b if b else b"\0")
        keep.append(buf)
        return pgs.Blob(C.cast(buf, C.POINTER(C.c_uint8)), len(b))
    arr = (pgs.ScanRequest * max(1, len(reqs)))()
    for i, q in enumerate(reqs):
        r = arr[i]
        r.start, r.stop = blob(q["start"]), blob(q["stop"])
        r.start_inclusive, r.stop_inclusive, r.reverse = int(q["start_inclusive"]), int(q["stop_inclusive"]), int(bool(q.get("reverse")))
        r.no_value, r.key_mode, r.return_expire_ts = int(q.get("no_value", 0)), q["key_mode"], int(q.get("return_expire_ts", 0))
        r.count_only, r.prefix_same_as_start = int(q.get("count_only", 0)), int(q.get("prefix", 0))
        r.reserved[0] = int(q.get("has_upper", 0))
        r.validate_hash, r.pidx, r.partition_version = int(q.get("validate_hash", 0)), q.get("pidx", 0), q.get("partition_version", -1)
        r.hash_filter_type, r.sort_filter_type = q.get("hft", 0), q.get("sft", 0)
        r.hash_filter, r.sort_filter = blob(q.get("hpat", b"")), blob(q.get("spat", b""))
        r.max_count, r.max_iter_count, r.max_iter_size = q["max_count"], q["max_iter_count"], q["max_iter_size"]
    keep.append(arr)
    return arr


def answer(r, arena, kvs, resume):
    """one pgs_scan_result + its kv records (key/value offsets into `arena`) -> the dict model_scan returns"""
    recs = [(arena[kv.key_off:kv.key_off + kv.key_len].tobytes(), arena[kv.value_off:kv.value_off + kv.value_len].tobytes(), kv.expire_ts)
            for kv in kvs]
    return dict(count=r.count, iter_count=r.iter_count, expire_count=r.expire_count, filter_count=r.filter_count, size=r.size,
                complete=bool(r.complete), iter_valid=bool(r.iter_valid),
                resume=bytes(resume[:r.resume_len]) if r.iter_valid and not r.complete else None, kvs=recs)


def diff(got, want):
    return {k: (got[k], want[k]) for k in want if got[k] != want[k]}


# ---- the packed read-back of a batch (pgs_range_scan / pgs_range_scan_many[_multi]) ---------------------------------------------
SLICE_MAX = 2**32 - 16  # pgs_kv's offsets are 32-bit: the most one request's slice holds


def round16(x):
    return (x + 15) & ~15


def slice_bytes(arena_stride):
    """the arena slice each request of a batch writes into"""
    return min(round16(arena_stride), SLICE_MAX)


def pack_offsets(used, n_kvs):
    """k_pack_offsets: request i's output at arena_base[i], each one rounded up to 16 bytes, and its kvs at kv_base[i]"""
    ab, kb = [0], [0]
    for u, k in zip(used, n_kvs):
        ab.append(ab[-1] + round16(u))
        kb.append(kb[-1] + k)
    return ab, kb


def model_batch(answers, arena_stride, kv_stride, arena_cap, kv_cap):
    """the status and (arena_base, kv_base) of a batch whose requests answer `answers` (model_scan dicts).  PGS_ABORTED when an
    output passes its slice or kv_stride records; else PGS_INCOMPLETE when the packed batch passes arena_cap or kv_cap; else
    PGS_OK.  A batch of one request is read back unpadded."""
    used = [sum(len(k) + len(v) for k, v, _ in a["kvs"]) for a in answers]
    n_kvs = [len(a["kvs"]) for a in answers]
    if any(u > slice_bytes(arena_stride) or k > kv_stride for u, k in zip(used, n_kvs)):
        return "ABORTED", None, None
    ab, kb = ([0, used[0]], [0, n_kvs[0]]) if len(answers) == 1 else pack_offsets(used, n_kvs)
    if ab[-1] > arena_cap or kb[-1] > kv_cap:
        return "INCOMPLETE", None, None
    return "OK", ab, kb


def check_packed(results, arena, kvs, ab, kb, answers, want_ab, want_kb):
    """a packed read-back against the model: the bases, every result's sizes, every kv's offsets, and the output bytes
    [ab[i], ab[i] + arena_used[i]) of every request (never the padding after them)"""
    assert [int(x) for x in ab] == want_ab and [int(x) for x in kb] == want_kb
    outs = {}  # a batch repeats its requests: each answer's bytes joined once
    for i, a in enumerate(answers):
        r, base = results[i], int(ab[i])
        out = outs.get(id(a))
        if out is None:
            out = outs[id(a)] = b"".join(k + v for k, v, _ in a["kvs"])
        assert (r.arena_used, r.n_kvs) == (len(out), len(a["kvs"])), i
        assert arena[base:base + len(out)].tobytes() == out, i
        off = 0
        for j, (k, v, ets) in enumerate(a["kvs"]):
            kv = kvs[int(kb[i]) + j]
            assert (kv.key_off, kv.key_len, kv.value_off, kv.value_len, kv.expire_ts) == (off, len(k), off + len(k), len(v), ets), (i, j)
            off += len(k) + len(v)
