"""Device tests of the range-scan kernels at the kernel boundary (pgs_range_scan / pgs_range_scan_many through a Partition),
compared with the Python model of tests/scan_model.py: k_scan_fwd for forward-only batches, k_scan for every batch that holds
a reverse request.  Runs of 1..32 with several block geometries, a hot key with hundreds of versions inside one run,
tombstones over older values, values larger than a block, user keys near 4096 bytes, runs rewritten by the GPU compaction,
every request flag, every way of batching the same requests, and the output-limit statuses."""
import ctypes as C

import numpy as np
import pytest

from incubator_pegasus_b200 import synth
from scan_model import answer, diff, filter_list, mirror, model_scan, next_key, raw_key, scan_list, scan_requests, value, visible

pytestmark = pytest.mark.gpu
NOW = synth.NOW
HKS = [b"h0", b"h1", b"h2", b"", bytes([0xFF, 0xFF])]
HOT = raw_key(b"h1", b"s0011")
RESUME = 4104  # >= the kernels' key slot for user keys of up to 4096 bytes


def build_db(pgs, seed, n_runs, long_keys=False, big=4096):
    """n_runs runs (oldest first) of random writes; every third run holds hundreds of versions of HOT; tombstones shadow
    values of older runs; 1 in 40 values is 1 to 1.5 times `big` bytes (the block size); long_keys adds user keys of
    4088..4096 bytes.  -> (Records per run, [(key, seq, type, value)] per run, newest first)"""
    rng = np.random.default_rng(seed)
    seq = 0
    runs_items = []
    for r in range(n_runs):
        items = {}

        def put(k, t, v):
            nonlocal seq
            seq += 1
            items[(k, -seq)] = (k, seq, t, v if t else b"")
        for hk in HKS:
            for s in range(24):
                if rng.random() < 0.5:
                    continue
                u = rng.random()
                ets = 0 if u < 0.6 else (NOW + 100 if u < 0.8 else NOW - 100)
                dl = int(rng.integers(0, 40)) if rng.random() < 0.975 else int(rng.integers(big + 1, big + big // 2 + 2))
                put(raw_key(hk, b"s%04d" % s), 0 if u < 0.2 else 1, value(ets, bytes(rng.integers(0, 256, dl, dtype=np.uint8))))
        if r % 3 == 0:
            for _ in range(int(rng.integers(200, 400))):
                put(HOT, 0 if rng.random() < 0.3 else 1, value(0, b"v%d" % seq))
        if long_keys and r % 2 == 0:
            for n in (4093, 4090, 4085):  # user keys of 4096 (a multiple of 8: the kernels' key slot), 4093 and 4088 bytes
                put(raw_key(b"L", bytes([97 + r % 3]) * n), 1, value(0, b"long%d" % r))
        runs_items.append([items[k] for k in sorted(items)])
    return [pgs.Records.from_list(it) for it in runs_items], runs_items[::-1]


def load(pgs, eng, recs, block_size, ri, compact_oldest=0):
    """a partition holding the runs (the oldest `compact_oldest` merged by the GPU with the filter off, not bottommost: the
    visible set stays the same, and k_scan reads the entry index k_emit wrote)"""
    part = eng.partition()
    ids = [part.upload(pgs.build_run(r, block_size, ri)) for r in recs]
    if compact_oldest:
        res = part.compact(ids[:compact_oldest], out_level=1, bottommost=0, now=NOW, enabled=False)
        assert res.new_run_id and res.dropped_expired == 0 and res.dropped_tombstone == 0
    return part


def run_scans(pgs, part, reqs, arena_stride=1 << 16, kv_stride=800, arena_cap=None, kv_cap=None, resume_stride=RESUME, resume=None):
    """one pgs_range_scan_many call -> (status, [answer dicts])"""
    n = len(reqs)
    keep = []
    arr = scan_requests(pgs, reqs, keep)
    arena = np.zeros(arena_cap if arena_cap is not None else n * arena_stride, np.uint8)
    kvs = (pgs.KV * max(1, kv_cap if kv_cap is not None else n * kv_stride))()
    resume = np.zeros(max(1, n * resume_stride), np.uint8) if resume is None else resume
    res = (pgs.ScanResult * n)()
    ab, kb = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint32)
    vp = C.c_void_p
    st = pgs.lib().pgs_range_scan_many(part.h, arr, n, NOW, arena_stride, kv_stride, arena.ctypes.data_as(vp), arena.shape[0], kvs,
                                       len(kvs), resume.ctypes.data_as(vp), resume_stride, res, ab.ctypes.data_as(vp), kb.ctypes.data_as(vp))
    if st != 0:
        return st, None
    return st, [answer(res[i], arena[int(ab[i]):], kvs[int(kb[i]):int(kb[i]) + res[i].n_kvs], resume[i * resume_stride:(i + 1) * resume_stride])
                for i in range(n)]


def run_one(pgs, part, q):
    keep = []
    arr = scan_requests(pgs, [q], keep)
    arena = np.zeros(1 << 20, np.uint8)
    kvs = (pgs.KV * 4096)()
    resume = np.zeros(RESUME, np.uint8)
    r = pgs.ScanResult()
    st = pgs.lib().pgs_range_scan(part.h, arr, NOW, arena.ctypes.data_as(C.c_void_p), arena.shape[0], kvs, len(kvs),
                                  resume.ctypes.data_as(C.c_void_p), RESUME, C.byref(r))
    assert st == 0, (st, q)
    return answer(r, arena, kvs[:r.n_kvs], resume)


def request_list(vis):
    """forward requests: the simulator's list, bounds around the stored keys, every filter, limits swept over every record
    (so that some land exactly on the last record of a chunk)"""
    full = dict(start=b"", stop=b"\xff" * 6, start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0,
                max_count=100000, max_iter_count=100000, max_iter_size=0)
    reqs = scan_list(HKS)
    longest = max((k for k, _ in vis), key=len)
    first, last = vis[0][0], vis[-1][0]
    for k in (longest, HOT, first, last):
        for ext in (b"\x00", b"\xff"):  # bounds longer than every stored key (longest + 1 byte: one past the key slot)
            for si in (True, False):
                for ti in (True, False):
                    reqs.append(dict(full, start=k + ext, start_inclusive=si, stop_inclusive=ti))
                    reqs.append(dict(full, stop=k + ext, start_inclusive=si, stop_inclusive=ti))
                    reqs.append(dict(full, start=k, stop=k + ext, start_inclusive=si, stop_inclusive=ti))
        for si in (True, False):
            for ti in (True, False):
                reqs.append(dict(full, start=k, stop=k, start_inclusive=si, stop_inclusive=ti))  # start == stop
    reqs += [dict(full, start=last, stop=first),                                 # empty: start > stop
             dict(full, start=b"", stop=b"\x00"), dict(full, start=b"", stop=b"", stop_inclusive=False),  # before every key
             dict(full, start=last + b"\x00", stop=b"\xff" * 6), dict(full, start=b"\xff" * 5)]          # after every key
    reqs += filter_list(full)
    sizes = np.cumsum([len(k) + len(v) - 12 for k, v in vis])
    for i in range(1, len(vis) + 2):
        reqs.append(dict(full, max_iter_count=i))
        reqs.append(dict(full, max_count=i, max_iter_count=len(vis) + 5))
    for s in sizes[:: max(1, len(sizes) // 150)]:
        reqs.append(dict(full, max_iter_size=int(s)))
        reqs.append(dict(full, max_iter_size=int(s) + 1))
    return reqs


def stride(vis):
    """an arena slice that holds the whole visible set"""
    return (sum(len(k) + len(v) for k, v in vis) + 4096 + 15) & ~15


def check(vis, reqs, got, what):
    for i, (q, g) in enumerate(zip(reqs, got)):
        w = model_scan(vis, q, NOW)
        assert g == w, (what, i, {k: v for k, v in q.items() if k not in ("start", "stop")}, q["start"][:40], q["stop"][:40], diff(g, w))


CASES = [  # runs, block size, restart interval, GPU-compacted oldest runs, long keys
    (1, 4096, 16, 0, False),
    (4, 256, 1, 0, True),
    (4, 16384, 16, 0, False),
    (9, 1024, 4, 5, False),
    (17, 1024, 16, 0, False),
    (32, 256, 4, 0, False),
]


@pytest.mark.parametrize("n_runs,block_size,ri,compacted,long_keys", CASES)
def test_scans_against_the_model(pgs, engine, n_runs, block_size, ri, compacted, long_keys):
    recs, items = build_db(pgs, 1000 + n_runs, n_runs, long_keys, block_size)
    vis, _ = visible(items)
    part = load(pgs, engine, recs, block_size, ri, compacted)
    try:
        assert len(part.runs()) == n_runs - (compacted - 1 if compacted else 0)
        fwd = request_list(vis)
        rev = [mirror(q) for q in fwd]
        n_unique = len(fwd)
        while len(fwd) < 2000:  # enough requests that the persistent CTA loops wrap
            fwd, rev = fwd + fwd[:2000 - len(fwd)], rev + rev[:2000 - len(rev)]
        st, got_fwd = run_scans(pgs, part, fwd, stride(vis))          # forward only: k_scan_fwd
        assert st == 0, st
        check(vis, fwd, got_fwd, "forward batch")
        st, got_rev = run_scans(pgs, part, rev, stride(vis))          # reverse only: k_scan
        assert st == 0, st
        check(vis, rev, got_rev, "reverse batch")
        st, got_mix = run_scans(pgs, part, fwd + rev[:1], stride(vis))  # one reverse request sends the forward ones through k_scan
        assert st == 0, st
        assert got_mix[:-1] == got_fwd and got_mix[-1] == got_rev[0]
        for i in range(n_unique):                                    # one request per call
            assert run_one(pgs, part, fwd[i]) == got_fwd[i], ("single forward", i)
            assert run_one(pgs, part, rev[i]) == got_rev[i], ("single reverse", i)
    finally:
        part.close()


def test_output_limits(pgs, engine):
    """a request's output larger than its arena / kv slice -> PGS_ABORTED; a packed batch larger than arena_cap / kv_cap ->
    PGS_INCOMPLETE; a resume slot shorter than a key -> no resume keys.  For both kernels."""
    recs, items = build_db(pgs, 77, 4)
    vis, _ = visible(items)
    part = load(pgs, engine, recs, 1024, 16)
    try:
        hk = dict(start=raw_key(b"h0", b""), stop=next_key(raw_key(b"h0", b"")), start_inclusive=True, stop_inclusive=False,
                  key_mode=1, prefix=1, max_count=3000, max_iter_count=3000, max_iter_size=0)
        want = model_scan(vis, hk)
        out = sum(len(k) + len(v) for k, v, _ in want["kvs"])
        assert want["count"] > 4 and out > 64
        for reverse in (False, True):
            reqs = [dict(hk, reverse=reverse)] * 3
            assert run_scans(pgs, part, reqs, arena_stride=64)[0] == pgs.ABORTED
            assert run_scans(pgs, part, reqs, kv_stride=2)[0] == pgs.ABORTED
            assert run_scans(pgs, part, reqs, arena_cap=2 * out)[0] == pgs.INCOMPLETE
            assert run_scans(pgs, part, reqs, kv_cap=2 * want["count"])[0] == pgs.INCOMPLETE
            st, got = run_scans(pgs, part, reqs, arena_cap=3 * (out + 15), kv_cap=3 * want["count"])
            assert st == 0 and all(g["kvs"] == model_scan(vis, q)["kvs"] for g, q in zip(got, reqs))
            limited = [dict(hk, reverse=reverse, max_count=2)] * 3
            resume = np.zeros(3 * 4, np.uint8)
            st, got = run_scans(pgs, part, limited, resume_stride=4, resume=resume)
            assert st == 0 and all(g["iter_valid"] and not g["complete"] for g in got)
            assert not resume.any()
    finally:
        part.close()


def test_where_not_supported_is_allowed(pgs, engine):
    """the only refusals: more than 32 runs (DESIGN §8) and, for reverse scans, runs of which one block each does not fit the
    staging pool (§8: dense 16 KB blocks in 17 runs); the forward scans of that stack still answer"""
    recs, items = build_db(pgs, 5, 33)
    part = load(pgs, engine, recs, 4096, 16)
    try:
        q = dict(start=b"", stop=b"\xff" * 4, start_inclusive=True, stop_inclusive=True, key_mode=0, max_count=10, max_iter_count=10, max_iter_size=0)
        for rev in (False, True):
            assert run_scans(pgs, part, [dict(q, reverse=rev)] * 2)[0] == pgs.NOT_SUPPORTED
    finally:
        part.close()
    recs, items = build_db(pgs, 6, 17, big=16384)
    vis, _ = visible(items)
    part = load(pgs, engine, recs, 16384, 1)
    try:
        reqs = [dict(q, max_count=50, max_iter_count=50)] * 2
        st, got = run_scans(pgs, part, reqs)
        assert st == 0
        check(vis, reqs, got, "forward over dense 16 KB blocks")
        assert run_scans(pgs, part, [mirror(x) for x in reqs])[0] == pgs.NOT_SUPPORTED
    finally:
        part.close()
