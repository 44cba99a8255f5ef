"""Device tests of the packed read-back of batched range scans (k_pack_offsets, k_pack_copy of read_kernels.cuh) through
pgs_range_scan, pgs_range_scan_many and pgs_range_scan_many_multi, against the packing model of tests/scan_model.py: batch sizes
around the warp and the 1024-thread CTA up to 70 000 requests, outputs at every length mod 16, arena_cap and kv_cap at exactly
the packed need and one below, a packed batch past 4 GiB, and one request whose output passes the 4 GiB - 16 slice."""
import ctypes as C

import numpy as np
import pytest

from incubator_pegasus_b200 import synth
from scan_model import SLICE_MAX, check_packed, mirror, model_batch, model_scan, next_key, raw_key, round16, scan_requests, value, visible
from test_scan_kernels_gpu import build_db, load, request_list

pytestmark = pytest.mark.gpu
NOW = synth.NOW
BATCHES = [1, 2, 31, 32, 33, 1023, 1024, 1025, 2049, 70000]
vp = C.c_void_p


def scan_batch(pgs, parts, reqs, req_part, arena_stride, kv_stride, arena_cap, kv_cap):
    """one pgs_range_scan_many (req_part None) or _multi call -> (status, results, packed arena, packed kvs, arena_base, kv_base)"""
    n = len(reqs)
    keep = []
    arr = scan_requests(pgs, reqs, keep)
    arena = np.empty(max(1, arena_cap), np.uint8)
    kvs = (pgs.KV * max(1, kv_cap))()
    res = (pgs.ScanResult * n)()
    ab, kb = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint32)
    tail = (arena_stride, kv_stride, arena.ctypes.data_as(vp), arena_cap, kvs, kv_cap, None, 0, res,
            ab.ctypes.data_as(vp), kb.ctypes.data_as(vp))
    if req_part is None:
        st = pgs.lib().pgs_range_scan_many(parts[0].h, arr, n, NOW, *tail)
    else:
        handles = (vp * len(parts))(*[p.h for p in parts])
        slots = np.ascontiguousarray(req_part, np.uint32)
        st = pgs.lib().pgs_range_scan_many_multi(handles, len(parts), arr, slots.ctypes.data_as(vp), n, NOW, *tail)
    return st, res, arena, kvs, ab, kb


def check_sweep(pgs, parts, reqs, models, slot_of=None):
    """every batch size: PGS_OK at exactly the packed need with every base, kv and output byte as the model; PGS_INCOMPLETE at
    one byte and at one kv below it.  The slice is the largest output, kv_stride the most kvs."""
    used = [sum(len(k) + len(v) for k, v, _ in m["kvs"]) for m in models]
    stride, kv_stride = max(used), max(len(m["kvs"]) for m in models)
    assert set(u % 16 for u in used) == set(range(16))
    at = 0
    for n in BATCHES:
        pick = [(at + j) % len(reqs) for j in range(n)]
        at += n
        q, m = [reqs[j] for j in pick], [models[j] for j in pick]
        req_part = None if slot_of is None else [slot_of[j] for j in pick]
        st, ab_want, kb_want = model_batch(m, stride, kv_stride, 2**64, 2**64)
        assert st == "OK"
        need_a, need_k = ab_want[-1], kb_want[-1]
        st, res, arena, kvs, ab, kb = scan_batch(pgs, parts, q, req_part, stride, kv_stride, need_a, need_k)
        assert st == pgs.OK, (n, st)
        check_packed(res, arena, kvs, ab, kb, m, ab_want, kb_want)
        if need_a:
            assert scan_batch(pgs, parts, q, req_part, stride, kv_stride, need_a - 1, need_k)[0] == pgs.INCOMPLETE, n
        if need_k:
            assert scan_batch(pgs, parts, q, req_part, stride, kv_stride, need_a, need_k - 1)[0] == pgs.INCOMPLETE, n


def lengths(full, n):
    return [dict(full, max_count=c) for c in range(1, n + 1)]


FULL = dict(start=b"", stop=b"\xff" * 6, start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0, max_count=100000,
            max_iter_count=100000, max_iter_size=0)


def test_sweep_many(pgs, engine):
    """pgs_range_scan_many: forward batches (k_scan_fwd), then forward and reverse requests interleaved (k_scan)"""
    recs, items = build_db(pgs, 2001, 4, False, 1024)
    vis, _ = visible(items)
    part = load(pgs, engine, recs, 1024, 16)
    try:
        fwd = lengths(FULL, 60) + request_list(vis)
        mixed = [q for pair in zip(fwd[0::2], [mirror(q) for q in fwd[1::2]]) for q in pair]
        for reqs in (fwd, mixed):
            check_sweep(pgs, [part], reqs, [model_scan(vis, q, NOW) for q in reqs])
    finally:
        part.close()


def test_sweep_many_multi(pgs, engine):
    """pgs_range_scan_many_multi: request i merges the runs of slot i % 3; slot 2 is an empty partition"""
    recs_a, items_a = build_db(pgs, 2002, 3, False, 1024)
    recs_b, items_b = build_db(pgs, 2003, 5, False, 512)
    parts = [load(pgs, engine, recs_a, 1024, 16), load(pgs, engine, recs_b, 512, 4), engine.partition()]
    try:
        vis_of = [visible(items_a)[0], visible(items_b)[0], []]
        base = lengths(FULL, 60) + request_list(vis_of[0])
        reqs = [q for q in base for _ in range(3)]
        slot_of = [i % 3 for i in range(len(reqs))]
        check_sweep(pgs, parts, reqs, [model_scan(vis_of[s], q, NOW) for s, q in zip(slot_of, reqs)], slot_of)
    finally:
        for p in parts:
            p.close()


def test_single_request(pgs, engine):
    """pgs_range_scan: one request read back unpadded; arena_cap is also the slice, so one byte below the output is
    PGS_INCOMPLETE or, when the rounded slice no longer holds it, PGS_ABORTED -- both as the model says"""
    recs, items = build_db(pgs, 2004, 3, False, 1024)
    vis, _ = visible(items)
    part = load(pgs, engine, recs, 1024, 16)
    try:
        names = {pgs.OK: "OK", pgs.INCOMPLETE: "INCOMPLETE", pgs.ABORTED: "ABORTED"}
        seen = set()
        for q in lengths(FULL, 40) + [mirror(q) for q in lengths(FULL, 20)]:
            m = model_scan(vis, q, NOW)
            out = b"".join(k + v for k, v, _ in m["kvs"])
            for cap in (len(out), len(out) - 1, len(out) + 1):
                for kv_cap in (len(m["kvs"]), len(m["kvs"]) - 1):
                    keep = []
                    arena = np.zeros(max(1, cap), np.uint8)
                    kvs = (pgs.KV * max(1, kv_cap))()
                    r = pgs.ScanResult()
                    st = pgs.lib().pgs_range_scan(part.h, scan_requests(pgs, [q], keep), NOW, arena.ctypes.data_as(vp), cap, kvs, kv_cap,
                                                  None, 0, C.byref(r))
                    want, ab, kb = model_batch([m], cap, kv_cap, cap, kv_cap)
                    assert names.get(st, st) == want, (cap, kv_cap, len(out))
                    seen.add(want)
                    if want == "OK":
                        check_packed([r], arena, kvs, [0, len(out)], [0, len(m["kvs"])], [m], ab, kb)
        assert seen == {"OK", "INCOMPLETE", "ABORTED"}
    finally:
        part.close()


# ---- past 4 GiB ---------------------------------------------------------------------------------------------------------------
VAL = 100 << 10  # 100 KiB of user data per record: a record per block, and k_scan's staging pool still holds a block of each


def big_hash_key(pgs, n, seed):
    """n records under hash key b"big" (sort keys s000000 ..), each value VAL bytes from a 1 MiB random pool at its own offset.
    -> (Records, sort keys (n, 7) uint8, user data (n, VAL) uint8)"""
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 256, 1 << 20, dtype=np.uint8)
    sk = np.frombuffer(b"".join(b"s%06d" % i for i in range(n)), np.uint8).reshape(n, 7)
    hk = raw_key(b"big", b"")
    keys = np.concatenate([np.tile(np.frombuffer(hk, np.uint8), (n, 1)), sk], axis=1)
    vals = np.empty((n, 12 + VAL), np.uint8)
    vals[:, :12] = np.frombuffer(value(0, b""), np.uint8)
    starts = rng.integers(0, pool.shape[0] - VAL, n)
    for i in range(n):
        vals[i, 12:] = pool[starts[i]:starts[i] + VAL]
    kw, vw = keys.shape[1], vals.shape[1]
    recs = pgs.Records(keys.reshape(-1), np.arange(n + 1, dtype=np.uint64) * kw, vals.reshape(-1), np.arange(n + 1, dtype=np.uint64) * vw,
                       np.arange(1, n + 1, dtype=np.uint64), np.ones(n, np.uint8))
    return recs, sk, vals[:, 12:]


def prefix_request(**kw):
    return dict(dict(start=raw_key(b"big", b""), stop=next_key(raw_key(b"big", b"")), start_inclusive=True, stop_inclusive=False,
                     key_mode=1, prefix=1, max_count=2**32 - 1, max_iter_count=2**32 - 1, max_iter_size=0), **kw)


def test_packed_batch_beyond_4_gib(pgs, engine):  # 9 GB of device memory, 5 GB of host memory
    """arena_base is 64-bit: 160 prefix scans of one hash key holding 28 MiB pack to 4.7 GB, across 2^32 inside the first 1024
    requests.  Every base is i times the rounded output, and every request's kvs and bytes are its own.  Needs about 9 GB of
    device memory and 5 GB of host memory."""
    n_rec, n = 287, 160
    recs, sk, data = big_hash_key(pgs, n_rec, 3)
    part = engine.partition()
    try:
        part.build_records(recs)
        rec = 7 + VAL
        out = n_rec * rec
        assert out % 16 and n * round16(out) > 2**32 and 1024 * round16(out) > 2**32
        st, res, arena, kvs, ab, kb = scan_batch(pgs, [part], [prefix_request()] * n, None, out, n_rec, n * round16(out), n * n_rec)
        assert st == pgs.OK, st
        assert np.array_equal(ab, np.arange(n + 1, dtype=np.uint64) * round16(out))
        assert np.array_equal(kb, np.arange(n + 1, dtype=np.uint32) * n_rec)
        kvs = np.frombuffer(kvs, np.uint32).reshape(-1, 5)
        want_kv = np.zeros((n_rec, 5), np.uint32)
        want_kv[:, 0] = np.arange(n_rec) * rec
        want_kv[:, 1], want_kv[:, 3] = 7, VAL
        want_kv[:, 2] = want_kv[:, 0] + 7
        want = np.concatenate([sk, data], axis=1).reshape(-1)
        for i in range(n):
            assert res[i].arena_used == out and res[i].n_kvs == n_rec, i
            assert np.array_equal(kvs[i * n_rec:(i + 1) * n_rec], want_kv), i
            assert np.array_equal(arena[int(ab[i]):int(ab[i]) + out], want), i
    finally:
        part.close()


def test_request_beyond_4_gib(pgs, engine):  # 14 GB of device memory at peak, 10 GB of host memory
    """pgs_kv's offsets are 32-bit: one request's slice holds at most 4 GiB - 16 bytes, whatever the stride.  43 000 records
    of 100 KiB under one hash key: the whole prefix is PGS_ABORTED with a 5 GiB stride, forward and reverse; cut by max_count
    just below 4 GiB - 16, it is PGS_OK with the last kv's offsets near 2^32 and every byte its own.  Needs about 14 GB of device
    memory while the run is built and 10 GB of host memory."""
    n_rec = 43000
    rec = 7 + VAL
    assert n_rec * rec > 2**32
    recs, sk, data = big_hash_key(pgs, n_rec, 4)
    part = engine.partition()
    try:
        part.build_records(recs)
        del recs
        cap = 5 << 30
        arena = np.empty(cap, np.uint8)
        kvs = np.empty((n_rec, 5), np.uint32)
        m = SLICE_MAX // rec
        assert m < n_rec and SLICE_MAX - m * rec < rec

        def one(q):
            keep = []
            r = pgs.ScanResult()
            st = pgs.lib().pgs_range_scan(part.h, scan_requests(pgs, [q], keep), NOW, arena.ctypes.data_as(vp), cap,
                                          kvs.ctypes.data_as(vp), n_rec, None, 0, C.byref(r))
            return st, r
        for reverse in (False, True):
            assert one(prefix_request(reverse=reverse))[0] == pgs.ABORTED, reverse
            st, r = one(prefix_request(reverse=reverse, max_count=m))
            assert st == pgs.OK and r.n_kvs == m and r.arena_used == m * rec, (reverse, st)
            rows = np.arange(m) if not reverse else np.arange(n_rec - 1, n_rec - 1 - m, -1)
            last = kvs[m - 1]
            assert int(last[0]) == (m - 1) * rec and int(last[2]) == (m - 1) * rec + 7 and int(last[2]) > 2**32 - 2 * rec
            assert np.array_equal(kvs[:m, 0], np.arange(m, dtype=np.uint64) * rec)
            got = arena[:m * rec].reshape(m, rec)
            assert np.array_equal(got[-1, 7:], data[rows[-1]])
            assert np.array_equal(got[:, :7], sk[rows])
            for lo in range(0, m, 4096):  # every record's bytes, a slab at a time
                assert np.array_equal(got[lo:lo + 4096, 7:], data[rows[lo:lo + 4096]]), (reverse, lo)
    finally:
        part.close()
