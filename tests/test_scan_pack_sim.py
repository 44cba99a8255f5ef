"""CPU check of the packed read-back of batched range scans (k_pack_offsets, k_pack_copy of
incubator_pegasus_b200/csrc/read_kernels.cuh) inside the host SIMT interpreter (tools/simt, see test_kernel_sim.py), against the
packing model of tests/scan_model.py:
  (i)  k_pack_offsets alone over made-up results: batch sizes around the warp and the 1024-thread CTA, outputs of 0 to 4 GiB - 16
       bytes, and packed totals below 4 GiB, exactly at it, across it inside the first 1024 requests, across it only between
       two groups of 1024, and past 8 GiB;
  (ii) whole batches read back as pgs_range_scan_many reads them: forward, reverse, mixed and multi-partition request lists at
       those batch sizes, with outputs at every length mod 16, and the statuses at the caps and strides.
The same check runs in the AddressSanitizer build:
    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_scan_pack_sim.py
    bash tools/simt/build.sh"""
import ctypes as C

import numpy as np
import pytest

from incubator_pegasus_b200 import synth
from scan_model import (SLICE_MAX, answer, check_packed, filter_list, make_db, mirror, model_batch, model_scan, next_key, pack_offsets,
                        raw_key, round16, scan_list, scan_requests, visible)
from test_kernel_sim import sim  # noqa: F401  (fixture)
from test_read_kernels_sim import run_args

NOW = synth.NOW
BATCHES = [1, 2, 31, 32, 33, 1023, 1024, 1025, 2049, 70000]


# ---- (i) k_pack_offsets against the model -------------------------------------------------------------------------------------
def made_up(rng, n, total):
    """arena_used / n_kvs of n requests: outputs of 0, 1, 15, 16, 17 and random bytes, some 5 MiB, a fifth with no kvs, then
    `total` places outputs of 4 GiB - 16 (or what is left below 4 GiB) so that the packed total lands where it names"""
    used = np.where(rng.random(n) < 0.5, rng.choice([0, 1, 15, 16, 17], n), rng.integers(0, 20000, n)).astype(np.uint64)
    used[rng.permutation(n)[:min(n // 4, 50)]] = 5 << 20
    kvs = rng.integers(1, 500, n).astype(np.uint64)
    none = rng.random(n) < 0.2
    used[none], kvs[none] = 0, 0
    first = min(n, 1024)
    pick = rng.permutation(first)
    rest = lambda skip: sum(round16(int(u)) for i, u in enumerate(used) if i not in skip)  # noqa: E731
    if total == "at":        # exactly 2^32
        used[pick[0]] = 2**32 - rest({pick[0]}) - int(rng.integers(0, 16))
    elif total == "first":   # across 2^32 inside the first 1024 requests
        used[pick[:2]] = SLICE_MAX
    elif total == "between":  # every 1024 requests below 2^32, the whole batch across it
        group = sum(round16(int(u)) for u in used[1:1024])
        used[0] = 2**32 - 32 - group
        used[1024 + int(rng.integers(0, n - 1024))] = 5 << 20
    elif total == "past":    # past 2^33
        used[rng.permutation(n)[:3]] = SLICE_MAX
    elif total == "single":
        used[0] = SLICE_MAX
    return used, kvs


def pack_cases():
    for n in BATCHES:
        yield n, "below"
        if n == 1:
            yield n, "single"
        if n >= 2:
            yield n, "at"
            yield n, "first"
        if n >= 3:
            yield n, "past"
        if n > 1024:
            yield n, "between"


@pytest.mark.parametrize("n,total", list(pack_cases()))
def test_pack_offsets(pgs, sim, n, total):
    rng = np.random.default_rng(n * 7 + len(total))
    used, n_kvs = made_up(rng, n, total)
    ab_want, kb_want = pack_offsets([int(u) for u in used], [int(k) for k in n_kvs])
    where = {"below": lambda: ab_want[-1] < 2**32, "at": lambda: ab_want[-1] == 2**32, "past": lambda: ab_want[-1] > 2**33,
             "single": lambda: True, "first": lambda: ab_want[min(n, 1024)] > 2**32,
             "between": lambda: ab_want[1024] < 2**32 < ab_want[-1] and ab_want[-1] - ab_want[1024] < 2**32}
    assert where[total](), (total, ab_want[-1])
    res = (pgs.ScanResult * n)()
    for i in range(n):
        res[i].arena_used, res[i].n_kvs = int(used[i]), int(n_kvs[i])
    ab, kb = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint32)
    sim.sim_pack_offsets(res, n, ab.ctypes.data_as(C.c_void_p), kb.ctypes.data_as(C.c_void_p))
    bad = np.nonzero(ab != np.array(ab_want, np.uint64))[0]
    assert bad.size == 0, ("arena_base", total, int(bad[0]), int(ab[bad[0]]), ab_want[bad[0]])
    assert np.array_equal(kb, np.array(kb_want, np.uint32))


# ---- (ii) whole batches through sim_scan_packed -------------------------------------------------------------------------------
def sim_batch(pgs, sim, args, reqs, arena_stride, kv_stride, arena_cap, kv_cap, lanes=0, rstride=512):
    """one batch read back as scan_many does -> (status name, results, packed arena, packed kvs, arena_base, kv_base, resume)"""
    n = len(reqs)
    keep = []
    arr = scan_requests(pgs, reqs, keep)
    arena = np.zeros(max(1, arena_cap), np.uint8)
    kvs = (pgs.KV * max(1, kv_cap))()
    resume = np.zeros(rstride * n, np.uint8)
    res = (pgs.ScanResult * n)()
    ab, kb = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint32)
    vp = C.c_void_p
    st = sim.sim_scan_packed(*args, arr, n, NOW, C.c_uint64(arena_stride), kv_stride, arena.ctypes.data_as(vp), C.c_uint64(arena_cap), kvs,
                             C.c_uint64(kv_cap), resume.ctypes.data_as(vp), rstride, res, ab.ctypes.data_as(vp), kb.ctypes.data_as(vp), lanes)
    name = {pgs.OK: "OK", pgs.INCOMPLETE: "INCOMPLETE", pgs.ABORTED: "ABORTED"}.get(st, st)
    return name, res, arena, kvs, ab, kb, resume


def check_batch(pgs, sim, args, reqs, models, lanes=0, caps=False, arena_stride=1 << 16, kv_stride=512, rstride=512):
    """the batch at exactly its packed need (PGS_OK, every answer and byte as the model); caps: also at one byte / one kv less"""
    n = len(reqs)
    _, ab_want, kb_want = model_batch(models, arena_stride, kv_stride, 2**64, 2**64)
    st, res, arena, kvs, ab, kb, resume = sim_batch(pgs, sim, args, reqs, arena_stride, kv_stride, ab_want[-1], kb_want[-1], lanes, rstride)
    assert st == "OK", st
    check_packed(res, arena, kvs, ab, kb, models, ab_want, kb_want)
    for i, (q, m) in enumerate(zip(reqs, models)):
        got = answer(res[i], arena[int(ab[i]):], kvs[int(kb[i]):int(kb[i + 1])], resume[i * rstride:(i + 1) * rstride])
        assert got == m, (i, q)
    if caps and ab_want[-1]:
        assert sim_batch(pgs, sim, args, reqs, arena_stride, kv_stride, ab_want[-1] - 1, kb_want[-1], lanes, rstride)[0] == "INCOMPLETE"
    if caps and kb_want[-1]:
        assert sim_batch(pgs, sim, args, reqs, arena_stride, kv_stride, ab_want[-1], kb_want[-1] - 1, lanes, rstride)[0] == "INCOMPLETE"
    return [len(b"".join(k + v for k, v, _ in m["kvs"])) % 16 for m in models]


def sweep(pgs, sim, args, reqs, models, sizes, lanes=0):
    """the list packed at each batch size (requests taken in turn, from where the last batch ended; the caps probed up to 2
    requests) and whole; every output length mod 16 occurs"""
    residues, at = set(), 0
    for n in sizes + [len(reqs)]:
        pick = [(at + j) % len(reqs) for j in range(n)]
        at += n
        residues |= set(check_batch(pgs, sim, args, [reqs[j] for j in pick], [models[j] for j in pick], lanes, n <= 2))
    assert residues == set(range(16)), residues


def db(pgs, seed, n_runs):
    rng = np.random.default_rng(seed)
    hks = [b"h%d" % i for i in range(4)] + [b"", bytes([0xff, 0xff])]
    runs, items = make_db(pgs, rng, n_runs, hks, 16, big=True)
    return hks, runs, items


def lengths(full, n):
    """a whole-range scan cut after 1 .. n records: outputs of every length mod 16"""
    return [dict(full, max_count=c) for c in range(1, n + 1)]


FULL = dict(start=b"", stop=b"\xff" * 4, start_inclusive=True, stop_inclusive=True, key_mode=0, max_count=1000, max_iter_count=1000,
            max_iter_size=0)


@pytest.mark.parametrize("direction", ["forward", "reverse", "mixed"])
def test_packed_batches(pgs, sim, direction):
    hks, runs, items = db(pgs, 11, 3)
    vis, _ = visible(items)
    args, keep = run_args(pgs, runs, block_size=512, ri=4)
    fwd = lengths(FULL, 40) + scan_list(hks) + filter_list(FULL)
    rev = [mirror(q) for q in fwd]
    reqs = {"forward": fwd, "reverse": rev, "mixed": [q for pair in zip(fwd[0::2], rev[1::2]) for q in pair]}[direction]
    sweep(pgs, sim, args, reqs, [model_scan(vis, q, NOW) for q in reqs], [1, 2, 31, 32, 33])


def test_packed_batches_of_the_device_tests(pgs, sim):
    """the request list of test_scan_kernels_gpu.py over its database shape (a hot key with hundreds of versions, values larger
    than a block), packed whole and at 2 and 33 requests"""
    from test_scan_kernels_gpu import build_db, request_list
    recs, items = build_db(pgs, 1003, 3, big=512)
    vis, _ = visible(items)
    args, keep = run_args(pgs, recs[::-1], block_size=512, ri=4)
    reqs = request_list(vis)
    sweep(pgs, sim, args, reqs, [model_scan(vis, q, NOW) for q in reqs], [2, 33])


def test_packed_multi_partition(pgs, sim):
    """pgs_range_scan_many_multi's shape: request i merges the runs of slot i % 3 (the third slot is empty)"""
    hks, runs, items = db(pgs, 12, 4)
    vis_of = [visible(items[:2])[0], visible(items[2:])[0], []]
    args, keep = run_args(pgs, runs, block_size=512, ri=4)
    reqs = []
    for q in lengths(FULL, 16) + scan_list(hks[:3]):
        reqs += [q, q, q]
    models = [model_scan(vis_of[i % 3], q, NOW) for i, q in enumerate(reqs)]
    residues = set(check_batch(pgs, sim, args, reqs, models, lanes=0x100))
    assert residues == set(range(16)), residues
    for n in (2, 31, 33):
        check_batch(pgs, sim, args, reqs[:n], models[:n], lanes=0x100, caps=n == 2)


@pytest.mark.parametrize("reverse", [False, True])
def test_packed_statuses(pgs, sim, reverse):
    """an output past its slice (the stride rounded up to 16) or kv_stride -> PGS_ABORTED; inside both -> PGS_OK; for both
    kernels"""
    hks, runs, items = db(pgs, 13, 2)
    vis, _ = visible(items)
    args, keep = run_args(pgs, runs, block_size=512, ri=4)
    hk = dict(start=raw_key(b"h1", b""), stop=next_key(raw_key(b"h1", b"")), start_inclusive=True, stop_inclusive=False, key_mode=1,
              prefix=1, max_count=3000, max_iter_count=3000, max_iter_size=0, reverse=reverse)
    reqs = [hk, dict(hk, max_count=3), hk]
    models = [model_scan(vis, q, NOW) for q in reqs]
    out = max(sum(len(k) + len(v) for k, v, _ in m["kvs"]) for m in models)
    n_kv = max(len(m["kvs"]) for m in models)
    assert n_kv > 4 and out % 16
    big = 1 << 20
    cases = {(out, n_kv): "OK", (round16(out) - 15, n_kv): "OK", (round16(out) - 16, n_kv): "ABORTED", (out, n_kv - 1): "ABORTED"}
    for (stride, kv_stride), want in cases.items():
        assert model_batch(models, stride, kv_stride, big, big)[0] == want
        assert sim_batch(pgs, sim, args, reqs, stride, kv_stride, big, big)[0] == want, (stride, kv_stride)
