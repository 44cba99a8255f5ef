"""CPU check of the READ kernels' logic (k_get, k_scan_fwd of incubator_pegasus_b200/csrc/read_kernels.cuh) inside the host SIMT
interpreter (tools/simt, see test_kernel_sim.py): random multi-version data over several runs, point lookups and forward
range scans with every flag of the request, compared with a plain Python model of RocksDB's visibility rules and of the
reference's iterator loop (src/server/pegasus_server_impl.cpp:617-756, 1266-1320).  Also: the Bloom filters built at upload and
by the compaction walker never reject a present key or hash-key prefix."""
import ctypes as C

import numpy as np
import pytest

from get_model import (check_results, compacted_run, flat_keys, key_slot, model_get, model_stats, query_keys, sweep_items, sweep_keys,
                       uploaded_run)
from incubator_pegasus_b200 import synth
from scan_model import answer, diff, filter_list, make_db, mirror, model_scan, next_key, raw_key, scan_list, scan_requests, visible
from test_kernel_sim import sim, sim_compact  # noqa: F401  (fixture + helper)

NOW = synth.NOW


def run_args(pgs, runs, block_size=4096, ri=16):
    brs = [pgs.build_run(r, block_size, ri) for r in runs]
    k = len(brs)
    return (k, (C.c_void_p * k)(*[b.data.ctypes.data for b in brs]), (C.c_uint64 * k)(*[b.data.shape[0] for b in brs]),
            (C.c_void_p * k)(*[b.blk_off.ctypes.data for b in brs]), (C.c_void_p * k)(*[b.blk_size.ctypes.data for b in brs]),
            (C.c_uint32 * k)(*[b.n_blocks for b in brs])), brs


@pytest.mark.parametrize("use_bloom", [1, 0])
def test_sim_get(pgs, sim, use_bloom):
    rng = np.random.default_rng(5)
    hks = [bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8)) for _ in range(12)] + [b""]
    runs, items = make_db(pgs, rng, 4, hks, 40, big=True)
    vis, best = visible(items)
    args, keep = run_args(pgs, runs, block_size=1024)
    present = list(best.keys())
    absent = [raw_key(h, b"s%04d" % s) for h in hks[:4] for s in (41, 77)] + [raw_key(b"zz", b""), b"", b"\x00", b"\x00\x05ab", b"\xff" * 300]
    keys = [present[i] for i in rng.permutation(len(present))[:300]] + absent
    flat = np.frombuffer(b"".join(keys), np.uint8).copy()
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    res = (pgs.GetResult * len(keys))()
    arena = np.zeros(1 << 20, np.uint8)
    stats = (C.c_uint64 * 3)()
    st = sim.sim_get(*args, flat.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), len(keys), NOW,
                     arena.ctypes.data_as(C.c_void_p), C.c_uint64(arena.shape[0]), res, stats, use_bloom)
    assert st == 0
    for i, k in enumerate(keys):
        r = res[i]
        if k not in best or best[k][1] == 0:
            assert r.status == pgs.NOT_FOUND and not r.expired, (i, k)
            continue
        v = best[k][2]
        ets = int.from_bytes(v[:4], "big")
        assert r.expire_ts == ets
        if 0 < ets <= NOW:
            assert r.status == pgs.NOT_FOUND and r.expired
        else:
            assert r.status == pgs.OK and arena[r.value_off:r.value_off + r.value_len].tobytes() == v[12:], (i, k)
    if use_bloom:
        assert stats[2] > 0                                     # some run probes were saved ...
    else:
        assert stats[2] == 0
    print("probes", stats[1], "skipped", stats[2])


def test_sim_get_multi_partition(pgs, sim):
    """pgs_get_batch_multi's kernel shape: one launch, every key looked up in the runs of its own partition slot only"""
    rng = np.random.default_rng(15)
    hks = [bytes(rng.integers(0, 256, int(rng.integers(1, 6)), dtype=np.uint8)) for _ in range(8)]
    runs, items = make_db(pgs, rng, 4, hks, 30)
    per_run = {}
    for key, seq, typ, val, run in [(k, s, t, v, r) for r, rr in enumerate(runs) for k, s, t, v in [(rr.key(i), int(rr.seq[i]), int(rr.type[i]), rr.value(i)) for i in range(rr.n)]]:
        per_run.setdefault(run, []).append((key, seq, typ, val))
    def best_of(run_ids):
        best = {}
        for r in run_ids:
            for k, s, t, v in per_run.get(r, []):
                if k not in best or s > best[k][0]:
                    best[k] = (s, t, v)
        return best
    slots = [best_of([0, 1]), best_of([2, 3]), {}]
    allkeys = sorted(set(k for b in slots for k in b))
    keys = [allkeys[i] for i in rng.permutation(len(allkeys))[:240]] + [b"", b"\x00\x09nothing"]
    flat = np.frombuffer(b"".join(keys), np.uint8).copy()
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    args, keep = run_args(pgs, runs, block_size=1024)
    res = (pgs.GetResult * len(keys))()
    arena = np.zeros(1 << 20, np.uint8)
    stats = (C.c_uint64 * 3)()
    assert sim.sim_get(*args, flat.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), len(keys), NOW,
                       arena.ctypes.data_as(C.c_void_p), C.c_uint64(arena.shape[0]), res, stats, 3) == 0
    hits = 0
    for i, k in enumerate(keys):
        best, r = slots[i % 3], res[i]
        if k not in best or best[k][1] == 0:
            assert r.status == pgs.NOT_FOUND and not r.expired, (i, k)
            continue
        v = best[k][2]
        ets = int.from_bytes(v[:4], "big")
        if 0 < ets <= NOW:
            assert r.status == pgs.NOT_FOUND and r.expired
        else:
            hits += 1
            assert r.status == pgs.OK and arena[r.value_off:r.value_off + r.value_len].tobytes() == v[12:], (i, k)
    assert hits > 30


def do_scans(pgs, sim, args, reqs, lanes=0, pool=0, rstride=512):
    n = len(reqs)
    keep = []
    arr = scan_requests(pgs, reqs, keep)
    astride, kstride = 1 << 16, 512
    arena = np.zeros(astride * n, np.uint8)
    kvs = (pgs.KV * (kstride * n))()
    resume = np.zeros(rstride * n, np.uint8)
    res = (pgs.ScanResult * n)()
    st = sim.sim_scan(*args, arr, n, NOW, C.c_uint64(astride), kstride, arena.ctypes.data_as(C.c_void_p), kvs,
                      resume.ctypes.data_as(C.c_void_p), rstride, res, lanes, pool)
    assert st == 0, st
    return [answer(res[i], arena[i * astride:(i + 1) * astride], kvs[i * kstride:i * kstride + res[i].n_kvs],
                   resume[i * rstride:(i + 1) * rstride]) for i in range(n)]


def check_scans(vis, reqs, got):
    for i, (q, g_) in enumerate(zip(reqs, got)):
        want = model_scan(vis, q, NOW)
        assert g_ == want, (i, q, diff(g_, want))


SCAN_HKS = [b"h%d" % i for i in range(7)] + [b"", b"h1x", bytes([0xff, 0xff])]


@pytest.mark.parametrize("n_runs,lanes,long_keys", [(4, 0, False), (1, 0, False), (6, 16, False), (3, 32, False), (2, 0, True)],
                         ids=["4-0", "1-0", "6-16", "3-32", "2-0-3k_keys"])
def test_sim_scan_forward(pgs, sim, n_runs, lanes, long_keys):
    """long_keys: a hash key of 3000 bytes, whose key rows do not fit k_scan_fwd's shared memory: the forward batch runs
    through k_scan, as in the library"""
    rng = np.random.default_rng(100 + n_runs)
    hks = SCAN_HKS[:3] + [b"L" * 3000] if long_keys else SCAN_HKS
    runs, items = make_db(pgs, rng, n_runs, hks, 12 if long_keys else 30)
    vis, best = visible(items)
    args, keep = run_args(pgs, runs, block_size=512, ri=4)
    full = dict(start=b"", stop=b"\xff" * 4, start_inclusive=True, stop_inclusive=True, key_mode=0, max_count=1000, max_iter_count=1000,
                max_iter_size=0)
    reqs = scan_list(hks) + filter_list(full)
    check_scans(vis, reqs, do_scans(pgs, sim, args, reqs, lanes, rstride=4096 if long_keys else 512))


@pytest.mark.parametrize("pool", ["product", "minimal"])
@pytest.mark.parametrize("n_runs", [1, 4, 9])
def test_sim_scan_reverse_and_mixed(pgs, sim, n_runs, pool):
    """k_scan: the forward list mirrored (all reverse), then forward and reverse requests interleaved in one batch, which
    sends the forward ones through k_scan too.  The minimal pool holds one block of every run, so chunks end after about
    one block and the far bound, the cursors and the look-ahead state cross a chunk boundary every few records."""
    rng = np.random.default_rng(200 + n_runs)
    hks = SCAN_HKS[:3] + SCAN_HKS[-3:] + [b"hlong0123"]  # its keys are 16 bytes long: the kernel's key slot
    runs, items = make_db(pgs, rng, n_runs, hks, 24, big=True)
    vis, best = visible(items)
    args, keep = run_args(pgs, runs, block_size=512, ri=4)
    fwd = scan_list(hks)
    full = dict(start=b"", stop=b"\xff" * 4, start_inclusive=True, stop_inclusive=True, key_mode=0, max_count=1000, max_iter_count=1000,
                max_iter_size=0)
    for k in [k for k, _ in vis if len(k) == 16][::5]:  # bounds one byte longer than the slot, equal to a stored key in it
        for si in (True, False):
            for ti in (True, False):
                fwd += [dict(full, start=k + b"\x00", start_inclusive=si, stop_inclusive=ti),
                        dict(full, stop=k + b"\x00", start_inclusive=si, stop_inclusive=ti)]
    fwd += filter_list(full)
    rev = [mirror(q) for q in fwd]
    p = 0 if pool == "product" else 1
    check_scans(vis, rev, do_scans(pgs, sim, args, rev, pool=p))
    mixed = [q for pair in zip(fwd[0::2], rev[1::2]) for q in pair]
    check_scans(vis, mixed, do_scans(pgs, sim, args, mixed, pool=p))


@pytest.mark.parametrize("n_runs,lanes", [(4, 0), (5, 16)])
def test_sim_scan_multi_partition(pgs, sim, n_runs, lanes):
    """pgs_range_scan_many_multi's kernel shape: one launch, every request merges the runs of its own partition slot only"""
    rng = np.random.default_rng(300 + n_runs)
    hks = [b"h%d" % i for i in range(5)] + [b"", bytes([0xff, 0xff])]
    runs, items = make_db(pgs, rng, n_runs, hks, 30, big=True)  # values of 600..1500 bytes among them: several copy rounds
    assert len(runs) == n_runs
    half = n_runs // 2
    vis_of = [visible(items[:half])[0], visible(items[half:])[0], []]
    args, keep = run_args(pgs, runs, block_size=512, ri=4)
    reqs = []
    for hk in hks + [b"nope"]:
        base = dict(start=raw_key(hk, b""), stop=next_key(raw_key(hk, b"")), start_inclusive=True, stop_inclusive=False, key_mode=1, prefix=1,
                    max_count=3000, max_iter_count=3000, max_iter_size=0)
        for q in (base, dict(base, max_count=7), dict(base, start=raw_key(hk, b"s0010"), stop=raw_key(hk, b"s0020"), stop_inclusive=True),
                  dict(base, sft=1, spat=b"01", count_only=1),
                  dict(base, key_mode=0, prefix=0, stop=raw_key(hk, b"\xff" * 8), return_expire_ts=1, max_count=11)):
            reqs += [q, q, q]   # the same request against each of the three slots
    got = do_scans(pgs, sim, args, reqs, lanes | 0x100)
    nonempty = 0
    for i, (q, g_) in enumerate(zip(reqs, got)):
        want = model_scan(vis_of[i % 3], q, NOW)
        nonempty += want["count"] > 0
        assert g_ == want, (i, i % 3, q, diff(g_, want))
    assert nonempty > 20


def test_sim_bloom_no_false_negatives(pgs, sim):
    rng = np.random.default_rng(9)
    runs = synth.compaction_runs(k=3, n_per_run=400, seed=9)
    out, x = sim_compact(pgs, sim, runs, bottommost=True, seg_weight=32 * 1024)
    got = pgs.decode_blocks(out)
    miss = 0
    for i in range(got.n):
        k = got.key(i)
        assert sim.sim_result_bloom_check(k, len(k)) == 1
        pl = 2 + int.from_bytes(k[:2], "big")
        assert sim.sim_result_bloom_check(k[:pl], pl) == 1
    for _ in range(2000):
        k = bytes(rng.integers(0, 256, 50, dtype=np.uint8))
        miss += sim.sim_result_bloom_check(k, len(k))
    assert miss < 200  # ~1 % expected at 10 bits per entry


# ---- k_get against tests/get_model.py: every result field and the exact probe / skip counts ---------------------------------
def sim_lookup(pgs, sim, args, keys, use_bloom=1):
    flat, off = flat_keys(keys)
    res = (pgs.GetResult * len(keys))()
    arena = np.zeros(1 << 22, np.uint8)
    stats = (C.c_uint64 * 3)()
    st = sim.sim_get(*args, flat.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), len(keys), NOW,
                     arena.ctypes.data_as(C.c_void_p), C.c_uint64(arena.shape[0]), res, stats, use_bloom)
    assert st == 0, st
    return res, arena, list(stats)


def sim_filter(sim, br):
    """the filter words the upload's k_index_walk builds for one run, in the simulator"""
    out = np.zeros(1 << 20, np.uint32)
    lines = sim.sim_run_bloom(br.data.ctypes.data_as(C.c_void_p), C.c_uint64(br.data.shape[0]), br.blk_off.ctypes.data_as(C.c_void_p),
                              br.blk_size.ctypes.data_as(C.c_void_p), br.n_blocks, out.ctypes.data_as(C.c_void_p), C.c_uint64(out.shape[0]))
    return out[:16 * lines]


def check_lookup(pgs, sim, args, runs, keys, use_bloom=1):
    res, arena, stats = sim_lookup(pgs, sim, args, keys, use_bloom)
    want = [model_get(runs, k, NOW) for k in keys]
    n_ok = check_results(res, arena, keys, want)
    assert stats[0] == sum((len(w["value"]) + 3) & ~3 for w in want if w["status"] == pgs.OK)
    assert stats[1:] == list(model_stats(runs, keys)), (stats, model_stats(runs, keys))
    return n_ok


def sample(rng, keys, n):
    return [keys[i] for i in sorted(rng.permutation(len(keys))[:n])] if len(keys) > n else keys


@pytest.mark.parametrize("n_runs,block_size,ri", [(1, 4096, 16), (4, 256, 1), (9, 512, 4)])
def test_sim_get_against_model(pgs, sim, n_runs, block_size, ri):
    """user keys of 0..300 bytes, hash keys of 0..140 bytes, 4 KB keys, values shorter than the header, expire_ts == now, and
    (256 B blocks) a hot key whose 300 versions span many blocks.  The filters the simulated upload builds equal the model's
    bit for bit, and the probe / skip counters equal model_stats."""
    rng = np.random.default_rng(40 + n_runs)
    items = sweep_items(rng, n_runs, sweep_keys(rng, long_keys=n_runs < 9), NOW, hot=300 if block_size == 256 else 0)
    args, brs = run_args(pgs, [pgs.Records.from_list(it) for it in items], block_size, ri)
    runs = [uploaded_run(b) for b in brs]
    for b, r in zip(brs, runs):
        assert np.array_equal(sim_filter(sim, b), r.bloom.words())
    keys = sample(rng, query_keys(runs), 1500)
    assert check_lookup(pgs, sim, args, runs, keys) > 100
    if n_runs > 1:  # without filters: no run is skipped, the answers stay the same
        res, arena, stats = sim_lookup(pgs, sim, args, keys[:300], use_bloom=0)
        check_results(res, arena, keys[:300], [model_get(runs, k, NOW) for k in keys[:300]])
        assert stats[2] == 0


def test_sim_get_multi_partition_against_model(pgs, sim):
    """pgs_get_batch_multi's kernel shape: slot 0 = the newest 3 runs, slot 1 = the other 3, slot 2 = an empty partition;
    one key slot for the whole launch, the counters summed over the slots"""
    rng = np.random.default_rng(77)
    items = sweep_items(rng, 6, sweep_keys(rng), NOW, hot=200)
    args, brs = run_args(pgs, [pgs.Records.from_list(it) for it in items], 256, 1)
    runs = [uploaded_run(b) for b in brs]
    slots = [runs[:3], runs[3:], []]
    ks = key_slot([runs])
    keys = sample(rng, query_keys(runs), 1200)
    res, arena, stats = sim_lookup(pgs, sim, args, keys, use_bloom=3)
    want = [model_get(slots[i % 3], k, NOW, ks=ks) for i, k in enumerate(keys)]
    assert check_results(res, arena, keys, want) > 100
    per_slot = [model_stats(slots[s], keys[s::3], ks) for s in range(3)]
    assert stats[1:] == [sum(p[0] for p in per_slot), sum(p[1] for p in per_slot)]


def test_sim_get_on_a_compacted_run(pgs, sim):
    """the oldest three of five runs merged by the simulated compaction: its filter (k_emit's builder, sized as compact.cu
    sizes it) equals the model's bit for bit, and lookups through it and the two newer uploaded runs match the model"""
    rng = np.random.default_rng(91)
    items = sweep_items(rng, 5, sweep_keys(rng, long_keys=False), NOW, hot=250)
    recs = [pgs.Records.from_list(it) for it in items]
    out, _ = sim_compact(pgs, sim, recs[2:], bottommost=False, enabled=False, block_size=512, restart_interval=4, seg_weight=16 * 1024)
    merged = compacted_run(out, [uploaded_run(pgs.build_run(r, 512, 4)) for r in recs[2:]])
    words = np.zeros(16 * merged.bloom.n_lines, np.uint32)
    assert sim.sim_result_bloom(words.ctypes.data_as(C.c_void_p), C.c_uint64(words.shape[0])) == merged.bloom.n_lines
    assert np.array_equal(words, merged.bloom.words())
    args, brs = run_args(pgs, recs[:2], 512, 4)
    runs = [uploaded_run(b) for b in brs] + [merged]
    keys = sample(rng, query_keys(runs), 1500)
    assert check_lookup(pgs, sim, args, runs, keys, use_bloom=5) > 100
