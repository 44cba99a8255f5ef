"""Device tests of the point-lookup kernel k_get at the kernel boundary (pgs_get_batch / pgs_get_batch_multi through a Partition),
compared field by field with the Python model of tests/get_model.py: status, expired, expire_ts, value length and bytes, the
arena bytes used, and the exact blocks-probed / runs-skipped counters, which pin the Bloom filters the device builds at upload
(k_index_walk) and at compaction (k_emit).  Runs of 1..32 with several block geometries, a hot key with hundreds of versions,
keys of every length, 4 KB keys, values shorter than their header, partial warps, batches that wrap the persistent CTA loop,
the arena-overflow contract, several partitions in one launch, data version 0, and the bench's own data set."""
import ctypes as C

import numpy as np
import pytest

from get_model import (INCOMPLETE, NOT_FOUND, OK, check_results, compacted_run, flat_keys, key_slot, model_get, model_stats,
                       prefix_len, query_keys, sweep_items, sweep_keys, unknown_filter_run, uploaded_run)
from incubator_pegasus_b200 import synth
from scan_model import model_scan, next_key, raw_key, visible
from test_scan_kernels_gpu import CASES, HOT, build_db, load, run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW


def get(pgs, part, keys, cap, now=NOW):
    """one pgs_get_batch call -> (status, results, arena, arena_used, (blocks probed, runs skipped))"""
    flat, off = flat_keys(keys)
    n = len(keys)
    res = (pgs.GetResult * max(1, n))()
    C.memset(res, 0xAB, C.sizeof(res))  # every field of every result must be written
    arena = np.zeros(max(1, cap), np.uint8)
    used = C.c_uint64()
    st = pgs.lib().pgs_get_batch(part.h, flat.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), n, now,
                                 arena.ctypes.data_as(C.c_void_p), C.c_uint64(cap), res, C.byref(used))
    return st, res, arena, used.value, (part.eng.last_blocks_probed, part.eng.last_runs_skipped)


def get_multi(pgs, parts, keys, key_part, cap, now=NOW):
    flat, off = flat_keys(keys)
    n = len(keys)
    res = (pgs.GetResult * max(1, n))()
    C.memset(res, 0xAB, C.sizeof(res))
    arena = np.zeros(max(1, cap), np.uint8)
    kp = np.ascontiguousarray(key_part, np.uint32)
    handles = (C.c_void_p * len(parts))(*[p.h for p in parts])
    used = C.c_uint64()
    st = pgs.lib().pgs_get_batch_multi(handles, len(parts), flat.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p),
                                       kp.ctypes.data_as(C.c_void_p), n, now, arena.ctypes.data_as(C.c_void_p), C.c_uint64(cap), res,
                                       C.byref(used))
    return st, res, arena, used.value, (parts[0].eng.last_blocks_probed, parts[0].eng.last_runs_skipped)


def need(want):
    return sum((len(w["value"]) + 3) & ~3 for w in want if w["status"] == OK)


def model_of(pgs, part, inputs=None):
    """the partition's runs, newest first, downloaded from the device: uploaded runs (level 0) with the upload's filter, a
    level-1 run with the filter of a compaction of `inputs` (uploaded runs)"""
    runs = []
    for rid in part.runs():
        br = part.download(rid)
        if part.run_info(rid).level == 0:
            runs.append(uploaded_run(br))
        else:
            runs.append(compacted_run(br, inputs) if inputs is not None else unknown_filter_run(br))
    return runs


def check_batch(pgs, part, runs, keys, data_version=1):
    """one launch over `keys`: every field, the arena bytes, the counters"""
    ks = key_slot([runs])
    want = [model_get(runs, k, NOW, data_version, ks) for k in keys]
    st, res, arena, used, stats = get(pgs, part, keys, need(want) + 64)
    assert st == 0, st
    n_ok = check_results(res, arena, keys, want, need(want) + 64)
    assert used == need(want)
    assert stats == model_stats(runs, keys, ks), (stats, model_stats(runs, keys, ks))
    return n_ok


@pytest.mark.parametrize("n_runs,block_size,ri,compacted,long_keys", CASES)
def test_get_against_the_model(pgs, engine, n_runs, block_size, ri, compacted, long_keys):
    recs, items = build_db(pgs, 2000 + n_runs, n_runs, long_keys, block_size)
    part = load(pgs, engine, recs, block_size, ri, compacted)
    try:
        inputs = [uploaded_run(pgs.build_run(r, block_size, ri)) for r in recs[:compacted]] if compacted else None
        runs = model_of(pgs, part, inputs)
        assert len(runs) == n_runs - (compacted - 1 if compacted else 0)
        keys = query_keys(runs)
        assert check_batch(pgs, part, runs, keys) > 20
        assert check_batch(pgs, part, runs, keys[::-1][:777]) > 10  # another order, another count
    finally:
        part.close()


@pytest.mark.parametrize("n_runs,block_size,ri,compact", [(1, 4096, 16, 0), (4, 256, 1, 0), (9, 1024, 4, 0), (6, 512, 4, 3)])
def test_get_key_length_sweep(pgs, engine, n_runs, block_size, ri, compact):
    """user keys of 0..300 bytes, hash keys of 0..140 bytes, 4 KB keys, values of 0..12 bytes, expire_ts == now, a hot key
    over many blocks; the compacted case merges the oldest runs on the device (k_emit's filter)"""
    rng = np.random.default_rng(500 + n_runs)
    items = sweep_items(rng, n_runs, sweep_keys(rng, long_keys=not compact), NOW, hot=300)
    recs = [pgs.Records.from_list(it) for it in items[::-1]]  # oldest first, as load uploads them
    part = load(pgs, engine, recs, block_size, ri, compact)
    try:
        runs = model_of(pgs, part, [uploaded_run(pgs.build_run(r, block_size, ri)) for r in recs[:compact]])
        assert check_batch(pgs, part, runs, query_keys(runs)) > 100
    finally:
        part.close()


def test_batch_shapes(pgs, engine):
    """partial warps and CTAs, a batch that wraps the ticket loop of every CTA, one key 10,000 times, an empty batch, a
    partition without runs"""
    n_runs, block_size, ri, compacted, long_keys = CASES[3]
    recs, items = build_db(pgs, 2100, n_runs, long_keys, block_size)
    part = load(pgs, engine, recs, block_size, ri, compacted)
    try:
        runs = model_of(pgs, part, [uploaded_run(pgs.build_run(r, block_size, ri)) for r in recs[:compacted]])
        keys = query_keys(runs)
        rng = np.random.default_rng(3)
        order = [keys[i] for i in rng.permutation(len(keys))]
        for n in (1, 2, 3, 5, 31, 33):
            check_batch(pgs, part, runs, order[:n])
        ks = key_slot([runs])
        per_key = {k: (model_get(runs, k, NOW, 1, ks), model_stats(runs, [k], ks)) for k in keys}
        big = (order * (300_000 // len(order) + 1))[:300_000]
        want = [per_key[k][0] for k in big]
        st, res, arena, used, stats = get(pgs, part, big, need(want))
        assert st == 0 and used == need(want)
        check_results(res, arena, big, want, need(want))
        assert stats == tuple(sum(per_key[k][1][j] for k in big) for j in range(2))
        assert any(HOT in r.newest for r in runs)
        check_batch(pgs, part, runs, [HOT] * 10_000)
        st, res, arena, used, stats = get(pgs, part, [], 16)
        assert st == 0 and used == 0
    finally:
        part.close()
    empty = engine.partition()
    try:
        keys = [b"", b"\x00\x02h1s0001", b"x" * 5000]
        st, res, arena, used, _ = get(pgs, empty, keys, 64)
        assert st == 0 and used == 0
        for i in range(len(keys)):
            r = res[i]
            assert (r.status, r.expired, r.expire_ts, r.value_off, r.value_len, list(r.reserved)) == (NOT_FOUND, 0, 0, 0, 0, [0, 0, 0])
    finally:
        empty.close()


def test_arena_overflow(pgs, engine):
    """an arena below the need: PGS_INCOMPLETE, arena_used = the whole need, every OK value exact, 4-aligned, inside the cap
    and disjoint, every other value that has data INCOMPLETE; a retry with arena_cap = arena_used answers every key"""
    recs, items = build_db(pgs, 2200, 4, False, 1024)
    part = load(pgs, engine, recs, 1024, 16)
    try:
        runs = model_of(pgs, part)
        keys = query_keys(runs) * 3
        want = [model_get(runs, k, NOW) for k in keys]
        total = need(want)
        assert total > 4096
        for cap in (total // 3, total - 4, 0):
            st, res, arena, used, _ = get(pgs, part, keys, cap)
            assert st == INCOMPLETE and used == total, (st, used, total)
            spans = []
            for i, w in enumerate(want):
                r = res[i]
                if w["status"] != OK:
                    assert (r.status, r.expired, r.expire_ts, r.value_len) == (w["status"], w["expired"], w["expire_ts"], 0)
                    continue
                assert r.expire_ts == w["expire_ts"] and r.expired == 0
                if r.status == OK:
                    assert r.value_len == len(w["value"]) and r.value_off % 4 == 0 and r.value_off + r.value_len <= cap
                    assert arena[r.value_off:r.value_off + r.value_len].tobytes() == w["value"]
                    if r.value_len:
                        spans.append((r.value_off, r.value_off + r.value_len))
                else:
                    assert r.status == INCOMPLETE and r.value_len == 0, (i, r.status)  # an empty value too, when its offset lies past the cap
            spans.sort()
            assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
            st, res, arena, used2, _ = get(pgs, part, keys, used)
            assert st == 0 and used2 == total
            check_results(res, arena, keys, want, used)
    finally:
        part.close()


def test_arena_beyond_4_gib(pgs, engine):  # the suite's largest test: 4.5 GB of device and of host memory
    """value offsets are 32-bit: a 4 MiB value looked up 1,030 times needs 4.3 GB of arena; with a cap above that, the values
    that would end past 4 GiB - 1 are PGS_INCOMPLETE and every OK value has its own bytes.  Needs about 4.5 GB of device memory
    and 4.5 GB of host memory."""
    val = np.random.default_rng(1).integers(0, 256, 4 << 20, dtype=np.uint8).tobytes()
    key = raw_key(b"big", b"v")
    part = engine.partition()
    try:
        part.upload(pgs.build_run(pgs.Records.from_list([(key, 1, 1, bytes(12) + val)])))
        n = 1030
        total = n * len(val)
        assert total > 1 << 32
        st, res, arena, used, _ = get(pgs, part, [key] * n, total + (64 << 20))
        assert st == INCOMPLETE and used == total, (st, used)
        want = np.frombuffer(val, np.uint8)
        offs = []
        for i in range(n):
            r = res[i]
            if r.status == OK:
                assert r.value_len == len(val) and r.value_off + r.value_len <= 0xFFFFFFFF
                offs.append(r.value_off)
            else:
                assert r.status == INCOMPLETE
        offs.sort()
        assert len(offs) == 0xFFFFFFFF // len(val)
        assert all(b - a >= len(val) for a, b in zip(offs, offs[1:])), "values share arena bytes"
        for o in offs:
            assert np.array_equal(arena[o:o + len(val)], want)
    finally:
        part.close()


def test_get_batch_multi(pgs, engine):
    """several partitions in one launch: different key slots (one holds 4 KB keys), an empty partition between full ones,
    the same partition listed twice; the counters are the sum over the slots.  Mixed data versions are refused."""
    rng = np.random.default_rng(9)
    a_recs, _ = build_db(pgs, 2300, 4, True, 256)
    b_items = sweep_items(rng, 3, sweep_keys(rng, long_keys=False), NOW, hot=100)
    A = load(pgs, engine, a_recs, 256, 1)
    B = load(pgs, engine, [pgs.Records.from_list(it) for it in b_items[::-1]], 512, 4)
    E = engine.partition()
    D0 = engine.partition(data_version=0)
    try:
        ra, rb = model_of(pgs, A), model_of(pgs, B)
        parts, slots = [B, E, A, B], [rb, [], ra, rb]
        ks = key_slot([ra, rb])
        pool = query_keys(ra) + query_keys(rb)
        keys = [pool[i] for i in rng.integers(0, len(pool), 6000)]
        kp = rng.integers(0, len(parts), len(keys)).astype(np.uint32)
        want = [model_get(slots[s], k, NOW, 1, ks) for k, s in zip(keys, kp)]
        st, res, arena, used, stats = get_multi(pgs, parts, keys, kp, need(want) + 64)
        assert st == 0 and used == need(want)
        assert check_results(res, arena, keys, want, need(want) + 64) > 500
        per = [model_stats(slots[s], [k for k, p in zip(keys, kp) if p == s], ks) for s in range(len(parts))]
        assert stats == (sum(p[0] for p in per), sum(p[1] for p in per))
        st, *_ = get_multi(pgs, [B, D0], keys[:10], np.zeros(10, np.uint32), 1 << 16)
        assert st == pgs.INVALID_ARGUMENT
    finally:
        for p in (A, B, E, D0):
            p.close()


def test_data_version_0(pgs, engine):
    """data version 0: a 4-byte value header"""
    rng = np.random.default_rng(10)
    items = sweep_items(rng, 3, sweep_keys(rng), NOW, hot=120)
    part = engine.partition(data_version=0)
    try:
        for it in items[::-1]:
            part.upload(pgs.build_run(pgs.Records.from_list(it), 512, 4))
        runs = model_of(pgs, part)
        assert check_batch(pgs, part, runs, query_keys(runs), data_version=0) > 100
    finally:
        part.close()


def test_bloom_of_deeper_generations(pgs, engine):
    """a compaction of a compaction output (its filter sized from k_emit's own counts), and that run uploaded again from
    pgs_run_download: no present key or hash-key prefix is rejected, and absent keys skip at least 95 % of the runs"""
    rng = np.random.default_rng(11)
    items = sweep_items(rng, 6, sweep_keys(rng, long_keys=False), NOW, hot=200)
    recs = [pgs.Records.from_list(it) for it in items[::-1]]
    part = engine.partition()
    other = engine.partition()
    try:
        ids = [part.upload(pgs.build_run(r, 512, 4)) for r in recs[:3]]
        first = part.compact(ids, out_level=1, bottommost=0, now=NOW, enabled=False).new_run_id
        more = [part.upload(pgs.build_run(r, 512, 4)) for r in recs[3:]]
        second = part.compact([first] + more, out_level=2, bottommost=0, now=NOW, enabled=False).new_run_id
        assert part.runs() == [second]
        other.upload(part.download(second))
        absent = [bytes(rng.integers(0, 256, int(rng.integers(2, 60)), dtype=np.uint8)) for _ in range(4000)]
        for p in (part, other):
            runs = model_of(pgs, p)
            present = sorted(runs[0].newest)
            present += sorted({k[:prefix_len(k)] for k in present if prefix_len(k)} - set(present))
            want = [model_get(runs, k, NOW) for k in present]
            st, res, arena, used, (probed, skipped) = get(pgs, p, present, need(want) + 64)
            assert st == 0 and skipped == 0
            check_results(res, arena, present, want)
            absent = [k for k in absent if k not in runs[0].newest]
            st, res, arena, used, (probed, skipped) = get(pgs, p, absent, 64)
            assert st == 0 and skipped >= 0.95 * len(absent), (skipped, len(absent))
    finally:
        part.close()
        other.close()


@pytest.mark.parametrize("compact", [0, 3])
def test_prefix_scans_over_the_key_length_sweep(pgs, engine, compact):
    """multi_get (prefix_same_as_start) of every hash key of the sweep: k_scan_fwd's prefix hash at every word and lane split,
    through the upload's filters and (compact) a filter k_emit built"""
    rng = np.random.default_rng(600 + compact)
    keys = sweep_keys(rng, long_keys=False)
    items = sweep_items(rng, 6, keys, NOW, hot=100)
    vis, _ = visible(items)
    part = load(pgs, engine, [pgs.Records.from_list(it) for it in items[::-1]], 512, 4, compact)
    try:
        hks = sorted({k[2:prefix_len(k)] for k in keys if prefix_len(k)})
        reqs = []
        for hk in hks + [b"zz-absent", b"p" * 30 + b"c"]:
            lo = raw_key(hk, b"")
            reqs.append(dict(start=lo, stop=next_key(lo), start_inclusive=True, stop_inclusive=False, key_mode=1, prefix=1,
                             max_count=3000, max_iter_count=3000, max_iter_size=0))
        st, got = run_scans(pgs, part, reqs, 1 << 16)
        assert st == 0, st
        nonempty = 0
        for i, (q, g) in enumerate(zip(reqs, got)):
            w = model_scan(vis, q, NOW)
            nonempty += w["count"] > 0
            assert g == w, (i, q["start"][:40])
        assert nonempty > 100
    finally:
        part.close()


def test_bench_scale_get(pgs, engine):
    """the bench's data set and get batch (4 runs of 2.5 M records, 262,144 keys): every result against the oracle's merged
    visible set (a bottommost compaction with the filter disabled keeps expired values)"""
    import bench
    import oracle_py as orc
    runs = bench.gen_runs(2_500_000, 1000)
    gk, _ = bench.read_workload(2_500_000, 262_144, 16_384, 1000)
    brs = [pgs.build_run(r) for r in runs]
    part = engine.partition()
    try:
        for br in brs:
            part.upload(br)
        bruns = [orc.BlockRunCPU.from_blocks(b) for b in reversed(brs)]
        out, _, _ = orc.compact_blocks(bruns, True, orc.filter_params(enabled=False), bench.NOW, 8)
        vis = out.decode().records()
        klen = gk.shape[1]
        assert np.all(np.diff(vis.key_off.astype(np.int64)) == klen)
        vkeys = vis.keys.reshape(-1, klen).view(f"S{klen}").ravel()
        qkeys = np.ascontiguousarray(gk).view(f"S{klen}").ravel()
        pos = np.minimum(np.searchsorted(vkeys, qkeys), len(vkeys) - 1)
        hit = vkeys[pos] == qkeys
        vo = vis.val_off.astype(np.int64)
        n = qkeys.shape[0]
        cap = n * (bench.VAL + 8)
        keys = [bytes(k) for k in gk]
        st, res, arena, used, _ = get(pgs, part, keys, cap, bench.NOW)
        assert st == 0
        found = 0
        for i in range(n):
            r = res[i]
            if not hit[i]:
                assert (r.status, r.expired, r.expire_ts) == (NOT_FOUND, 0, 0), i
                continue
            v = vis.vals[vo[pos[i]]:vo[pos[i] + 1]]
            ets = int.from_bytes(v[:4].tobytes(), "big")
            assert r.expire_ts == ets, i
            if 0 < ets <= bench.NOW:
                assert (r.status, r.expired, r.value_len) == (NOT_FOUND, 1, 0), i
            else:
                found += 1
                assert r.status == OK and r.expired == 0 and r.value_len == v.shape[0] - 12, i
                assert np.array_equal(arena[r.value_off:r.value_off + r.value_len], v[12:]), i
        assert found > n // 2
    finally:
        part.close()
