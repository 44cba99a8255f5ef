"""Runs whose bytes lie past 2^32 on the device: the moved runs of tests/far_runs.py through upload, upload_many, download,
get_batch, scans, the merge and the split; and a merge whose OUTPUT passes 4 GiB, read back across 2^32 by gets, scans, a
second merge and a split.  tests/test_far_runs_sim.py runs the moved runs through the same kernel sources on the host.

Every partition is closed as soon as its test is done: a moved run costs the device its whole span (4.3 GB, 8.6 GB for hi2).
Measured on an H100 80GB HBM3 at a 700 W power limit: the file takes about 5 minutes; device memory in use peaked at 37 GB
(the uploads of moved runs, whose freed buffers the engine keeps for reuse) and host memory at 28 GB (the merge past 4 GiB)."""
import hashlib

import numpy as np
import pytest

import far_runs as fr
import foreign_blocks as fb
import split_model as sm
from get_model import (check_results, check_run_format, emit_geometry, flat_keys, model_get, model_stats, query_keys, sweep_items, sweep_keys,
                       uploaded_run)
from incubator_pegasus_b200 import synth
from scan_model import filter_list, make_db, mirror, model_scan, raw_key, scan_list, value, visible
from test_far_runs_sim import FULL, SCAN_HKS, inputs, merge_records, moved
from test_merge_geometry_gpu import smem_budget
from test_scan_kernels_gpu import run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW
INFO_FIELDS = ("n_blocks", "n_records", "n_tombstones", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len", "max_block_size",
               "max_block_records", "smallest_seq", "largest_seq")


def check_download(part, rid, far):
    """pgs_run_download returns the handles as they came and every byte up to the end of the last block: the blocks where
    they were, zeros between them"""
    got = part.download(rid)
    assert got.blk_off.tolist() == far.blk_off.tolist() and got.blk_size.tolist() == far.blk_size.tolist()
    assert got.data.shape[0] == far.data.shape[0] and np.array_equal(got.data, far.data)


@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_upload_and_download_of_moved_runs(pgs, engine, name):
    """upload and upload_many (where the gap of gap_spans_segments is one copy chunk): run_info is the compact upload's but
    for data_bytes; the download gives back the moved run.  Needs up to 9 GB of device memory and 9 GB of host memory."""
    part = engine.partition()
    try:
        for data, br in inputs(pgs).items():
            want = part.run_info(part.upload(br))
            far = moved(br, name)
            rids = [part.upload(far)] if data != "tiny" else part.upload_many([br, far, br])[1:2]
            info = part.run_info(rids[0])
            for f in INFO_FIELDS:
                assert getattr(info, f) == getattr(want, f), (data, f)
            assert info.data_bytes == far.data.shape[0]
            check_download(part, rids[0], far)
            for rid in part.runs():
                part.drop(rid)
            del far
    finally:
        part.close()


@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_reads_of_moved_runs(pgs, engine, name):
    """get_batch with its probe / skip counters over three runs, the newest moved; forward, reverse and mixed scans over two
    runs, the newest moved; and one multi-partition launch that holds the moved run in slot 0"""
    rng = np.random.default_rng(80 + fr.LAYOUTS.index(name))
    items = sweep_items(rng, 3, sweep_keys(rng), NOW, hot=250)
    brs = [pgs.build_run(pgs.Records.from_list(it), 1024, 4) for it in items]
    runs = [uploaded_run(b) for b in brs]
    part = engine.partition()
    try:
        for br in [brs[2], brs[1], moved(brs[0], name)]:   # the newest last
            part.upload(br)
        keys = query_keys(runs)
        flat, off = flat_keys(keys)
        st, res, arena, _used = part.get_batch(flat, off, NOW, arena_cap=1 << 24)
        assert st == 0
        assert check_results(res, arena, keys, [model_get(runs, k, NOW) for k in keys]) > 100
        assert (engine.last_blocks_probed, engine.last_runs_skipped) == model_stats(runs, keys)
    finally:
        part.close()
    rng = np.random.default_rng(950 + fr.LAYOUTS.index(name))
    recs, items = make_db(pgs, rng, 2, SCAN_HKS, 24)
    a, b = engine.partition(pidx=0), engine.partition(pidx=1)
    try:
        a.upload(pgs.build_run(recs[1], 512, 4))
        a.upload(moved(pgs.build_run(recs[0], 512, 4), name))
        b.upload(pgs.build_run(recs[1], 512, 4))
        vis = visible(items)[0]
        fwd = scan_list(SCAN_HKS) + filter_list(FULL)
        rev = [mirror(q) for q in fwd]
        for reqs in (fwd, rev, [q for pair in zip(fwd[0::2], rev[1::2]) for q in pair]):
            st, got = run_scans(pgs, a, reqs)
            assert st == 0
            for q, g_ in zip(reqs, got):
                assert g_ == model_scan(vis, q, NOW), q
        sb = pgs.ScanBatch(None, SCAN_HKS * 2, 200, 96 * 1024, parts=[a, b], req_part=[0] * len(SCAN_HKS) + [1] * len(SCAN_HKS))
        assert sb.run(NOW) == 0
        vis_b = visible(items[1:])[0]
        for j, hk in enumerate(SCAN_HKS * 2):
            v = vis if j < len(SCAN_HKS) else vis_b
            want = [(k[2 + len(hk):], x[12:]) for k, x in v if k[:2 + len(hk)] == len(hk).to_bytes(2, "big") + hk
                    and not 0 < int.from_bytes(x[:4], "big") <= NOW]
            assert sb.records(j) == want, (j, hk)
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_merge_and_split_of_moved_inputs(pgs, oracle, engine, name):
    """the newer input moved: the merge gives the oracle's records (both decoders), counters and run_info, in the block
    format check_run_format reads; then a split of the moved run gives split_model's children"""
    recs = merge_records()
    brs = [pgs.build_run(r, 4096, 16) for r in recs]
    part = engine.partition()
    try:
        ids = [part.upload(brs[1]), part.upload(moved(brs[0], name))][::-1]   # newest first
        res = part.compact(ids, out_level=1, bottommost=1, now=NOW, default_ttl=50)
        want_run, st = oracle.compact([oracle.Run.from_records(r) for r in recs], True, oracle.filter_params(default_ttl=50), NOW)
        want = want_run.records()
        raw = part.download(res.new_run_id)
        got = pgs.decode_blocks(raw)
        assert got.same_as(want) and got.same_as(oracle.Run.from_blocks(raw).records())
        for f in ("in_records", "out_records", "in_bytes", "out_bytes", "dropped_shadowed", "dropped_tombstone", "dropped_expired",
                  "dropped_user", "dropped_stale", "ttl_rewritten"):
            assert getattr(res, f) == getattr(st, f), f
        info, m = part.run_info(res.new_run_id), fb.model_index(raw)
        for f in INFO_FIELDS + ("data_bytes",):
            assert getattr(info, f) == m["info"][f], f
        geo = emit_geometry(4096, 16, info.max_ukey_len, smem_budget())
        check_run_format(raw, 16, geo["block_size"])
    finally:
        part.close()
    br = pgs.build_run(recs[0], 4096, 16)
    items = fb.decode(br).to_list()
    parent = engine.partition(app_id=5, pidx=0)
    kids = [engine.partition(app_id=6, pidx=i) for i in range(4)]
    try:
        parent.upload(moved(br, name), level=1)
        parent.split(1, 4, kids)
        want, _dropped = sm.split_items(items, 1, 4)
        for c, kid in enumerate(kids):
            got = [pgs.decode_blocks(kid.download(r)).to_list() for r in kid.runs()]
            assert got == ([want[c]] if want[c] else []), c
    finally:
        parent.close()
        for k in kids:
            k.close()


# ---- a merge whose output passes 4 GiB --------------------------------------------------------------------------------------------
N_HK, PER_HK = 2000, 19_600   # 39.2 M records of 15-byte keys and 100-byte values: about 4.5 GB of blocks
BIG = 20_000                   # values larger than k_emit's block buffer (its in-place path) that k_scan still stages


def big_records(pgs):
    """run A: N_HK hash keys h0000.. of PER_HK sort keys s0000000.., each value 12 header bytes and 88 random bytes, built
    with numpy (no per-record Python)"""
    rng = np.random.default_rng(12)
    n = N_HK * PER_HK
    hk = np.repeat(np.arange(N_HK), PER_HK)
    sk = np.tile(np.arange(PER_HK), N_HK)
    keys = np.empty((n, 15), np.uint8)
    keys[:, 0], keys[:, 1], keys[:, 2] = 0, 5, ord("h")
    for d in range(4):
        keys[:, 6 - d] = ord("0") + (hk // 10 ** d) % 10
    keys[:, 7] = ord("s")
    for d in range(7):
        keys[:, 14 - d] = ord("0") + (sk // 10 ** d) % 10
    pool = rng.integers(0, 256, (4096, 88), dtype=np.uint8)
    vals = np.empty((n, 100), np.uint8)
    vals[:, :12] = np.frombuffer(value(0, b""), np.uint8)
    for lo in range(0, n, 1 << 20):
        hi = min(n, lo + (1 << 20))
        vals[lo:hi, 12:] = pool[rng.integers(0, 4096, hi - lo)]
    recs = pgs.Records(keys.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 15, vals.reshape(-1), np.arange(n + 1, dtype=np.uint64) * 100,
                       np.arange(1, n + 1, dtype=np.uint64), np.ones(n, np.uint8))
    return recs


def key_of(i):
    return raw_key(b"h%04d" % (i // PER_HK), b"s%07d" % (i % PER_HK))


def newer_records(pgs, seq0, picks, rng):
    """a newer run over record indices `picks` of run A: values of BIG bytes, tombstones, short new values"""
    items = []
    for j, i in enumerate(sorted(set(picks))):
        seq0 += 1
        if j % 3 == 0:
            items.append((key_of(i), seq0, 1, value(0, bytes(rng.integers(0, 256, BIG, dtype=np.uint8)))))
        elif j % 3 == 1:
            items.append((key_of(i), seq0, 0, b""))
        else:
            items.append((key_of(i), seq0, 1, value(0, b"new%d" % i)))
    return pgs.Records.from_list(items)


def digest(r):
    h = hashlib.blake2b(digest_size=16)
    for a in (r.key_off, r.keys, r.val_off, r.vals, r.seq, r.type):
        h.update(np.ascontiguousarray(a).view(np.uint8).data)
    return h.hexdigest()


def child_records_match(got, want, child_of_hk, c):
    """got (Records) holds exactly the records of want whose hash key routes to child c, in order: keys are 15 bytes, so the
    selection is vectorised; values are compared a slab of records at a time"""
    hk = (want.keys.reshape(-1, 15)[:, 3:7].astype(np.int64) - ord("0")) @ np.array([1000, 100, 10, 1])
    sel = child_of_hk[hk] == c
    assert got.n == int(sel.sum())
    assert np.array_equal(got.keys.reshape(-1, 15), want.keys.reshape(-1, 15)[sel])
    assert np.array_equal(got.seq, want.seq[sel]) and np.array_equal(got.type, want.type[sel])
    wl = np.diff(want.val_off.astype(np.int64))
    assert np.array_equal(np.diff(got.val_off.astype(np.int64)), wl[sel])
    at = 0
    for lo in range(0, want.n, 1 << 20):
        hi = min(want.n, lo + (1 << 20))
        part = want.vals[int(want.val_off[lo]):int(want.val_off[hi])][np.repeat(sel[lo:hi], wl[lo:hi])]
        assert np.array_equal(got.vals[at:at + part.shape[0]], part), lo
        at += part.shape[0]
    assert at == got.vals.shape[0]


def test_merge_output_beyond_4_gib(pgs, oracle, engine):
    """39.2 M entries of 115 bytes and 460 newer ones (a third of them 20 KB values, a third tombstones) merge into a run of
    about 4.5 GB: k_emit's batch stores and its in-place path write past 2^32.  The output equals oracle.compact_blocks
    (digest), its data_bytes pass 2^32 and the block holding byte 2^32 has many entries.  On that output: gets and
    forward / reverse scans of the blocks on either side of 2^32; a second merge with a newer run (k_walk and its head
    windows read across 2^32) against the oracle; and a split of it into two children against split_model.  Needs about 20 GB
    of device memory and 28 GB of host memory (measured on an H100 80GB HBM3, 700 W: 18 GB and 28 GB, 155 s)."""
    rng = np.random.default_rng(13)
    n = N_HK * PER_HK
    recs_a = big_records(pgs)
    picks = rng.integers(0, n, 400).tolist() + rng.integers(n - n // 32, n, 60).tolist()   # some in the last 4 %: past 2^32
    recs_b = newer_records(pgs, n, picks, rng)
    part = engine.partition()
    kids = []
    try:
        ida = part.build_records(recs_a)
        idb = part.upload(pgs.build_run(recs_b))
        fp = oracle.filter_params()
        cpu_b = oracle.BlockRunCPU.from_run(oracle.Run.from_records(recs_b))
        cpu_a = oracle.BlockRunCPU.from_run(oracle.Run.from_records(recs_a))
        del recs_a
        res = part.compact([idb, ida], out_level=1, bottommost=1, now=NOW)
        want_b, st, _ = oracle.compact_blocks([cpu_b, cpu_a], True, fp, NOW, threads=16)
        del cpu_a
        for f in ("in_records", "out_records", "in_bytes", "out_bytes", "dropped_shadowed", "dropped_tombstone", "dropped_expired"):
            assert getattr(res, f) == getattr(st, f), f
        want = want_b.decode().records()
        raw = part.download(res.new_run_id)
        assert raw.data.shape[0] > fr.G4
        got = pgs.decode_blocks(raw)
        assert got.n == want.n and digest(got) == digest(want)
        del got
        # the blocks on either side of 2^32
        b = fr.boundary_block(raw)
        assert b is not None and len(fr.block_entries(raw, b)) > 1
        near = [(e.key[:-8], e.value) for x in (b - 1, b, b + 1) for e in fr.block_entries(raw, x)]
        del raw
        keys = [k for k, _ in near]
        flat, off = flat_keys(keys)
        st_, gres, arena, _used = part.get_batch(flat, off, NOW, arena_cap=1 << 24)
        assert st_ == 0
        for i, (k, v) in enumerate(near):
            assert gres[i].status == pgs.OK and arena[gres[i].value_off:gres[i].value_off + gres[i].value_len].tobytes() == v[12:], i
        vis = sorted(near)
        span = dict(FULL, start=vis[0][0], stop=vis[-1][0], max_count=100000, max_iter_count=100000)
        reqs = [span, dict(span, start_inclusive=False), dict(span, stop=vis[len(vis) // 2][0], stop_inclusive=False)]
        reqs += [mirror(q) for q in reqs]
        for rev in (False, True):
            batch = [q for q in reqs if bool(q.get("reverse")) == rev]
            st_, got_s = run_scans(pgs, part, batch, arena_stride=(sum(len(k) + len(v) for k, v in vis) + 4096 + 15) & ~15, kv_stride=len(vis) + 8)
            assert st_ == 0
            for q, g_ in zip(batch, got_s):
                assert g_ == model_scan(vis, q, NOW), (rev, q["start"], q["stop"])
        # a second generation across 2^32
        picks2 = rng.integers(0, n, 300).tolist()
        recs_c = newer_records(pgs, n + 1000, picks2, rng)
        idc = part.upload(pgs.build_run(recs_c))
        res2 = part.compact([idc, res.new_run_id], out_level=1, bottommost=1, now=NOW)
        want2_b, st2, _ = oracle.compact_blocks([oracle.BlockRunCPU.from_run(oracle.Run.from_records(recs_c)), want_b], True, fp, NOW, threads=16)
        del want_b, want
        assert (res2.in_records, res2.out_records, res2.dropped_shadowed, res2.dropped_tombstone) == \
            (st2.in_records, st2.out_records, st2.dropped_shadowed, st2.dropped_tombstone)
        want2 = want2_b.decode().records()
        del want2_b
        raw2 = part.download(res2.new_run_id)
        assert raw2.data.shape[0] > fr.G4
        got2 = pgs.decode_blocks(raw2)
        del raw2
        assert digest(got2) == digest(want2)
        del got2
        # a split of the output into two children
        kids = [engine.partition(app_id=9, pidx=i) for i in range(2)]
        child_of_hk = np.array([sm.child_of(raw_key(b"h%04d" % h, b"s0000000"), 1, 2) for h in range(N_HK)])
        assert set(child_of_hk.tolist()) == {0, 1}
        part.split(1, 2, kids)
        for c, kid in enumerate(kids):
            rids = kid.runs()
            assert len(rids) == 1
            child_records_match(pgs.decode_blocks(kid.download(rids[0])), want2, child_of_hk, c)
    finally:
        part.close()
        for k in kids:
            k.close()
