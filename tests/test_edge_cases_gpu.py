"""GPU edge cases against the oracle: long keys, big values (blocks larger than the staging slots), many runs,
several versions of one key inside a run, multi-chunk scans, corrupt / oversized input handling."""
import ctypes as C
import random

import numpy as np
import pytest

from incubator_pegasus_b200 import synth
from rrdb_harness import Backend, next_blob, raw_key, same_response

pytestmark = pytest.mark.gpu
NOW = 200_000_000


def val(user: bytes, ets: int = 0) -> bytes:
    return ets.to_bytes(4, "big") + bytes(8) + user


def compact_both(pgs, oracle, engine, runs, bottommost=True, **kw):
    part = engine.partition()
    try:
        ids = [part.upload_records(r) for r in runs]
        res = part.compact(ids, out_level=1, bottommost=1 if bottommost else 0, now=NOW, **kw)
        want, st = oracle.compact([oracle.Run.from_records(r) for r in runs], bottommost,
                                  oracle.filter_params(default_ttl=kw.get("default_ttl", 0)), NOW)
        w = want.records()
        if w.n == 0:
            assert res.new_run_id == 0
            return res
        got = pgs.decode_blocks(part.download(res.new_run_id))
        assert got.same_as(w)
        assert res.out_records == st.out_records and res.dropped_shadowed == st.dropped_shadowed
        return res
    finally:
        part.close()


def test_long_keys_and_big_values(pgs, oracle, engine):
    rnd = random.Random(3)
    runs, seq = [], 1
    for i in range(3):
        items = {}
        for _ in range(300):
            hk = bytes(rnd.getrandbits(8) for _ in range(rnd.choice([1, 40, 300])))
            sk = bytes(rnd.getrandbits(8) for _ in range(rnd.choice([0, 5, 700])))
            key = raw_key(hk, sk)
            user = bytes(rnd.getrandbits(8) for _ in range(rnd.choice([0, 10, 3000, 20000])))
            items[key] = (key, seq, 1, val(user, rnd.choice([0, NOW + 9, NOW - 9])))
            seq += 1
        runs.append(pgs.Records.from_list(sorted(items.values())))
    compact_both(pgs, oracle, engine, runs, bottommost=True)
    compact_both(pgs, oracle, engine, runs, bottommost=False, default_ttl=77)


def test_many_runs(pgs, oracle, engine):
    runs = synth.compaction_runs(k=12, n_per_run=1500, seed=31, dup_frac=0.3, tomb_frac=0.05)
    res = compact_both(pgs, oracle, engine, runs)
    assert res.dropped_shadowed > 0


def test_versions_of_one_key_inside_a_run(pgs, oracle, engine):
    k = lambda i: raw_key(b"h", b"%03d" % i)
    run_a = pgs.Records.from_list([
        (k(1), 9, 1, val(b"new")), (k(1), 5, 0, b""), (k(1), 2, 1, val(b"old")),
        (k(2), 8, 0, b""), (k(2), 7, 1, val(b"gone")),
        (k(3), 6, 1, val(b"three")),
    ])
    run_b = pgs.Records.from_list([(k(1), 1, 1, val(b"older")), (k(2), 3, 1, val(b"x")), (k(4), 4, 1, val(b"four", NOW - 1))])
    for bottom in (True, False):
        compact_both(pgs, oracle, engine, [run_a, run_b], bottommost=bottom)


def test_reads_over_many_runs_and_big_values(engine):
    g, o = Backend("gpu", engine, opts={"l0_compaction_trigger": 100}), Backend("oracle", opts={"l0_compaction_trigger": 100})
    rnd = random.Random(11)
    try:
        for round_ in range(11):  # 11 L0 runs
            for be in (g, o):
                be.decree = round_ * 1000
            kvs = {b"s%04d" % rnd.randrange(400): bytes(rnd.getrandbits(8) for _ in range(rnd.choice([3, 900, 6000]))) for _ in range(60)}
            for be in (g, o):
                be.multi_put(b"big", kvs, expire_ts=rnd.choice([0, NOW + 100]))
                be.multi_remove(b"big", [b"s%04d" % (round_ * 7 + j) for j in range(3)])
                be.flush(NOW)
        for sk in [b"s0000", b"s0007", b"s0100", b"s0399", b"nope"]:
            rg, ro = g.get(b"big", sk, now=NOW), o.get(b"big", sk, now=NOW)
            assert same_response(rg, ro)[0]
        # multi-chunk scans: ~300 live records of up to 6 KB
        (kg, bg), (ko, bo) = g.scan_all(b"big", batch_size=1000, now=NOW), o.scan_all(b"big", batch_size=1000, now=NOW)
        assert kg == ko and len(bg) == len(bo)
        for kw in [dict(), dict(reverse=True), dict(max_kv_size=20000), dict(max_kv_count=17, reverse=True), dict(no_value=True),
                   dict(start=b"s0100", stop=b"s0300", stop_inclusive=True, reverse=True)]:
            rg, ro = g.multi_get(b"big", now=NOW, **kw), o.multi_get(b"big", now=NOW, **kw)
            ok, d = same_response(rg, ro)
            assert ok, (kw, d[0]["error"], d[1]["error"], len(d[0]["kvs"]), len(d[1]["kvs"]))
        assert same_response(g.sortkey_count(b"big", now=NOW), o.sortkey_count(b"big", now=NOW))[0]
        for be in (g, o):
            be.manual_compact(NOW)
        (kg, _), (ko, _) = g.scan_all(b"big", batch_size=50, now=NOW), o.scan_all(b"big", batch_size=50, now=NOW)
        assert kg == ko
    finally:
        g.close()
        o.close()


def test_reverse_reads_over_many_runs_of_tombstones(engine):
    """11 L0 runs of ~2,000 short tombstones each (multi_remove + flush): a 4 KB block holds ~320 records, so k_scan could
    not stage one block of every run, and 11 runs stay under the read-triggered fold at 12.  Reverse reads must still
    answer (the server folds L0 for them first); forward reads and counts as well."""
    g, o = Backend("gpu", engine, opts={"l0_compaction_trigger": 100}), Backend("oracle", opts={"l0_compaction_trigger": 100})
    try:
        for round_ in range(11):
            for be in (g, o):
                be.decree = round_ * 1000
                be.multi_put(b"t", {b"%d" % (round_ * 37 + j): b"v%d" % round_ for j in range(5)})
                assert be.multi_remove(b"t", [b"%d" % (i * 11 + round_) for i in range(2000)])[0] == 0
                be.flush(NOW)
        for kw in [dict(reverse=True), dict(), dict(reverse=True, max_kv_count=3), dict(start=b"200", stop=b"300", reverse=True)]:
            rg, ro = g.multi_get(b"t", now=NOW, **kw), o.multi_get(b"t", now=NOW, **kw)
            assert rg["error"] == ro["error"] and same_response(rg, ro)[0], (kw, rg["error"], ro["error"])
        assert same_response(g.sortkey_count(b"t", now=NOW), o.sortkey_count(b"t", now=NOW))[0]
    finally:
        g.close()
        o.close()


def test_corrupt_and_unsupported_uploads(pgs, engine):
    run = pgs.build_run(synth.compaction_runs(k=1, n_per_run=500, seed=5)[0])
    part = engine.partition()
    try:
        bad = pgs.BlockRun(run.data.copy(), run.blk_off, run.blk_size)
        bad.data[int(run.blk_off[1]) + 1] = 0xFF  # non_shared varint of the first entry of block 1 runs past the block
        bad.data[int(run.blk_off[1]) + 2] = 0xFF
        with pytest.raises(pgs.PegasusError) as e:
            part.upload(bad)
        assert e.value.code == pgs.CORRUPTION
        bad2 = pgs.BlockRun(run.data.copy(), run.blk_off, run.blk_size.copy())
        bad2.data[int(run.blk_off[0]) + int(run.blk_size[0]) - 4] = 0  # restart count 0
        with pytest.raises(pgs.PegasusError) as e:
            part.upload(bad2)
        assert e.value.code == pgs.CORRUPTION
        off = run.blk_off.copy()
        off[1] += 1  # misaligned handle
        with pytest.raises(pgs.PegasusError) as e:
            part.upload(pgs.BlockRun(run.data, off, run.blk_size))
        assert e.value.code == pgs.INVALID_ARGUMENT
        huge = pgs.Records.from_list([(raw_key(b"h" * 5000, b""), 1, 1, val(b"v"))])
        with pytest.raises(pgs.PegasusError) as e:
            part.upload_records(huge)
        assert e.value.code == pgs.NOT_SUPPORTED
        assert part.runs() == []  # nothing half-installed
        rid = part.upload(run)
        assert part.runs() == [rid]
        with pytest.raises(pgs.PegasusError) as e:
            part.compact([rid, rid])
        assert e.value.code == pgs.INVALID_ARGUMENT
        with pytest.raises(pgs.PegasusError) as e:
            part.compact([rid + 12345])
        assert e.value.code == pgs.NOT_FOUND
    finally:
        part.close()


def test_upload_many_is_all_or_nothing(pgs, engine):
    """a damaged run in the middle of a pipelined upload: the call fails, no run of it stays installed, the partition still works;
    a multi-chunk run (> 32 MB) goes through the chunked copy + per-chunk index pass"""
    runs = [pgs.build_run(r) for r in synth.compaction_runs(k=3, n_per_run=800, seed=6)]
    part = engine.partition()
    try:
        bad = pgs.BlockRun(runs[1].data.copy(), runs[1].blk_off, runs[1].blk_size)
        bad.data[int(bad.blk_off[2]) + 1] = 0xFF
        bad.data[int(bad.blk_off[2]) + 2] = 0xFF
        with pytest.raises(pgs.PegasusError) as e:
            part.upload_many([runs[0], bad, runs[2]])
        assert e.value.code == pgs.CORRUPTION and part.runs() == []
        ids = part.upload_many(runs + [pgs.BlockRun(np.zeros(0, np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint32))])
        assert ids[3] == 0 and sorted(part.runs()) == sorted(ids[:3])
        for rid, r in zip(ids, runs):
            assert pgs.decode_blocks(part.download(rid)).same_as(pgs.decode_blocks(r))
        big = pgs.build_run(synth.compaction_runs(k=1, n_per_run=150_000, seed=9)[0])  # ~48 MB of blocks: two chunks
        assert big.data.shape[0] > (32 << 20)
        rid = part.upload_many([big])[0]
        info = part.run_info(rid)
        assert info.n_records == 150_000 and info.n_blocks == big.n_blocks
        assert pgs.decode_blocks(part.download(rid)).same_as(pgs.decode_blocks(big))
    finally:
        part.close()


def test_get_batch_over_several_partitions(pgs, engine):
    """pgs_get_batch_multi: one launch answers keys of several replicas; the same answers as one pgs_get_batch per partition"""
    rng = np.random.default_rng(8)
    parts, keysets = [], []
    try:
        for p, n_runs in enumerate((1, 3, 5, 0)):  # the last partition holds nothing
            part = engine.partition(app_id=4, pidx=p)
            parts.append(part)
            runs = synth.compaction_runs(k=max(1, n_runs), n_per_run=3000, seed=40 + p)[:n_runs]
            for r in runs:
                part.upload_records(r)
            ks = [r.key(int(i)) for r in runs for i in rng.integers(0, r.n, 150)]
            keysets.append(ks + [raw_key(b"absent%d" % p, b"x")])
        keys, slot = [], []
        for p, ks in enumerate(keysets):          # every partition is also asked for the other partitions' keys
            for q in range(len(parts)):
                keys += keysets[q][:40]
                slot += [p] * len(keysets[q][:40])
        order = rng.permutation(len(keys))
        keys, slot = [keys[i] for i in order], np.array([slot[i] for i in order], np.uint32)
        flat = np.frombuffer(b"".join(keys), np.uint8).copy()
        off = np.zeros(len(keys) + 1, np.uint32)
        off[1:] = np.cumsum([len(k) for k in keys])
        arena = np.zeros(len(keys) * 400, np.uint8)
        st, res, arena, used = pgs.get_batch_multi(parts, flat, off, slot, synth.NOW, arena)
        assert st == 0 and used > 0
        for p, part in enumerate(parts):
            sel = np.nonzero(slot == p)[0]
            sub = [keys[i] for i in sel]
            f2 = np.frombuffer(b"".join(sub), np.uint8).copy()
            o2 = np.zeros(len(sub) + 1, np.uint32)
            o2[1:] = np.cumsum([len(k) for k in sub])
            st2, res2, arena2, _ = part.get_batch(f2, o2, synth.NOW)
            assert st2 == 0
            for j, i in enumerate(sel):
                a, b = res[int(i)], res2[j]
                assert (a.status, a.expire_ts, a.expired, a.value_len) == (b.status, b.expire_ts, b.expired, b.value_len), (p, j)
                if a.status == pgs.OK:
                    assert arena[a.value_off:a.value_off + a.value_len].tobytes() == arena2[b.value_off:b.value_off + b.value_len].tobytes()
        assert sum(1 for i in range(len(keys)) if res[i].status == pgs.OK) > 100
        bad = slot.copy(); bad[0] = 9
        assert pgs.get_batch_multi(parts, flat, off, bad, synth.NOW, arena)[0] == pgs.INVALID_ARGUMENT
    finally:
        for part in parts:
            part.close()


def test_empty_partition_reads(engine):
    g, o = Backend("gpu", engine), Backend("oracle")
    try:
        assert same_response(g.get(b"a", b"b", now=NOW), o.get(b"a", b"b", now=NOW))[0]
        assert same_response(g.multi_get(b"a", now=NOW), o.multi_get(b"a", now=NOW))[0]
        assert same_response(g.sortkey_count(b"a", now=NOW), o.sortkey_count(b"a", now=NOW))[0]
        rg, ro = g.get_scanner(raw_key(b"", b""), b"\xff\xff", full_scan=True, now=NOW), o.get_scanner(raw_key(b"", b""), b"\xff\xff", full_scan=True, now=NOW)
        assert same_response(rg, ro)[0]
        for be in (g, o):
            be.manual_compact(NOW)
            be.flush(NOW)
        assert same_response(g.batch_get([(b"a", b"b")], now=NOW), o.batch_get([(b"a", b"b")], now=NOW))[0]
    finally:
        g.close()
        o.close()


def test_prefix_scans_over_several_partitions(pgs, engine):
    """pgs_range_scan_many_multi: one launch answers multi_get-shaped scans of several replicas, with the same records as one
    pgs_range_scan_many per partition"""
    rng = np.random.default_rng(9)
    parts, hksets = [], []
    try:
        for p, n_runs in enumerate((2, 4, 0, 7)):  # partition 2 holds nothing
            part = engine.partition(app_id=5, pidx=p)
            parts.append(part)
            runs = synth.compaction_runs(k=max(1, n_runs), n_per_run=3000, seed=60 + p)[:n_runs]
            for r in runs:
                part.upload_records(r)
            hks = set()
            for r in runs:
                for i in rng.integers(0, r.n, 40):
                    k = r.key(int(i))
                    hks.add(k[2:2 + int.from_bytes(k[:2], "big")])
            hksets.append(sorted(hks)[:60] + [b"absent%d" % p])
        hashkeys, slot = [], []
        for p in range(len(parts)):               # every partition is also asked for the other partitions' hash keys
            for q in range(len(parts)):
                hashkeys += hksets[q][:25]
                slot += [p] * len(hksets[q][:25])
        order = rng.permutation(len(hashkeys))
        hashkeys, slot = [hashkeys[i] for i in order], np.array([slot[i] for i in order], np.uint32)
        multi = pgs.ScanBatch(None, hashkeys, 200, 65536, parts=parts, req_part=slot)
        assert multi.run(synth.NOW) == 0
        total = 0
        for p, part in enumerate(parts):
            sel = np.nonzero(slot == p)[0]
            one = part.prefix_scan_batch([hashkeys[i] for i in sel], max_records=200, arena_stride=65536)
            assert one.run(synth.NOW) == 0
            for j, i in enumerate(sel):
                a, b = multi.results[int(i)], one.results[j]
                assert (a.count, a.iter_count, a.expire_count, a.filter_count, a.size, a.complete, a.iter_valid) == \
                       (b.count, b.iter_count, b.expire_count, b.filter_count, b.size, b.complete, b.iter_valid), (p, j)
                assert multi.records(int(i)) == one.records(j), (p, j)
                total += a.count
        assert total > 200
        bad = slot.copy(); bad[0] = 9
        assert pgs.ScanBatch(None, hashkeys, 200, 65536, parts=parts, req_part=bad).run(synth.NOW) == pgs.INVALID_ARGUMENT
        multi.reqs[0].reverse = 1
        assert multi.run(synth.NOW) == pgs.NOT_SUPPORTED
    finally:
        for part in parts:
            part.close()


def test_run_count_limits_are_reported(pgs, engine):
    """more than 16 runs in one merge launch and more than 32 runs under one read are refused with NOT_SUPPORTED (DESIGN §8),
    not answered wrongly; 16 / 32 themselves work"""
    runs = synth.compaction_runs(k=33, n_per_run=200, seed=77)
    part = engine.partition(app_id=6, pidx=0)
    try:
        ids = [part.upload_records(r) for r in runs]
        key = runs[0].key(0)
        flat = np.frombuffer(key, np.uint8).copy()
        off = np.array([0, len(key)], np.uint32)
        assert part.get_batch(flat, off, synth.NOW)[0] == pgs.NOT_SUPPORTED
        sb = part.prefix_scan_batch([key[2:2 + int.from_bytes(key[:2], "big")]], max_records=50, arena_stride=32768)
        assert sb.run(synth.NOW) == pgs.NOT_SUPPORTED
        with pytest.raises(pgs.PegasusError) as e:
            part.compact(ids[:17])
        assert e.value.code == pgs.NOT_SUPPORTED
        assert len(part.runs()) == 33  # nothing was consumed by the refused merge
        res = part.compact(ids[:16])
        assert res.out_records > 0 and len(part.runs()) == 33 - 16 + 1
        st, r, arena, _ = part.get_batch(flat, off, synth.NOW)  # 18 runs: served
        assert st == 0
        assert sb.run(synth.NOW) == 0
    finally:
        part.close()
