"""The fused compaction filter on the device (Partition.compact -> k_walk's dev_filter / dev_user_ops), against
tests/filter_model.py and the oracle: the reference's rule and operation tables, seeded random ops tables, inputs of many
tiles and segments (the compiled kernel's own registers and local memory run the out-of-line table walk), a long table,
data_version 0, values on k_emit's in-place path, and one replica end to end."""
import numpy as np
import pytest

import filter_cases as fc
import filter_model as fm
from incubator_pegasus_b200 import synth

pytestmark = pytest.mark.gpu


def run_gpu_case(pgs, oracle, engine, runs, ops, *, bottommost, now=fc.NOW, data_version=1, **kw):
    """merge runs (newest first) on the device; compare records and the ten counters with the oracle and the model"""
    part = engine.partition(data_version=data_version)
    try:
        ids = [part.upload_records(fc.to_records(pgs, r)) for r in runs[::-1]]  # the later upload is the newer run
        text = fm.to_json(ops) if ops else None
        res = part.compact(ids, out_level=1, bottommost=1 if bottommost else 0, now=now, data_version=data_version,
                           ops=pgs.parse_ops(text, data_version) if text else None, **kw)
        oops = oracle.Ops(text, data_version) if text else None
        want_run, ost = oracle.compact([oracle.Run.from_records(fc.to_records(pgs, r)) for r in runs], bottommost,
                                       oracle.filter_params(ops=oops, data_version=data_version, **kw), now)
        want, st = fm.compact(runs, bottommost, fc.model_params(ops, data_version=data_version, **kw), now)
        assert want_run.records().to_list() == want
        got = pgs.decode_blocks(part.download(res.new_run_id)).to_list() if res.new_run_id else []
        assert got == want
        for f in fm.STAT_FIELDS:
            assert getattr(res, f) == getattr(ost, f) == st[f], f
        return got, st
    finally:
        part.close()


@pytest.mark.parametrize("table", fc.GOLDEN_TABLES)
def test_gpu_golden_table_rows(pgs, oracle, engine, table):
    recs, ops, now, want = fc.golden_case(table)
    out, st = run_gpu_case(pgs, oracle, engine, [recs], ops, bottommost=False, now=now)
    assert fc.verdicts(out, recs) == ["drop" if w == "expired" else w for w in want]
    run_gpu_case(pgs, oracle, engine, [recs], ops, bottommost=True, now=now)


@pytest.mark.parametrize("seed", range(6))
def test_gpu_seeded_ops_tables(pgs, oracle, engine, seed):
    rng = np.random.default_rng(1000 + seed)
    now = fc.NEAR_WRAP_NOW if seed % 2 else fc.NOW
    runs = fc.random_records(rng, now)
    ops = fc.random_ops(rng, now)
    for i, kw in enumerate(fc.filter_settings()):
        run_gpu_case(pgs, oracle, engine, runs, ops, bottommost=(i + seed) % 2 == 0, now=now, **kw)


def _many_records(rng, n_runs, per_run, now):
    hks = [b"", b"a", b"ab", b"abc", b"ba", b"user%d" % 7, b"x" * 20]
    ets_c = [0, 0, now - 1, now, now + 1, now + 30, 0xFFFFFFFF, now + 100000]
    runs, seq = [], 1
    for r in range(n_runs):
        idx = np.sort(rng.choice(per_run * 3, per_run, replace=False))
        recs = []
        for i in idx:
            hk = hks[i % len(hks)]
            key = fc.ukey(hk, b"s%07d" % i + (b"ab" if i % 11 == 0 else b""))
            ets = int(ets_c[rng.integers(len(ets_c))])
            typ = 0 if i % 23 == 0 else 1
            recs.append((key, seq, typ, b"" if typ == 0 else fc.value(ets, b"v" * int(i % 13))))
            seq += 1
        runs.append(sorted(recs, key=lambda x: x[0]))
    return runs[::-1]


def test_gpu_many_tiles_and_segments(pgs, oracle, engine):
    """>= 200 k records: many tiles and segments, every walker running the table walk in the compiled kernel"""
    rng = np.random.default_rng(71)
    runs = _many_records(rng, 4, 60_000, fc.NOW)
    for seed, bm in ((2, True), (5, False)):
        ops = fc.random_ops(np.random.default_rng(1000 + seed), fc.NOW)
        ops.append(fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"ab")], fm.TTL_FROM_CURRENT, 9))
        ops.append(fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_HASHKEY, fm.MATCH_PREFIX, b"ab"), fm.Rule(fm.RULE_TTL_RANGE, start_ttl=0, stop_ttl=40)]))
        _, st = run_gpu_case(pgs, oracle, engine, runs, ops, bottommost=bm, default_ttl=40, validate_hash=True, pidx=1, partition_version=3)
        assert st["in_records"] >= 200_000 and st["dropped_user"] > 1000 and st["ttl_rewritten"] > 1000


def test_gpu_long_table(pgs, oracle, engine):
    """64 ops of 8 rules with patterns of up to 4 KB, over keys that some of them match"""
    rng = np.random.default_rng(13)
    body = bytes(rng.integers(97, 100, 10_000, dtype=np.uint8))
    recs = []
    for i in range(3000):
        off = int(rng.integers(0, 5000))
        sk = body[off:off + int(rng.integers(1, 3000))]
        recs.append((fc.ukey(b"h%02d" % (i % 50), sk), i + 1, 1, fc.value(int(rng.choice([0, fc.NOW + 50, fc.NOW - 3])), b"x" * (i % 9))))
    recs = sorted({r[0]: r for r in recs}.values(), key=lambda r: r[0])
    ops = []
    for o in range(64):
        rules = []
        for r in range(8):
            if r == 7:
                rules.append(fm.Rule(fm.RULE_TTL_RANGE, start_ttl=0, stop_ttl=100) if o % 3 else fm.Rule(fm.RULE_TTL_RANGE))
                continue
            if r < 6 and o % 4 != 0:  # most ops carry patterns that never match (long ones, or inside a rule set that fails)
                pl = int(rng.integers(1, 4097))
                off = int(rng.integers(0, 10_000 - pl))
                rules.append(fm.Rule(fm.RULE_SORTKEY, int(rng.integers(0, 3)), body[off:off + pl]))
            else:
                rules.append(fm.Rule(fm.RULE_SORTKEY, fm.MATCH_ANYWHERE, body[o * 50:o * 50 + 1 + o % 3]))
        ops.append(fm.Op(fm.OP_DELETE, rules) if o % 5 == 0 else fm.Op(fm.OP_UPDATE_TTL, rules, o % 3, 1000 + o))
    for bm in (True, False):
        _, st = run_gpu_case(pgs, oracle, engine, [recs], ops, bottommost=bm, default_ttl=40)
    assert st["ttl_rewritten"] > 0


def test_gpu_data_version_0_with_ops(pgs, oracle, engine):
    rng = np.random.default_rng(77)
    runs = fc.random_records(rng, fc.NOW, n_runs=3, per_run=2000, data_version=0)
    R = fm.Rule
    ops = [fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_HASHKEY, fm.MATCH_ANYWHERE, b"a")], fm.TTL_FROM_NOW, 10),
           fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_SORTKEY, fm.MATCH_PREFIX, b"a")], fm.TTL_FROM_CURRENT, 2**32 - 3),
           fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"b")], fm.TTL_TIMESTAMP, 7),
           fm.Op(fm.OP_DELETE, [R(fm.RULE_TTL_RANGE, start_ttl=2**32 - 100, stop_ttl=100), R(fm.RULE_HASHKEY, fm.MATCH_POSTFIX, b"b")])]
    for dt, bm in ((0, True), (40, False), (40, True)):
        _, st = run_gpu_case(pgs, oracle, engine, runs, ops, bottommost=bm, data_version=0, default_ttl=dt)
        assert st["ttl_rewritten"] > 0 and st["dropped_user"] > 0


def test_gpu_rewrites_on_the_in_place_path(pgs, oracle, engine):
    """values larger than k_emit's block buffer, rewritten by default_ttl and by an op; shadowed older versions"""
    rng = np.random.default_rng(9)
    new, old = [], []
    for i in range(3000):
        key = fc.ukey(b"k", b"%05d" % i)
        vl = int(rng.choice([4100, 8000, 70_000])) if i % 41 == 7 else int(rng.integers(0, 6))
        new.append((key, 10_000 + i, 1, fc.value(0 if i % 2 else fc.NOW + 500, bytes(rng.integers(0, 256, vl, dtype=np.uint8)))))
        if i % 5 == 0:
            old.append((key, 1 + i, 1, fc.value(0, b"old")))
    ops = [fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"0")], fm.TTL_FROM_NOW, 3600)]
    out, st = run_gpu_case(pgs, oracle, engine, [new, old], ops, bottommost=True, default_ttl=40)
    assert any(len(r[3]) > 4096 and fm.expire_ts(r[3]) == fc.NOW + 3600 for r in out)
    assert any(len(r[3]) > 4096 and fm.expire_ts(r[3]) == fc.NOW + 40 for r in out)


def test_gpu_replica_user_specified_compaction_with_ttl_updates(engine):
    """a replica with default_ttl and FROM_CURRENT / TIMESTAMP update ops in its envs, after a manual compaction: every read
    handler against the oracle backend"""
    from rrdb_harness import Backend, raw_key, same_response

    def both(fn, *a, **kw):
        return getattr(pair[0], fn)(*a, **kw), getattr(pair[1], fn)(*a, **kw)

    def check(fn, *a, **kw):
        rg, ro = both(fn, *a, **kw)
        ok, detail = same_response(rg, ro)
        assert ok, (fn, a, kw, detail)
        return rg
    now = synth.NOW
    R = fm.Rule
    ops = fm.to_json([fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_HASHKEY, fm.MATCH_PREFIX, b"cur")], fm.TTL_FROM_CURRENT, 500),
                      fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"_ts")], fm.TTL_TIMESTAMP, fm.EPOCH_BEGIN + now + 77),
                      fm.Op(fm.OP_DELETE, [R(fm.RULE_TTL_RANGE, start_ttl=0, stop_ttl=20), R(fm.RULE_HASHKEY, fm.MATCH_PREFIX, b"cur")])])
    pair = (Backend("gpu", engine), Backend("oracle"))
    try:
        for be in pair:
            for hk in (b"cur_1", b"cur_2", b"other"):
                be.multi_put(hk, {b"a": b"1", b"b_ts": b"2"}, expire_ts=now + 10)
                be.multi_put(hk, {b"c": b"3", b"d_ts": b"4"}, expire_ts=now + 1000)
                be.multi_put(hk, {b"e": b"5", b"f_ts": b"6"}, expire_ts=0)
            be.flush(now)
            be.update_envs({"user_specified_compaction": ops, "default_ttl": "300"})
            be.manual_compact(now)
        for hk in (b"cur_1", b"cur_2", b"other"):
            check("multi_get", hk, now=now)
            check("sortkey_count", hk, now=now)
            for sk in (b"a", b"b_ts", b"c", b"d_ts", b"e", b"f_ts"):
                check("get", hk, sk, now=now)
                check("ttl", hk, sk, now=now)
            (kg, _), (ko, _) = both("scan_all", hk, return_expire_ts=True, now=now)
            assert kg == ko
        assert check("ttl", b"cur_1", b"c", now=now)["ttl"] == 1500  # FROM_CURRENT: 1000 + 500
        assert check("ttl", b"other", b"d_ts", now=now)["ttl"] == 77  # TIMESTAMP
        assert check("ttl", b"other", b"e", now=now)["ttl"] == 300  # default_ttl
        assert check("get", b"cur_1", b"a", now=now)["error"] == 1  # deleted by the range op
        full = (raw_key(b"", b""), b"\xff\xff")
        rg, ro = both("get_scanner", *full, full_scan=True, batch_size=1000, now=now)
        assert same_response(rg, ro)[0]
    finally:
        for be in pair:
            be.close()
