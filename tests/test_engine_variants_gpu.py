"""GPU parity with the oracle for every lane-group width of the compaction walker (PGS_WALK_G; the default is 4, wider groups are
what long keys fall back to), with the same comparison as test_compaction_gpu, and for the read path over overlapping L0 runs
through the rrdb surface."""
import random

import pytest

from incubator_pegasus_b200 import synth
from rrdb_harness import Backend, same_response
from test_compaction_gpu import run_case

NOW = synth.NOW

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("lanes", [1, 2, 8, 16])
@pytest.mark.parametrize("bottommost", [True, False])
def test_compaction_group_widths(pgs, oracle, engine, monkeypatch, lanes, bottommost):
    monkeypatch.setenv("PGS_WALK_G", str(lanes))  # read per pgs_compact call
    runs = synth.compaction_runs(k=4, n_per_run=30_000)
    run_case(pgs, oracle, engine, runs, bottommost=bottommost, default_ttl=3600 if bottommost else 0)


def test_long_keys_pick_a_wider_group(pgs, oracle, engine):
    """2 KB user keys: the per-group shared memory no longer fits the narrow shape, the geometry widens the groups"""
    import numpy as np
    rng = np.random.default_rng(3)
    runs = []
    seq = 1
    for i in range(3):
        items = {}
        for j in range(300):
            hk = b"h%03d" % rng.integers(0, 40)
            sk = bytes(rng.integers(97, 100, int(rng.integers(1500, 2000))).astype(np.uint8))
            key = len(hk).to_bytes(2, "big") + hk + sk
            items[key] = (key, seq, 1, (0).to_bytes(4, "big") + bytes(8) + b"v%d" % j)
            seq += 1
        runs.append(pgs.Records.from_list([items[k] for k in sorted(items)]))
    run_case(pgs, oracle, engine, runs, bottommost=True)


def test_reads_variants(engine):
    """gets, multi_gets (forward / reverse / limited), sortkey_count and scans through the rrdb surface over 4 overlapping L0 runs"""
    g, o = Backend("gpu", engine, opts={"l0_compaction_trigger": 100}), Backend("oracle", opts={"l0_compaction_trigger": 100})
    rnd = random.Random(5)
    try:
        for round_ in range(4):  # 4 overlapping L0 runs
            for be in (g, o):
                be.decree = round_ * 1000
            for hk in (b"h1", b"h2", b"h3"):
                kvs = {b"s%04d" % rnd.randrange(300): bytes(rnd.getrandbits(8) for _ in range(rnd.choice([5, 120, 700]))) for _ in range(80)}
                ets = rnd.choice([0, NOW + 100, NOW - 5])
                for be in (g, o):
                    be.multi_put(hk, kvs, expire_ts=ets)
            for be in (g, o):
                be.multi_remove(b"h2", [b"s%04d" % (round_ * 5 + j) for j in range(4)])
                be.flush(NOW)
        for hk in (b"h1", b"h2", b"h3", b"none"):
            for sk in [b"s0000", b"s0007", b"s0150", b"s0299", b"nope"]:
                ok, d = same_response(g.get(hk, sk, now=NOW), o.get(hk, sk, now=NOW))
                assert ok, (hk, sk, d)
            for kw in [dict(), dict(reverse=True), dict(max_kv_size=5000), dict(max_kv_count=9, reverse=True), dict(no_value=True),
                       dict(start=b"s0050", stop=b"s0200", stop_inclusive=True)]:
                ok, d = same_response(g.multi_get(hk, now=NOW, **kw), o.multi_get(hk, now=NOW, **kw))
                assert ok, (hk, kw, d[0]["error"], d[1]["error"], len(d[0]["kvs"]), len(d[1]["kvs"]))
            assert same_response(g.sortkey_count(hk, now=NOW), o.sortkey_count(hk, now=NOW))[0]
            (kg, _), (ko, _) = g.scan_all(hk, batch_size=37, now=NOW), o.scan_all(hk, batch_size=37, now=NOW)
            assert kg == ko
    finally:
        g.close()
        o.close()
