"""pgs_run_build_unsorted on the device against pgs_run_build of the same records sorted first: for shuffled, sorted and reversed
inputs the downloaded run and its pgs_run_info (all but the run id) are identical, and point lookups and forward and reverse
batched scans answer exactly as over the pre-sorted run.  2.5 M shuffled config #2 records give the digest of the pre-sorted
build.  Every refusal leaves the run list as it was."""
import random

import pytest

from incubator_pegasus_b200 import synth
from test_run_build_gpu import _digest, _gets, _same_run, _scans
from test_run_build_sim import edge_items
from test_run_build_unsorted_sim import (ikey_sorted, long_prefix_items, one_key_items, prefix_items, version_items,
                                         window_edge_items)

pytestmark = pytest.mark.gpu


def _orders(items, seed):
    want = ikey_sorted(items)
    shuffled = list(items)
    random.Random(seed).shuffle(shuffled)
    return want, [shuffled, want, want[::-1]]


def _check(pgs, eng, items, seed=0, queries=True):
    want, orders = _orders(items, seed)
    a = eng.partition(app_id=11, pidx=0)
    try:
        recs = pgs.Records.from_list(want)
        ia = a.build_records(recs)
        for o in orders:
            b = eng.partition(app_id=11, pidx=1)
            try:
                ib = b.build_records_unsorted(pgs.Records.from_list(o))
                if not items:
                    assert ib == 0 and b.runs() == []
                    continue
                assert pgs.run_build_last_sort_ms() > 0 and all(ms >= 0 for ms in pgs.run_build_last_ms())
                _same_run(a, ia, b, ib)
                if queries:
                    keys = [recs.key(i) for i in range(0, recs.n, max(1, recs.n // 3000))] + [b"\x00\x01zz-missing", b"\x00"]
                    assert _gets(a, keys) == _gets(b, keys)
                    assert _scans(pgs, a, recs) == _scans(pgs, b, recs)
            finally:
                b.close()
    finally:
        a.close()


@pytest.mark.parametrize("bs,ri", [(4096, 16), (512, 2), (16384, 1)])
def test_edge_items(pgs, bs, ri):
    eng = pgs.Engine(block_size=bs, restart_interval=ri)
    try:
        _check(pgs, eng, edge_items(bs + ri), seed=bs)
    finally:
        eng.close()


@pytest.mark.parametrize("case", ["window_edges", "prefixes", "versions", "one_key", "long_prefix", "config2", "n0", "n1", "n2"])
def test_cases(pgs, engine, case):
    items = {
        "window_edges": window_edge_items, "prefixes": prefix_items, "versions": version_items,
        "one_key": lambda: one_key_items(20_000), "long_prefix": long_prefix_items,
        "config2": lambda: synth.compaction_runs(k=1, n_per_run=20_000, seed=3)[0].to_list(),
        "n0": lambda: [], "n1": lambda: [(b"\x00\x01a", 3, 1, b"x")],
        "n2": lambda: [(b"\x00\x01b", 3, 1, b"x"), (b"\x00\x01a", 3, 0, b"")],
    }[case]()
    _check(pgs, engine, items, seed=len(items))


def test_config2_shuffled_digest(pgs, engine):
    """config #2: 2.5 M records of 318 bytes, shuffled"""
    recs = synth.compaction_runs(k=1, n_per_run=2_500_000)[0]
    shuffled = synth.shuffled(recs)
    a, b = engine.partition(app_id=12, pidx=0), engine.partition(app_id=12, pidx=1)
    try:
        ia, ib = a.build_records(recs, 1), b.build_records_unsorted(shuffled, 1)
        assert _digest(a.download(ia)) == _digest(b.download(ib))
        x, y = a.run_info(ia), b.run_info(ib)
        assert y.n_records == 2_500_000 and x.level == y.level == 1
        keys = [recs.key(i) for i in range(0, recs.n, 997)]
        assert _gets(a, keys) == _gets(b, keys)
    finally:
        a.close()
        b.close()


def test_refusals_leave_the_run_list(pgs, engine):
    part = engine.partition(app_id=13)
    try:
        base = part.build_records_unsorted(synth.compaction_runs(k=1, n_per_run=500, seed=4)[0])
        before = part.runs()
        assert before == [base]
        ok = [(b"\x00\x01k%04d" % i, 5, 1, b"v") for i in range(300)]
        random.Random(1).shuffle(ok)
        k4097 = (b"\x00\x01c" + bytes(4094), 5, 1, b"v")
        dup = ok[:50] + [(ok[10][0], 5, 1, b"w")] + ok[50:]

        def bad_offsets(items):
            recs = pgs.Records.from_list(items)
            recs.key_off[3], recs.key_off[4] = recs.key_off[4], recs.key_off[3]
            return recs

        cases = [
            (pgs.Records.from_list(ok[:200] + [k4097] + ok[200:]), pgs.NOT_SUPPORTED),
            (pgs.Records.from_list(dup), pgs.INVALID_ARGUMENT),
            (bad_offsets(ok), pgs.INVALID_ARGUMENT),
            (bad_offsets(dup + [k4097]), pgs.INVALID_ARGUMENT),   # offsets first
            (pgs.Records.from_list(dup + [k4097]), pgs.NOT_SUPPORTED),  # then a long key, before a duplicate
        ]
        for recs, want in cases:
            with pytest.raises(pgs.PegasusError) as e:
                part.build_records_unsorted(recs)
            assert e.value.code == want
            assert part.runs() == before
        assert part.build_records_unsorted(pgs.Records.from_list([])) == 0
        assert part.runs() == before
    finally:
        part.close()
