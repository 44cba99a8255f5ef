"""GPU: pgs_rrdb_split, the replica-level partition split.  After a randomized write history that leaves data in runs and in
the memtable, every child answers every read handler (get, ttl, multi_get, batch_get, sortkey_count, get_scanner / scan)
for its keys as the parent does; then writes, flushes and a manual compaction go on on each child and on a CPU-oracle
replica that replayed the parent's history restricted to the child's keys, and both keep answering alike.  The decrees,
last_seq (a child's write overrides a copied version) and the refusals are checked, and a writer thread that keeps
writing to the parent during the split leaves children that hold exactly the writes up to the returned decree."""
import threading

import numpy as np
import pytest

import split_model as sm
from incubator_pegasus_b200 import synth
from rrdb_harness import Backend, raw_key

pytestmark = pytest.mark.gpu

NOW = synth.NOW
HKS = [b"h%03d" % i for i in range(40)] + [b""]  # the empty hash key: its records are routed by the sort key


def history(rng, n):
    ops = []
    for _ in range(n):
        hk, sk = HKS[int(rng.integers(len(HKS)))], b"s%02d" % int(rng.integers(16))
        r = rng.random()
        if r < 0.75:
            ets = 0 if rng.random() < 0.8 else NOW + int(rng.integers(-200, 2000))  # some already expired
            ops.append(("put", hk, sk, bytes(rng.integers(97, 123, int(rng.integers(1, 40)), dtype=np.uint8)), ets))
        elif r < 0.97:
            ops.append(("remove", hk, sk))
        else:
            ops.append(("flush",))
    return ops


def apply(b, op):
    if op[0] == "put":
        assert b.put(op[1], op[2], op[3], expire_ts=op[4], now=NOW) == 0
    elif op[0] == "remove":
        assert b.remove(op[1], op[2], now=NOW) == 0
    else:
        assert b.flush(NOW) == 0


def child_of(hk, sk, src, dst):
    return sm.child_of(raw_key(hk, sk), src, dst)


def mine(op, c, src, dst):
    return op[0] == "flush" or child_of(op[1], op[2], src, dst) == c


def strip(r):
    r = dict(r)
    for k in ("app_id", "partition_index", "context_id", "ctx_class"):
        r.pop(k, None)
    return r


def same_reads(a, b, keys, hks):
    """a's and b's answers to every read handler over the keys (hk, sk) and the non-empty hash keys hks"""
    for hk, sk in keys:
        assert strip(a.get(hk, sk, now=NOW)) == strip(b.get(hk, sk, now=NOW)), (hk, sk)
        assert strip(a.ttl(hk, sk, now=NOW)) == strip(b.ttl(hk, sk, now=NOW)), (hk, sk)
    if keys:
        assert strip(a.batch_get(keys, now=NOW)) == strip(b.batch_get(keys, now=NOW))
    for hk in hks:
        assert strip(a.multi_get(hk, now=NOW)) == strip(b.multi_get(hk, now=NOW)), hk
        assert strip(a.sortkey_count(hk, now=NOW)) == strip(b.sortkey_count(hk, now=NOW)), hk
        ka, _ = a.scan_all(hk, batch_size=7, now=NOW)
        kb, _ = b.scan_all(hk, batch_size=7, now=NOW)
        assert ka == kb, hk


@pytest.mark.parametrize("dst", [2, 4])
def test_rrdb_split_reads_writes_and_decrees(engine, dst):
    rng = np.random.default_rng(dst)
    ops = history(rng, 1500)
    parent = Backend("gpu", engine, app_id=6, pidx=0)
    kids = [Backend("gpu", engine, app_id=6, pidx=i) for i in range(dst)]
    orcs = []
    try:
        for op in ops:
            apply(parent, op)
        parent.put(b"h001", b"mem", b"in the memtable", now=NOW)  # the split flushes it
        ops.append(("put", b"h001", b"mem", b"in the memtable", 0))
        decree = synth_split(parent, kids, 1, dst)
        assert decree == parent.decree
        assert parent.f("rrdb_last_flushed_decree")(parent.h) == decree
        keys = sorted({(op[1], op[2]) for op in ops if op[0] != "flush"})
        for c, kid in enumerate(kids):
            assert kid.f("rrdb_last_committed_decree")(kid.h) == decree
            assert kid.f("rrdb_last_flushed_decree")(kid.h) == decree
            assert kid.f("rrdb_last_durable_decree")(kid.h) == 0
            ck = [k for k in keys if child_of(*k, 1, dst) == c]
            hks = sorted({hk for hk, _ in ck if hk})
            same_reads(kid, parent, ck, hks)
            # the oracle replica: the parent's history restricted to the child's keys
            orc = Backend("orc", app_id=6, pidx=c)
            orcs.append(orc)
            for op in ops:
                if mine(op, c, 1, dst):
                    apply(orc, op)
            same_reads(kid, orc, ck, hks)
            # new writes on the child win over the copied versions (its last_seq is the parent's)
            kid.decree = decree
            old = next(k for k in ck if k[0])
            assert kid.put(old[0], old[1], b"newer", now=NOW) == 0
            assert orc.put(old[0], old[1], b"newer", now=NOW) == 0
            assert kid.get(*old, now=NOW)["kvs"][0][1] == b"newer"
            more = [op for op in history(np.random.default_rng(100 + c), 400) if mine(op, c, 1, dst)]
            for op in more:
                apply(kid, op)
                apply(orc, op)
            assert kid.manual_compact(NOW) == 0 and orc.manual_compact(NOW) == 0
            ck2 = sorted(set(ck) | {(op[1], op[2]) for op in more if op[0] != "flush"} | {old})
            same_reads(kid, orc, ck2, sorted({hk for hk, _ in ck2 if hk}))
    finally:
        for b in kids + orcs + [parent]:
            b.close()


def synth_split(parent, kids, src, dst):
    import incubator_pegasus_b200 as pgs
    return pgs.rrdb_split(parent.h, src, dst, [k.h if k is not None else None for k in kids])


def test_rrdb_split_online_shape_and_refusals(engine):
    """the online split {NULL, child}; a child that is not empty, has the wrong index or is the parent is refused and
    nothing changes"""
    import incubator_pegasus_b200 as pgs
    rng = np.random.default_rng(3)
    parent = Backend("gpu", engine, app_id=7, pidx=1)
    ops = history(rng, 300)
    good = Backend("gpu", engine, app_id=7, pidx=3)
    wrong = Backend("gpu", engine, app_id=7, pidx=2)
    used = Backend("gpu", engine, app_id=7, pidx=3)
    try:
        for op in ops:
            apply(parent, op)
        used.put(b"x", b"y", b"z", now=NOW)
        for kids, code in (([None, wrong], pgs.INVALID_ARGUMENT), ([None, used], pgs.INVALID_ARGUMENT), ([None, good, None], pgs.INVALID_ARGUMENT)):
            with pytest.raises(pgs.PegasusError) as e:
                pgs.rrdb_split(parent.h, 2, 4, [k.h if k is not None else None for k in kids])
            assert e.value.code == code
        with pytest.raises(pgs.PegasusError) as e:
            pgs.rrdb_split(parent.h, 2, 4, [None, parent.h])
        assert e.value.code == pgs.INVALID_ARGUMENT
        assert good.f("rrdb_last_committed_decree")(good.h) == 0 and wrong.f("rrdb_last_committed_decree")(wrong.h) == 0
        assert used.get(b"x", b"y", now=NOW)["kvs"][0][1] == b"z"
        decree = pgs.rrdb_split(parent.h, 2, 4, [None, good.h])
        keys = sorted({(op[1], op[2]) for op in ops if op[0] != "flush"})
        ck = [k for k in keys if child_of(*k, 2, 4) == 1]
        same_reads(good, parent, ck, sorted({hk for hk, _ in ck if hk}))
        assert good.f("rrdb_last_committed_decree")(good.h) == decree
    finally:
        for b in (good, wrong, used, parent):
            b.close()


def test_rrdb_split_with_a_concurrent_writer(engine):
    """a thread keeps writing new keys to the parent during the split: each child holds exactly the writes up to the
    split's decree"""
    import incubator_pegasus_b200 as pgs
    parent = Backend("gpu", engine, app_id=9, pidx=0)
    kids = [Backend("gpu", engine, app_id=9, pidx=i) for i in range(2)]
    log, stop = [], threading.Event()
    for i in range(3000):  # a base in runs and in the memtable
        parent.put(b"base%03d" % (i % 200), b"s%04d" % i, b"v%d" % i, now=NOW)
        if i == 2000:
            parent.flush(NOW)

    def writer():
        i = 0
        while not stop.is_set() and i < 200_000:
            parent.put(b"w%03d" % (i % 97), b"k%06d" % i, b"x%d" % i, now=NOW)
            log.append((parent.decree, b"w%03d" % (i % 97), b"k%06d" % i))
            i += 1
    t = threading.Thread(target=writer)
    t.start()
    try:
        while len(log) < 2000:
            pass
        decree = pgs.rrdb_split(parent.h, 1, 2, [k.h for k in kids])
    finally:
        stop.set()
        t.join()
    try:
        before = [(hk, sk) for d, hk, sk in log if d <= decree]
        after = [(hk, sk) for d, hk, sk in log if d > decree]
        assert before and after  # the writer ran on both sides of the split
        for c, kid in enumerate(kids):
            for hk, sk in before[::7] + before[-50:]:
                if child_of(hk, sk, 1, 2) == c:
                    assert strip(kid.get(hk, sk, now=NOW)) == strip(parent.get(hk, sk, now=NOW)), (hk, sk)
            absent = strip(kid.get(b"never", b"written", now=NOW))
            for hk, sk in after[:50] + after[-50:]:
                if child_of(hk, sk, 1, 2) == c:
                    assert strip(kid.get(hk, sk, now=NOW)) == absent, (hk, sk)
            hks = sorted({b"w%03d" % i for i in range(97)} | {b"base%03d" % i for i in range(200)})
            for hk in hks[::5]:
                want = [kv for kv in parent.multi_get(hk, now=NOW)["kvs"]]
                if child_of(hk, b"", 1, 2) != c:
                    continue
                got = kid.multi_get(hk, now=NOW)["kvs"]
                written = {sk for d, h, sk in log if h == hk and d > decree}
                assert got == [kv for kv in want if kv[0] not in written], hk
    finally:
        for b in kids + [parent]:
            b.close()
