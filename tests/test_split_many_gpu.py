"""GPU: pgs_partition_split_many against pgs_partition_split on twin partitions.  Every parent has a twin holding the same
uploaded runs (1 to 7 runs over levels 0..3, one parent without runs); the twins are split one by one, the originals in one
call.  Every child must hold the same runs with the same decoded records, the same counters, and answer gets and forward
and reverse scans alike; the call launches the same kernels for 1 parent as for 64; every refusal launches nothing and
changes no child; a call past 4 GiB of values gives the single splits' children.  The replica layer: pgs_rrdb_split_many
against pgs_rrdb_split on twin replicas with write histories, including the online shape (child 0 not built)."""
import hashlib

import numpy as np
import pytest

import split_model as sm
from incubator_pegasus_b200 import synth
from rrdb_harness import Backend
from test_rrdb_split_gpu import apply, child_of, history, same_reads
from test_scan_kernels_gpu import run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW
CHILD_FIELDS = ("records", "tombstones", "raw_bytes", "runs")
RES_FIELDS = ("in_records", "in_bytes", "dropped_empty")
INFO_FIELDS = ("level", "n_records", "n_tombstones", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len",
               "smallest_seq", "largest_seq")


def parent_runs(i, n_per_run=400):
    """parent i's runs (oldest first) and their levels; parent 3 has none"""
    if i == 3:
        return [], []
    k = 1 + i % 7
    runs = synth.compaction_runs(k=k, n_per_run=n_per_run, seed=300 + i)
    return runs, [min(3, k - 1 - r) for r in range(k)]


def load(engine, n, app_id, src=1, n_per_run=400):
    """parent i: index i % src of a table of src partitions"""
    out = []
    for i in range(n):
        p = engine.partition(app_id=app_id, pidx=i % src)
        runs, levels = parent_runs(i, n_per_run)
        for r, lvl in zip(runs, levels):
            p.upload_records(r, lvl)
        out.append(p)
    return out


def kids_of(engine, parents, src, dst, app_id, online=False):
    S = dst // src
    return [[None if online and c == 0 else engine.partition(app_id=app_id, pidx=i % src + c * src) for c in range(S)]
            for i in range(len(parents))]


def child_runs(pgs, kid):
    return [(kid.run_info(r).level, pgs.decode_blocks(kid.download(r)).to_list(), kid.run_info(r)) for r in kid.runs()]


def reads(pgs, part, keys):
    if not keys:
        return None
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    st, res, arena, _ = part.get_batch(np.frombuffer(b"".join(keys), np.uint8).copy(), off, NOW, arena_cap=64 << 20)
    assert st == 0
    gets = [(r.status, r.expire_ts, arena[r.value_off:r.value_off + r.value_len].tobytes() if r.status == 0 else b"") for r in res]
    full = dict(start=b"", stop=b"\xff" * 8, start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0,
                max_count=1 << 20, max_iter_count=1 << 20, max_iter_size=0, return_expire_ts=1)
    mid = keys[len(keys) // 3]
    reqs = [full, dict(full, reverse=1), dict(full, start=mid, max_count=40), dict(full, stop=mid, reverse=1, max_count=40)]
    st, ans = run_scans(pgs, part, reqs, arena_stride=8 << 20, kv_stride=1 << 14)
    assert st == 0
    return gets, ans


def close(*groups):
    for g in groups:
        for x in g:
            if isinstance(x, list):
                close(x)
            elif x is not None:
                x.close()


@pytest.mark.parametrize("src,dst", [(1, 2), (2, 8), (1, 8)])
def test_split_many_matches_one_by_one(pgs, engine, src, dst):
    n = 9
    S = dst // src
    orig, twins = load(engine, n, 600, src), load(engine, n, 601, src)
    ka, kb = kids_of(engine, orig, src, dst, 602), kids_of(engine, twins, src, dst, 603)
    try:
        res_one = [t.split(src, dst, k) for t, k in zip(twins, kb)]
        before = engine.launches
        res_many = engine.split_many(list(zip(orig, ka)), src, dst)
        assert engine.launches - before == pgs.SPLIT_MANY_LAUNCHES
        for i in range(len(orig)):
            a, b = res_many[i], res_one[i]
            assert a.n_launches == pgs.SPLIT_MANY_LAUNCHES
            for f in RES_FIELDS:
                assert getattr(a, f) == getattr(b, f), (i, f)
            keys = sorted({r.key(x) for r in parent_runs(i)[0] for x in range(r.n)})
            for c in range(S):
                for f in CHILD_FIELDS:
                    assert getattr(a.child[c], f) == getattr(b.child[c], f), (i, c, f)
                ra, rb = child_runs(pgs, ka[i][c]), child_runs(pgs, kb[i][c])
                assert [(lvl, recs) for lvl, recs, _ in ra] == [(lvl, recs) for lvl, recs, _ in rb], (i, c)
                for (_, _, ia), (_, _, ib) in zip(ra, rb):
                    for f in INFO_FIELDS:
                        assert getattr(ia, f) == getattr(ib, f), (i, c, f)
                mine = [k for k in keys if sm.child_of(k, src, dst) == c]
                assert reads(pgs, ka[i][c], mine) == reads(pgs, kb[i][c], mine), (i, c)
    finally:
        close(orig, twins, ka, kb)


@pytest.mark.parametrize("n", [1, 16, 64])
def test_launches_do_not_grow_with_jobs(pgs, engine, n):
    parents = load(engine, n, 610, n_per_run=60)
    kids = kids_of(engine, parents, 1, 2, 611)
    try:
        before = engine.launches
        res = engine.split_many(list(zip(parents, kids)), 1, 2)
        assert engine.launches - before == pgs.SPLIT_MANY_LAUNCHES
        assert all(r.n_launches == pgs.SPLIT_MANY_LAUNCHES for r in res)
        assert engine.split_many([], 1, 2) == []
        assert engine.launches - before == pgs.SPLIT_MANY_LAUNCHES
    finally:
        close(parents, kids)


def test_refusals(pgs, engine):
    parents = load(engine, 4, 620, n_per_run=100)  # parents[3] holds no runs
    kids = kids_of(engine, parents, 1, 2, 621)
    other = pgs.Engine()
    extra = []
    try:
        held = [[k.runs() for k in row] for row in kids]

        def refused(code, jobs, src=1, dst=2):
            before = engine.launches
            with pytest.raises(pgs.PegasusError) as e:
                engine.split_many(jobs, src, dst)
            assert e.value.code == code
            assert engine.launches == before
            assert [[k.runs() for k in row] for row in kids] == held

        ok = [(parents[0], kids[0])]
        refused(pgs.INVALID_ARGUMENT, ok + [(parents[0], kids[1])])                  # the same parent twice
        refused(pgs.INVALID_ARGUMENT, ok + [(parents[1], [kids[0][0], kids[1][1]])])  # the same child in two jobs
        refused(pgs.INVALID_ARGUMENT, ok + [(kids[0][0], kids[1])])                    # a child reused as a parent
        empty = [(parents[3], kids[3])]
        refused(pgs.INVALID_ARGUMENT, empty + [(parents[1], [parents[3], kids[1][1]])])  # a parent reused as a child
        far = other.partition(app_id=622, pidx=1)
        extra.append(far)
        refused(pgs.INVALID_ARGUMENT, ok + [(parents[1], [kids[1][0], far])])          # a child on another engine
        far_parent = other.partition(app_id=623, pidx=0)
        extra.append(far_parent)
        refused(pgs.INVALID_ARGUMENT, ok + [(far_parent, kids[1])])                    # a parent on another engine
        full = engine.partition(app_id=624, pidx=1)
        full.upload_records(synth.compaction_runs(k=1, n_per_run=50)[0])
        extra.append(full)
        refused(pgs.INVALID_ARGUMENT, ok + [(parents[1], [kids[1][0], full])])         # a child that holds runs
        wrong = engine.partition(app_id=625, pidx=0)
        extra.append(wrong)
        refused(pgs.INVALID_ARGUMENT, ok + [(parents[1], [kids[1][0], wrong])])        # a wrong child index
        v2 = engine.partition(app_id=626, pidx=1, data_version=0)
        extra.append(v2)
        refused(pgs.NOT_SUPPORTED, ok + [(parents[1], [kids[1][0], v2])])              # another data_version
        many = [engine.partition(app_id=627, pidx=i) for i in range(64)]
        extra += many
        refused(pgs.NOT_SUPPORTED, [(parents[2], many)], 1, 64)                        # beyond PGS_SPLIT_MAX_CHILDREN
        refused(pgs.NOT_SUPPORTED, [(parents[0], kids[0])] * (pgs.SPLIT_MANY_MAX_JOBS + 1))  # n over the limit
        res = engine.split_many(list(zip(parents, kids)), 1, 2)  # the good call still goes through
        assert [r.in_records for r in res] == [sum(r.n for r in parent_runs(i, 100)[0]) for i in range(4)]
    finally:
        close(parents, kids, extra)
        other.close()


def _digest(pgs, kid):
    h = hashlib.sha256()
    for r in kid.runs():
        d = pgs.decode_blocks(kid.download(r))
        for a in (d.keys, d.key_off, d.vals, d.val_off, d.seq, d.type):
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def test_split_many_past_4_gib(pgs, engine):
    """five parents of one run of 1 000 records with 1 MB values (5 GB of values, every record its own hash key) split
    1 -> 2 together and one by one: every child's decoded records are the same"""
    rng = np.random.default_rng(4)
    chunk = rng.integers(0, 256, 1 << 26, np.uint8)
    parents = []
    for j in range(5):
        n = 1000
        vals = np.tile(np.roll(chunk, j), 16)[: n << 20]
        keys = np.frombuffer(b"".join(b"\x00\x04%04d-j%d" % (x, j) for x in range(n)), np.uint8).copy()
        klen = len(b"\x00\x040000-j0")
        recs = pgs.Records(keys, np.arange(n + 1, dtype=np.uint64) * klen, vals, np.arange(n + 1, dtype=np.uint64) << 20,
                           np.arange(n, 0, -1).astype(np.uint64) + 10, np.ones(n, np.uint8))
        p = engine.partition(app_id=630, pidx=0)
        p.build_records(recs)
        parents.append(p)
        del vals, recs
    ka = [[engine.partition(app_id=631, pidx=c) for c in range(2)] for _ in parents]
    try:
        res = engine.split_many(list(zip(parents, ka)), 1, 2)
        assert sum(r.in_bytes for r in res) > 4 << 30
        da = [[_digest(pgs, k) for k in row] for row in ka]
        assert all(r.child[0].records and r.child[1].records for r in res)
    finally:
        close(ka)
    kb = [[engine.partition(app_id=632, pidx=c) for c in range(2)] for _ in parents]
    try:
        for p, row in zip(parents, kb):
            p.split(1, 2, row)
        assert [[_digest(pgs, k) for k in row] for row in kb] == da
    finally:
        close(parents, kb)


def test_rrdb_split_many_matches_rrdb_split(pgs, engine):
    """replicas with write histories (data in runs and in the memtable): split together and their twins one by one, 1 -> 4
    with every child built and 2 -> 4 in the online shape; decrees, reads and writes after the split agree"""
    for src, dst, online in ((1, 4, False), (2, 4, True)):
        S = dst // src
        n = 3 if src == 1 else 1
        pa = [Backend("gpu", engine, app_id=650 + src, pidx=src - 1 if src > 1 else 0) for _ in range(n)]
        pb = [Backend("gpu", engine, app_id=660 + src, pidx=src - 1 if src > 1 else 0) for _ in range(n)]
        ka = [[None if online and c == 0 else Backend("gpu", engine, app_id=670 + src, pidx=(src - 1) + c * src) for c in range(S)]
              for _ in range(n)]
        kb = [[None if online and c == 0 else Backend("gpu", engine, app_id=680 + src, pidx=(src - 1) + c * src) for c in range(S)]
              for _ in range(n)]
        try:
            ops = []
            for i in range(n):
                o = history(np.random.default_rng(40 + i), 800)
                o.append(("put", b"h001", b"mem%d" % i, b"in the memtable", 0))
                ops.append(o)
                for op in o:
                    apply(pa[i], op)
                    apply(pb[i], op)
            decrees = pgs.rrdb_split_many([b.h for b in pa], src, dst, [[k.h if k else None for k in row] for row in ka])
            one = [pgs.rrdb_split(pb[i].h, src, dst, [k.h if k else None for k in kb[i]]) for i in range(n)]
            assert decrees == one
            for i in range(n):
                keys = sorted({(op[1], op[2]) for op in ops[i] if op[0] != "flush"})
                for c in range(S):
                    a, b = ka[i][c], kb[i][c]
                    if a is None:
                        continue
                    for f in ("rrdb_last_committed_decree", "rrdb_last_flushed_decree", "rrdb_last_durable_decree"):
                        assert a.f(f)(a.h) == b.f(f)(b.h), (i, c, f)
                    ck = [k for k in keys if child_of(*k, src, dst) == c]
                    hks = sorted({hk for hk, _ in ck if hk})
                    same_reads(a, b, ck, hks)
                    # writes after the split: a child's write wins over every copied version on both sides
                    a.decree = b.decree = decrees[i]
                    more = [op for op in history(np.random.default_rng(90 + 7 * i + c), 200) if op[0] == "flush" or child_of(op[1], op[2], src, dst) == c]
                    for op in more:
                        apply(a, op)
                        apply(b, op)
                    ck2 = sorted(set(ck) | {(op[1], op[2]) for op in more if op[0] != "flush"})
                    same_reads(a, b, ck2, sorted({hk for hk, _ in ck2 if hk}))
        finally:
            for b in pa + pb + [k for row in ka + kb for k in row if k is not None]:
                b.close()


def test_rrdb_split_many_refusals(pgs, engine):
    p = Backend("gpu", engine, app_id=690, pidx=0)
    q = Backend("gpu", engine, app_id=691, pidx=0)
    kids = [Backend("gpu", engine, app_id=692, pidx=c) for c in range(2)]
    try:
        p.put(b"h", b"s", b"v", now=NOW)
        for parents, rows in (([p.h, p.h], [[kids[0].h, None], [None, kids[1].h]]),  # a parent given twice
                              ([p.h, q.h], [[None, kids[1].h], [None, kids[1].h]]),  # a child given twice
                              ([p.h], [[None, q.h]])):                               # a child with the wrong index
            with pytest.raises(pgs.PegasusError) as e:
                pgs.rrdb_split_many(parents, 1, 2, rows)
            assert e.value.code == pgs.INVALID_ARGUMENT
        assert all(k.f("rrdb_last_committed_decree")(k.h) == 0 for k in kids)
    finally:
        for b in [p, q] + kids:
            b.close()
