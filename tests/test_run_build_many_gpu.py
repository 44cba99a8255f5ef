"""pgs_run_build_many on the device: every job's run equals pgs_run_build of the same records in a twin partition (downloads,
run info but the id, point gets, forward and reverse batched scans); the call launches 2 * R + 7 kernels for 1 job as for 64;
every refusal launches nothing and changes no run list; a call whose values pass 4 GiB builds the per-partition runs.  The
replica layer: pgs_rrdb_flush_many against pgs_rrdb_flush on twin replicas."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

from incubator_pegasus_b200 import synth
from test_run_build_gpu import _gets, _same_run, _scans
from test_run_build_many_sim import job_records
from test_run_build_sim import INFO_FIELDS

pytestmark = pytest.mark.gpu
NOW = synth.NOW


def _launches_expected(n_records):
    return 2 * max(1, math.ceil(math.log2(n_records))) + 7


def test_64_jobs_equal_single_builds(pgs, engine):
    recs = job_records(pgs, 64, seed=21)
    recs[10] = synth.compaction_runs(k=1, n_per_run=20_000, seed=2)[0]
    many = [engine.partition(app_id=70, pidx=i) for i in range(64)]
    one = [engine.partition(app_id=71, pidx=i) for i in range(64)]
    try:
        ids = engine.build_many([(p, r, i % 3) for i, (p, r) in enumerate(zip(many, recs))])
        for i, r in enumerate(recs):
            want = one[i].build_records(r, i % 3)
            if r.n == 0:
                assert ids[i] == 0 and many[i].runs() == []
                continue
            assert many[i].runs() == [ids[i]]
            _same_run(many[i], ids[i], one[i], want)
            keys = [r.key(x) for x in range(0, r.n, max(1, r.n // 500))] + [b"\x00\x01zz-missing"]
            assert _gets(many[i], keys) == _gets(one[i], keys)
            if i % 4 == 2 or i == 10:
                assert _scans(pgs, many[i], r) == _scans(pgs, one[i], r)
        assert len(set(x for x in ids if x)) == sum(1 for r in recs if r.n)
    finally:
        for p in many + one:
            p.close()


def test_launches_do_not_depend_on_the_job_count(pgs, engine):
    base = synth.compaction_runs(k=1, n_per_run=64 * 300, seed=8)[0]
    items = base.to_list()
    split = [pgs.Records.from_list(items[i * 300:(i + 1) * 300]) for i in range(64)]
    for jobs_recs in ([base], split):
        parts = [engine.partition(app_id=72, pidx=i) for i in range(len(jobs_recs))]
        try:
            before = engine.launches
            engine.build_many([(p, r, 0) for p, r in zip(parts, jobs_recs)])
            assert engine.launches - before == _launches_expected(base.n), len(jobs_recs)
        finally:
            for p in parts:
                p.close()


def test_refusals_launch_nothing_and_change_no_run_list(pgs, engine):
    L = pgs.lib()
    parts = [engine.partition(app_id=73, pidx=i) for i in range(4)]
    other = pgs.Engine()
    foreign = other.partition(app_id=73, pidx=9)
    try:
        ok = [pgs.Records.from_list([(b"\x00\x01k%02d-%04d" % (i, x), 5, 1, b"v") for x in range(100)]) for i in range(4)]
        base = [p.build_records(r) for p, r in zip(parts, ok)]
        lists = [p.runs() for p in parts]

        def call(jobs, n=None):
            arr = (pgs.RunBuildJob * max(1, len(jobs)))(*jobs)
            ids = np.zeros(max(1, len(jobs)), np.uint64)
            before = engine.launches
            st = L.pgs_run_build_many(arr, len(jobs) if n is None else n, ids.ctypes.data_as(C.POINTER(C.c_uint64)))
            return st, engine.launches - before

        J = pgs.RunBuildJob.of
        no_part = J(None, ok[0])
        neg = J(parts[0], ok[0], -1)
        no_seq = J(parts[1], ok[1])
        no_seq.seq = None
        cases = [
            ([J(parts[0], ok[0]), no_part], pgs.INVALID_ARGUMENT),
            ([neg], pgs.INVALID_ARGUMENT),
            ([no_seq], pgs.INVALID_ARGUMENT),
            ([J(parts[0], ok[0]), J(parts[0], ok[1])], pgs.INVALID_ARGUMENT),  # one partition in two jobs
            ([J(parts[0], ok[0]), J(foreign, ok[1])], pgs.INVALID_ARGUMENT),  # another engine
        ]
        for jobs, want in cases:
            assert call(jobs) == (want, 0)
        st, launched = call([J(parts[0], ok[0])], n=4097)  # more jobs than one call takes
        assert (st, launched) == (pgs.NOT_SUPPORTED, 0)
        assert L.pgs_run_build_many(None, 3, None) == pgs.INVALID_ARGUMENT
        assert [p.runs() for p in parts] == lists
        # a device-found error in one job: no run list changes, and the same valid call then succeeds
        bad = pgs.Records.from_list(ok[2].to_list()[:50] + [(b"\x00\x01a", 5, 1, b"")] + ok[2].to_list()[50:])
        jobs = [(parts[0], ok[0], 1), (parts[1], ok[1], 1), (parts[2], bad, 1), (parts[3], ok[3], 1)]
        with pytest.raises(pgs.PegasusError) as e:
            engine.build_many(jobs)
        assert e.value.code == pgs.INVALID_ARGUMENT and "job 2" in str(e.value)
        assert [p.runs() for p in parts] == lists
        jobs[2] = (parts[2], ok[2], 1)
        ids = engine.build_many(jobs)
        assert [p.runs() for p in parts] == [lists[i] + [ids[i]] for i in range(4)]
        assert base == [x[0] for x in lists]
    finally:
        for p in parts + [foreign]:
            p.close()
        other.close()


def _digest(run):
    h = hashlib.sha256()
    for x in (run.data, run.blk_off, run.blk_size):
        h.update(x.tobytes())
    return h.hexdigest()


def test_values_past_4_gib(pgs, engine):
    """five jobs of 1 000 records with 1 MB values: 5 GB of values in one call"""
    rng = np.random.default_rng(4)
    chunk = rng.integers(0, 256, 1 << 26, np.uint8)
    recs = []
    for j in range(5):
        n = 1000
        vals = np.tile(np.roll(chunk, j), 16)[: n << 20]
        keys = np.frombuffer(b"".join(b"\x00\x02j%d-%06d" % (j, x) for x in range(n)), np.uint8).copy()
        klen = len(b"\x00\x02j0-000000")
        recs.append(pgs.Records(keys, np.arange(n + 1, dtype=np.uint64) * klen, vals, np.arange(n + 1, dtype=np.uint64) << 20,
                                np.arange(n, 0, -1).astype(np.uint64) + 10, np.ones(n, np.uint8)))
    assert sum(int(r.val_off[-1]) for r in recs) > 4 << 30
    parts = [engine.partition(app_id=74, pidx=i) for i in range(5)]
    try:
        ids = engine.build_many([(p, r, 0) for p, r in zip(parts, recs)])
        got = []
        for p, i in zip(parts, ids):
            got.append((_digest(p.download(i)), p.run_info(i)))
            p.drop(i)
        for j, (p, r) in enumerate(zip(parts, recs)):
            i = p.build_records(r)
            assert _digest(p.download(i)) == got[j][0], j
            info = p.run_info(i)
            assert all(getattr(info, f) == getattr(got[j][1], f) for f in INFO_FIELDS), j
            p.drop(i)
    finally:
        for p in parts:
            p.close()


def test_replicas_flush_many(pgs, engine):
    """replicas with puts, removes, TTLs and per-replica envs, some one flush below the L0 trigger: pgs_rrdb_flush_many
    against pgs_rrdb_flush on twin replicas"""
    from rrdb_harness import Backend, same_response

    n = 7
    envs = [{}, {"default_ttl": "500"}, {}, {"default_ttl": "40"}, {}, {}, {"default_ttl": "90"}]
    opts = {"l0_compaction_trigger": 3}
    multi = [Backend("gpu", engine, app_id=75, pidx=i, opts=opts) for i in range(n)]
    twin = [Backend("gpu", engine, app_id=76, pidx=i, opts=opts) for i in range(n)]
    L = pgs.lib()
    try:
        for i in range(n):
            rounds = i % 4  # flushes before the compared one: 0 to 3, so some replicas reach the trigger with it
            for be in (multi[i], twin[i]):
                be.update_envs(envs[i], NOW)
                r2 = np.random.default_rng(200 + i)
                for rd in range(rounds + 1):
                    for x in range(0 if i == 5 else 60):  # replica 5: an empty memtable
                        hk, sk = b"h%02d" % r2.integers(0, 8), b"s%04d" % r2.integers(0, 60)
                        u = r2.random()
                        if u < 0.15:
                            be.remove(hk, sk, now=NOW)
                        else:
                            ets = 0 if u < 0.6 else (NOW + 100 if u < 0.8 else NOW - 5)
                            be.put(hk, sk, b"v%d_%d" % (rd, x) * int(r2.integers(1, 40)), expire_ts=ets, now=NOW)
                    if rd < rounds:
                        be.flush(NOW)
        for be in twin:
            be.flush(NOW)
        handles = (C.c_void_p * n)(*[be.h.value for be in multi])
        assert L.pgs_rrdb_flush_many(handles, n, NOW) == 0
        compacted = 0
        for i in range(n):
            assert L.pgs_rrdb_last_flushed_decree(multi[i].h) == L.pgs_rrdb_last_flushed_decree(twin[i].h)
            pm = pgs.Partition(engine, 0, 0, 0, handle=L.pgs_rrdb_partition(multi[i].h))
            pt = pgs.Partition(engine, 0, 0, 0, handle=L.pgs_rrdb_partition(twin[i].h))
            rm, rt = pm.runs(), pt.runs()
            assert [pm.run_info(x).level for x in rm] == [pt.run_info(x).level for x in rt], i
            compacted += any(pm.run_info(x).level == 1 for x in rm)
            assert [pgs.decode_blocks(pm.download(x)).to_list() for x in rm] == [pgs.decode_blocks(pt.download(x)).to_list() for x in rt]
            for hk in (b"h%02d" % h for h in range(8)):
                for fn, a in (("multi_get", (hk,)), ("sortkey_count", (hk,)), ("get", (hk, b"s0007")), ("get", (hk, b"s0042"))):
                    rm_, rt_ = (dict(getattr(be, fn)(*a, now=NOW), app_id=0) for be in (multi[i], twin[i]))
                    ok, detail = same_response(rm_, rt_)
                    assert ok, (i, fn, a, detail)
                (km, _), (kt, _) = multi[i].scan_all(hk, now=NOW), twin[i].scan_all(hk, now=NOW)
                assert km == kt
        assert compacted >= 2
        # refusals: a replica twice, and a replica of another engine
        assert L.pgs_rrdb_flush_many((C.c_void_p * 2)(multi[0].h.value, multi[0].h.value), 2, NOW) == pgs.INVALID_ARGUMENT
        other = pgs.Engine()
        try:
            far = Backend("gpu", other, app_id=77, pidx=0, opts=opts)
            try:
                assert L.pgs_rrdb_flush_many((C.c_void_p * 2)(multi[0].h.value, far.h.value), 2, NOW) == pgs.INVALID_ARGUMENT
            finally:
                far.close()
        finally:
            other.close()
    finally:
        for be in multi + twin:
            be.close()
