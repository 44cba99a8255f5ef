"""pgs_compact_many on the device: every job's partition has a twin holding the same uploaded runs, the twins are compacted
one by one with pgs_compact_ex and the originals in one pgs_compact_many.  Both sides must hold the same records, counters
and run info (block layout aside) and answer every read the same way; the call launches as much for 1 job as for 64;
every refusal launches nothing and changes no run list.  The replica layer: pgs_rrdb_manual_compact_many against
pgs_rrdb_manual_compact on twin replicas."""
import ctypes as C

import numpy as np
import pytest

import compact_many_jobs as cm
from incubator_pegasus_b200 import synth
from test_scan_kernels_gpu import run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW
CMP_FIELDS = ("in_records", "out_records", "in_bytes", "out_bytes", "in_block_bytes", "dropped_shadowed", "dropped_tombstone",
              "dropped_expired", "dropped_user", "dropped_stale", "ttl_rewritten")
INFO_FIELDS = ("level", "n_records", "n_tombstones", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len",
               "smallest_seq", "largest_seq")


def job_kw(pgs, j):
    kw = dict(j["kw"])
    ops_json = kw.pop("ops_json", None)
    if ops_json:
        kw["ops"] = pgs.parse_ops(ops_json)
    return kw


def load(pgs, engine, jobs, app_id):
    """one partition per job holding its runs (the oldest uploaded first) -> [(partition, run ids)]"""
    out = []
    for i, j in enumerate(jobs):
        p = engine.partition(app_id=app_id, pidx=i)
        out.append((p, [p.upload_records(r) for r in j["runs"]]))
    return out


def records_of(pgs, part):
    ids = part.runs()
    assert len(ids) <= 1
    return pgs.decode_blocks(part.download(ids[0])).to_list() if ids else []


def all_keys(jobs_runs):
    keys = sorted({r.key(i) for r in jobs_runs for i in range(r.n)})
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    return np.frombuffer(b"".join(keys), np.uint8).copy() if keys else np.zeros(1, np.uint8), off


def reads(pgs, part, j):
    """every key through pgs_get_batch, and forward and reverse scans of the whole range and of a window"""
    keys, off = all_keys(j["runs"])
    st, res, arena, _ = part.get_batch(keys, off, NOW, arena_cap=64 << 20)
    assert st == 0
    gets = [(r.status, r.expire_ts, arena[r.value_off:r.value_off + r.value_len].tobytes() if r.status == 0 else b"")
            for r in res]
    full = dict(start=b"", stop=b"\xff" * 8, start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0,
                max_count=1 << 20, max_iter_count=1 << 20, max_iter_size=0, return_expire_ts=1)
    mid = keys[int(off[len(off) // 3]):int(off[len(off) // 3 + 1])].tobytes()
    reqs = [full, dict(full, reverse=1), dict(full, start=mid, max_count=40), dict(full, stop=mid, reverse=1, max_count=40)]
    st, ans = run_scans(pgs, part, reqs, arena_stride=8 << 20, kv_stride=1 << 14)
    assert st == 0
    return gets, ans


def compare(pgs, jobs, orig, twins, res_many, res_one, check_reads=True):
    for i, j in enumerate(jobs):
        (p, _), (t, _) = orig[i], twins[i]
        a, b = res_many[i], res_one[i]
        for f in CMP_FIELDS:
            assert getattr(a, f) == getattr(b, f), (i, f, getattr(a, f), getattr(b, f))
        assert records_of(pgs, p) == records_of(pgs, t), i
        assert (a.new_run_id != 0) == (b.new_run_id != 0), i
        if a.new_run_id:
            ia, ib = p.run_info(a.new_run_id), t.run_info(b.new_run_id)
            for f in INFO_FIELDS:
                assert getattr(ia, f) == getattr(ib, f), (i, f)
            assert a.out_block_bytes == ia.data_bytes
        if check_reads:
            assert reads(pgs, p, j) == reads(pgs, t, j), i


def run_mix(pgs, engine, jobs, app):
    orig, twins = load(pgs, engine, jobs, app), load(pgs, engine, jobs, app + 1)
    res_one = [t.compact(ids, out_level=1, bottommost=1 if j["bottommost"] else 0, now=NOW, **job_kw(pgs, j))
               for (t, ids), j in zip(twins, jobs)]
    before = engine.launches
    res_many = engine.compact_many([(p, ids, 1, 1 if j["bottommost"] else 0, job_kw(pgs, j)) for (p, ids), j in zip(orig, jobs)], NOW)
    assert engine.launches - before == 6
    assert all(r.n_launches == 6 for r in res_many)
    return orig, twins, res_many, res_one


def close_all(*groups):
    for g in groups:
        for p, _ in g:
            p.close()


def test_mix_matches_one_by_one(pgs, engine):
    jobs = cm.mix_main(scale=4)
    orig, twins, res_many, res_one = run_mix(pgs, engine, jobs, 500)
    try:
        compare(pgs, jobs, orig, twins, res_many, res_one)
        assert res_many[4].new_run_id == 0 and orig[4][0].runs() == []  # the job whose output is empty
    finally:
        close_all(orig, twins)


def test_long_keys_widen_every_job(pgs, engine):
    jobs = cm.mix_long_keys()
    orig, twins, res_many, res_one = run_mix(pgs, engine, jobs, 510)
    try:
        compare(pgs, jobs, orig, twins, res_many, res_one)
    finally:
        close_all(orig, twins)


@pytest.mark.parametrize("n", [1, 64])
def test_launches_do_not_grow_with_jobs(pgs, engine, n):
    """64 partitions of several runs each (bottommost derived per partition) cost the six launches of one"""
    jobs = [cm.job(synth.compaction_runs(k=1 + i % 5, n_per_run=200, seed=100 + i), True, default_ttl=(i % 3) * 100,
                   validate_hash=i % 2 == 1, pidx=i % 4, partition_version=3) for i in range(n)]
    orig, twins = load(pgs, engine, jobs, 520), load(pgs, engine, jobs, 521)
    try:
        res_one = [t.compact(ids, out_level=2, bottommost=-1, now=NOW, **job_kw(pgs, j)) for (t, ids), j in zip(twins, jobs)]
        before = engine.launches
        res_many = engine.compact_many([(p, ids, 2, -1, job_kw(pgs, j)) for (p, ids), j in zip(orig, jobs)], NOW)
        assert engine.launches - before == 6
        compare(pgs, jobs, orig, twins, res_many, res_one, check_reads=n == 1)
    finally:
        close_all(orig, twins)


def test_keep_inputs_and_discard_output_leave_the_partitions(pgs, engine):
    jobs = cm.mix_main()
    orig = load(pgs, engine, jobs, 530)
    try:
        lists = [p.runs() for p, _ in orig]
        keep_inputs_discard_output = 3  # PGS_COMPACT_KEEP_INPUTS | PGS_COMPACT_DISCARD_OUTPUT
        res = engine.compact_many([(p, ids, 1, 1, job_kw(pgs, j)) for (p, ids), j in zip(orig, jobs)], NOW,
                                  flags=keep_inputs_discard_output)
        assert [p.runs() for p, _ in orig] == lists
        assert sum(r.out_records for r in res) > 0
    finally:
        close_all(orig)


def test_refusals_launch_nothing(pgs, engine):
    jobs = cm.mix_main()
    orig = load(pgs, engine, jobs[:3], 540)
    other = pgs.Engine()
    try:
        lists = [p.runs() for p, _ in orig]
        good = [(p, ids, 1, 1, job_kw(pgs, j)) for (p, ids), j in zip(orig, jobs)]
        L = pgs.lib()

        def refused(job_list, code, n=None):
            before = engine.launches
            arr = (pgs.CompactJob * max(1, len(job_list)))()
            keep = []
            for i, (p, ids, lvl, bot, kw) in enumerate(job_list):
                a = np.array(ids, np.uint64)
                fp = pgs._filter_params(**kw)
                keep += [a, fp]
                arr[i] = pgs.CompactJob(p.h.value, a.ctypes.data_as(C.POINTER(C.c_uint64)), len(ids), lvl, bot, C.pointer(fp))
            res = (pgs.CompactResult * max(1, len(job_list)))()
            st = L.pgs_compact_many(arr, len(job_list) if n is None else n, NOW, 0, res)
            assert st == code, (st, L.pgs_last_error())
            assert engine.launches == before
            assert [p.runs() for p, _ in orig] == lists

        assert L.pgs_compact_many(None, 3, NOW, 0, None) == pgs.INVALID_ARGUMENT
        before = engine.launches
        assert L.pgs_compact_many(None, 0, NOW, 0, None) == 0 and engine.launches == before  # n == 0
        p0, ids0, *_ = good[0]
        refused([good[0], (good[1][0], good[1][1], -1, 1, {})], pgs.INVALID_ARGUMENT)          # negative level
        refused([good[0], (good[1][0], [], 1, 1, {})], pgs.INVALID_ARGUMENT)                    # k == 0
        refused([good[0], good[1], (p0, ids0, 1, 1, {})], pgs.INVALID_ARGUMENT)                 # a partition twice
        stranger = other.partition(app_id=9, pidx=0)
        sid = stranger.upload_records(jobs[0]["runs"][0])
        refused([good[0], (stranger, [sid], 1, 1, {})], pgs.INVALID_ARGUMENT)                  # another engine
        refused([good[0], (good[1][0], [good[1][1][0], 987654321], 1, 1, {})], pgs.NOT_FOUND)  # an unknown run
        bad_ops = np.array([5, 0, 0, 0, 1, 2, 3], np.uint8)
        refused([good[0], (good[1][0], good[1][1], 1, 1, dict(ops=bad_ops))], pgs.INVALID_ARGUMENT)  # a malformed ops table
        deep = engine.partition(app_id=541, pidx=0)
        dids = [deep.upload_records(r) for r in synth.compaction_runs(k=17, n_per_run=5, seed=7)]
        refused([good[0], (deep, dids, 1, 1, {})], pgs.NOT_SUPPORTED)                           # 17 runs
        refused(good, pgs.NOT_SUPPORTED, n=5000)  # more jobs than one call takes (checked before the job array is read)
        wide = load(pgs, engine, cm.mix_too_wide(), 542)
        refused([(p, ids, 1, 1, {}) for p, ids in wide], pgs.NOT_SUPPORTED)                    # joint geometry
        close_all(wide)
        deep.close()
        stranger.close()
    finally:
        close_all(orig)
        other.close()


def test_replicas_manual_compact_many(pgs, engine):
    """replicas with puts, removes, TTLs and per-replica envs, one with more than 16 runs: pgs_rrdb_manual_compact_many
    against pgs_rrdb_manual_compact on twin replicas"""
    from rrdb_harness import Backend, same_response

    n = 5
    envs = [{}, {"default_ttl": "500"}, {"user_specified_compaction": cm.OPS_DELETE}, {"default_ttl": "40"}, {}]
    opts = {"l0_compaction_trigger": 1000}
    multi = [Backend("gpu", engine, app_id=60, pidx=i, opts=opts) for i in range(n)]
    twin = [Backend("gpu", engine, app_id=61, pidx=i, opts=opts) for i in range(n)]
    try:
        for i in range(n):
            rounds = 20 if i == 4 else 3  # replica 4: 20 flushed runs, a stack deeper than one merge
            for be in (multi[i], twin[i]):
                be.update_envs(envs[i], NOW)
                r2 = np.random.default_rng(100 + i)
                for rd in range(rounds):
                    for x in range(40):
                        hk, sk = b"h%02d" % r2.integers(0, 8), b"s%04d" % r2.integers(0, 60)
                        u = r2.random()
                        if u < 0.15:
                            be.remove(hk, sk, now=NOW)
                        else:
                            ets = 0 if u < 0.6 else (NOW + 100 if u < 0.8 else NOW - 5)
                            be.put(hk, sk, b"v%d_%d" % (rd, x), expire_ts=ets, now=NOW)
                    if rd + 1 < rounds:
                        be.flush(NOW)
        for be in twin:
            assert be.manual_compact(NOW) == 0
        handles = (C.c_void_p * n)(*[be.h.value for be in multi])
        res = (pgs.CompactResult * n)()
        assert pgs.lib().pgs_rrdb_manual_compact_many(handles, n, NOW, res) == 0
        L = pgs.lib()
        for i in range(n):
            pm = pgs.Partition(engine, 0, 0, 0, handle=L.pgs_rrdb_partition(multi[i].h))
            pt = pgs.Partition(engine, 0, 0, 0, handle=L.pgs_rrdb_partition(twin[i].h))
            rm, rt = pm.runs(), pt.runs()
            assert len(rm) == len(rt) == 1, (i, rm, rt)
            assert pm.run_info(rm[0]).level == pt.run_info(rt[0]).level
            assert res[i].out_records == pm.run_info(rm[0]).n_records
            for hk in (b"h%02d" % h for h in range(8)):
                for fn, a in (("multi_get", (hk,)), ("sortkey_count", (hk,)), ("get", (hk, b"s0007")), ("get", (hk, b"s0042"))):
                    rm_, rt_ = (dict(getattr(be, fn)(*a, now=NOW), app_id=0) for be in (multi[i], twin[i]))  # twins: app 60 / 61
                    ok, detail = same_response(rm_, rt_)
                    assert ok, (i, fn, a, detail)
                (km, _), (kt, _) = multi[i].scan_all(hk, now=NOW), twin[i].scan_all(hk, now=NOW)
                assert km == kt
        # manual_compact_last_finish_ms is set: a `once` trigger older than the compaction does not fire again
        trig = str(NOW + 1451606400 - 5)
        for i in range(n):
            for be in (multi[i], twin[i]):
                be.put(b"late", b"x", b"v", now=NOW)
                be.flush(NOW)
                be.update_envs(dict(envs[i], **{"manual_compact.once.trigger_time": trig}), NOW)
                part = pgs.Partition(engine, 0, 0, 0, handle=L.pgs_rrdb_partition(be.h))
                assert len(part.runs()) == 2, i
    finally:
        for be in multi + twin:
            be.close()
