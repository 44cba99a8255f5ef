"""The multi-job compaction kernels (k_plan_many ... k_emit_many of csrc/compact_kernels.cuh) in the kernel simulator: several
jobs planned and launched together through compact_many_geometry / compact_launch_many, with a small segment weight so that
segments of different jobs meet in one warp's tickets.  Every job's output is compared with the oracle's merge of that job's
runs and with the single-job launch (sim_compact) of the same runs: the same records and counters."""
import ctypes as C

import numpy as np
import pytest

import compact_many_jobs as cm
from incubator_pegasus_b200 import synth
from test_kernel_sim import STAT_FIELDS, check, sim  # noqa: F401  (sim is a fixture)

# sim_result_stats fields that do not depend on where blocks are cut (15, 16: largest block and its records, 19: index keys)
SAME_STATS = list(range(15)) + [17, 18]


def read_result(pgs, sim):
    """the run sim_result_* read: (BlockRun, stats)"""
    db, nblk, nseg = C.c_uint64(), C.c_uint32(), C.c_uint32()
    sim.sim_result_sizes(C.byref(db), C.byref(nblk), C.byref(nseg))
    n = nblk.value
    out = pgs.BlockRun(np.zeros(db.value + 16, np.uint8), np.zeros(n + 1, np.uint64), np.zeros(n, np.uint32))
    stats = (C.c_uint64 * 20)()
    sim.sim_result_stats(stats)
    sim.sim_result_copy(out.data.ctypes.data_as(C.c_void_p), out.blk_off.ctypes.data_as(C.c_void_p), out.blk_size.ctypes.data_as(C.c_void_p),
                        None, None, None, None)
    out.blk_off = out.blk_off[:n].copy()
    return out, list(stats), nseg.value


def sim_compact_many(pgs, sim, jobs, *, lanes=0, seg_weight=0, block_size=4096, restart_interval=16, now=synth.NOW, status=0):
    """every job through one sim_compact_many; returns [(BlockRun, stats, segments)] per job and the launch count"""
    brs = [[pgs.build_run(r, block_size, restart_interval) for r in j["runs"]] for j in jobs]
    flat = [b for bs in brs for b in bs]
    t = len(flat)
    data = (C.c_void_p * t)(*[b.data.ctypes.data for b in flat])
    nbytes = (C.c_uint64 * t)(*[b.data.shape[0] for b in flat])
    off = (C.c_void_p * t)(*[b.blk_off.ctypes.data for b in flat])
    size = (C.c_void_p * t)(*[b.blk_size.ctypes.data for b in flat])
    nb = (C.c_uint32 * t)(*[b.n_blocks for b in flat])
    n = len(jobs)
    k = (C.c_uint32 * n)(*[len(bs) for bs in brs])
    bottom = (C.c_int32 * n)(*[1 if j["bottommost"] else 0 for j in jobs])
    fps = (pgs.FilterParams * n)()
    keep = []
    for i, j in enumerate(jobs):
        kw = dict(j["kw"])
        ops_json = kw.pop("ops_json", None)
        fp = pgs._filter_params(ops=pgs.parse_ops(ops_json) if ops_json else None, **kw)
        keep.append(fp)
        fps[i] = fp
    launches = C.c_uint32()
    st = sim.sim_compact_many(n, k, data, nbytes, off, size, nb, block_size, restart_interval, bottom, fps, now, lanes,
                              C.c_uint64(seg_weight), C.byref(launches))
    assert st == status, st
    if st:
        return None, launches.value
    out = []
    for i in range(n):
        assert sim.sim_compact_many_select(i) == 0
        out.append(read_result(pgs, sim))
    return out, launches.value


def check_mix(pgs, oracle, sim, jobs, *, lanes, seg_weight):
    got, launches = sim_compact_many(pgs, sim, jobs, lanes=lanes, seg_weight=seg_weight)
    assert launches == 6
    for i, j in enumerate(jobs):
        kw = dict(j["kw"])
        # the single-job launch of the same runs, checked against the oracle (records, counters, run format)
        want = check(pgs, oracle, sim, j["runs"], bottommost=j["bottommost"], lanes=lanes, seg_weight=seg_weight, **kw)
        run, stats, nseg = got[i]
        assert nseg >= 1
        assert [stats[x] for x in SAME_STATS] == [want["stats"][x] for x in SAME_STATS], i
        if not want["got"]:
            assert run.n_blocks == 0, i
            continue
        recs = pgs.decode_blocks(run)
        assert recs.to_list() == want["got"], i
        assert recs.same_as(oracle.Run.from_blocks(run).records())  # the oracle's own decoder of the raw blocks
        assert sim.sim_compact_many_select(i) == 0  # (check ran sim_compact since)
        for key in {r[0] for r in want["got"]}:  # every surviving key is in the job's own Bloom filter
            assert sim.sim_result_bloom_check(key, len(key)) == 1, i


@pytest.mark.parametrize("lanes", [1, 8])
def test_many_jobs_match_each_job_alone(pgs, oracle, sim, lanes):
    """pidx / partition_version with validate_hash, default_ttl and ops tables per job, bottommost 0 and 1, one run and 16
    runs, an empty output: 4 KB segments, so that a warp's tickets cross from one job into the next"""
    check_mix(pgs, oracle, sim, cm.mix_main(), lanes=lanes, seg_weight=4096)


def test_long_keys_widen_every_job(pgs, oracle, sim):
    """one job of 2 KB keys sizes the key rows of all of them"""
    check_mix(pgs, oracle, sim, cm.mix_long_keys(), lanes=0, seg_weight=8192)


def test_joint_geometry_that_does_not_fit(pgs, sim):
    """a 16-run job next to a job of 2 KB keys: PGS_NOT_SUPPORTED, while each fits a launch of its own"""
    jobs = cm.mix_too_wide()
    sim_compact_many(pgs, sim, jobs, status=pgs.NOT_SUPPORTED)
    for j in jobs:
        got, _ = sim_compact_many(pgs, sim, [j])
        assert got[0][1][1] > 0


def test_one_job_is_the_single_launch(pgs, oracle, sim):
    """n == 1 plans exactly what sim_compact plans: the same segments and the same blocks, byte for byte"""
    j = cm.mix_main()[0]
    got, _ = sim_compact_many(pgs, sim, [j], lanes=4, seg_weight=8192)
    want = check(pgs, oracle, sim, j["runs"], bottommost=j["bottommost"], lanes=4, seg_weight=8192, **j["kw"])
    run, stats, nseg = got[0]
    assert nseg == want["nseg"]
    assert stats == want["stats"]
    assert pgs.decode_blocks(run).to_list() == want["got"]


def test_bad_jobs_are_refused(pgs, sim):
    """a job of no runs, or of more runs than one merge takes"""
    j = cm.mix_main()[0]
    sim_compact_many(pgs, sim, [j, dict(j, runs=[])], status=pgs.INVALID_ARGUMENT)
    many = synth.compaction_runs(k=17, n_per_run=5, seed=3)
    sim_compact_many(pgs, sim, [j, dict(j, runs=many)], status=pgs.NOT_SUPPORTED)
