"""pgs_run_build_many's kernels (build_kernels.cuh: k_build_*_many, index_kernel.cuh: k_index_walk_many) inside the host SIMT
interpreter, planned and launched through the library's build_many_* and index_launch_many functions.  Every job's run equals
the single-run build of the same records (sim_run_build) and the host builder's (pgs.build_run) byte for byte, and so does its
pgs_run_info.  A device-found error gives the status pgs_run_build gives that job, and the call returns the lowest failing job's.

The file also passes against the AddressSanitizer build of the simulator:

    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_run_build_many_sim.py
    bash tools/simt/build.sh"""
import ctypes as C
import random

import numpy as np
import pytest

from test_run_build_sim import INFO_FIELDS, _sorted, bsim, sim_build, upload_status  # noqa: F401  (bsim is a fixture)

vp = C.c_void_p


@pytest.fixture(scope="module")
def msim(pgs, bsim):  # noqa: F811
    bsim.sim_run_build_many.argtypes = [C.POINTER(pgs.RunBuildJob), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
    bsim.sim_run_build_many_info.argtypes = [C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), vp]
    bsim.sim_run_build_many_copy.argtypes = [C.c_uint32, vp, vp, vp]
    return bsim


def build_many(pgs, msim, recs_list, block_size, ri, grid_cap=4):
    """-> (status, failed job, [(BlockRun, RunInfo)] per job or None)"""
    arr = (pgs.RunBuildJob * len(recs_list))(*[pgs.RunBuildJob.of(None, r) for r in recs_list])
    failed = C.c_uint32()
    st = msim.sim_run_build_many(arr, len(recs_list), block_size, ri, grid_cap, C.byref(failed))
    if st:
        return st, failed.value, None
    out = []
    for j in range(len(recs_list)):
        nbytes, nb, info = C.c_uint64(), C.c_uint32(), pgs.RunInfo()
        msim.sim_run_build_many_info(j, C.byref(nbytes), C.byref(nb), C.byref(info))
        data, off, size = np.zeros(nbytes.value, np.uint8), np.zeros(nb.value, np.uint64), np.zeros(nb.value, np.uint32)
        msim.sim_run_build_many_copy(j, data.ctypes.data, off.ctypes.data, size.ctypes.data)
        out.append((pgs.BlockRun(data, off, size), info))
    return st, failed.value, out


def shifted(pgs, recs, pad):
    """the same records with `pad` bytes in front of the first key and value (key_off[0] = val_off[0] = pad)"""
    return pgs.Records(np.concatenate([np.full(pad, 0xAB, np.uint8), recs.keys]), recs.key_off + np.uint64(pad),
                       np.concatenate([np.full(pad, 0xCD, np.uint8), recs.vals]), recs.val_off + np.uint64(pad), recs.seq, recs.type)


def job_records(pgs, n_jobs, seed):
    """jobs of 0, 1, a few and a few hundred records; keys drawn from one space, so a job's first key often sorts below the
    previous job's last key; every fifth job's offsets start past 0"""
    rng = random.Random(seed)
    out = []
    for j in range(n_jobs):
        n = rng.choice([0, 1, 3, 40, 250]) if j else 250
        items = [(b"\x00\x02k%05d" % rng.randrange(3000) + rng.randbytes(rng.randrange(0, 20)), rng.randrange(1, 1 << 40),
                  rng.choice([0, 1, 1]), rng.randbytes(rng.choice([0, 5, 60, 900, 5000]))) for _ in range(n)]
        recs = pgs.Records.from_list(_sorted(items))
        out.append(shifted(pgs, recs, 3 + j) if j % 5 == 4 and recs.n else recs)
    return out


def check_jobs(pgs, msim, recs_list, bs, ri, grid_cap=4):
    st, _, got = build_many(pgs, msim, recs_list, bs, ri, grid_cap)
    assert st == 0
    for j, recs in enumerate(recs_list):
        run, info = got[j]
        if recs.n == 0:
            assert run.n_blocks == 0
            continue
        st1, one, info1 = sim_build(pgs, msim, recs, bs, ri, grid_cap)
        want_st, want, want_info = upload_status(pgs, msim, recs, bs, ri)
        assert st1 == want_st == 0
        for ref, ref_info in ((one, info1), (want, want_info)):
            assert np.array_equal(run.blk_off, ref.blk_off) and np.array_equal(run.blk_size, ref.blk_size), j
            assert run.data.shape == ref.data.shape and np.array_equal(run.data, ref.data), j
            for f in INFO_FIELDS:
                assert getattr(info, f) == getattr(ref_info, f), (j, f)


@pytest.mark.parametrize("bs,ri", [(4096, 16), (512, 2), (16384, 1)])
@pytest.mark.parametrize("n_jobs", [1, 2, 17, 64])
def test_jobs_equal_single_builds(pgs, msim, bs, ri, n_jobs):
    check_jobs(pgs, msim, job_records(pgs, n_jobs, seed=n_jobs * 7 + bs + ri), bs, ri)


def test_one_thread_per_record_grids(pgs, msim):
    """the product's grids as well as the capped grids of the other tests"""
    check_jobs(pgs, msim, job_records(pgs, 9, seed=5), 512, 2, grid_cap=0)


def test_only_empty_jobs(pgs, msim):
    st, _, got = build_many(pgs, msim, [pgs.Records.from_list([])] * 3, 4096, 16)
    assert st == 0 and all(run.n_blocks == 0 for run, _ in got)


def _ok(i):
    return [(b"\x00\x01j%02d-%04d" % (i, x), 5, 1, b"v") for x in range(30)]


def test_order_error_in_one_job(pgs, msim):
    jobs = [_ok(i) for i in range(9)]
    jobs[5] = jobs[5][:10] + [(b"\x00\x01a", 5, 1, b"")] + jobs[5][10:]
    st, failed, _ = build_many(pgs, msim, [pgs.Records.from_list(j) for j in jobs], 4096, 16)
    assert (st, failed) == (pgs.INVALID_ARGUMENT, 5)


def test_lowest_failing_job_wins(pgs, msim):
    """a long key in job 3 (kNotSupported) and an order error in job 7 (kInvalidArgument): job 3's status"""
    jobs = [_ok(i) for i in range(9)]
    jobs[3] = jobs[3][:4] + [(jobs[3][3][0] + bytes(4096), 5, 1, b"")] + jobs[3][4:]
    jobs[7] = jobs[7][:1] + [(jobs[7][0][0], 6, 1, b"")] + jobs[7][1:]  # an ascending trailer
    st, failed, _ = build_many(pgs, msim, [pgs.Records.from_list(j) for j in jobs], 512, 2)
    assert (st, failed) == (pgs.NOT_SUPPORTED, 3)


def test_bad_offsets_checked_inside_the_job(pgs, msim):
    """a record whose key ends past its own job's keys is refused, though the next job's bytes lie behind them"""
    jobs = [pgs.Records.from_list(_ok(i)) for i in range(3)]
    jobs[1].key_off[15] = jobs[1].key_off[30] + np.uint64(5)  # record 14 ends 5 bytes past the job's keys
    st, failed, _ = build_many(pgs, msim, jobs, 4096, 16)
    assert (st, failed) == (pgs.INVALID_ARGUMENT, 1)
