"""The multi-job split (split_kernels.cuh: k_plan_many, k_seg_bounds_many, k_seg_layout_many, k_split_walk_many<count /
write>, then k_seg_scan_many and k_emit_many over every built child) inside the host SIMT interpreter, through
split_many_plan / split_many_buffers / split_many_child / split_many_launch as pgs_partition_split_many runs them.  Several
parents -- builder runs, foreign_blocks runs, tombstones and empty writes, a parent of 2 KB keys that widens every job's key
rows -- are split together; every child equals tests/split_model.py record for record and the single-run split of the same
run in its records and counters, its pgs_run_info, index and Bloom filter match its own blocks, and foreign_blocks.classify
accepts it.

The file also passes against the AddressSanitizer build of the simulator:

    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_split_many_sim.py
    bash tools/simt/build.sh"""
import ctypes as C

import numpy as np
import pytest

import foreign_blocks as fb
import merge_inputs
import split_model as sm
from test_split_sim import INFO_FIELDS, _mixed, sim_split, ssim  # noqa: F401  (ssim: the simulator fixture)

LAUNCHES = 7
# the pgs_run_info fields that do not depend on where blocks are cut
RECORD_FIELDS = ("n_records", "n_tombstones", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len", "smallest_seq",
                 "largest_seq")


@pytest.fixture(scope="module")
def msim(ssim):
    ssim.sim_split_many.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                    C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint32)]
    ssim.sim_split_many_select.argtypes = [C.c_uint32]
    return ssim


def _children(pgs, ssim, S):
    """the children sim_split_child_* read: {child: BlockRun + index arrays + info}"""
    out = {}
    for c in range(S):
        info, q, kb = pgs.RunInfo(), C.c_uint32(), C.c_uint64()
        if not ssim.sim_split_child_info(c, C.byref(info), C.byref(q), C.byref(kb)):
            continue
        nb = info.n_blocks
        data, off, size = np.zeros(info.data_bytes, np.uint8), np.zeros(nb + 1, np.uint64), np.zeros(nb, np.uint32)
        blk_rec, ikey_off, ikeys = np.zeros(nb + 1, np.uint32), np.zeros(nb + 1, np.uint32), np.zeros(kb.value + 1, np.uint8)
        ssim.sim_split_child_copy(c, data.ctypes.data, off.ctypes.data, size.ctypes.data, blk_rec.ctypes.data, ikey_off.ctypes.data,
                                  ikeys.ctypes.data)
        out[c] = dict(run=pgs.BlockRun(data, off[:nb].copy(), size), info=info, blk_rec=blk_rec, ikey_off=ikey_off,
                      ikeys=ikeys[:kb.value], segments=q.value)
    return out


def sim_split_many(pgs, ssim, runs, wants, src, dst, seg_weight=0, block_size=4096, restart_interval=16):
    """-> (status, [per run: {child: ...}], [per run: dropped], launches)"""
    n = len(runs)
    ptrs = lambda xs: (C.c_void_p * max(1, n))(*xs)  # noqa: E731
    data = ptrs([r.data.ctypes.data for r in runs])
    nbytes = np.array([r.data.shape[0] for r in runs], np.uint64)
    off = ptrs([r.blk_off.ctypes.data for r in runs])
    size = ptrs([r.blk_size.ctypes.data for r in runs])
    nblk = np.array([r.n_blocks for r in runs], np.uint32)
    want = np.array(wants, np.uint32)
    dropped = np.zeros(max(1, n), np.uint64)
    launches = C.c_uint32()
    st = ssim.sim_split_many(n, data, nbytes.ctypes.data, off, size, nblk.ctypes.data, want.ctypes.data, block_size, restart_interval, src,
                             dst, seg_weight, dropped.ctypes.data, C.byref(launches))
    if st:
        return st, [], [], launches.value
    got = []
    for i in range(n):
        assert ssim.sim_split_many_select(i) == 0
        got.append(_children(pgs, ssim, dst // src))
    return st, got, [int(x) for x in dropped[:n]], launches.value


def check_child(ssim, x, items, c):
    """child x (of the selected run) holds exactly `items`; its info, index and filter match its blocks"""
    run = x["run"]
    assert fb.classify(run) == fb.OK, c
    recs = fb.decode(run)
    assert recs.to_list() == items, c
    m = fb.model_index(run)
    assert x["blk_rec"].tolist() == m["blk_rec"] and x["ikey_off"].tolist() == m["ikey_off"] and x["ikeys"].tobytes() == m["ikeys"]
    for f in INFO_FIELDS:
        assert getattr(x["info"], f) == m["info"][f], (c, f, getattr(x["info"], f), m["info"][f])
    for k, _s, _t, _v in items:
        assert ssim.sim_split_child_bloom_check(c, k, len(k)), (c, k)
        pl = 2 + int.from_bytes(k[:2], "big") if len(k) >= 2 else 0
        if 2 < pl <= len(k):
            assert ssim.sim_split_child_bloom_check(c, k[:pl], pl), (c, k[:pl])


def _long_key_run(pgs):
    recs = merge_inputs.long_keys(3)[0]
    return pgs.build_run(recs, 4096, 16)


def _parents(pgs):
    """parent -> its runs (BlockRun, records): builder runs, foreign_blocks runs of several encodings, a parent of 2 KB keys,
    and a parent without runs"""
    P = []
    P.append([pgs.build_run(pgs.Records.from_list(_mixed(s, 300)), 4096, 16) for s in (1, 2, 3)])
    foreign = []
    for i, policy in enumerate(list(fb.GRID)[:3]):
        recs = pgs.Records.from_list(_mixed(10 + i, 250))
        foreign.append(fb.encode_run(recs, seed=i, **fb.GRID[policy]))
    P.append(foreign)
    P.append([pgs.build_run(pgs.Records.from_list(_mixed(20, 400)), 16384, 1)])
    P.append([_long_key_run(pgs)])
    P.append([])
    return P


@pytest.mark.parametrize("src,dst", [(1, 2), (2, 8), (1, 8), (1, 32)])
def test_sim_split_many_matches_model_and_single(pgs, msim, src, dst):
    S = dst // src
    parents = _parents(pgs)
    full = (1 << S) - 1
    # some children are not built: the online split's parent half (child 0), and one more in another parent
    pwant = [full, full & ~1, full & ~(1 << (S - 1)), full, full]
    runs, wants = [], []
    for p, rs in enumerate(parents):
        for r in rs:
            runs.append(r)
            wants.append(pwant[p])
    st, got, dropped, launches = sim_split_many(pgs, msim, runs, wants, src, dst, seg_weight=3000)
    assert st == 0 and launches == LAUNCHES
    for i, (r, want) in enumerate(zip(runs, wants)):
        items = fb.decode(r).to_list()
        parts, want_dropped = sm.split_items(items, src, dst)
        assert dropped[i] == want_dropped
        st1, single, dropped1 = sim_split(pgs, msim, r, src, dst, want, seg_weight=3000)
        assert st1 == 0 and dropped1 == dropped[i]
        assert msim.sim_split_many_select(i) == 0
        for c in range(S):
            built = (want >> c) & 1 and parts[c]
            assert (c in got[i]) == bool(built), (i, c)
            assert (c in single) == bool(built), (i, c)
            if not built:
                continue
            check_child(msim, got[i][c], parts[c], c)
            assert fb.decode(got[i][c]["run"]).to_list() == fb.decode(single[c]["run"]).to_list()
            for f in RECORD_FIELDS:
                assert getattr(got[i][c]["info"], f) == getattr(single[c]["info"], f), (i, c, f)
    # segments of different parents meet in one warp's tickets: many segments per run, several runs
    assert sum(max((x["segments"] for x in g.values()), default=0) for g in got) > 20


def test_sim_split_many_one_job_is_the_single_launch(pgs, msim):
    """with one job the joint plan is the single plan: the children are byte for byte sim_split's"""
    br = pgs.build_run(pgs.Records.from_list(_mixed(7, 500)), 4096, 16)
    for dst, want, w in [(4, 0b1111, 0), (8, 0b10110110, 2500)]:
        st, got, dropped, launches = sim_split_many(pgs, msim, [br], [want], 1, dst, seg_weight=w)
        st1, single, dropped1 = sim_split(pgs, msim, br, 1, dst, want, seg_weight=w)
        assert st == 0 and st1 == 0 and dropped == [dropped1] and launches == LAUNCHES
        assert sorted(got[0]) == sorted(single)
        for c, x in single.items():
            y = got[0][c]
            assert np.array_equal(x["run"].data, y["run"].data) and np.array_equal(x["run"].blk_off, y["run"].blk_off)
            assert x["segments"] == y["segments"]
            for f in INFO_FIELDS:
                assert getattr(x["info"], f) == getattr(y["info"], f), (c, f)


def test_sim_split_many_no_child_record(pgs, msim):
    """runs whose records all go to children that are not built: the counting phase only"""
    items = [it for it in _mixed(4, 200) if it[0] and sm.child_of(it[0], 1, 2) == 1]
    br = pgs.build_run(pgs.Records.from_list(items))
    st, got, dropped, launches = sim_split_many(pgs, msim, [br, br], [0b01, 0b01], 1, 2)
    assert st == 0 and launches == 4 and got == [{}, {}] and dropped == [0, 0]


def test_sim_split_many_refusals(pgs, msim):
    br = pgs.build_run(pgs.Records.from_list(_mixed(1, 20)))
    # more child runs than one launch takes: 129 parent runs into 32 built children each
    st, *_ = sim_split_many(pgs, msim, [br] * 129, [0xFFFFFFFF] * 129, 1, 32)
    assert st == pgs.NOT_SUPPORTED
    # a joint plan over more parent runs than one launch plans, though no child is built
    one = pgs.build_run(pgs.Records.from_list(_mixed(2, 1)))
    st, *_ = sim_split_many(pgs, msim, [one] * 4097, [0] * 4097, 1, 2)
    assert st == pgs.NOT_SUPPORTED
    # more children than a split has
    st, *_ = sim_split_many(pgs, msim, [br], [1], 1, 64)
    assert st == pgs.NOT_SUPPORTED
