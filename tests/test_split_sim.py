"""The partition split kernels (split_kernels.cuh: k_split_walk's counting and writing passes, then k_seg_scan and k_emit per
child) inside the host SIMT interpreter, through split_plan / split_buffers / split_child / split_launch as
pgs_partition_split runs them.  Each child equals tests/split_model.py record for record; its reported pgs_run_info, index
and Bloom filter match its own blocks, and foreign_blocks.classify accepts them.

The file also passes against the AddressSanitizer build of the simulator:

    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_split_sim.py
    bash tools/simt/build.sh"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import foreign_blocks as fb
import merge_inputs
import split_model as sm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM_DIR = os.path.join(ROOT, "tools", "simt")


@pytest.fixture(scope="module")
def ssim():
    so = os.path.join(SIM_DIR, "libpgs_sim.so")
    srcs = [os.path.join(SIM_DIR, f) for f in ("sim_compact.cpp", "simt.h")]
    srcs += [os.path.join(ROOT, "incubator_pegasus_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "incubator_pegasus_b200", "csrc"))]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["bash", os.path.join(SIM_DIR, "build.sh")])
    L = C.CDLL(so)
    L.sim_split.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                            C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64)]
    L.sim_split_child_info.argtypes = [C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    L.sim_split_child_copy.argtypes = [C.c_uint32] + [C.c_void_p] * 6
    L.sim_split_child_bloom_check.argtypes = [C.c_uint32, C.c_char_p, C.c_uint32]
    return L


def sim_split(pgs, ssim, br, src, dst, want=None, seg_weight=0, block_size=4096, restart_interval=16):
    """-> (status, {child: BlockRun + index arrays + info}, dropped)"""
    S = dst // src
    want = (1 << S) - 1 if want is None else want
    dropped = C.c_uint64()
    st = ssim.sim_split(br.data.ctypes.data, br.data.shape[0], br.blk_off.ctypes.data, br.blk_size.ctypes.data, br.n_blocks, block_size,
                        restart_interval, src, dst, want, seg_weight, C.byref(dropped))
    out = {}
    if st:
        return st, out, dropped.value
    for c in range(S):
        info, q, kb = pgs.RunInfo(), C.c_uint32(), C.c_uint64()
        if not ssim.sim_split_child_info(c, C.byref(info), C.byref(q), C.byref(kb)):
            continue
        nb = info.n_blocks
        data, off, size = np.zeros(info.data_bytes, np.uint8), np.zeros(nb + 1, np.uint64), np.zeros(nb, np.uint32)
        blk_rec, ikey_off, ikeys = np.zeros(nb + 1, np.uint32), np.zeros(nb + 1, np.uint32), np.zeros(kb.value + 1, np.uint8)
        ssim.sim_split_child_copy(c, data.ctypes.data, off.ctypes.data, size.ctypes.data, blk_rec.ctypes.data, ikey_off.ctypes.data,
                                  ikeys.ctypes.data)
        out[c] = dict(run=pgs.BlockRun(data, off[:nb].copy(), size), info=info, blk_rec=blk_rec, ikey_off=ikey_off, ikeys=ikeys[:kb.value],
                      segments=q.value)
    return st, out, dropped.value


INFO_FIELDS = ("n_blocks", "n_records", "n_tombstones", "data_bytes", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len",
               "max_block_size", "max_block_records", "smallest_seq", "largest_seq")


def check_split(pgs, ssim, br, src, dst, want=None, **kw):
    """split br in the simulator and compare every built child with the model; returns the children"""
    items = fb.decode(br).to_list()
    want_items, want_dropped = sm.split_items(items, src, dst)
    S = dst // src
    mask = (1 << S) - 1 if want is None else want
    st, got, dropped = sim_split(pgs, ssim, br, src, dst, want, **kw)
    assert st == 0
    assert dropped == want_dropped
    for c in range(S):
        built = (mask >> c) & 1 and want_items[c]
        assert (c in got) == bool(built), c
        if not built:
            continue
        x = got[c]
        run = x["run"]
        assert fb.classify(run) == fb.OK, c
        recs = pgs.decode_blocks(run)
        assert recs.to_list() == want_items[c], c
        assert recs.same_as(fb.decode(run))
        m = fb.model_index(run)
        assert x["blk_rec"].tolist() == m["blk_rec"] and x["ikey_off"].tolist() == m["ikey_off"] and x["ikeys"].tobytes() == m["ikeys"]
        for f in INFO_FIELDS:
            assert getattr(x["info"], f) == m["info"][f], (c, f, getattr(x["info"], f), m["info"][f])
        for k, _s, _t, _v in want_items[c]:
            assert ssim.sim_split_child_bloom_check(c, k, len(k)), (c, k)
            pl = 2 + int.from_bytes(k[:2], "big") if len(k) >= 2 else 0
            if 2 < pl <= len(k):
                assert ssim.sim_split_child_bloom_check(c, k[:pl], pl), (c, k[:pl])
    return got


def test_model_hash_is_the_library_hash(pgs):
    rng = np.random.default_rng(5)
    keys = [b"", b"\x00", b"\x00\x00", b"\x00\x00sort", b"\x00\x05hk", b"\x00\x02hkrest", b"\xff\xff" + b"x" * 40]
    keys += [bytes(rng.integers(0, 256, int(rng.integers(0, 60)), dtype=np.uint8)) for _ in range(200)]
    for k in keys:
        assert sm.key_hash(k) == pgs.lib().pgs_key_hash(k, len(k)), k


def test_model_routes_by_the_reference_formula():
    """the children of (src, dst) partition the parent's records in order; splitting 1 -> 2 -> 4 step by step ends where
    1 -> 4 does (child i of partition p is p + i * src_count)"""
    rng = np.random.default_rng(9)
    items = sorted({(b"\x00\x02%02d" % int(rng.integers(0, 60)) + b"s%d" % i, i + 1, 1, b"v") for i in range(400)})
    four, _ = sm.split_items(items, 1, 4)
    two, _ = sm.split_items(items, 1, 2)
    for p in range(2):
        sub, _ = sm.split_items(two[p], 2, 4)
        for i in range(2):
            assert sub[i] == four[p + 2 * i]
    assert sorted(sum(four, [])) == sorted(items)


def _mixed(seed, n=700):
    """several versions per key, tombstones, empty hash keys (hashed on the sort key), the empty write, one hash key's
    records over many blocks"""
    rng = np.random.default_rng(seed)
    items = {}
    seq = 0
    for i in range(n):
        r = rng.random()
        if r < 0.15:
            key = b"\x00\x00" + b"sk%04d" % int(rng.integers(0, 300))
        elif r < 0.3:
            key = b"\x00\x03hot" + b"%05d" % int(rng.integers(0, 2000))
        else:
            hk = b"h%03d" % int(rng.integers(0, 120))
            key = len(hk).to_bytes(2, "big") + hk + b"s%03d" % int(rng.integers(0, 40))
        for _ in range(int(rng.integers(1, 4))):
            seq += 1
            t = 0 if rng.random() < 0.15 else 1
            items[(key, -seq)] = (key, seq, t, (bytes(4) + bytes(rng.integers(0, 256, int(rng.integers(0, 60)), dtype=np.uint8))) if t else b"")
    items[(b"", -1)] = (b"", 1_000_000, 1, b"")
    return [items[k] for k in sorted(items)]


@pytest.mark.parametrize("src,dst", [(1, 2), (1, 8), (4, 16)])
@pytest.mark.parametrize("block_size,ri", [(4096, 16), (16384, 1)])
def test_sim_split_builder_runs(pgs, ssim, src, dst, block_size, ri):
    recs = pgs.Records.from_list(_mixed(src * 10 + dst))
    br = pgs.build_run(recs, block_size, ri)
    check_split(pgs, ssim, br, src, dst, block_size=block_size, restart_interval=ri)
    # forced small segments: boundaries fall inside a hash key's records
    got = check_split(pgs, ssim, br, src, dst, seg_weight=3000, block_size=block_size, restart_interval=ri)
    assert max(x["segments"] for x in got.values()) > 10


@pytest.mark.parametrize("name", ["ragged_records", "long_keys", "empty_hash_keys", "long_restart_arrays", "edge"])
def test_sim_split_edge_inputs(pgs, ssim, name):
    """keys of 0..4096 bytes, values past k_emit's block buffer (its big-entry path), restart interval 1, tiny entries"""
    recs = fb.edge_records(3) if name == "edge" else getattr(merge_inputs, name)(7)[0]
    for ri in (1, 16):
        br = pgs.build_run(recs, 4096, ri)
        check_split(pgs, ssim, br, 1, 4, restart_interval=ri)
        check_split(pgs, ssim, br, 1, 2, seg_weight=2000, restart_interval=ri)


@pytest.mark.parametrize("policy", list(fb.GRID))
def test_sim_split_foreign_runs(pgs, ssim, policy):
    """short, zero or random shared prefixes, padded varints, irregular restart arrays, gaps between blocks"""
    for i, (name, recs) in enumerate(fb.record_sets().items()):
        br = fb.encode_run(recs, seed=i, **fb.GRID[policy])
        check_split(pgs, ssim, br, 1, 8, seg_weight=4000 if i % 2 else 0)


def test_sim_split_null_and_empty_children(pgs, ssim):
    """a child that is not built (the online split's parent half) and a child that receives nothing get no run"""
    items = [it for it in _mixed(4) if it[0] and sm.child_of(it[0], 1, 4) != 2]
    br = pgs.build_run(pgs.Records.from_list(items))
    got = check_split(pgs, ssim, br, 1, 4, want=0b1011)
    assert 2 not in got and 3 in got
    got = check_split(pgs, ssim, br, 1, 4, want=0b0010)
    assert list(got) == [1]


def test_sim_split_refuses_too_many_children(pgs, ssim):
    br = pgs.build_run(pgs.Records.from_list(_mixed(1, 50)))
    st, _got, _d = sim_split(pgs, ssim, br, 1, 64)
    assert st == pgs.NOT_SUPPORTED
