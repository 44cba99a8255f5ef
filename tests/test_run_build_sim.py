"""The device run builder (build_kernels.cuh: record, next-block, chain, scan and block passes, then the upload's index passes)
inside the host SIMT interpreter, through build_plan / build_buffers / build_launch_plan / build_launch_blocks as pgs_run_build
runs them.  Every built run equals the host builder's (pgs.build_run) byte for byte -- blocks, padding, blk_off and blk_size --
and its pgs_run_info equals that of the host-built run as the upload indexes it.  Inputs the host path refuses get the host
path's status: the builder's kInvalidArgument for records out of order, the upload's kNotSupported for a user key over 4096
bytes.

The file also passes against the AddressSanitizer build of the simulator:

    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_run_build_sim.py
    bash tools/simt/build.sh"""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from incubator_pegasus_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM_DIR = os.path.join(ROOT, "tools", "simt")
vp = C.c_void_p


@pytest.fixture(scope="module")
def bsim():
    so = os.path.join(SIM_DIR, "libpgs_sim.so")
    srcs = [os.path.join(SIM_DIR, f) for f in ("sim_compact.cpp", "simt.h")]
    srcs += [os.path.join(ROOT, "incubator_pegasus_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "incubator_pegasus_b200", "csrc"))]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["bash", os.path.join(SIM_DIR, "build.sh")])
    L = C.CDLL(so)
    L.sim_run_build.argtypes = [C.c_uint64, vp, vp, vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32]
    L.sim_run_build_info.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), vp]
    L.sim_run_build_copy.argtypes = [vp, vp, vp]
    L.sim_run_index.argtypes = [vp, C.c_uint64, vp, vp, C.c_uint32, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), vp, vp,
                                C.c_uint64, vp, C.c_uint64, vp, C.c_uint64, vp, C.c_uint64]
    return L


INFO_FIELDS = ("n_blocks", "n_records", "n_tombstones", "data_bytes", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len",
               "max_block_size", "max_block_records", "smallest_seq", "largest_seq")


def sim_build(pgs, bsim, recs, block_size, ri, grid_cap=4):
    """-> (status, BlockRun or None, RunInfo or None)"""
    st = bsim.sim_run_build(recs.n, recs.keys.ctypes.data, recs.key_off.ctypes.data, recs.vals.ctypes.data, recs.val_off.ctypes.data,
                            recs.seq.ctypes.data, recs.type.ctypes.data, block_size, ri, grid_cap)
    if st:
        return st, None, None
    nbytes, nb, info = C.c_uint64(), C.c_uint32(), pgs.RunInfo()
    bsim.sim_run_build_info(C.byref(nbytes), C.byref(nb), C.byref(info))
    data, off, size = np.zeros(nbytes.value, np.uint8), np.zeros(nb.value, np.uint64), np.zeros(nb.value, np.uint32)
    bsim.sim_run_build_copy(data.ctypes.data, off.ctypes.data, size.ctypes.data)
    return st, pgs.BlockRun(data, off, size), info


def upload_status(pgs, bsim, recs, block_size, ri):
    """the host path: builder, then the upload's handle rule and index passes -> (status, BlockRun or None, RunInfo or None)"""
    try:
        br = pgs.build_run(recs, block_size, ri)
    except pgs.PegasusError as e:
        return e.code, None, None
    info, ne, bl = pgs.RunInfo(), C.c_uint64(), C.c_uint32()
    st = bsim.sim_run_index(br.data.ctypes.data, br.data.shape[0], br.blk_off.ctypes.data, br.blk_size.ctypes.data, br.n_blocks, C.byref(info),
                            C.byref(ne), C.byref(bl), None, None, 0, None, 0, None, 0, None, 0)
    return st, br, info


def check_identity(pgs, bsim, recs, block_size, ri, grid_cap=4):
    want_st, want, want_info = upload_status(pgs, bsim, recs, block_size, ri)
    st, got, info = sim_build(pgs, bsim, recs, block_size, ri, grid_cap)
    assert st == want_st == 0
    assert got.n_blocks == want.n_blocks
    assert np.array_equal(got.blk_off, want.blk_off) and np.array_equal(got.blk_size, want.blk_size)
    assert got.data.shape == want.data.shape and np.array_equal(got.data, want.data)
    for f in INFO_FIELDS:
        assert getattr(info, f) == getattr(want_info, f), f
    return got


def _sorted(items):
    """internal-key order: user key ascending, then seq << 8 | type descending (duplicates of a trailer dropped)"""
    seen, out = set(), []
    for k, s, t, v in sorted(items, key=lambda x: (x[0], -((x[1] << 8) | x[2]))):
        if (k, (s << 8) | t) not in seen:
            seen.add((k, (s << 8) | t))
            out.append((k, s, t, v))
    return out


def edge_items(seed=0):
    """the empty user key, many versions of one key, tombstones, empty values, values larger than a 16 KB block, long shared
    prefixes, 4096-byte user keys, and user keys that are prefixes of the next one so that the shared prefix of the internal
    keys runs into the trailer"""
    rng = random.Random(seed)
    it = [(b"", 90, 1, b"e"), (b"", 80, 0, b""), (b"", 2, 1, b"")]
    hot = b"\x00\x03hotkey"
    it += [(hot, s, 0 if s % 5 == 0 else 1, rng.randbytes(rng.randrange(0, 30))) for s in range(700, 100, -1)]
    long_base = b"\x00\x20" + bytes([0x61]) * 1500
    it += [(long_base + b"%06d" % i, 7, 1, rng.randbytes(rng.randrange(0, 9))) for i in range(120)]
    it += [(b"\x00\x02big%02d" % i, 9, 1, rng.randbytes(rng.choice([300, 5000, 17000, 40000]))) for i in range(8)]
    k4096 = b"\x00\x04" + bytes(rng.randrange(256) for _ in range(4094))
    it += [(k4096, 5, 1, b"v"), (k4096, 4, 0, b""), (k4096[:-1] + b"\xff", 3, 1, rng.randbytes(100))]
    for i in range(40):  # "ab" with type t, then "ab" + t + seq byte: the internal keys share 4 bytes and more
        uk = b"\x00\x02pre%02d" % i
        it += [(uk, 0x105, 1, b"x"), (uk + b"\x01\x05", 3, 1, b"y"), (uk + b"\x01\x05\x01", 2, 0, b""),
               (uk + b"\x01\x05\x01\x00", 9, 1, b"z" * i)]
    it += [(b"\x00\x01z%04d" % i, rng.randrange(1, 1 << 40), rng.choice([0, 1]), b"" if i % 3 == 0 else rng.randbytes(rng.randrange(1, 200)))
           for i in range(400)]
    return _sorted(it)


@pytest.mark.parametrize("block_size", [256, 512, 4096, 16384])
@pytest.mark.parametrize("ri", [1, 2, 16])
def test_edge_records_byte_identical(pgs, bsim, block_size, ri):
    check_identity(pgs, bsim, pgs.Records.from_list(edge_items(block_size + ri)), block_size, ri)


@pytest.mark.parametrize("block_size,ri", [(256, 1), (4096, 16), (16384, 2)])
def test_single_record(pgs, bsim, block_size, ri):
    for item in [(b"", 1, 1, b""), (b"\x00\x01k", 3, 0, b""), (b"\x00\x01k", 3, 1, bytes(50000))]:
        check_identity(pgs, bsim, pgs.Records.from_list([item]), block_size, ri)


def test_one_thread_per_record_grids(pgs, bsim):
    """the product's grids (one thread per record, one warp per block) as well as the capped grids of the other tests"""
    check_identity(pgs, bsim, pgs.Records.from_list(edge_items(7)[:700]), 512, 2, grid_cap=0)


@pytest.mark.parametrize("block_size,ri", [(4096, 16), (512, 1)])
def test_synth_thousands_of_blocks(pgs, bsim, block_size, ri):
    recs = synth.compaction_runs(k=1, n_per_run=15_000 if block_size == 4096 else 3_000, seed=11)[0]
    got = check_identity(pgs, bsim, recs, block_size, ri, grid_cap=16)
    assert got.n_blocks >= 1000


def _refusal(pgs, bsim, items, want):
    recs = pgs.Records.from_list(items)
    for block_size, ri in [(4096, 16), (256, 1)]:
        host, _, _ = upload_status(pgs, bsim, recs, block_size, ri)
        st, _, _ = sim_build(pgs, bsim, recs, block_size, ri)
        assert host == want and st == want


@pytest.mark.parametrize("at", [1, 2, 150, 399])
def test_descending_user_key_refused(pgs, bsim, at):
    items = [(b"\x00\x01k%05d" % i, 10, 1, b"v%d" % i) for i in range(400)]
    # a smaller key, or a proper prefix of the key before (smaller too)
    items[at] = (b"\x00\x01j" if at % 2 else items[at - 1][0][:-1], 10, 1, b"w")
    _refusal(pgs, bsim, items, pgs.INVALID_ARGUMENT)


@pytest.mark.parametrize("second", [(5, 1), (5, 2), (6, 0)])
def test_non_descending_trailer_refused(pgs, bsim, second):
    items = [(b"\x00\x01a", 9, 1, b""), (b"\x00\x01k", 5, 1, b"v"), (b"\x00\x01k",) + second + (b"w",), (b"\x00\x01m", 1, 1, b"")]
    _refusal(pgs, bsim, items, pgs.INVALID_ARGUMENT)


def test_key_over_4096_refused(pgs, bsim):
    items = [(b"\x00\x01a", 9, 1, b""), (b"\x00\x01b" + bytes(4094), 5, 1, b"v"), (b"\x00\x01c", 1, 1, b"")]
    _refusal(pgs, bsim, items, pgs.NOT_SUPPORTED)
    # the order rule is the builder's and comes first, wherever the long key is
    items2 = [(b"\x00\x01b" + bytes(4094), 5, 1, b"v"), (b"\x00\x01c", 1, 1, b""), (b"\x00\x01a", 9, 1, b"")]
    _refusal(pgs, bsim, items2, pgs.INVALID_ARGUMENT)


def test_no_records(pgs, bsim):
    st, run, _ = sim_build(pgs, bsim, pgs.Records.from_list([]), 4096, 16)
    assert st == 0 and run is not None and run.n_blocks == 0
