"""The device sort (sort_kernels.cuh: check, per-round key, radix and settle passes, gather) followed by the device run build, inside
the host SIMT interpreter, through sort_plan / sort_buffers / sort_launch as pgs_run_build_unsorted runs them.  For every input,
random permutations of the records give a run whose blocks, handles and pgs_run_info equal sim_run_build's on the records sorted
in Python, and the host builder's.  Refusals follow the documented precedence: offsets first (kInvalidArgument), then a user key
over 4096 bytes (kNotSupported), then a duplicate internal key (kInvalidArgument).

The file also passes against the AddressSanitizer build of the simulator:

    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_run_build_unsorted_sim.py
    bash tools/simt/build.sh"""
import ctypes as C
import random

import numpy as np
import pytest

from incubator_pegasus_b200 import synth
from test_run_build_sim import INFO_FIELDS, bsim, check_identity, edge_items, sim_build  # noqa: F401  (bsim: the module's fixture)

M56 = 1 << 56


@pytest.fixture(scope="module")
def usim(bsim):  # noqa: F811
    vp = C.c_void_p
    bsim.sim_run_build_unsorted.argtypes = [C.c_uint64, vp, vp, vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
    return bsim


def ikey_sorted(items):
    """internal-key order: user key ascending (bytewise, a prefix first), then seq << 8 | type descending"""
    return sorted(items, key=lambda x: (x[0], -(((x[1] << 8) | x[2]) & ((1 << 64) - 1))))


def unsorted_build(pgs, usim, recs, block_size, ri, grid_cap=4):
    """-> (status, BlockRun or None, RunInfo or None, launches)"""
    launches = C.c_uint32()
    st = usim.sim_run_build_unsorted(recs.n, recs.keys.ctypes.data, recs.key_off.ctypes.data, recs.vals.ctypes.data,
                                     recs.val_off.ctypes.data, recs.seq.ctypes.data, recs.type.ctypes.data, block_size, ri, grid_cap,
                                     C.byref(launches))
    if st:
        return st, None, None, launches.value
    nbytes, nb, info = C.c_uint64(), C.c_uint32(), pgs.RunInfo()
    usim.sim_run_build_info(C.byref(nbytes), C.byref(nb), C.byref(info))
    data, off, size = np.zeros(nbytes.value, np.uint8), np.zeros(nb.value, np.uint64), np.zeros(nb.value, np.uint32)
    usim.sim_run_build_copy(data.ctypes.data, off.ctypes.data, size.ctypes.data)
    return st, pgs.BlockRun(data, off, size), info, launches.value


def check_orders(pgs, usim, items, block_size=4096, ri=16, perms=2, seed=0, extra_orders=()):
    """sim_run_build of the Python-sorted records (checked against the host builder) against the unsorted build of random
    permutations, and of each order in extra_orders ("sorted", "reversed")"""
    want_items = ikey_sorted(items)
    want = check_identity(pgs, usim, pgs.Records.from_list(want_items), block_size, ri) if items else None
    want_st, _, want_info = sim_build(pgs, usim, pgs.Records.from_list(want_items), block_size, ri)
    assert want_st == 0
    rng = random.Random(seed)
    orders = []
    for _ in range(perms):
        o = list(items)
        rng.shuffle(o)
        orders.append(o)
    for name in extra_orders:
        orders.append(want_items if name == "sorted" else want_items[::-1])
    for o in orders:
        st, got, info, _ = unsorted_build(pgs, usim, pgs.Records.from_list(o), block_size, ri)
        assert st == 0
        if want is None:
            assert got.n_blocks == 0
            continue
        assert np.array_equal(got.blk_off, want.blk_off) and np.array_equal(got.blk_size, want.blk_size)
        assert got.data.shape == want.data.shape and np.array_equal(got.data, want.data)
        for f in INFO_FIELDS:
            assert getattr(info, f) == getattr(want_info, f), f


@pytest.mark.parametrize("block_size,ri", [(4096, 16), (256, 1), (16384, 2)])
def test_edge_items(pgs, usim, block_size, ri):
    check_orders(pgs, usim, edge_items(block_size + ri), block_size, ri, seed=block_size, extra_orders=("sorted", "reversed"))


def test_config2_like_records(pgs, usim):
    recs = synth.compaction_runs(k=1, n_per_run=3000, seed=5)[0]
    check_orders(pgs, usim, recs.to_list(), 4096, 16, perms=1, seed=1, extra_orders=("reversed",))


def window_edge_items():
    """keys that differ only at bytes 7 / 8 and 15 / 16: the last byte of a window and the first of the next"""
    base = bytes(range(0x30, 0x30 + 24))
    items = []
    for at in (7, 8, 15, 16):
        for v in (0x00, 0x01, 0x7F, 0x80, 0xFF):
            k = bytearray(base)
            k[at] = v
            items.append((bytes(k), 3, 1, b"v%d" % at))
    items = list({k: (k, s, t, v) for k, s, t, v in items}.values())
    return items + [(base[:n], 2, 1, b"p") for n in (7, 8, 9, 15, 16, 17)]  # the same bytes ending at each side of an edge


def prefix_items():
    """"k" < "k\\0" < "k\\0\\0", the empty user key first, 0xFF bytes last"""
    return [(b"k", 5, 1, b"a"), (b"k\x00", 5, 1, b"b"), (b"k\x00\x00", 5, 1, b"c"), (b"k\x00" * 4, 1, 0, b""),
            (b"", 9, 1, b"e"), (b"", 8, 0, b""), (b"\xff", 1, 1, b"f"), (b"\xff" * 9, 1, 1, b"g"), (b"\xff" * 8, 2, 1, b"h"),
            (b"\xfe\xff", 1, 1, b""), (b"k\xff", 4, 1, b"i"), (b"\x00", 1, 1, b""), (b"\x00" * 8, 1, 1, b""), (b"\x00" * 9, 1, 1, b"")]


def version_items():
    """many versions of one key with seqs near 2^56, and equal seqs with types 0 and 1"""
    rng = random.Random(3)
    items = [(b"\x00\x03hot", M56 - 1 - i, rng.choice([0, 1]), rng.randbytes(rng.randrange(0, 20))) for i in range(0, 1500, 3)]
    items += [(b"\x00\x03hot", 77, 0, b""), (b"\x00\x03hot", 77, 1, b"x"), (b"\x00\x03hou", 5, 1, b""), (b"\x00\x03hos", M56 - 1, 1, b"")]
    return items + [(b"\x00\x03eq", s, t, b"%d" % t) for s in (1, 1000, M56 - 2) for t in (0, 1)]


def one_key_items(n=2500):
    return [(b"\x00\x04only", s, s & 1, b"v" * (s % 7)) for s in range(1, n)]


def long_prefix_items():
    """4096-byte keys sharing a 4000-byte prefix: about 500 rounds in which nothing splits, then the tails"""
    rng = random.Random(9)
    prefix = bytes(rng.randrange(256) for _ in range(4000))
    items = [(prefix + rng.randbytes(96), 3, 1, rng.randbytes(rng.randrange(0, 40))) for _ in range(40)]
    return items + [(items[0][0], 2, 0, b""), (items[1][0][:4090], 4, 1, b"short")]


def test_window_edges(pgs, usim):
    check_orders(pgs, usim, window_edge_items(), 256, 1, perms=3, extra_orders=("sorted", "reversed"))


def test_prefix_and_zero_bytes(pgs, usim):
    check_orders(pgs, usim, prefix_items(), 256, 2, perms=4, extra_orders=("sorted", "reversed"))


def test_versions_near_2_pow_56(pgs, usim):
    check_orders(pgs, usim, version_items(), 512, 16, perms=2, extra_orders=("reversed",))


def test_one_user_key_only(pgs, usim):
    check_orders(pgs, usim, one_key_items(), 4096, 16, perms=1, extra_orders=("sorted", "reversed"))


def test_long_shared_prefix_4096_byte_keys(pgs, usim):
    check_orders(pgs, usim, long_prefix_items(), 16384, 16, perms=1, extra_orders=("reversed",))


@pytest.mark.parametrize("n", [0, 1, 2])
def test_tiny(pgs, usim, n):
    items = [(b"\x00\x01b", 4, 1, b"x"), (b"\x00\x01a", 9, 0, b"")][:n]
    check_orders(pgs, usim, items, 4096, 16, perms=1, extra_orders=("sorted", "reversed"))


def test_product_grids(pgs, usim):
    """the product's grids (one thread per record) as well as the capped grids of the other tests"""
    items = edge_items(5)[:900]
    want = check_identity(pgs, usim, pgs.Records.from_list(items), 512, 2, grid_cap=0)
    rng = random.Random(2)
    rng.shuffle(items)
    st, got, _, _ = unsorted_build(pgs, usim, pgs.Records.from_list(items), 512, 2, grid_cap=0)
    assert st == 0 and np.array_equal(got.data, want.data) and np.array_equal(got.blk_off, want.blk_off)


# ---- refusals --------------------------------------------------------------------------------------------------------------------
def _ok(n=300):
    items = [(b"\x00\x01k%04d" % i, 5, 1, b"v") for i in range(n)]
    random.Random(n).shuffle(items)
    return items


def _bad_offsets(recs, which="key", at=None):
    at = recs.n // 2 if at is None else at
    off = recs.key_off if which == "key" else recs.val_off
    off[at], off[at + 1] = off[at + 1], off[at]  # not ascending (when the record is not empty)
    return recs


def _status(pgs, usim, recs):
    return [unsorted_build(pgs, usim, recs, bs, ri)[0] for bs, ri in [(4096, 16), (256, 1)]]


def test_refusals_in_precedence(pgs, usim):
    long_key = (b"\x00\x01b" + bytes(4095), 5, 1, b"v")   # 4098 bytes
    k4097 = (b"\x00\x01c" + bytes(4094), 5, 1, b"v")      # 4097 bytes
    ok = _ok()
    dup = ok[:50] + [(ok[10][0], ok[10][1], ok[10][2], b"other value")] + ok[50:]
    cases = [
        (pgs.Records.from_list(ok[:100] + [k4097] + ok[100:]), pgs.NOT_SUPPORTED),
        (pgs.Records.from_list([long_key]), pgs.NOT_SUPPORTED),
        (pgs.Records.from_list(dup), pgs.INVALID_ARGUMENT),
        (pgs.Records.from_list([(b"", 1, 1, b""), (b"", 1, 1, b"")]), pgs.INVALID_ARGUMENT),
        (_bad_offsets(pgs.Records.from_list(ok)), pgs.INVALID_ARGUMENT),
        (_bad_offsets(pgs.Records.from_list(ok), "val"), pgs.INVALID_ARGUMENT),
        # combinations: offsets before a long key before a duplicate
        (_bad_offsets(pgs.Records.from_list(ok[:10] + [k4097] + ok[10:])), pgs.INVALID_ARGUMENT),
        (_bad_offsets(pgs.Records.from_list(dup + [k4097])), pgs.INVALID_ARGUMENT),
        (pgs.Records.from_list(dup + [k4097]), pgs.NOT_SUPPORTED),
        (pgs.Records.from_list([k4097] + dup), pgs.NOT_SUPPORTED),
    ]
    for recs, want in cases:
        assert _status(pgs, usim, recs) == [want, want]


def test_offsets_past_the_bytes_refused(pgs, usim):
    """an offset past key_off[n] / val_off[n] (the copied bytes), and a last offset before an earlier one"""
    for which in ("key", "val"):
        recs = pgs.Records.from_list(_ok(40))
        off = recs.key_off if which == "key" else recs.val_off
        off[5] = off[-1] + 7
        assert _status(pgs, usim, recs) == [pgs.INVALID_ARGUMENT] * 2
    recs = pgs.Records.from_list(_ok(40))
    recs.key_off[-1] = 3
    assert _status(pgs, usim, recs) == [pgs.INVALID_ARGUMENT] * 2


def test_duplicate_among_versions_refused(pgs, usim):
    items = [(b"\x00\x02hk", s, 1, b"") for s in range(100, 0, -1)] + [(b"\x00\x02hk", 50, 1, b"again")]
    random.Random(4).shuffle(items)
    assert _status(pgs, usim, pgs.Records.from_list(items)) == [pgs.INVALID_ARGUMENT] * 2
    # equal seq, different type: not a duplicate
    check_orders(pgs, usim, [(b"\x00\x02hk", 50, 1, b""), (b"\x00\x02hk", 50, 0, b"")], 4096, 16, perms=2)
