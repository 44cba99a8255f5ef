"""CPU check of the compaction KERNELS' logic: the same sources nvcc compiles for sm_90a
(incubator_pegasus_b200/csrc/compact_kernels.cuh, group.cuh) are compiled by g++ against tools/simt/simt.h, a host-side SIMT
interpreter (every CUDA thread a fiber, shuffles / ballots / barriers as rendezvous), and their output is compared with the
oracle.  This says nothing about timing or the memory model -- the `-m gpu` tests do -- but it runs the merge, filter,
prefix-compression and block-assembly code bit for bit without a GPU.  The simulator is test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import merge_inputs
from get_model import SIM_SMEM, check_run_format, emit_geometry
from incubator_pegasus_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM_DIR = os.path.join(ROOT, "tools", "simt")


@pytest.fixture(scope="session")
def sim():
    so = os.path.join(SIM_DIR, "libpgs_sim.so")
    srcs = [os.path.join(SIM_DIR, f) for f in ("sim_compact.cpp", "simt.h")]
    srcs += [os.path.join(ROOT, "incubator_pegasus_b200", "csrc", f)
             for f in ("compact_kernels.cuh", "index_kernel.cuh", "read_kernels.cuh", "scan_kernel.cuh", "group.cuh", "device_util.cuh",
                       "format.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                               os.path.join(SIM_DIR, "sim_compact.cpp"), "-o", so])
    return C.CDLL(so)


def sim_compact(pgs, sim, runs, *, bottommost, now=synth.NOW, default_ttl=0, validate_hash=False, pidx=0, partition_version=-1,
                ops=None, enabled=True, block_size=4096, restart_interval=16, lanes=0, seg_weight=0):
    brs = [pgs.build_run(r, block_size, restart_interval) for r in runs]
    k = len(brs)
    data = (C.c_void_p * k)(*[b.data.ctypes.data for b in brs])
    nbytes = (C.c_uint64 * k)(*[b.data.shape[0] for b in brs])
    off = (C.c_void_p * k)(*[b.blk_off.ctypes.data for b in brs])
    size = (C.c_void_p * k)(*[b.blk_size.ctypes.data for b in brs])
    nb = (C.c_uint32 * k)(*[b.n_blocks for b in brs])
    fp = pgs.FilterParams()
    fp.enabled = 1 if enabled else 0
    fp.validate_hash = 1 if validate_hash else 0
    fp.data_version = 1
    fp.default_ttl = default_ttl
    fp.pidx = pidx
    fp.partition_version = partition_version
    if ops is not None and len(ops):
        fp.ops = ops.ctypes.data_as(C.POINTER(C.c_uint8))
        fp.ops_len = len(ops)
    crc = (C.c_uint64 * 256)(*crc_table()) if validate_hash else None
    st = sim.sim_compact(k, data, nbytes, off, size, nb, block_size, restart_interval, 1 if bottommost else 0, C.byref(fp), now,
                         lanes, C.c_uint64(seg_weight), crc)
    assert st == 0, st
    db, nblk, nseg = C.c_uint64(), C.c_uint32(), C.c_uint32()
    sim.sim_result_sizes(C.byref(db), C.byref(nblk), C.byref(nseg))
    n = nblk.value
    out = pgs.BlockRun(np.zeros(db.value + 16, np.uint8), np.zeros(n + 1, np.uint64), np.zeros(n, np.uint32))
    blk_rec = np.zeros(n + 1, np.uint32)
    ikey_off = np.zeros(n + 1, np.uint32)
    stats = (C.c_uint64 * 20)()
    sim.sim_result_stats(stats)
    ikeys = np.zeros(int(stats[19]) + 16, np.uint8)
    rec_off = np.zeros(int(stats[1]) + 1, np.uint32)
    sim.sim_result_copy(out.data.ctypes.data_as(C.c_void_p), out.blk_off.ctypes.data_as(C.c_void_p), out.blk_size.ctypes.data_as(C.c_void_p),
                        blk_rec.ctypes.data_as(C.c_void_p), ikey_off.ctypes.data_as(C.c_void_p), ikeys.ctypes.data_as(C.c_void_p),
                        rec_off.ctypes.data_as(C.c_void_p))
    end = int(out.blk_off[n])
    out.blk_off = out.blk_off[:n].copy()
    return out, dict(stats=list(stats), blk_rec=blk_rec, ikey_off=ikey_off, ikeys=ikeys, rec_off=rec_off, end=end, nseg=nseg.value)


def entry_offsets(data, off, size):
    """offsets of the entries of the block at data[off:off + size], from its headers (shared, non_shared, value length)"""
    nr = int.from_bytes(data[off + size - 4:off + size].tobytes(), "little")
    limit, p, out = size - 4 - 4 * nr, 0, []
    while p < limit:
        out.append(p)
        h, lens = 0, []
        for _ in range(3):
            v = sh = 0
            while True:
                c = int(data[off + p + h])
                h += 1
                v |= (c & 127) << sh
                sh += 7
                if c < 128:
                    break
            lens.append(v)
        p += h + lens[1] + lens[2]
    return out


def crc_table():
    poly = 0x9a6c9329ac4bc9b5
    tab = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ poly if c & 1 else c >> 1
        tab.append(c)
    return tab


STAT_FIELDS = ("in_records", "out_records", "in_bytes", "out_bytes", "dropped_shadowed", "dropped_tombstone", "dropped_expired",
               "dropped_user", "dropped_stale", "ttl_rewritten")


def check(pgs, oracle, sim, runs, *, bottommost, ops_json=None, **kw):
    if "lanes" not in kw:  # the one-thread-per-segment shape and a lane-group shape of the same source
        check(pgs, oracle, sim, runs, bottommost=bottommost, ops_json=ops_json, lanes=8, **kw)
        kw["lanes"] = 1
    ops_bin = pgs.parse_ops(ops_json) if ops_json else None
    got_run, x = sim_compact(pgs, sim, runs, bottommost=bottommost, ops=ops_bin, **kw)
    okw = {k: v for k, v in kw.items() if k in ("enabled", "default_ttl", "validate_hash", "pidx", "partition_version")}
    oops = oracle.Ops(ops_json) if ops_json else None  # keeps the parsed table alive across orc_compact
    fp = oracle.filter_params(ops=oops, **okw)
    want_run, st = oracle.compact([oracle.Run.from_records(r) for r in runs], bottommost, fp, kw.get("now", synth.NOW))
    want = want_run.records()
    for i, f in enumerate(STAT_FIELDS):
        assert x["stats"][i] == getattr(st, f), (f, x["stats"][i], getattr(st, f))
    if want.n == 0:
        assert got_run.n_blocks == 0
        return x
    got = pgs.decode_blocks(got_run)
    assert got.n == want.n, (got.n, want.n)
    assert got.same_as(want)
    assert got.same_as(oracle.Run.from_blocks(got_run).records())  # independent decoder of the raw blocks
    # the new run's index: block layout, cumulative record counts, last user key per block, entry offsets
    n = got_run.n_blocks
    assert int(x["blk_rec"][n]) == want.n and int(x["blk_rec"][0]) == 0
    assert np.all(got_run.blk_off % 16 == 0)
    ends = got_run.blk_off + ((got_run.blk_size.astype(np.uint64) + 15) & ~np.uint64(15))
    assert np.array_equal(ends[:-1], got_run.blk_off[1:]) and int(ends[-1]) == x["end"]  # contiguous, ordered
    for b in range(n):
        last = int(x["blk_rec"][b + 1]) - 1
        assert x["ikeys"][int(x["ikey_off"][b]):int(x["ikey_off"][b + 1])].tobytes() == want.key(last)
    # restart arrays, the cut rule at the block size the geometry leaves, padding
    max_ukey = max(int(np.diff(r.key_off.astype(np.int64)).max(initial=0)) for r in runs)
    geo = emit_geometry(kw.get("block_size", 4096), kw.get("restart_interval", 16), max_ukey, SIM_SMEM)
    counts = check_run_format(got_run, kw.get("restart_interval", 16), geo["block_size"])
    assert counts == np.diff(x["blk_rec"][:n + 1].astype(np.int64)).tolist()
    # entry offsets: walking each block entry by entry must land on its rec_off entries
    for b in range(n):
        walk = entry_offsets(got_run.data, int(got_run.blk_off[b]), int(got_run.blk_size[b]))
        assert walk == [int(v) for v in x["rec_off"][int(x["blk_rec"][b]):int(x["blk_rec"][b + 1])]], b
    assert x["stats"][10] == int(np.sum(want.type == 0))
    assert x["stats"][11] == want.keys.shape[0] and x["stats"][12] == want.vals.shape[0]
    return x


OPS_JSON = (
    '{"ops":[{"type":"COT_DELETE","params":"","rules":[{"type":"FRT_HASHKEY_PATTERN","params":'
    '"{\\"pattern\\":\\"\\\\u0001\\",\\"match_type\\":\\"SMT_MATCH_PREFIX\\"}"}]},'
    '{"type":"COT_UPDATE_TTL","params":"{\\"type\\":\\"UTOT_FROM_NOW\\",\\"value\\":10000}","rules":['
    '{"type":"FRT_SORTKEY_PATTERN","params":"{\\"pattern\\":\\"7\\",\\"match_type\\":\\"SMT_MATCH_POSTFIX\\"}"},'
    '{"type":"FRT_TTL_RANGE","params":"{\\"start_ttl\\":0,\\"stop_ttl\\":50000}"}]}]}'
)

OPS_ANYWHERE_JSON = (
    '{"ops":[{"type":"COT_DELETE","params":"","rules":[{"type":"FRT_SORTKEY_PATTERN","params":'
    '"{\\"pattern\\":\\"01\\",\\"match_type\\":\\"SMT_MATCH_ANYWHERE\\"}"}]}]}'
)


@pytest.mark.parametrize("bottommost", [True, False])
def test_sim_l0_to_l1(pgs, oracle, sim, bottommost):
    runs = synth.compaction_runs(k=4, n_per_run=600)
    x = check(pgs, oracle, sim, runs, bottommost=bottommost, seg_weight=24 * 1024)
    assert x["nseg"] > 8


@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 16])
def test_sim_group_widths(pgs, oracle, sim, lanes):
    runs = synth.compaction_runs(k=3, n_per_run=300, seed=5)
    check(pgs, oracle, sim, runs, bottommost=True, lanes=lanes, seg_weight=16 * 1024)


def test_sim_filter_variants(pgs, oracle, sim):
    runs = synth.compaction_runs(k=3, n_per_run=400, seed=7)
    x = check(pgs, oracle, sim, runs, bottommost=True, default_ttl=3600, seg_weight=32 * 1024)
    assert x["stats"][9] > 0
    x = check(pgs, oracle, sim, runs[:2], bottommost=True, validate_hash=True, pidx=1, partition_version=3, seg_weight=32 * 1024)
    assert x["stats"][8] > 0
    x = check(pgs, oracle, sim, runs, bottommost=False, ops_json=OPS_JSON, seg_weight=32 * 1024)
    check(pgs, oracle, sim, runs, bottommost=True, enabled=False, seg_weight=32 * 1024)


def test_sim_ragged_records(pgs, oracle, sim):
    """keys of 0..300 bytes, values of 0..9000 bytes (blocks of one entry, entries larger than the block buffer),
    several versions of a key inside one run, tombstones, restart interval 1 and 3, small blocks."""
    runs = merge_inputs.ragged_records(11)
    for ri, bs in ((1, 256), (3, 512), (16, 4096)):
        for bm in (True, False):
            check(pgs, oracle, sim, runs, bottommost=bm, restart_interval=ri, block_size=bs, seg_weight=8 * 1024, default_ttl=50)


def test_sim_long_restart_arrays_and_near_buffer_values(pgs, oracle, sim):
    """restart interval 1 with tiny entries: a 4 KB block holds ~270 entries and spans many emit batches, so its restart
    array is carried across batches; values just below / above the emit block buffer switch between the batch and the
    in-place path right after such a block."""
    runs = merge_inputs.long_restart_arrays(5)
    for ri in (1, 2, 16):
        check(pgs, oracle, sim, runs, bottommost=True, restart_interval=ri, block_size=4096, seg_weight=64 * 1024)


def test_sim_single_run_and_empty_output(pgs, oracle, sim):
    runs = synth.compaction_runs(k=1, n_per_run=500, seed=3)
    check(pgs, oracle, sim, runs, bottommost=True, seg_weight=16 * 1024)
    # everything expired -> no output run
    check(pgs, oracle, sim, runs, bottommost=True, now=synth.NOW + 10_000_000, default_ttl=1, seg_weight=16 * 1024)


def test_sim_long_keys_widen_the_groups(pgs, oracle, sim):
    """2 KB user keys: a narrow group's key rows no longer fit shared memory, the geometry falls back to wider groups"""
    runs = merge_inputs.long_keys(3)
    check(pgs, oracle, sim, runs, bottommost=True, lanes=0, seg_weight=64 * 1024)


def test_sim_anywhere_rule_and_empty_hash_keys(pgs, oracle, sim):
    """a delete rule whose pattern matches inside the sort key ("01" of s0001, s0010..s0019, never at its start), and
    validate_hash over records with an empty hash key, whose sort key is hashed instead"""
    runs = merge_inputs.empty_hash_keys(21)
    x = check(pgs, oracle, sim, runs, bottommost=True, ops_json=OPS_ANYWHERE_JSON, seg_weight=16 * 1024)
    assert x["stats"][7] > 0
    x = check(pgs, oracle, sim, runs, bottommost=True, validate_hash=True, pidx=1, partition_version=3, seg_weight=16 * 1024)
    assert x["stats"][8] > 0


@pytest.mark.parametrize("block_size,ri", [(1024, 1), (1024, 2), (512, 3)])
def test_sim_carried_restart_arrays(pgs, oracle, sim, block_size, ri):
    """a block that spans batches closes in a batch in which the next block records restart points: the closed block's
    restart array keeps the offsets of its own entries (check_run_format)"""
    check(pgs, oracle, sim, merge_inputs.carried_restart_arrays(31), bottommost=True, restart_interval=ri, block_size=block_size,
          seg_weight=64 * 1024)
