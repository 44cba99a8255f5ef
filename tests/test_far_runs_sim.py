"""Runs whose bytes lie past 2^32 (tests/far_runs.py) inside the host SIMT interpreter: the upload's index and filter, k_get,
k_scan_fwd and k_scan, the merge and the split read a moved run exactly as they read the same blocks at offset 0.  The
simulator runs the device sources with the library's plans, and 64-bit positions are 64-bit here too, so a truncation to
32 bits shows up as it would on the device.

Host memory: a far run spans 4.3 GB (8.6 GB for hi2), nearly all of it zeros.  The relocated numpy copy touches only its
blocks' pages, and the simulator holds a run of a gigabyte or more in a lazily zeroed mapping into which it copies only the
non-zero pages (load_run), so neither side pays for the span.  Measured for the whole file: a peak RSS of 0.9 GB and about
5 minutes on eight cores.  The `enough_memory` fixture skips a test when the machine has less than NEED_GB available.

A merge whose OUTPUT passes 4 GiB is not run here: it would take gigabytes of values through the interpreter's byte-wise
copies and about 15 GB of host memory; tests/test_far_runs_gpu.py runs it on the device."""
import os

import numpy as np
import pytest

import far_runs as fr
import foreign_blocks as fb
import split_model as sm
from far_runs import Layout, relocate
from get_model import query_keys, sweep_items, sweep_keys, uploaded_run
from incubator_pegasus_b200 import Records, RunInfo, synth
from scan_model import filter_list, make_db, mirror, model_scan, scan_list, visible
from test_foreign_blocks_sim import FULL, SCAN_HKS, args_of, check_same_merge, sim_index
from test_kernel_sim import sim, sim_compact  # noqa: F401  (fixture + helper)
from test_read_kernels_sim import check_lookup, check_scans, do_scans, sample
from test_split_sim import check_split, ssim  # noqa: F401  (fixture + helper)

NOW = synth.NOW
NEED_GB = 4
SEG_WEIGHT, SEG_REC_COST = 128 << 10, 256   # kSegWeight, kSegRecCost (compact_kernels.cuh): the simulator's default budget


@pytest.fixture(autouse=True)
def enough_memory():
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail < NEED_GB << 30:
        pytest.skip("the far runs' merges and splits need %d GB of host memory, %.1f GB available" % (NEED_GB, avail / 2**30))


# ---- the inputs ---------------------------------------------------------------------------------------------------------------
def hot_records(seed):
    """a key with 300 versions (tombstones among them) over many blocks, 4 KB keys, keys of 0..300 bytes"""
    rng = np.random.default_rng(seed)
    return Records.from_list(sweep_items(rng, 1, sweep_keys(rng), NOW, hot=300)[0])


def inputs(pgs):
    """name -> BlockRun at offset 0: the builder's blocks of the edge set, of 1300 tiny entries, of a hot key"""
    return {"edge": pgs.build_run(fb.edge_records(1), 4096, 16), "tiny": pgs.build_run(fb.tiny_records(2), 4096, 16),
            "hot": pgs.build_run(hot_records(3), 512, 4)}


def layout_for(br, name):
    """a Layout of br for `name` around the middle of the run: for shift_cross / hi2 the first block from the middle on with
    eight entries or more, the boundary inside a value in the middle of it; for end_at the first block whose size is a
    multiple of 16, else the one before the middle"""
    nb = br.n_blocks
    mid = nb // 2
    if name in ("shift_cross", "hi2"):
        for b in list(range(mid, nb)) + list(range(mid)):
            n = len(fr.block_entries(br, b))
            if n >= 8:
                try:
                    fr._crossing_value(br, b, n // 2, 2 * fr.G4)
                    return Layout(name, b, n // 2)
                except AssertionError:
                    continue
        raise AssertionError("no block of eight entries holds a value across a multiple of 16")
    if name == "end_at":
        return Layout(name, next((b for b in list(range(mid, nb - 1)) + list(range(mid)) if int(br.blk_size[b]) % 16 == 0), max(0, mid - 1)))
    if name == "all_above":
        return Layout(name, 0, 5)
    return Layout(name, max(0, min(mid, nb - 2)))


def moved(br, name):
    return relocate(br, layout_for(br, name))


# ---- k_index_walk and the filter ------------------------------------------------------------------------------------------------
INFO_FIELDS = [f for f, _ in RunInfo._fields_ if f not in ("run_id", "level", "data_bytes")]


@pytest.mark.parametrize("data", ["edge", "tiny", "hot"])
@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_sim_index_of_a_moved_run(pgs, sim, name, data):
    """blk_rec, ikey_off, the index keys, rec_off and the Bloom filter are the compact run's bit for bit; run_info differs only
    in data_bytes, which is the moved run's end"""
    br = inputs(pgs)[data]
    m = fb.model_index(br)
    n_lines = uploaded_run(br).bloom.n_lines
    st, want = sim_index(pgs, sim, br, len(m["rec_off"]), len(m["ikeys"]), n_lines, arrays=True)
    assert st == 0
    far = moved(br, name)
    st, got = sim_index(pgs, sim, far, len(m["rec_off"]), len(m["ikeys"]), n_lines, arrays=True)
    assert st == 0
    for k in ("blk_rec", "ikey_off", "ikeys", "rec_off", "bloom"):
        assert np.array_equal(got[k], want[k]), k
    assert (got["n_bloom_entries"], got["bloom_lines"]) == (want["n_bloom_entries"], want["bloom_lines"])
    for f in INFO_FIELDS:
        assert getattr(got["info"], f) == getattr(want["info"], f), f
    assert got["info"].data_bytes == far.data.shape[0] > fr.G4


# ---- k_get ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_sim_get_on_a_moved_run(pgs, sim, name):
    """three runs, the newest moved (a sweep of keys of 0..300 bytes, 4 KB keys, a hot key of 250 versions in the oldest run):
    answers, arena use and the probe / skip counters equal the model's.  For shift_cross and hi2 the entry whose value holds
    the boundary is looked up and found."""
    rng = np.random.default_rng(80 + fr.LAYOUTS.index(name))
    items = sweep_items(rng, 3, sweep_keys(rng), NOW, hot=250)
    brs = [pgs.build_run(pgs.Records.from_list(it), 1024, 4) for it in items]
    runs = [uploaded_run(b) for b in brs]
    lay = layout_for(brs[0], name)
    far = relocate(brs[0], lay)
    keys = sample(rng, query_keys(runs), 1500)
    if name in ("shift_cross", "hi2"):
        e = fr.block_entries(brs[0], lay.block)[fr._crossing_value(brs[0], lay.block, lay.entry, 2 * fr.G4)[0]]
        k = e.key[:-8]
        assert runs[0].newest[k][0] == 1   # the newest version of its key, a value
        keys.append(k)
    assert check_lookup(pgs, sim, args_of([far] + brs[1:]), runs, keys) > 100


# ---- k_scan_fwd, k_scan -------------------------------------------------------------------------------------------------------------
def scan_db(pgs, seed, n_runs, name):
    """make_db's runs in 512-byte blocks, the newest moved"""
    rng = np.random.default_rng(seed)
    recs, items = make_db(pgs, rng, n_runs, SCAN_HKS, 24)
    brs = [pgs.build_run(r, 512, 4) for r in recs]
    return [moved(brs[0], name)] + brs[1:], items


@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_sim_scan_forward_on_a_moved_run(pgs, sim, name):
    """k_scan_fwd over three runs; the layouts take 8, 16 and 32 lanes per group in turn"""
    i = fr.LAYOUTS.index(name)
    brs, items = scan_db(pgs, 900 + i, 3, name)
    reqs = scan_list(SCAN_HKS)[::2] + filter_list(FULL)
    check_scans(visible(items)[0], reqs, do_scans(pgs, sim, args_of(brs), reqs, (8, 16, 32)[i % 3]))


@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_sim_scan_reverse_on_a_moved_run(pgs, sim, name):
    """k_scan with the minimal staging pool (about one block of every run per chunk, so chunk boundaries fall next to 2^32):
    all reverse, and forward and reverse interleaved"""
    brs, items = scan_db(pgs, 950 + fr.LAYOUTS.index(name), 2, name)
    vis = visible(items)[0]
    fwd = scan_list(SCAN_HKS)[::4] + filter_list(FULL)[::3]
    rev = [mirror(q) for q in fwd]
    check_scans(vis, rev, do_scans(pgs, sim, args_of(brs), rev, pool=1))
    mixed = [q for pair in zip(fwd[0::2], rev[1::2]) for q in pair]
    check_scans(vis, mixed, do_scans(pgs, sim, args_of(brs), mixed, pool=1))


@pytest.mark.parametrize("name", ["shift_cross", "gap_spans_segments"])
def test_sim_scan_multi_partition_with_a_moved_run(pgs, sim, name):
    """one launch over two partitions: slot 0 holds the moved run, slot 1 a run at offset 0, slot 2 nothing"""
    brs, items = scan_db(pgs, 990, 2, name)
    vis_of = [visible(items[:1])[0], visible(items[1:])[0], []]
    reqs = [q for q in scan_list(SCAN_HKS)[::3] for _ in range(3)]
    got = do_scans(pgs, sim, args_of(brs), reqs, 0x100)
    for i, (q, g_) in enumerate(zip(reqs, got)):
        assert g_ == model_scan(vis_of[i % 3], q, NOW), (i, q)


# ---- k_walk + k_emit --------------------------------------------------------------------------------------------------------------
def merge_records():
    """the edge set (4 KB keys, twelve versions of two keys, tombstones) over 600 tiny entries"""
    return [fb.edge_records(7), fb.tiny_records(4, 600)]


@pytest.mark.parametrize("name", fr.LAYOUTS)
def test_sim_merge_of_moved_inputs_as_one_segment(pgs, oracle, sim, name):
    """the newer input moved: as one segment the output is byte-identical to the merge of the compact inputs (and is the
    oracle's); the layouts take 1, 4 and 16 lanes per group in turn, so every width meets two of them"""
    recs = merge_records()
    brs = [pgs.build_run(r, 4096, 16) for r in recs]
    inp = [moved(brs[0], name), brs[1]]
    i = fr.LAYOUTS.index(name)
    lanes = (1, 4, 16)[i % 3]
    assert check_same_merge(pgs, oracle, sim, recs, inp, bottommost=i % 2 == 0, default_ttl=50, seg_weight=1 << 40, lanes=lanes) == 1


def planned_segments(brs):
    """compact_geometry's segment count at the default budget: every run weighs its data_bytes (the end of its last block,
    gaps and the offset of its first block included) and 256 per record"""
    w = sum(((int(b.blk_off[-1]) + int(b.blk_size[-1]) + 15) & ~15) + SEG_REC_COST * len(fb.model_index(fr.compact(b))["rec_off"]) for b in brs)
    return (w + SEG_WEIGHT - 1) // SEG_WEIGHT


@pytest.mark.parametrize("name", ["shift_cross", "gap_spans_segments"])
def test_sim_merge_of_moved_inputs_planned(pgs, oracle, sim, name):
    """the default planner over a moved input: tens of thousands of segments, nearly all of them over bytes no block holds,
    and the oracle's records.  The run's weight counts from offset 0, so the segments in front of its first block and (for
    gap_spans_segments) those over the gap are empty."""
    newer = Records.from_list([(k, s + 10_000, t, v) for k, s, t, v in fb.tiny_records(6, 2000).to_list()])
    recs = [newer, fb.tiny_records(4, 3000)]   # short keys: the scratch of 32 768 segments stays small (4 KB keys need GBs)
    brs = [pgs.build_run(r, 4096, 16) for r in recs]
    inp = [moved(brs[0], name), brs[1]]
    nseg = check_same_merge(pgs, oracle, sim, recs, inp, bottommost=False, seg_weight=0, lanes=4)
    assert nseg == planned_segments(inp) > fr.G4 // SEG_WEIGHT


# ---- the split ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["shift_cross", "end_at", "hi2", "gap_spans_segments"])
def test_sim_split_of_a_moved_run(pgs, ssim, name):
    """k_split_walk's descriptors carry 40-bit value offsets as the merge's do: every child is split_model's.  The edge set
    (4 KB keys) as one segment; for gap_spans_segments also tiny entries under the default planner (tens of thousands of
    segments, which would need gigabytes of scratch with 4 KB keys)"""
    cases = [(fb.edge_records(9), dict(seg_weight=1 << 40))]
    if name == "gap_spans_segments":
        cases.append((fb.tiny_records(5, 3000), {}))
    for recs, kw in cases:
        br = pgs.build_run(recs, 4096, 16)
        items = fb.decode(br).to_list()
        assert sum(1 for c in sm.split_items(items, 1, 4)[0] if c) >= 3
        check_split(pgs, ssim, moved(br, name), 1, 4, items=items, **kw)
