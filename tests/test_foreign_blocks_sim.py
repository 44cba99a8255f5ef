"""The device decoders on runs the library's builder never writes (tests/foreign_blocks.py), inside the host SIMT
interpreter: k_index_walk (upload), cur_decode of k_get / k_scan_fwd, the head-window decoder of k_walk and the staging
decoder of k_scan all read short and zero shared prefixes, padded varints, irregular restart arrays, ragged block sizes,
gaps between blocks and bytes behind the last one; the upload's verdict on damaged blocks equals foreign_blocks.classify,
and whatever it accepts, the readers decode as foreign_blocks.decode does.

The file also passes against the AddressSanitizer build of the simulator, which checks every load of the decoders against
the exact sizes the library allocates (a decoder that reads past a block shows up as a report with a source line):

    bash tools/simt/build.sh asan
    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_foreign_blocks_sim.py
    bash tools/simt/build.sh

Key ORDER and record types inside a run are not validated by the upload; a damaged copy that the model accepts is read
back only when its records are still in order and of the two known types (foreign_blocks.readable)."""
import ctypes as C

import numpy as np
import pytest

import foreign_blocks as fb
import merge_inputs
from get_model import Bloom, prefix_len, query_keys, sweep_items, sweep_keys, uploaded_run
from incubator_pegasus_b200 import synth
from scan_model import filter_list, make_db, mirror, model_scan, scan_list, visible
from test_kernel_sim import STAT_FIELDS, sim, sim_compact  # noqa: F401  (fixture + helper)
from test_read_kernels_sim import check_lookup, check_scans, do_scans, sample

NOW = synth.NOW

GRID, POLICIES, record_sets = fb.GRID, fb.POLICIES, fb.record_sets


def args_of(brs):
    k = len(brs)
    return (k, (C.c_void_p * k)(*[b.data.ctypes.data for b in brs]), (C.c_uint64 * k)(*[b.data.shape[0] for b in brs]),
            (C.c_void_p * k)(*[b.blk_off.ctypes.data for b in brs]), (C.c_void_p * k)(*[b.blk_size.ctypes.data for b in brs]),
            (C.c_uint32 * k)(*[b.n_blocks for b in brs]))


def sim_index(pgs, sim, br, n_rec=0, n_key=0, n_lines=0, arrays=False):
    """sim_run_index -> (status, what the upload built).  arrays: copy the index arrays and the filter out too; n_rec, n_key
    and n_lines are then the model's record count, index-key bytes and filter lines, which size the buffers"""
    info, nbe, lines = pgs.RunInfo(), C.c_uint64(), C.c_uint32()
    nb = br.n_blocks
    blk_rec, ikey_off = np.zeros(nb + 1, np.uint32), np.zeros(nb + 1, np.uint32)
    ikeys, rec_off, bloom = np.zeros(n_key + 1, np.uint8), np.zeros(n_rec + 1, np.uint32), np.zeros(16 * n_lines + 16, np.uint32)
    p = (lambda a: a.ctypes.data_as(C.c_void_p)) if arrays else (lambda a: None)
    st = sim.sim_run_index(br.data.ctypes.data_as(C.c_void_p), C.c_uint64(br.data.shape[0]), br.blk_off.ctypes.data_as(C.c_void_p),
                           br.blk_size.ctypes.data_as(C.c_void_p), nb, C.byref(info), C.byref(nbe), C.byref(lines), p(blk_rec), p(ikey_off),
                           C.c_uint64(nb + 1), p(ikeys), C.c_uint64(n_key), p(rec_off), C.c_uint64(n_rec), p(bloom), C.c_uint64(bloom.shape[0]))
    return st, dict(info=info, n_bloom_entries=nbe.value, bloom_lines=lines.value, blk_rec=blk_rec, ikey_off=ikey_off, ikeys=ikeys[:n_key],
                    rec_off=rec_off[:n_rec], bloom=bloom[:16 * n_lines])


# ---- the writer itself ----------------------------------------------------------------------------------------------------
def test_writer_round_trips_through_three_decoders(pgs, oracle):
    """for every policy row and record set: the library's host decoder, the oracle's and foreign_blocks.decode return the
    input records; over all of them the block sizes take the residues 0, 1 and 15 mod 16, blocks of one entry and a block
    of more than a thousand occur"""
    residues, counts = set(), set()
    sets = dict(record_sets(), tiny=fb.tiny_records(2))
    for name, recs in sets.items():
        for pi, pol in enumerate(POLICIES + [dict(POLICIES[0], block_cut=60_000)]):
            br = fb.encode_run(recs, seed=pi, **pol)
            assert fb.classify(br) == fb.OK
            for got in (pgs.decode_blocks(br), oracle.Run.from_blocks(br).records(), fb.decode(br)):
                assert got.same_as(recs), (name, pol)
            residues |= set((br.blk_size % 16).tolist())
            counts |= set(np.diff(fb.model_index(br)["blk_rec"]).tolist())
    assert {0, 1, 15} <= residues and 1 in counts and max(counts) >= 1000


def test_named_mutants_get_the_verdict_they_were_built_for():
    all_ = list(fb.mutants(fb.mutant_base(1), 3))
    for name, m, want in all_:
        assert fb.classify(m) == want, name
    names = [n for n, _m, _st in all_]
    assert len(names) == len(set(names)) and sum(n.startswith("byte_") for n in names) == fb.N_RANDOM
    assert {fb.OK, fb.CORRUPTION} <= {st for n, _m, st in all_ if n.startswith("byte_")}


# ---- k_index_walk ---------------------------------------------------------------------------------------------------------
def check_index(pgs, sim, br):
    m, f = fb.model_index(br), uploaded_run(br)
    st, x = sim_index(pgs, sim, br, len(m["rec_off"]), len(m["ikeys"]), f.bloom.n_lines, arrays=True)
    assert st == 0
    assert x["rec_off"].tolist() == m["rec_off"] and x["blk_rec"].tolist() == m["blk_rec"]
    assert x["ikey_off"].tolist() == m["ikey_off"] and x["ikeys"].tobytes() == m["ikeys"]
    for name, want in m["info"].items():
        assert getattr(x["info"], name) == want, (name, getattr(x["info"], name), want)
    # the filter: sized by pass 1's count, filled by pass 2 -- both follow the rule of get_model.uploaded_run, bit for bit
    assert x["n_bloom_entries"] == f.n_bloom_entries and x["bloom_lines"] == f.bloom.n_lines
    assert np.array_equal(x["bloom"], f.bloom.words())
    # and the words the simulated upload wrote reject no stored key and no hash-key prefix of one
    built = Bloom(f.bloom.n_lines)
    built.lines = [sum(int(w) << (32 * i) for i, w in enumerate(x["bloom"][16 * li:16 * li + 16])) for li in range(built.n_lines)]
    for k in f.newest:
        assert built.may_contain(k) and (not prefix_len(k) or built.may_contain(k[:prefix_len(k)])), k


@pytest.mark.parametrize("policy", list(GRID))
def test_sim_index_of_foreign_runs(pgs, sim, policy):
    for i, (name, recs) in enumerate(record_sets().items()):
        check_index(pgs, sim, fb.encode_run(recs, seed=i, **GRID[policy]))


def test_sim_index_of_a_block_of_1300_entries_and_a_2mib_value(pgs, sim):
    check_index(pgs, sim, fb.encode_run(fb.tiny_records(2), seed=1, **dict(GRID["random-pad-rirr-irr-gaps"], block_cut=60_000)))
    check_index(pgs, sim, fb.encode_run(fb.edge_records(5, big_value=(2 << 20) + 5), seed=2, **GRID["cap3-pad-r1-256-gaps"]))


# ---- k_get ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_runs", [1, 4])
def test_sim_get_on_foreign_runs(pgs, sim, n_runs):
    """the key sweep of the get tests (user keys of 0..300 bytes, hash keys of 0..140, 4 KB keys) over 1..4 foreign runs, each
    with another policy row: answers, arena use and the probe / skip counters equal the model's"""
    rng = np.random.default_rng(60 + n_runs)
    items = sweep_items(rng, n_runs, sweep_keys(rng, long_keys=n_runs < 4), NOW, hot=120)
    brs = [fb.encode_run(pgs.Records.from_list(it), seed=i, **POLICIES[(3 * n_runs + i) % len(POLICIES)]) for i, it in enumerate(items)]
    runs = [uploaded_run(b) for b in brs]
    keys = sample(rng, query_keys(runs), 400)
    assert check_lookup(pgs, sim, args_of(brs), runs, keys) > 40


# ---- k_scan_fwd, k_scan -----------------------------------------------------------------------------------------------------
SCAN_HKS = [b"h%d" % i for i in range(5)] + [b"", b"h1x", bytes([0xff, 0xff]), b"W" * 130]
FULL = dict(start=b"", stop=b"\xff" * 4, start_inclusive=True, stop_inclusive=True, key_mode=0, max_count=1000, max_iter_count=1000,
            max_iter_size=0)


def scan_db(pgs, seed, n_runs, first=0, canonical=()):
    rng = np.random.default_rng(seed)
    recs, items = make_db(pgs, rng, n_runs, SCAN_HKS, 24)  # small values: k_scan's pool must hold one block of every run
    brs = [pgs.build_run(r, 512, 4) if i in canonical else fb.encode_run(r, seed=i, **POLICIES[(first + i) % len(POLICIES)])
           for i, r in enumerate(recs)]
    return brs, items


@pytest.mark.parametrize("n_runs,lanes,first", [(1, 0, 1), (3, 16, 4), (2, 32, 8)])
def test_sim_scan_forward_on_foreign_runs(pgs, sim, n_runs, lanes, first):
    brs, items = scan_db(pgs, 400 + n_runs, n_runs, first)
    reqs = scan_list(SCAN_HKS)[::2] + filter_list(FULL)
    check_scans(visible(items)[0], reqs, do_scans(pgs, sim, args_of(brs), reqs, lanes))


@pytest.mark.parametrize("n_runs,first,pool", [(1, 1, "minimal"), (3, 5, "product"), (4, 0, "minimal")])
def test_sim_scan_reverse_on_foreign_runs(pgs, sim, n_runs, first, pool):
    """a reverse request sends the batch through k_scan, whose staging decoder reaches every entry through rec_off: all
    reverse, and forward and reverse interleaved"""
    brs, items = scan_db(pgs, 500 + n_runs, n_runs, first)
    vis = visible(items)[0]
    fwd = scan_list(SCAN_HKS)[::2] + filter_list(FULL)[::2]
    rev = [mirror(q) for q in fwd]
    p = 0 if pool == "product" else 1
    check_scans(vis, rev, do_scans(pgs, sim, args_of(brs), rev, pool=p))
    mixed = [q for pair in zip(fwd[0::2], rev[1::2]) for q in pair]
    check_scans(vis, mixed, do_scans(pgs, sim, args_of(brs), mixed, pool=p))


def test_sim_scan_multi_partition_foreign_and_canonical(pgs, sim):
    """one launch over two partitions: slot 0 holds a foreign run, slot 1 one the library's builder wrote"""
    brs, items = scan_db(pgs, 600, 2, first=1, canonical=(1,))
    vis_of = [visible(items[:1])[0], visible(items[1:])[0], []]
    reqs = [q for q in scan_list(SCAN_HKS)[::3] for _ in range(3)]
    got = do_scans(pgs, sim, args_of(brs), reqs, 0x100)
    for i, (q, g_) in enumerate(zip(reqs, got)):
        assert g_ == model_scan(vis_of[i % 3], q, NOW), (i, q)


# ---- k_walk + k_emit ----------------------------------------------------------------------------------------------------------
def merged(pgs, sim, runs, **kw):
    out, x = sim_compact(pgs, sim, runs, **kw)
    return out.data.tobytes(), out.blk_off.tolist(), out.blk_size.tolist(), x["stats"]


def check_same_merge(pgs, oracle, sim, recs, foreign, **kw):
    """the merge depends on the records, not on how its inputs were encoded: the builder's encoding and the foreign ones give
    the same records, counters and run statistics, which are the oracle's.  Segments are cut at input block boundaries, so
    the output BYTES (where blocks end) are compared when both merges ran as one segment, and are identical then."""
    want, xw = sim_compact(pgs, sim, recs, **kw)
    got, xg = sim_compact(pgs, sim, foreign, **kw)
    layout_free = list(range(15)) + [17, 18]  # the counters of pgs_compact_result and the run statistics but block sizes / counts
    assert [xg["stats"][i] for i in layout_free] == [xw["stats"][i] for i in layout_free], (xg["stats"], xw["stats"])
    if xw["nseg"] == 1 and xg["nseg"] == 1:
        assert xg["stats"] == xw["stats"]
        assert got.blk_off.tolist() == want.blk_off.tolist() and got.blk_size.tolist() == want.blk_size.tolist()
        assert got.data.tobytes() == want.data.tobytes()
    okw = {k: v for k, v in kw.items() if k in ("enabled", "default_ttl")}
    orun, st = oracle.compact([oracle.Run.from_records(r) for r in recs], kw["bottommost"], oracle.filter_params(**okw), kw.get("now", NOW))
    for i, f in enumerate(STAT_FIELDS):
        assert xg["stats"][i] == getattr(st, f), f
    assert (got.n_blocks == 0) == (orun.records().n == 0)
    if got.n_blocks:
        assert pgs.decode_blocks(got).same_as(orun.records())
    return xg["nseg"]


MERGE_INPUTS = {"ragged": lambda: merge_inputs.ragged_records(11), "window_keys": lambda: merge_inputs.window_key_lengths(3),
                "crossings": lambda: merge_inputs.window_block_crossings(4), "empty_hash_keys": lambda: merge_inputs.empty_hash_keys(21),
                "synth": lambda: synth.compaction_runs(k=3, n_per_run=250, seed=5)}


def foreign_runs(recs, first):
    return [fb.encode_run(r, seed=i, **POLICIES[(first + 3 * i) % len(POLICIES)]) for i, r in enumerate(recs)]


@pytest.mark.parametrize("n,inputs", list(enumerate(MERGE_INPUTS)), ids=list(MERGE_INPUTS))
def test_sim_merge_of_foreign_runs(pgs, oracle, sim, n, inputs):
    """every input set under three policy rows, TTL filter on: as one segment (byte-identical output), and in segments of 8 KB
    that end inside foreign blocks, the oldest run in the builder's encoding"""
    recs = MERGE_INPUTS[inputs]()
    foreign = foreign_runs(recs, n)
    lanes = (1, 2, 4, 8, 16)
    assert check_same_merge(pgs, oracle, sim, recs, foreign, bottommost=True, default_ttl=50, seg_weight=1 << 40, lanes=lanes[n % 5]) == 1
    assert check_same_merge(pgs, oracle, sim, recs, foreign[:-1] + [recs[-1]], bottommost=False, default_ttl=50, seg_weight=8 * 1024,
                            lanes=lanes[(n + 2) % 5], block_size=512, restart_interval=4) > 4


@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 16])
def test_sim_merge_of_foreign_runs_at_every_group_width(pgs, oracle, sim, lanes):
    recs = merge_inputs.empty_hash_keys(21)
    one = lanes in (2, 8)  # as one segment, or in segments of 4 KB
    nseg = check_same_merge(pgs, oracle, sim, recs, foreign_runs(recs, lanes), bottommost=lanes % 3 == 1, seg_weight=1 << 40 if one else 4 * 1024,
                            lanes=lanes)
    assert nseg == 1 if one else nseg > 4


@pytest.mark.parametrize("shared", ["zero", "random", "exact_minus_one", ("cap", 10)], ids=str)
def test_sim_merge_shadow_fallback_inside_one_run(pgs, oracle, sim, shared):
    """one run that holds up to twelve versions of its keys, stored with less than the exact shared length: every older
    version is dropped as shadowed by the compare, not by the `shared` shortcut"""
    recs = [fb.edge_records(7)]
    foreign = [fb.encode_run(recs[0], seed=9, shared=shared, varints="minimal", restart="single", block_cut=300)]
    assert check_same_merge(pgs, oracle, sim, recs, foreign, bottommost=True, enabled=False, seg_weight=1 << 40, lanes=1) == 1
    check_same_merge(pgs, oracle, sim, recs, foreign, bottommost=True, enabled=False, seg_weight=4 * 1024, lanes=8)


# ---- the validator ------------------------------------------------------------------------------------------------------------
def test_sim_upload_verdicts_and_reads_of_accepted_mutants(pgs, oracle, sim):
    """every damaged copy gets classify's status from the simulated upload.  A copy the model accepts (a changed byte that
    left a decodable block) is then read by every decoder -- k_get for every key, a whole-range scan forward (k_scan_fwd)
    and in reverse (k_scan), a one-run compaction -- and each returns what foreign_blocks.decode returns (every eighth such
    copy: the interpreter is slow)."""
    base = fb.mutant_base(1)
    read_back = 0
    for name, m, want in fb.mutants(base, 3):
        st, _ = sim_index(pgs, sim, m)
        assert st == want, (name, st, want)
        if want != fb.OK or not name.startswith("byte_"):
            continue
        recs = fb.decode(m)
        if not fb.readable(recs):
            continue
        read_back += 1
        if read_back % 8:
            continue
        check_index(pgs, sim, m)
        run = uploaded_run(m)
        check_lookup(pgs, sim, args_of([m]), [run], sorted(run.newest) + [b"", b"\x00\x06mutant"])
        vis = visible([recs.to_list()])[0]
        reqs = [FULL, mirror(FULL)]
        check_scans(vis, reqs[:1], do_scans(pgs, sim, args_of([m]), reqs[:1]))
        check_scans(vis, reqs[1:], do_scans(pgs, sim, args_of([m]), reqs[1:]))
        check_same_merge(pgs, oracle, sim, [recs], [m], bottommost=False, enabled=False, lanes=4, seg_weight=1 << 40)
    assert read_back > 40
