"""The runs of tests/foreign_blocks.py on the device, through the C ABI: upload (run info, download), get_batch with its
counters, forward, reverse and multi-partition scans, compaction, SST export / ingest, a checkpoint, and the upload's verdict on damaged blocks.

RULE OF THIS FILE.  The purpose of the damaged copies is a status code.  Every read k_index_walk makes is bounded by the
block's own handle, and a bad handle is refused on the host, so a damaged block is answered, not faulted on.  No test here
issues a get, scan or compaction on a run the model rejects.  If the device accepts a run the model rejects (or the reverse)
the test fails at that assertion and does nothing further with the run; such a disagreement is reproduced in the simulator
(tests/test_foreign_blocks_sim.py runs the same copies, also under AddressSanitizer), not by repeating the device run.  The
simulator file is green, plain and under AddressSanitizer, before this file is run."""
import ctypes as C

import numpy as np
import pytest

import foreign_blocks as fb
import merge_inputs
from foreign_blocks import GRID, POLICIES, record_sets
from get_model import check_results, flat_keys, model_get, model_stats, query_keys, sweep_items, sweep_keys, uploaded_run
from incubator_pegasus_b200 import synth
from scan_model import filter_list, make_db, mirror, model_scan, scan_list, visible
from test_scan_kernels_gpu import run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW


def check_upload(pgs, part, br, rid):
    m = fb.model_index(br)
    info = part.run_info(rid)
    for f, want in m["info"].items():
        assert getattr(info, f) == want, (f, getattr(info, f), want)
    # pgs_run_download: the run's bytes up to the 16-aligned end of its last block, as uploaded (gaps kept), and its handles
    got = part.download(rid)
    n = m["info"]["data_bytes"]
    assert got.blk_off.tolist() == br.blk_off.tolist() and got.blk_size.tolist() == br.blk_size.tolist()
    for o, s in zip(br.blk_off.tolist(), br.blk_size.tolist()):
        assert got.data[o:o + s].tobytes() == br.data[o:o + s].tobytes()
    keep = min(n, br.data.shape[0])
    assert got.data.shape[0] == n and got.data[:keep].tobytes() == br.data[:keep].tobytes() and not got.data[keep:].any()
    assert pgs.decode_blocks(got).same_as(fb.decode(br))


@pytest.mark.parametrize("policy", list(GRID))
def test_upload_of_foreign_runs(pgs, engine, policy):
    part = engine.partition()
    sets = list(record_sets().values())
    brs = [fb.encode_run(r, seed=i, **GRID[policy]) for i, r in enumerate(sets)]
    for br in brs[:3]:
        check_upload(pgs, part, br, part.upload(br))
    # one pipelined call that mixes foreign runs and runs of the library's builder
    mixed = brs[3:] + [pgs.build_run(sets[0]), fb.encode_run(fb.tiny_records(2), seed=1, **dict(GRID[policy], block_cut=60_000))]
    for br, rid in zip(mixed, part.upload_many(mixed)):
        check_upload(pgs, part, br, rid)
    part.close()


@pytest.mark.parametrize("n_runs", [1, 4])
def test_get_batch_on_foreign_runs(pgs, engine, n_runs):
    rng = np.random.default_rng(60 + n_runs)
    items = sweep_items(rng, n_runs, sweep_keys(rng), NOW, hot=300)
    brs = [fb.encode_run(pgs.Records.from_list(it), seed=i, **POLICIES[(3 * n_runs + i) % len(POLICIES)]) for i, it in enumerate(items)]
    part = engine.partition()
    for br in brs[::-1]:  # the newest run is uploaded last
        part.upload(br)
    runs = [uploaded_run(b) for b in brs]
    keys = query_keys(runs)
    flat, off = flat_keys(keys)
    st, res, arena, used = part.get_batch(flat, off, NOW, arena_cap=1 << 24)
    assert st == 0
    want = [model_get(runs, k, NOW) for k in keys]
    assert check_results(res, arena, keys, want) > 100
    assert (engine.last_blocks_probed, engine.last_runs_skipped) == model_stats(runs, keys)
    part.close()


FULL = dict(start=b"", stop=b"\xff" * 4, start_inclusive=True, stop_inclusive=True, key_mode=0, max_count=1000, max_iter_count=1000,
            max_iter_size=0)
SCAN_HKS = [b"h%d" % i for i in range(5)] + [b"", bytes([0xff, 0xff]), b"W" * 130]


def test_scans_on_foreign_runs(pgs, engine):
    """forward batches (k_scan_fwd), reverse and mixed batches (k_scan, which reaches every entry through rec_off), and one
    multi-partition launch over a partition of foreign runs and one of runs the library's builder wrote"""
    rng = np.random.default_rng(700)
    recs, items = make_db(pgs, rng, 4, SCAN_HKS, 24)
    a, b = engine.partition(pidx=0), engine.partition(pidx=1)
    for i, r in list(enumerate(recs))[::-1]:  # newest last
        (a if i < 2 else b).upload(fb.encode_run(r, seed=i, **POLICIES[(1 + 3 * i) % len(POLICIES)]) if i < 2 else pgs.build_run(r, 512, 4))
    vis_a, vis_b = visible(items[:2])[0], visible(items[2:])[0]
    fwd = scan_list(SCAN_HKS) + filter_list(FULL)
    rev = [mirror(q) for q in fwd]
    for reqs in (fwd, rev, [q for pair in zip(fwd[0::2], rev[1::2]) for q in pair]):
        st, got = run_scans(pgs, a, reqs)
        assert st == 0
        for q, g_ in zip(reqs, got):
            assert g_ == model_scan(vis_a, q, NOW), q
    sb = pgs.ScanBatch(None, SCAN_HKS * 2, 200, 96 * 1024, parts=[a, b], req_part=[0] * len(SCAN_HKS) + [1] * len(SCAN_HKS))
    assert sb.run(NOW) == 0
    for j, hk in enumerate(SCAN_HKS * 2):
        vis = vis_a if j < len(SCAN_HKS) else vis_b
        want = [(k[2 + len(hk):], v[12:]) for k, v in vis if k[:2 + len(hk)] == len(hk).to_bytes(2, "big") + hk
                and not 0 < int.from_bytes(v[:4], "big") <= NOW]
        assert sb.records(j) == want, (j, hk)
    a.close(); b.close()


@pytest.mark.parametrize("block_size", [0, 16384])
def test_compact_foreign_runs(pgs, oracle, block_size):
    """the compaction of foreign runs gives the oracle's records and counters.  Segments are cut at input block boundaries,
    so the output BYTES depend on where the input blocks end and on nothing else of the encoding: foreign runs cut where the
    builder cuts (other shared lengths, restart points and gaps) give the bytes the builder's runs give."""
    recs = merge_inputs.empty_hash_keys(21)
    want, st = oracle.compact([oracle.Run.from_records(r) for r in recs], True, oracle.filter_params(default_ttl=50), NOW)
    canonical = [pgs.build_run(r) for r in recs]
    same_cuts = [fb.encode_run(r, seed=i, shared=("random", "zero", "exact_minus_one")[i % 3], restart=("irregular", 1, "single")[i % 3], gaps=2,
                               block_cut=np.diff(fb.model_index(c)["blk_rec"]).tolist()) for i, (r, c) in enumerate(zip(recs, canonical))]
    other_cuts = [fb.encode_run(r, seed=i, **POLICIES[(1 + 3 * i) % len(POLICIES)]) for i, r in enumerate(recs)]
    with pgs.Engine(block_size=block_size) as eng:
        outs = []
        for brs in (canonical, same_cuts, other_cuts):
            part = eng.partition()
            ids = [part.upload(b) for b in brs[::-1]][::-1]
            res = part.compact(ids, out_level=1, bottommost=1, now=NOW, default_ttl=50)
            out = part.download(res.new_run_id)
            assert pgs.decode_blocks(out).same_as(want.records())
            for f in ("in_records", "out_records", "dropped_shadowed", "dropped_tombstone", "dropped_expired", "ttl_rewritten"):
                assert getattr(res, f) == getattr(st, f), f
            outs.append((out, res.n_tiles))
            part.close()
        (a, na), (b, nb), _ = outs
        assert na == nb and a.blk_off.tolist() == b.blk_off.tolist() and a.blk_size.tolist() == b.blk_size.tolist()
        assert a.data.tobytes() == b.data.tobytes()


def big_run(pgs):
    """40 MB of 1 KB values in 4 KB blocks with gaps: the pipelined upload moves it in two chunks"""
    rng = np.random.default_rng(8)
    pool = rng.integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    items = [(b"\x00\x03big%07d" % i, i + 1, 1, bytes(4) + pool[(i * 37) % 1000000:][:1020]) for i in range(40_000)]
    br = fb.encode_run(pgs.Records.from_list(items), seed=5, shared="random", varints="padded", restart="irregular", block_cut=4096, gaps=3, tail=9)
    off = br.blk_off.tolist()
    cut = next(b for b in range(1, br.n_blocks) if off[b] - off[0] >= 32 << 20)  # upload_stage_a's first chunk is [0, cut)
    assert cut < br.n_blocks - 8 and off[cut] >= off[cut - 1] + int(br.blk_size[cut - 1]) + 16, "no gap at the chunk boundary"
    return br, cut


def test_upload_of_a_run_of_two_chunks_with_a_gap_at_the_boundary(pgs, engine):
    part = engine.partition()
    br, cut = big_run(pgs)
    check_upload(pgs, part, br, part.upload(br))
    # a damaged block in the SECOND chunk of the run in the middle of an upload_many: nothing of the call stays installed
    bad = pgs.BlockRun(br.data.copy(), br.blk_off, br.blk_size)
    b = cut + 3
    bad.data[int(br.blk_off[b]) + int(br.blk_size[b]) - 4:int(br.blk_off[b]) + int(br.blk_size[b])] = 0  # restart count 0
    assert fb.walk_block(fb.run_blocks(bad)[b])[0] == fb.CORRUPTION
    small = fb.mutant_base(1)
    before = part.runs()
    with pytest.raises(pgs.PegasusError) as e:
        part.upload_many([small, bad, small])
    assert e.value.code == fb.CORRUPTION and part.runs() == before
    part.close()


def test_sst_export_and_ingest_of_a_foreign_run(pgs, engine):
    """pgs_sst_export of a resident foreign run -> pgs_sst_ingest re-enters the upload path: the same records"""
    L = pgs.lib()
    L.pgs_sst_export.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.pgs_sst_ingest.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    a, b = engine.partition(pidx=0), engine.partition(pidx=1)
    for i, (name, recs) in enumerate(record_sets().items()):
        rid = a.upload(fb.encode_run(recs, seed=i, **POLICIES[i % len(POLICIES)]))
        n = C.c_uint64()
        assert L.pgs_sst_export(a.h, rid, None, 0, C.byref(n)) == pgs.INCOMPLETE
        img = np.zeros(n.value, np.uint8)
        assert L.pgs_sst_export(a.h, rid, img.ctypes.data, img.shape[0], C.byref(n)) == 0
        rid2 = C.c_uint64()
        assert L.pgs_sst_ingest(b.h, 1, img.ctypes.data, n.value, C.byref(rid2)) == 0
        assert pgs.decode_blocks(b.download(rid2.value)).same_as(recs), name
    a.close(); b.close()


def test_checkpoint_of_a_replica_that_holds_a_foreign_run(pgs, engine, tmp_path):
    """a replica with a foreign run writes a checkpoint, a second replica applies it (the upload path again): it holds the
    same records and answers the same multi_get"""
    import os
    from rrdb_harness import Backend, same_response
    recs = merge_inputs.empty_hash_keys(21)[0]
    g, g2 = Backend("gpu", engine, pidx=23), Backend("gpu", engine, pidx=23)
    try:
        g.put(b"h1", b"written", b"v", now=NOW)
        g.flush(NOW)
        part = pgs.Partition(engine, 1, 23, 1, handle=pgs.lib().pgs_rrdb_partition(g.h))
        part.upload(fb.encode_run(recs, seed=2, **GRID["random-pad-rirr-irr-gaps"]), level=1)
        d = C.c_int64()
        base = str(tmp_path / "ckpt").encode()
        assert g.f("rrdb_sync_checkpoint")(g.h, base, NOW, C.byref(d)) == 0
        assert g2.f("rrdb_apply_checkpoint")(g2.h, os.path.join(base.decode(), "checkpoint.%d" % d.value).encode()) == 0
        part2 = pgs.Partition(engine, 1, 23, 1, handle=pgs.lib().pgs_rrdb_partition(g2.h))
        held = [pgs.decode_blocks(part2.download(r)) for r in part2.runs()]
        assert any(h.same_as(recs) for h in held)
        for hk in (b"", b"h1", b"a01b", b"h22"):
            for kw in (dict(), dict(reverse=True, max_kv_count=7)):
                ok, diff_ = same_response(g.multi_get(hk, now=NOW, **kw), g2.multi_get(hk, now=NOW, **kw))
                assert ok, (hk, kw, diff_)
    finally:
        g.close(); g2.close()


def test_upload_verdicts_equal_the_model(pgs, engine):
    """every damaged copy of foreign_blocks.mutants: the status of pgs_run_upload is classify's, an accepted copy decodes to
    the model's records after a download, and nothing else is done with any of them (see the rule above)"""
    part = engine.partition()
    base = fb.mutant_base(1)
    for name, m, want in fb.mutants(base, 3):
        try:
            rid = part.upload(m)
            got = fb.OK
        except pgs.PegasusError as e:
            got = e.code
        assert got == want, (name, got, want)
        if got == fb.OK:
            assert pgs.decode_blocks(part.download(rid)).same_as(fb.decode(m)), name
            part.drop(rid)
    assert part.runs() == []
    part.close()


def test_damaged_run_in_the_middle_of_upload_many_installs_nothing(pgs, engine):
    part = engine.partition()
    base = fb.mutant_base(1)
    bad = [m for n, m, _ in fb.mutants(base, 3) if n == "damage_in_last_cta"][0]
    with pytest.raises(pgs.PegasusError) as e:
        part.upload_many([base, pgs.build_run(fb.edge_records(1)), bad, base])
    assert e.value.code == fb.CORRUPTION and part.runs() == []
    part.close()
