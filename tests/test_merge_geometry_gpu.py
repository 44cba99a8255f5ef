"""The compaction kernels on the device at every block size and restart interval where k_emit / compact_geometry branch, fed
the edge inputs the simulator runs (tests/merge_inputs.py).  The simulator runs the same sources, but its bulk copies,
barriers and proxy fences are synchronous stand-ins: a missing fence, a stage rewritten before a store has read it or a
stale barrier phase can only fail here.  For every geometry and input: the merge against the oracle with both decoders,
every counter and run_info field, and the block format the decoders do not read (check_run_format: restart arrays, the cut
rule, padding); point lookups and forward / reverse scans of the merged run against the models; a second generation that
walks the GPU-written blocks through their entry index; and the same merge twice, byte for byte."""
import numpy as np
import pytest

import merge_inputs
from get_model import check_run_format, compacted_run, emit_geometry, key_slot, prefix_len, query_keys, uploaded_run
from incubator_pegasus_b200 import synth
from scan_model import mirror, model_scan, scan_list
from test_compaction_gpu import run_case
from test_get_kernel_gpu import check_batch
from test_kernel_sim import OPS_ANYWHERE_JSON
from test_scan_kernels_gpu import run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW
KEEP_INPUTS = 1  # PGS_COMPACT_KEEP_INPUTS (include/pegasus_b200.h)

GEOMETRIES = [  # block size, restart interval: the branch of k_emit / compact_geometry each one reaches
    (64, 1),          # a block smaller than almost every entry: emit_big for nearly all, one-entry blocks
    (256, 1),         # several blocks close per batch
    (512, 4),
    (4096, 1),        # ~270 tiny entries per block: restart offsets carried across batches
    (4096, 16),       # the default
    (4096, 128),      # one restart point per block
    (16384, 16),      # two CTAs of 3 warps per SM
    (65536, 16),      # one warp per CTA
    (80_000, 1),      # cut to ~74 KB
    (1 << 20, 1),
    (110_800, 16),    # cut to ~110 KB
    (1 << 20, 16),
]
CUT = {(80_000, 1), (1 << 20, 1), (110_800, 16), (1 << 20, 16)}

# name -> (the runs, filter arguments of the merge): the simulator's seeds and sizes
INPUTS = {
    "ragged": (lambda g: merge_inputs.ragged_records(11), dict(default_ttl=50)),
    "long_restart_arrays": (lambda g: merge_inputs.long_restart_arrays(5), {}),
    "long_keys": (lambda g: merge_inputs.long_keys(3), {}),
    "empty_hash_keys": (lambda g: merge_inputs.empty_hash_keys(21), dict(ops_json=OPS_ANYWHERE_JSON)),
    "window_key_lengths": (lambda g: merge_inputs.window_key_lengths(21), {}),
    "window_block_crossings": (lambda g: merge_inputs.window_block_crossings(22), {}),
    "window_end_of_buffer": (lambda g: merge_inputs.window_end_of_buffer(23), {}),
    "carried_restart_arrays": (lambda g: merge_inputs.carried_restart_arrays(31), {}),
    "huge_blocks": (lambda g: merge_inputs.huge_blocks(17), {}),
    "df_big_threshold": (lambda g: merge_inputs.df_big_threshold(41, g["blk_buf"]), {}),
}


def smem_budget():
    """compact_smem_budget: the device's opt-in shared memory per CTA less 1 KB"""
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 1024


@pytest.fixture(scope="module", params=GEOMETRIES, ids=lambda g: "bs%d-ri%d" % g)
def geo_engine(pgs, request):
    bs, ri = request.param
    eng = pgs.Engine(block_size=bs, restart_interval=ri)
    yield eng, bs, ri
    eng.close()


def max_ukey(runs):
    return max(int(np.diff(r.key_off.astype(np.int64)).max(initial=0)) for r in runs)


def test_restated_shapes_reach_their_branches():
    """the CTA shapes nothing in the ABI reports, from the restated rule with this device's shared memory"""
    smem = smem_budget()
    assert emit_geometry(4096, 16, 7, smem)["warps"] == 4
    assert emit_geometry(16384, 16, 7, smem) == dict(blk_buf=16416, block_size=16384, warps=3, twice=True)
    assert emit_geometry(65536, 16, 7, smem)["warps"] == 1
    for bs, ri in CUT:
        g = emit_geometry(bs, ri, 7, smem)
        assert g["block_size"] < bs and abs(g["block_size"] - (74_000 if ri == 1 else 110_000)) < 2_000, (bs, ri, g)


# ---- reads of the merged run -------------------------------------------------------------------------------------------
K_SCAN_STATIC = 5888  # k_scan's static shared memory (DESIGN §3.5)


def reverse_staging_fits(raw, counts, ks):
    """DESIGN §8: k_scan stages one largest block of every run (one run here): scan_min_pool and the key rows must fit the
    dynamic shared memory the device leaves it (scan_dyn_bytes, scan_max_dyn)"""
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    one = ((int(raw.blk_size.max()) + 15) & ~15) + 32 + max(counts) * (ks + 48)
    min_pool = one + 64 + 16 + 8 * (ks + 48)
    fixed = 5 * ((ks + 8 + 15) & ~15)
    return fixed + min_pool <= optin - K_SCAN_STATIC - 256


def scan_requests_for(model, vis):
    """whole-range scans, bounds on the first and last key of blocks across the run, iteration limits, multi_get over some
    hash keys; each also reversed"""
    full = dict(start=b"", stop=b"\xff" * 6, start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0,
                max_count=100000, max_iter_count=100000, max_iter_size=0)
    reqs = [full, dict(full, stop=b"\xff" * 400)]
    blocks = model.blocks
    for b in range(0, len(blocks), max(1, len(blocks) // 12)):
        first, last = blocks[b][0][0], blocks[b][-1][0]
        nxt = blocks[b + 1][0][0] if b + 1 < len(blocks) else last + b"\x00"
        for si in (True, False):
            reqs.append(dict(full, start=first, stop=last, start_inclusive=si, stop_inclusive=not si))
            reqs.append(dict(full, start=last, stop=nxt, start_inclusive=si, stop_inclusive=si))
    for n in (1, 2, 33, max(1, len(vis) // 2)):
        reqs.append(dict(full, max_iter_count=n))
    hks = sorted({k[2:prefix_len(k)] for k in model.newest if prefix_len(k)})
    reqs += scan_list(hks[:: max(1, len(hks) // 4)][:4])
    return reqs + [mirror(q) for q in reqs]


def check_reads(pgs, part, runs, raw, counts, bs, ri):
    model = compacted_run(raw, [uploaded_run(pgs.build_run(r, bs, ri)) for r in runs])
    check_batch(pgs, part, [model], query_keys([model]))
    vis = [(k, v) for k, (t, v) in sorted(model.newest.items()) if t == 1]
    reqs = scan_requests_for(model, vis)
    fits = reverse_staging_fits(raw, counts, key_slot([[model]]))
    arena = (sum(len(k) + len(v) for k, v in vis) + 4096 + 15) & ~15
    for rev in (False, True):
        batch = [q for q in reqs if bool(q.get("reverse")) == rev]
        st, got = run_scans(pgs, part, batch, arena, kv_stride=len(vis) + 8)
        if st == pgs.NOT_SUPPORTED:
            assert not fits, ("refused although the staging pool fits", rev)
            continue
        assert st == 0 and (fits or not rev), (st, rev, fits)
        for i, (q, g) in enumerate(zip(batch, got)):
            assert g == model_scan(vis, q, NOW), ("reverse" if rev else "forward", i, q["start"][:20], q["stop"][:20])


# ---- the merge at one geometry -------------------------------------------------------------------------------------------
def newer_runs(pgs, mid):
    """two L0 runs newer than a merge output: new values of every third key, tombstones of every fifth"""
    items = mid.to_list()
    s0 = int(mid.seq.max()) + 1
    a = [(k, s0 + i, 1, (v[:4] if t == 1 and len(v) >= 4 else bytes(4)) + b"2nd" + v[4:40]) for i, (k, _s, t, v) in enumerate(items) if i % 3 == 0]
    b = [(k, s0 + len(items) + i, 0, b"") for i, (k, _s, _t, _v) in enumerate(items) if i % 5 == 1]
    return [pgs.Records.from_list(a), pgs.Records.from_list(b)]


@pytest.mark.parametrize("name", list(INPUTS))
def test_merge_at_geometry(pgs, oracle, geo_engine, name):
    eng, bs, ri = geo_engine
    if name == "huge_blocks" and (bs, ri) not in CUT:
        pytest.skip("the huge-block input runs at the cut geometries only")
    smem = smem_budget()
    make, kw = INPUTS[name]
    g = emit_geometry(bs, ri, 7, smem)
    runs = make(g)
    g = emit_geometry(bs, ri, max_ukey(runs), smem)
    if name == "df_big_threshold":
        assert emit_geometry(bs, ri, 7, smem) == g
    seen = {}

    def inspect(part, res, raw, want):
        counts = check_run_format(raw, ri, g["block_size"])
        info = part.run_info(res.new_run_id)
        assert info.max_block_records == max(counts) and sum(counts) == want.n
        multi = [int(s) for s, c in zip(raw.blk_size, counts) if c > 1]
        seen["blocks"] = counts, multi
        if not seen.get("reads"):  # the reads run over the first merge, which keeps tombstones
            seen["reads"] = True
            check_reads(pgs, part, runs, raw, counts, bs, ri)

    for bm in (False, True):
        res, _ = run_case(pgs, oracle, eng, runs, bottommost=bm, build=(bs, ri), inspect=inspect, **kw)
        counts, multi = seen.pop("blocks")
        # the branch each geometry is there for, from what the test can see
        if bs == 64:  # at most four of the smallest entries (11 bytes and a restart offset) fit; larger ones stand alone
            assert max(counts) <= 4 and (1 in counts or name not in ("long_restart_arrays", "df_big_threshold")), counts[:50]
        if (bs, ri) == (4096, 1) and name == "long_restart_arrays":
            assert max(counts) > 32, "a block spans several batches"
        if (bs, ri) in CUT and name == "huge_blocks":
            assert max(multi) <= g["block_size"] < bs, (max(multi), g)

    # a second generation: k_walk walks the blocks k_emit wrote, through their entry index
    fp = oracle.filter_params()
    part = eng.partition()
    try:
        ids = [part.upload(pgs.build_run(r, bs, ri)) for r in runs]
        r1 = part.compact(ids, out_level=1, bottommost=0, now=NOW)
        mid, _ = oracle.compact([oracle.Run.from_records(r) for r in runs], False, fp, NOW)
        newer = newer_runs(pgs, mid.records())
        ids2 = [part.upload(pgs.build_run(r, bs, ri)) for r in newer]
        r2 = part.compact(ids2 + [r1.new_run_id], out_level=1, bottommost=1, now=NOW)
        want, _ = oracle.compact([oracle.Run.from_records(r) for r in newer] + [mid], True, fp, NOW)
        raw2 = part.download(r2.new_run_id)
        assert pgs.decode_blocks(raw2).same_as(want.records())
        check_run_format(raw2, ri, g["block_size"])
    finally:
        part.close()

    # determinism: the same merge twice (segment plans and prefix sums are deterministic: a difference is a race in k_emit)
    part = eng.partition()
    try:
        ids = [part.upload(pgs.build_run(r, bs, ri)) for r in runs]
        a = part.download(part.compact(ids, out_level=1, bottommost=0, now=NOW, flags=KEEP_INPUTS).new_run_id)
        b = part.download(part.compact(ids, out_level=1, bottommost=0, now=NOW, flags=KEEP_INPUTS).new_run_id)
        for x, y in ((a.data, b.data), (a.blk_off, b.blk_off), (a.blk_size, b.blk_size)):
            assert np.array_equal(x, y)
    finally:
        part.close()
