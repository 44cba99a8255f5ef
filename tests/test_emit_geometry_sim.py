"""Block sizes so large that k_emit's two block-sized buffers per warp (output buffer and value stage) and the open block's
restart offsets do not fit a CTA's shared memory: the geometry cuts the blocks down to the largest buffer that fits, and the
merge still matches the oracle, in the simulator (tools/simt)."""
import pytest

import merge_inputs
from get_model import SIM_SMEM, emit_geometry
from test_kernel_sim import check, sim  # noqa: F401  (sim: the session fixture that builds the simulator)


def test_sim_huge_block_sizes_are_cut_to_fit(pgs, oracle, sim):
    """restart interval 1 (the largest restart arrays per block byte) and 16; tiny entries, so that a cut block spans many
    emit batches, and values of 30..90 KB on both sides of the cut block buffer (about 74 KB at interval 1)."""
    runs = merge_inputs.huge_blocks(17)
    for ri, bs in ((1, 1 << 20), (1, 80_000), (16, 110_800)):
        check(pgs, oracle, sim, runs, bottommost=True, restart_interval=ri, block_size=bs, seg_weight=512 * 1024)


def test_restated_geometry_cuts_where_the_design_says():
    """emit_geometry, the tests' restatement of compact_geometry's block-buffer rule, with an H100's shared memory: blocks
    are cut to about 74 KB at restart interval 1 and 110 KB at 16 (DESIGN §3.3), and the warps per CTA follow the block size:
    4 at 4 KB blocks, two CTAs of 3 at 16 KB, one warp at 64 KB"""
    for bs in (80_000, 1 << 20):
        g = emit_geometry(bs, 1, 7, SIM_SMEM)
        assert 73_000 <= g["block_size"] <= 75_500 and g["blk_buf"] == g["block_size"] + 24, g
        assert g["warps"] == 1
    for bs in (110_800, 1 << 20):
        g = emit_geometry(bs, 16, 7, SIM_SMEM)
        assert 109_000 <= g["block_size"] < 110_800 and g["blk_buf"] == g["block_size"] + 24, g
    assert emit_geometry(4096, 16, 7, SIM_SMEM) == dict(blk_buf=4128, block_size=4096, warps=4, twice=True)
    assert emit_geometry(16384, 16, 7, SIM_SMEM) == dict(blk_buf=16416, block_size=16384, warps=3, twice=True)
    assert emit_geometry(65536, 16, 7, SIM_SMEM) == dict(blk_buf=65568, block_size=65536, warps=1, twice=False)


@pytest.mark.parametrize("block_size,ri", [(64, 1), (512, 4), (4096, 1), (4096, 16), (80_000, 1)])
def test_sim_df_big_threshold(pgs, oracle, sim, block_size, ri):
    """entries one byte under, at and over the size that sends them to k_emit's in-place path, between runs of tiny ones"""
    blk_buf = emit_geometry(block_size, ri, 7, SIM_SMEM)["blk_buf"]
    runs = merge_inputs.df_big_threshold(41, blk_buf)
    for bm in (True, False):
        check(pgs, oracle, sim, runs, bottommost=bm, restart_interval=ri, block_size=block_size, seg_weight=64 * 1024)
