"""The compaction walker's head window in the kernel simulator (group.cuh, kHeadWin): every next entry's head is staged in a
96-byte window, and heads that do not fit take the global path.  These inputs put entries on both sides of that line --
heads that straddle the window's end, restart points with long deltas, tombstones (no value bytes, no expire_ts), blocks
of every entry count up to a few (so the window serves the first entry of the next block from every position), and a run
whose last entry lies right at the end of its buffer -- and compare the merge with the oracle.  Under tools/simt/build.sh asan
every window fetch is checked against the exact size of the run buffer, 256 bytes of slack included."""
import pytest

import merge_inputs
from test_kernel_sim import check, sim  # noqa: F401  (helper + fixture)


@pytest.mark.parametrize("lanes", [1, 4, 16])
def test_sim_window_key_lengths(pgs, oracle, sim, lanes):
    """user keys of 40..100 bytes around the window's limit (a restart point's head fits up to ~60 bytes of key), sharing
    long prefixes so that non-restart entries carry short deltas; values of 4..7 bytes and tombstones (no value bytes)"""
    runs = merge_inputs.window_key_lengths(21)
    for ri in (1, 4, 16):
        check(pgs, oracle, sim, runs, bottommost=False, restart_interval=ri, block_size=512, seg_weight=8 * 1024, lanes=lanes)


def test_sim_window_block_crossings(pgs, oracle, sim):
    """blocks of 1, 2, 3, ... entries: values just under and over the block size cut blocks of one entry, runs of short
    ones fill blocks of a few, so the next block's first entry is fetched from every position of a block"""
    runs = merge_inputs.window_block_crossings(22)
    for bs in (256, 384):
        check(pgs, oracle, sim, runs, bottommost=True, restart_interval=2, block_size=bs, seg_weight=8 * 1024)


def test_sim_window_end_of_buffer(pgs, oracle, sim):
    """runs that end in tiny entries (4-byte values, a tombstone of a one- or two-byte key): the window of the last entry
    of the last block reaches past the blocks into the buffer's slack"""
    runs = merge_inputs.window_end_of_buffer(23)
    for ri in (1, 16):
        check(pgs, oracle, sim, runs, bottommost=False, restart_interval=ri, block_size=256, seg_weight=4 * 1024)
