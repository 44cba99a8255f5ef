"""The compaction walker's head window in the kernel simulator (group.cuh, kHeadWin): every next entry's head is staged in a
96-byte window, and heads that do not fit take the global path.  These inputs put entries on both sides of that line --
heads that straddle the window's end, restart points with long deltas, tombstones (no value bytes, no expire_ts), blocks
of every entry count up to a few (so the window serves the first entry of the next block from every position), and a run
whose last entry lies right at the end of its buffer -- and compare the merge with the oracle.  Under tools/simt/build.sh asan
every window fetch is checked against the exact size of the run buffer, 256 bytes of slack included."""
import numpy as np
import pytest

from test_kernel_sim import check, sim  # noqa: F401  (helper + fixture)


def records(pgs, items):
    return pgs.Records.from_list(sorted(items, key=lambda r: (r[0], -r[1])))


def value(rng, vl):
    """a value of vl >= 4 bytes: the 4-byte expire_ts header (0, no TTL), then random bytes"""
    return bytes(4) + bytes(rng.integers(0, 256, vl - 4, dtype=np.uint8))


@pytest.mark.parametrize("lanes", [1, 4, 16])
def test_sim_window_key_lengths(pgs, oracle, sim, lanes):
    """user keys of 40..100 bytes around the window's limit (a restart point's head fits up to ~60 bytes of key), sharing
    long prefixes so that non-restart entries carry short deltas; values of 4..7 bytes and tombstones (no value bytes)"""
    rng = np.random.default_rng(21)
    runs, seq = [], 0
    for r in range(3):
        items = []
        for i in range(160):
            kl = 40 + (i * 7 + r * 3) % 61
            key = (b"P" * (kl - 6) + b"%06d" % (i * 3 + r))[:kl]
            seq += 1
            t = 0 if i % 11 == 5 else 1
            items.append((key, seq, t, value(rng, int(rng.integers(4, 8))) if t else b""))
        runs.append(records(pgs, items))
    for ri in (1, 4, 16):
        check(pgs, oracle, sim, runs, bottommost=False, restart_interval=ri, block_size=512, seg_weight=8 * 1024, lanes=lanes)


def test_sim_window_block_crossings(pgs, oracle, sim):
    """blocks of 1, 2, 3, ... entries: values just under and over the block size cut blocks of one entry, runs of short
    ones fill blocks of a few, so the next block's first entry is fetched from every position of a block"""
    rng = np.random.default_rng(22)
    runs, seq = [], 0
    for r in range(3):
        items = []
        pattern = [300, 5, 300, 5, 5, 300, 5, 5, 5, 300, 40, 40, 40, 40, 600, 4, 0]
        for i in range(200):
            key = b"blk%05d" % (i * 3 + r)
            seq += 1
            vl = pattern[(i + r) % len(pattern)]
            items.append((key, seq, 1, value(rng, vl)) if vl else (key, seq, 0, b""))
        runs.append(records(pgs, items))
    for bs in (256, 384):
        check(pgs, oracle, sim, runs, bottommost=True, restart_interval=2, block_size=bs, seg_weight=8 * 1024)


def test_sim_window_end_of_buffer(pgs, oracle, sim):
    """runs that end in tiny entries (4-byte values, a tombstone of a one- or two-byte key): the window of the last entry
    of the last block reaches past the blocks into the buffer's slack"""
    rng = np.random.default_rng(23)
    runs, seq = [], 0
    for r in range(2):
        items = []
        for i in range(120):
            key = b"e%04d" % (i * 2 + r)
            seq += 1
            items.append((key, seq, 1, value(rng, int(rng.integers(4, 30)) if i < 110 else 4)))
        items.append((b"\xff" * (1 + r), seq + 1, 0, b""))
        seq += 1
        runs.append(records(pgs, items))
    for ri in (1, 16):
        check(pgs, oracle, sim, runs, bottommost=False, restart_interval=ri, block_size=256, seg_weight=4 * 1024)
