"""Block sizes so large that k_emit's two block-sized buffers per warp (output buffer and value stage) and the open block's
restart offsets do not fit a CTA's shared memory: the geometry cuts the blocks down to the largest buffer that fits, and the
merge still matches the oracle, in the simulator (tools/simt)."""
import numpy as np

from test_kernel_sim import check, sim  # noqa: F401  (sim: the session fixture that builds the simulator)


def test_sim_huge_block_sizes_are_cut_to_fit(pgs, oracle, sim):
    """restart interval 1 (the largest restart arrays per block byte) and 16; tiny entries, so that a cut block spans many
    emit batches, and values of 30..90 KB on both sides of the cut block buffer (about 74 KB at interval 1)."""
    rng = np.random.default_rng(17)
    def mk(seq0, n, big_every):
        recs = []
        for i in range(n):
            key = b"h%06d" % (i * 2 + seq0 % 2)
            seq0 += 1
            vl = int(rng.integers(30_000, 90_000)) if big_every and i % big_every == big_every - 1 else int(rng.integers(4, 24))
            recs.append((key, seq0, 1, (0).to_bytes(4, "big") + bytes(rng.integers(0, 256, vl - 4, dtype=np.uint8))))
        return seq0, pgs.Records.from_list(sorted(recs, key=lambda r: (r[0], -r[1])))
    seq, a = mk(0, 6000, 0)
    seq, b = mk(seq, 3000, 250)
    for ri, bs in ((1, 1 << 20), (1, 80_000), (16, 110_800)):
        check(pgs, oracle, sim, [b, a], bottommost=True, restart_interval=ri, block_size=bs, seg_weight=512 * 1024)
