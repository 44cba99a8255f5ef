"""The get model of tests/get_model.py pinned to the oracle: on the same runs and keys, model_get finds the same keys and the
same number of user-data bytes as the oracle's lookup over block runs (orc_blockruns_get_many, on_get's Get -> TTL check ->
header strip).  The oracle is itself pinned to the reference's tables (test_oracle_golden.py)."""
import numpy as np
import pytest

from get_model import OK, bloom_lines_for, flat_keys, model_get, prefix_len, query_keys, uploaded_run
from incubator_pegasus_b200 import synth
from scan_model import make_db

NOW = synth.NOW


@pytest.mark.parametrize("n_runs,block_size,ri", [(1, 4096, 16), (4, 256, 1), (9, 1024, 4)])
def test_model_get_matches_the_oracle(pgs, oracle, n_runs, block_size, ri):
    rng = np.random.default_rng(70 + n_runs)
    hks = [bytes(rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8)) for _ in range(10)] + [b"", b"h" * 140]
    runs, _ = make_db(pgs, rng, n_runs, hks, 40, big=True)  # newest first; every value carries the 12-byte header
    brs = [pgs.build_run(r, block_size, ri) for r in runs]
    model = [uploaded_run(b) for b in brs]
    keys = query_keys(model)
    want = [model_get(model, k, NOW) for k in keys]
    found = sum(w["status"] == OK for w in want)
    vbytes = sum(len(w["value"]) for w in want if w["status"] == OK)
    assert found > 100
    flat, off = flat_keys(keys)
    got_found, got_bytes, _ = oracle.get_many([oracle.BlockRunCPU.from_blocks(b) for b in brs], flat, off, NOW)
    assert (got_found, got_bytes) == (found, vbytes)


def test_sizing_formula_and_prefix_length():
    """10 bits per entry in 512-bit lines plus one; the HashkeyTransform prefix is 2 + BE16 bytes, 0 when the key is shorter"""
    assert [bloom_lines_for(n) for n in (0, 1, 51, 52, 1000)] == [1, 2, 2, 3, 21]
    assert [prefix_len(k) for k in (b"", b"\x00", b"\x00\x00", b"\x00\x03ab", b"\x00\x02ab", b"\x00\x02abc")] == [0, 0, 2, 0, 4, 4]
