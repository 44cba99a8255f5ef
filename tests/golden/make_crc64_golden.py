#!/usr/bin/env python
"""Regenerates crc64_reference.json: crc64 of seeded random inputs, computed by the reference's own
src/utils/crc.cpp (built into oracle/_ref by `make -C oracle` where the reference tree is present).
The inputs and answers are committed, so tests/test_oracle_selfcheck.py compares against them anywhere."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))


def main():
    import oracle_py
    ref = oracle_py.ref_crc()
    if ref is None:
        sys.exit("oracle/_ref/libref_crc.so not built (reference tree absent); the fixture is already committed")
    rng = np.random.default_rng(1)
    cases = []
    for n in [0, 1, 2, 7, 15, 16, 17, 31, 64, 1000, 4097]:
        b = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        for init in (0, 0x1234567890ABCDEF):
            cases.append({"data": b.hex(), "init": "%016x" % init, "crc64": "%016x" % ref.ref_crc64(b, n, init)})
    out = {"source": "reference src/utils/crc.cpp dsn::utils::crc64_calc", "cases": cases}
    with open(os.path.join(HERE, "crc64_reference.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("cases:", len(cases))


if __name__ == "__main__":
    main()
