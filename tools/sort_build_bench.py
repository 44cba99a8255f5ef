"""Runs from records in any order: pgs_run_build_unsorted (device sort + device build) against the host sort plus host builder plus
pgs_run_upload, with pgs_run_build on the pre-sorted records beside them for the build cost without a sort.  ABI-level, in one
process, the three paths alternating on the same records.

Shapes: config #2 records (50-byte keys, 268-byte values) shuffled, as one 64 MB memtable (200 924 records; the memtable counts
key + value + 16 bytes per record) and one run of 2.5 M records, each from pageable numpy arrays and from pinned ones; and two
worst cases for the sort: 4096-byte keys that share a 4000-byte prefix, and one user key with 200 000 versions.

The host sort is numpy's stable argsort (timsort) of the fixed-width keys as a bytes dtype, after a stable argsort of
~(seq << 8 | type); every shape here has fixed-width keys, for which this is internal-key order.  The host path is timed as
sort, gather of the sorted arrays, encode (pgs_run_builder_add_many + finish) and upload ("pinned": the blocks are uploaded from
pinned memory; the copy into it is not timed).  The unsorted device path is split into its CUDA-event phases: input copy, sort
(with the gather of the sorted copy), block plan, block writing, index.

Per configuration: the median of --reps timed calls after --warmup calls of each path.  Every call's run is dropped again, and
every device run is checked against the host path's blocks once.  The card's name, power limit and SM clock are read in the same
run.  Writes one JSON line.

    python tools/sort_build_bench.py [--reps 9] [--warmup 2] [--out /tmp/sort_build_bench.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import incubator_pegasus_b200 as pgs  # noqa: E402
from incubator_pegasus_b200 import synth  # noqa: E402
from build_bench import gpu_facts, median, pinned  # noqa: E402

HOST_SORT = "numpy stable argsort (timsort) of ~(seq << 8 | type), then of the fixed-width keys as an 'S' dtype"


def host_sort(recs):
    """-> the records in internal-key order (fixed-width keys)"""
    n = recs.n
    kw = int(recs.key_off[1] - recs.key_off[0]) if n else 0
    trailer = (recs.seq << np.uint64(8)) | recs.type.astype(np.uint64)
    order = np.argsort(~trailer, kind="stable")
    keys = recs.keys[:n * kw].view(f"S{kw}") if kw else np.zeros(n, "S1")
    order = order[np.argsort(keys[order], kind="stable")]
    vlen = np.diff(recs.val_off.astype(np.int64))[order]
    voff = np.zeros(n + 1, np.uint64)
    voff[1:] = np.cumsum(vlen)
    src = np.repeat(recs.val_off[:-1].astype(np.int64)[order] - voff[:-1].astype(np.int64), vlen) + np.arange(int(voff[-1]))
    ks = recs.keys[:n * kw].reshape(n, kw)[order].reshape(-1)
    return pgs.Records(np.ascontiguousarray(ks), recs.key_off.copy(), recs.vals[src], voff, recs.seq[order], recs.type[order])


def host_path(part, recs, pin):
    t0 = time.perf_counter()
    srt = host_sort(recs)
    t1 = time.perf_counter()
    run = pgs.build_run(srt)
    t2 = time.perf_counter()
    if pin:
        run = pgs.BlockRun(pinned(run.data), pinned(run.blk_off), pinned(run.blk_size))
    t3 = time.perf_counter()
    rid = part.upload(run)
    t4 = time.perf_counter()
    part.drop(rid)
    return {"total_ms": (t2 - t0 + t4 - t3) * 1e3, "sort_and_gather_ms": (t1 - t0) * 1e3, "encode_ms": (t2 - t1) * 1e3,
            "upload_ms": (t4 - t3) * 1e3}


def presorted_path(part, recs):
    t0 = time.perf_counter()
    rid = part.build_records(recs)
    t1 = time.perf_counter()
    ph = pgs.run_build_last_ms()
    part.drop(rid)
    return {"total_ms": (t1 - t0) * 1e3, "copy_ms": ph[0], "plan_ms": ph[1], "blocks_ms": ph[2], "index_ms": ph[3]}


def unsorted_path(part, recs, check=None):
    t0 = time.perf_counter()
    rid = part.build_records_unsorted(recs)
    t1 = time.perf_counter()
    ph, sort_ms = pgs.run_build_last_ms(), pgs.run_build_last_sort_ms()
    if check is not None:
        got = part.download(rid)
        assert np.array_equal(got.data, check.data) and np.array_equal(got.blk_off, check.blk_off), "device run differs"
    part.drop(rid)
    return {"total_ms": (t1 - t0) * 1e3, "copy_ms": ph[0], "sort_ms": sort_ms, "plan_ms": ph[1], "blocks_ms": ph[2],
            "index_ms": ph[3]}


def shapes():
    per_rec = 50 + 268 + 16
    c2 = lambda n: synth.compaction_runs(k=1, n_per_run=n, seed=21)[0]  # noqa: E731
    yield "memtable_64MB", c2((64 << 20) // per_rec), (False, True)
    yield "run_2.5M", c2(2_500_000), (False, True)
    rng = np.random.default_rng(5)
    n = 20_000  # 4096-byte keys sharing 4000 bytes
    keys = np.empty((n, 4096), np.uint8)
    keys[:, :4000] = rng.integers(0, 256, 4000, dtype=np.uint8)
    keys[:, 4000:] = rng.integers(0, 256, (n, 96), dtype=np.uint8)
    keys = keys[np.lexsort(keys[:, ::-1].T)]
    vals = rng.integers(0, 256, (n, 100), dtype=np.uint8)
    yield "long_prefix_4096B_keys", synth.fixed_records(keys, vals, np.full(n, 7, np.uint64), np.ones(n, np.uint8)), (True,)
    n = 200_000  # one user key, 200 000 versions
    keys = np.tile(np.frombuffer(b"\x00\x10" + b"h" * 16 + b"s" * 32, np.uint8), (n, 1))
    vals = rng.integers(0, 256, (n, 268), dtype=np.uint8)
    yield "one_key_200k_versions", synth.fixed_records(keys, vals, np.arange(n, 0, -1, dtype=np.uint64), np.ones(n, np.uint8)), (True,)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"gpu": gpu_facts(), "reps": args.reps, "warmup": args.warmup, "host_sort": HOST_SORT, "configs": {}}
    with pgs.Engine(device=0) as eng:
        part = eng.partition(app_id=9)
        for name, recs, pins in shapes():
            shuf = synth.shuffled(recs, seed=3)
            want = pgs.build_run(recs)
            host_bytes = sum(a.nbytes for a in (recs.keys, recs.key_off, recs.vals, recs.val_off, recs.seq, recs.type))
            for pin in pins:
                arrays = lambda r: [pinned(a) for a in (r.keys, r.key_off, r.vals, r.val_off, r.seq, r.type)]  # noqa: E731
                src, ssrc = (pgs.Records(*arrays(recs)), pgs.Records(*arrays(shuf))) if pin else (recs, shuf)
                unsorted_path(part, ssrc, check=want)
                for _ in range(args.warmup):
                    host_path(part, shuf, pin)
                    presorted_path(part, src)
                    unsorted_path(part, ssrc)
                hrows, prows, urows = [], [], []
                for _ in range(args.reps):  # alternating
                    hrows.append(host_path(part, shuf, pin))
                    prows.append(presorted_path(part, src))
                    urows.append(unsorted_path(part, ssrc))
                res["configs"][f"{name}/{'pinned' if pin else 'pageable'}"] = {
                    "records": recs.n, "input_bytes": host_bytes, "block_bytes": int(want.data.nbytes),
                    "host_sort_builder_upload": median(hrows), "device_build_presorted": median(prows),
                    "device_build_unsorted": median(urows)}
                print(name, "pinned" if pin else "pageable", json.dumps(res["configs"][f"{name}/{'pinned' if pin else 'pageable'}"]),
                      file=sys.stderr, flush=True)
        part.close()
    res["gpu_after"] = gpu_facts()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
