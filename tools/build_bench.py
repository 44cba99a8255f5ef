"""Run build on the device (pgs_run_build) against the host path it replaces (host builder + pgs_run_upload), at the ABI level,
in one process, the two alternating.

Inputs are config #2 records (50-byte keys, 268-byte values): the records of one 64 MB memtable (what a replica flushes; the
memtable counts key + value + 16 bytes per record) and one run of 2.5 M records.  The records are given from pageable numpy
arrays and from pinned ones.  For the host path "pinned" means the finished blocks are uploaded from pinned memory (the copy
into pinned memory is not timed); its encode time is the same either way.

Per configuration: the median of --reps timed calls after --warmup calls of each path, the host path split into encode and
upload, the device build into its phases (CUDA events inside pgs_run_build: input copy, block plan, block writing, index).
Every call's run is dropped again.  The card's name, power limit and SM clock are read in the same run.  Writes one JSON line.

    python tools/build_bench.py [--reps 9] [--warmup 2] [--out /tmp/build_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import incubator_pegasus_b200 as pgs  # noqa: E402
from incubator_pegasus_b200 import synth  # noqa: E402


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.splitlines()[0].split(",")])) if out else {}


class Pinned(np.ndarray):
    pass


def pinned(a):
    import torch
    t = torch.empty(max(1, a.nbytes), dtype=torch.uint8, pin_memory=True)
    p = t.numpy()[:a.nbytes].view(a.dtype).view(Pinned)
    p[:] = a
    p.owner = t
    return p


def host_path(part, recs, pin):
    t0 = time.perf_counter()
    run = pgs.build_run(recs)
    t1 = time.perf_counter()
    if pin:
        run = pgs.BlockRun(pinned(run.data), pinned(run.blk_off), pinned(run.blk_size))
    t2 = time.perf_counter()
    rid = part.upload(run)
    t3 = time.perf_counter()
    part.drop(rid)
    return {"total_ms": (t1 - t0 + t3 - t2) * 1e3, "encode_ms": (t1 - t0) * 1e3, "upload_ms": (t3 - t2) * 1e3}


def device_path(part, recs):
    t0 = time.perf_counter()
    rid = part.build_records(recs)
    t1 = time.perf_counter()
    ph = pgs.run_build_last_ms()
    part.drop(rid)
    return {"total_ms": (t1 - t0) * 1e3, "copy_ms": ph[0], "plan_ms": ph[1], "blocks_ms": ph[2], "index_ms": ph[3]}


def median(rows):
    return {k: statistics.median(r[k] for r in rows) for k in rows[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    facts = gpu_facts()
    per_rec = 50 + 268 + 16
    sizes = {"memtable_64MB": (64 << 20) // per_rec, "run_2.5M": 2_500_000}
    res = {"gpu": facts, "reps": args.reps, "warmup": args.warmup, "configs": {}}
    with pgs.Engine(device=0) as eng:
        part = eng.partition(app_id=9)
        for name, n in sizes.items():
            recs = synth.compaction_runs(k=1, n_per_run=n, seed=21)[0]
            host_bytes = sum(a.nbytes for a in (recs.keys, recs.key_off, recs.vals, recs.val_off, recs.seq, recs.type))
            block_bytes = pgs.build_run(recs).data.nbytes
            for pin in (False, True):
                src = pgs.Records(*[pinned(a) for a in (recs.keys, recs.key_off, recs.vals, recs.val_off, recs.seq, recs.type)]) if pin else recs
                for _ in range(args.warmup):
                    host_path(part, recs, pin)
                    device_path(part, src)
                hrows, drows = [], []
                for _ in range(args.reps):  # alternating
                    hrows.append(host_path(part, recs, pin))
                    drows.append(device_path(part, src))
                res["configs"][f"{name}/{'pinned' if pin else 'pageable'}"] = {
                    "records": n, "input_bytes": host_bytes, "block_bytes": block_bytes,
                    "host_builder_plus_upload": median(hrows), "device_build": median(drows)}
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
