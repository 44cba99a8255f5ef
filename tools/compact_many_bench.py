"""Measures what one pgs_compact_many saves over one pgs_compact per partition.

For N partitions that each hold 5 runs of the manual-compaction sweep's records (BASELINE.json configs[3]: 16-byte hash keys,
32-byte sort keys, 256-byte values, 30 % of them expired) at MB megabytes per run, both ways merge every partition's 5 runs,
bottommost forced, TTL filter on, with KEEP_INPUTS | DISCARD_OUTPUT so that a call can be repeated:
  seq    one pgs_compact per partition, in sequence (each synchronises before it returns);
  many   one pgs_compact_many over the N partitions.
Each is timed on device events (the calls' device_ms: summed over the sequence, the one call's for many) and on the host wall
clock around the calls and a final synchronise, after warm-ups.  Merged GB/s = user-key + value bytes of the inputs / time.
Before timing, the records of the first partitions merged both ways (without DISCARD_OUTPUT) are compared.  A shape whose
device memory does not fit is reported as such.

    python tools/compact_many_bench.py [--n 1 16 64 256] [--mb 8 32] [--warmup 1] [--repeats 3]

Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import incubator_pegasus_b200 as pgs  # noqa: E402
from incubator_pegasus_b200 import synth  # noqa: E402

NOW = 300_000_000
HK, SK, VAL = 16, 32, 256
KEEP_INPUTS, DISCARD_OUTPUT = 1, 2


def card():
    """the device's name and power limit (W), read with the numbers"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1])}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "power_limit_w": None, "error": str(e)}


def sweep_runs(mb):
    """5 runs of `mb` MB each, 30 % of the values expired (the sweep of bench.py)"""
    n = max(1000, (mb << 20) // (2 + HK + SK + 12 + VAL))
    rng = np.random.default_rng(900 + mb)
    runs = synth.compaction_runs(k=5, n_per_run=n, hk_len=HK, sk_len=SK, user_len=VAL, now=NOW, seed=2000 + mb)
    for r in runs:
        nv = r.val_off.shape[0] - 1
        has = (r.val_off[1:] - r.val_off[:-1]) >= 4
        pick = np.nonzero(has & (rng.random(nv) < 0.30))[0]
        ets = (NOW - rng.integers(1, 86401, pick.size)).astype(">u4").view(np.uint8).reshape(-1, 4)
        for j in range(4):
            r.vals[(r.val_off[pick] + j).astype(np.int64)] = ets[:, j]
    return [pgs.build_run(r) for r in runs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="*", default=[1, 16, 64, 256])
    ap.add_argument("--mb", type=int, nargs="*", default=[8, 32])
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    eng = pgs.Engine()
    out = {"device": card(), "what": "5 runs per partition, 30 % expired, bottommost forced; seq = one pgs_compact per "
                                     "partition, many = one pgs_compact_many", "shapes": []}
    for mb in args.mb:
        blocks = sweep_runs(mb)
        for n in args.n:
            row = {"run_mb": mb, "partitions": n}
            parts = []
            try:
                for i in range(n):
                    p = eng.partition(app_id=7, pidx=i)
                    parts.append((p, p.upload_many(blocks, levels=[4, 3, 2, 1, 0])))
                eng.sync()
                jobs = [(p, ids, 4, 1, {}) for p, ids in parts]
                # the same records both ways, on the first partitions (outputs installed, compared, dropped)
                for p, ids in parts[:2]:
                    a = p.compact(ids, out_level=4, bottommost=1, now=NOW, flags=KEEP_INPUTS)
                    ra = pgs.decode_blocks(p.download(a.new_run_id))
                    p.drop(a.new_run_id)
                    b = eng.compact_many([(p, ids, 4, 1, {})], NOW, flags=KEEP_INPUTS)[0]
                    rb = pgs.decode_blocks(p.download(b.new_run_id))
                    p.drop(b.new_run_id)
                    if not ra.same_as(rb):
                        raise SystemExit(f"compact_many_bench: records differ at {mb} MB x {n}")
                row["records_checked"] = True
                seq_dev, seq_wall, many_dev, many_wall = [], [], [], []
                for rep in range(args.warmup + args.repeats):
                    t0 = time.perf_counter()
                    dev = 0.0
                    res_seq = []
                    for p, ids in parts:
                        r = p.compact(ids, out_level=4, bottommost=1, now=NOW, flags=KEEP_INPUTS | DISCARD_OUTPUT)
                        dev += r.device_ms
                        res_seq.append(r)
                    eng.sync()
                    t1 = time.perf_counter()
                    res_many = eng.compact_many(jobs, NOW, flags=KEEP_INPUTS | DISCARD_OUTPUT)
                    eng.sync()
                    t2 = time.perf_counter()
                    if rep >= args.warmup:
                        seq_dev.append(dev)
                        seq_wall.append((t1 - t0) * 1e3)
                        many_dev.append(res_many[0].device_ms)
                        many_wall.append((t2 - t1) * 1e3)
                for a, b in zip(res_seq, res_many):
                    if (a.in_records, a.out_records, a.dropped_expired, a.out_bytes) != (b.in_records, b.out_records, b.dropped_expired, b.out_bytes):
                        raise SystemExit(f"compact_many_bench: counters differ at {mb} MB x {n}")
                merged = sum(r.in_bytes for r in res_many)
                med = lambda v: float(np.median(v))  # noqa: E731
                row.update({"merged_bytes": int(merged), "tiles": int(sum(r.n_tiles for r in res_many)),
                            "seq_device_ms": med(seq_dev), "seq_wall_ms": med(seq_wall),
                            "many_device_ms": med(many_dev), "many_wall_ms": med(many_wall),
                            "seq_device_GBps": merged / med(seq_dev) / 1e6, "many_device_GBps": merged / med(many_dev) / 1e6,
                            "seq_wall_GBps": merged / med(seq_wall) / 1e6, "many_wall_GBps": merged / med(many_wall) / 1e6})
            except pgs.PegasusError as e:
                row["not_run"] = str(e)
            finally:
                for p, _ in parts:
                    p.close()
                eng.sync()
            out["shapes"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
