"""Partition split benchmark (pgs_partition_split) at config #2: 4 x 2.5 M records (16 B hash key, 32 B sort key, 268 B
value; synth.compaction_runs), once as four L0 runs and once as the one L1 run their compaction writes (without the versions it shadows).  Each shape is split
into 2 and into 8 children: the median of --reps splits after --warmup warm-ups, as CUDA-event kernel time and whole-call
time (and its phases: planner + counting walk, writing walk, k_seg_scan + k_emit of the children), with GB/s over the algorithmic bytes (sum(key + value) read plus the same written) and that rate's fraction of the
H100 SXM data-sheet 3.35 TB/s.  pgs_compact of the same runs (inputs kept, output discarded) alternates with the splits in
the same process for scale.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/split_bench.py [--records 2500000] [--reps 9] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import incubator_pegasus_b200 as pgs  # noqa: E402
from incubator_pegasus_b200 import synth  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:  # the numbers are reported without it rather than not at all
        return "unknown (%s)" % e, "unknown"


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=2_500_000)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    t0 = time.time()
    runs = synth.compaction_runs(k=4, n_per_run=a.records)
    gen_s = time.time() - t0
    eng = pgs.Engine()
    l0 = eng.partition(app_id=1, pidx=0)
    for r in runs:
        l0.upload_records(r, 0)
    l1 = eng.partition(app_id=2, pidx=0)
    for r in runs:
        l1.upload_records(r, 0)
    l1.compact(l1.runs(), out_level=1, bottommost=0, enabled=False)  # the same records merged into one L1 run (older versions go)
    name, power = card()
    out = dict(card=name, power_limit=power, records=4 * a.records, gen_s=round(gen_s, 1), shapes={})
    for shape, part in (("4xL0", l0), ("1xL1", l1)):
        r = {}
        for S in (2, 8):
            kern, call, comp, phases = [], [], [], []
            res = None
            for it in range(a.warmup + a.reps):
                kids = [eng.partition(app_id=1 if part is l0 else 2, pidx=i) for i in range(S)]
                eng.sync()
                t = time.perf_counter()
                res = part.split(1, S, kids)
                dt = time.perf_counter() - t
                for k in kids:
                    k.close()
                c = part.compact(part.runs(), out_level=1, bottommost=0, enabled=False, flags=3)  # alternating, for scale
                if it >= a.warmup:
                    kern.append(res.kernel_ms)
                    call.append(dt * 1e3)
                    comp.append(c.device_ms)
                    phases.append((res.count_ms, res.walk_ms, res.emit_ms))
            algo = 2 * (res.in_bytes)  # read once, written once (nothing is dropped in config #2)
            km = median(kern)
            r["S%d" % S] = dict(kernel_ms=round(km, 3), call_ms=round(median(call), 3), device_ms_last=round(res.device_ms, 3),
                                algo_bytes=algo, gbps=round(algo / km / 1e6, 1), frac_peak=round(algo / (km * 1e-3) / PEAK_BPS, 3),
                                compact_device_ms=round(median(comp), 3), launches=res.n_launches,
                                count_ms=round(median([x[0] for x in phases]), 3), walk_ms=round(median([x[1] for x in phases]), 3),
                                emit_ms=round(median([x[2] for x in phases]), 3))
        out["shapes"][shape] = r
    out["oracle_split"] = "not measured"
    print(json.dumps(out))
    l0.close()
    l1.close()
    eng.close()


if __name__ == "__main__":
    main()
