"""Measures what one pgs_partition_split_many saves over one pgs_partition_split per parent.

N parent partitions each hold 5 runs of the manual-compaction sweep's records (BASELINE.json configs[3], as
tools/compact_many_bench.py builds them) at MB megabytes per run.  Both ways split every parent 1 -> S (S = 2 and 8) into
new, empty children:
  seq    one pgs_partition_split per parent, in sequence (each synchronises before it returns);
  many   one pgs_partition_split_many over the N parents.
Each is timed on device events (the calls' device_ms: summed over the sequence, the one call's for many) and on the host wall
clock around the calls, after warm-ups; the children are made before and closed after each timed call.  Merged GB/s = user
key + value bytes of the parents / time.  In every repetition the counters of every parent must agree between the two ways,
and in the first one the decoded records of every child of the first two parents.  A shape whose parents and children do
not fit device memory is reported as not run.

    python tools/split_many_bench.py [--n 1 16 64 256] [--mb 8 32] [--children 2 8] [--warmup 1] [--repeats 3]

Prints one JSON object.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import incubator_pegasus_b200 as pgs  # noqa: E402
from compact_many_bench import card, sweep_runs  # noqa: E402

DEVICE_BUDGET = 60 << 30  # parents and both ways' children at once


def children(eng, n, S, app):
    return [[eng.partition(app_id=app, pidx=c) for c in range(S)] for _ in range(n)]


def close(rows):
    for row in rows:
        for k in row:
            k.close()


def records(kid):
    return [pgs.decode_blocks(kid.download(r)).to_list() for r in kid.runs()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="*", default=[1, 16, 64, 256])
    ap.add_argument("--mb", type=int, nargs="*", default=[8, 32])
    ap.add_argument("--children", type=int, nargs="*", default=[2, 8])
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    eng = pgs.Engine()
    out = {"device": card(), "what": "5 runs per parent, 1 -> S; seq = one pgs_partition_split per parent, many = one "
                                     "pgs_partition_split_many", "shapes": []}
    for mb in args.mb:
        blocks = sweep_runs(mb)
        for n in args.n:
            if 3 * n * 5 * (mb << 20) > DEVICE_BUDGET:
                for S in args.children:
                    out["shapes"].append({"run_mb": mb, "parents": n, "children": S, "not_run": "does not fit device memory"})
                continue
            parents = []
            try:
                for i in range(n):
                    p = eng.partition(app_id=8, pidx=0)
                    p.upload_many(blocks, levels=[4, 3, 2, 1, 0])
                    parents.append(p)
                eng.sync()
                for S in args.children:
                    row = {"run_mb": mb, "parents": n, "children": S}
                    seq_dev, seq_wall, many_dev, many_wall = [], [], [], []
                    for rep in range(args.warmup + args.repeats):
                        ka, kb = children(eng, n, S, 9), children(eng, n, S, 10)
                        try:
                            eng.sync()
                            t0 = time.perf_counter()
                            res_seq = [p.split(1, S, row_) for p, row_ in zip(parents, ka)]
                            eng.sync()
                            t1 = time.perf_counter()
                            res_many = eng.split_many(list(zip(parents, kb)), 1, S)
                            eng.sync()
                            t2 = time.perf_counter()
                            for a, b in zip(res_seq, res_many):
                                ca = [(x.records, x.tombstones, x.raw_bytes, x.runs) for x in a.child[:S]]
                                cb = [(x.records, x.tombstones, x.raw_bytes, x.runs) for x in b.child[:S]]
                                if (a.in_records, a.in_bytes, a.dropped_empty, ca) != (b.in_records, b.in_bytes, b.dropped_empty, cb):
                                    raise SystemExit(f"split_many_bench: counters differ at {mb} MB x {n} x {S}")
                            if rep == 0:
                                for ra, rb in zip(ka[:2], kb[:2]):
                                    for x, y in zip(ra, rb):
                                        if records(x) != records(y):
                                            raise SystemExit(f"split_many_bench: records differ at {mb} MB x {n} x {S}")
                                row["records_checked"] = True
                        finally:
                            close(ka)
                            close(kb)
                            eng.sync()
                        if rep >= args.warmup:
                            seq_dev.append(sum(r.device_ms for r in res_seq))
                            seq_wall.append((t1 - t0) * 1e3)
                            many_dev.append(res_many[0].device_ms)
                            many_wall.append((t2 - t1) * 1e3)
                    merged = sum(r.in_bytes for r in res_many)
                    med = lambda v: float(np.median(v))  # noqa: E731
                    row.update({"merged_bytes": int(merged), "seq_launches": int(sum(r.n_launches for r in res_seq)),
                                "many_launches": int(res_many[0].n_launches),
                                "seq_device_ms": med(seq_dev), "seq_wall_ms": med(seq_wall),
                                "many_device_ms": med(many_dev), "many_wall_ms": med(many_wall),
                                "seq_device_GBps": merged / med(seq_dev) / 1e6, "many_device_GBps": merged / med(many_dev) / 1e6,
                                "seq_wall_GBps": merged / med(seq_wall) / 1e6, "many_wall_GBps": merged / med(many_wall) / 1e6})
                    out["shapes"].append(row)
                    print(json.dumps(row), file=sys.stderr, flush=True)
            except pgs.PegasusError as e:
                out["shapes"].append({"run_mb": mb, "parents": n, "not_run": str(e)})
            finally:
                for p in parents:
                    p.close()
                eng.sync()
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
