#!/usr/bin/env python
"""Diagnostics: compaction kernel times (k_walk, k_emit, planner) at BASELINE config #2 for a list of environment settings.
Usage: python tools/variants.py SPEC [SPEC ...]   where SPEC = "default" or "KEY=VAL,KEY=VAL" (e.g. PGS_WALK_G=8)

Per SPEC: the medians over the timed compactions (after 3 warm-ups) of the merge kernels, k_walk, k_emit and the planner,
and the bytes k_emit moves with the rate they give at its median time: the values it reads, the descriptors (16 B) and
key-stream records (trailer + user key padded to 4 B; rewritten expiry stamps not counted) it reads, the blocks it writes."""
import os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: F401  (device init)
import incubator_pegasus_b200 as pgs
from incubator_pegasus_b200 import synth

args = sys.argv[1:]
n = int(os.environ.get("VAR_RECORDS", "2500000"))
timed = int(os.environ.get("VAR_TIMED", "9"))
HK, SK = 16, 32
runs = synth.compaction_runs(k=4, n_per_run=n, hk_len=HK, sk_len=SK, user_len=256, now=synth.NOW, seed=1000)
ukey = 2 + HK + SK  # every user key of this workload: 2-byte hash-key length | hash key | sort key
host_runs = [pgs.build_run(r) for r in runs]
eng = pgs.Engine(device=0)
part = eng.partition(app_id=1, pidx=0)
ids = [part.upload(h) for h in host_runs]
for spec in args:
    saved = {}
    for kv in spec.split(","):
        if "=" in kv:
            k, v = kv.split("=", 1); saved[k] = os.environ.get(k); os.environ[k] = v
    rs = []
    for i in range(3 + timed):
        res = part.compact(ids, out_level=1, bottommost=1, now=synth.NOW, enabled=True, flags=3)
        if i >= 3: rs.append(res)
    med = lambda f: statistics.median(f(r) for r in rs)
    kern, walk, emit = med(lambda r: r.merge_kernel_ms), med(lambda r: r.walk_ms), med(lambda r: r.emit_ms)
    plan = med(lambda r: r.device_ms - r.merge_kernel_ms)
    print(f"== {spec}: kernel_ms {kern:.3f} (min {min(r.merge_kernel_ms for r in rs):.3f}) walk {walk:.3f} "
          f"(min {min(r.walk_ms for r in rs):.3f} max {max(r.walk_ms for r in rs):.3f}) emit {emit:.3f} "
          f"(min {min(r.emit_ms for r in rs):.3f} max {max(r.emit_ms for r in rs):.3f}) plan {plan:.3f} segs {res.n_tiles}", flush=True)
    val_rd = res.out_bytes - res.out_records * ukey
    meta_rd = res.out_records * (16 + 8 + (ukey + 3) // 4 * 4)
    wr = res.out_block_bytes
    tot = val_rd + meta_rd + wr
    print(f"   k_emit bytes: values read {val_rd / 1e9:.3f} GB, descriptors + key stream read {meta_rd / 1e9:.3f} GB, "
          f"blocks written {wr / 1e9:.3f} GB; {tot / 1e9:.3f} GB in {emit:.3f} ms = {tot / emit / 1e6:.0f} GB/s", flush=True)
    for k, v in saved.items():
        if v is None: os.environ.pop(k, None)
        else: os.environ[k] = v
