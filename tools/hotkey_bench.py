"""Cost of hot-key detection on the read path: the config #3 get pass (BASELINE.json configs[2] on one GPU: a 256-partition
table, 262 144 YCSB-C zipfian(0.99) gets in one pgs_get_batch_multi launch) with the READ collectors off, coarse and fine,
alternated round by round in one process.  Prints one JSON line: per phase the end-to-end pass time (host clock around the
call, which ends in a device synchronise) and the k_get time (CUDA events), plus k_hotkey_capture's kernel time from a
separate torch.profiler pass, and the card's name and power limit.
    python tools/hotkey_bench.py [--rounds 5] [--passes 10] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import incubator_pegasus_b200 as pgs  # noqa: E402
from incubator_pegasus_b200 import sharding, synth  # noqa: E402

HK, SK, VAL, NOW, T0 = 16, 16, 100, synth.NOW, 1000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--partitions", type=int, default=256)
    ap.add_argument("--table-hashkeys", type=int, default=65536)
    ap.add_argument("--n-get", type=int, default=262144)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = pgs.lib()
    eng = pgs.Engine(device=0)
    table = sharding.Table(partition_count=a.partitions, n_hash=a.table_hashkeys, sortkeys_per_hash=64, hk_len=HK, sk_len=SK,
                           user_len=VAL, now=NOW)
    servers, parts = [], []
    opts = pgs.ServerOptions()
    opts.prefix_filter = 1
    for p in range(a.partitions):
        h = C.c_void_p()
        assert L.pgs_rrdb_start(eng.h, 2, p, C.byref(opts), None, 0, C.byref(h)) == 0
        servers.append(h)
        part = pgs.Partition(eng, 2, p, 1, handle=L.pgs_rrdb_partition(h))
        runs = table.partition_runs(p)
        if runs:
            part.upload_many([pgs.build_run(r) for _, r in runs], levels=[lvl for lvl, _ in runs])
        parts.append(part)
    gh, gs, _ = table.requests(a.n_get, 0)
    owner = table.pidx[gh.astype(np.int64)].astype(np.uint32)
    keys = synth.make_keys(gh, gs, HK, SK, table.seed)
    flat = np.ascontiguousarray(keys.reshape(-1))
    off = np.arange(a.n_get + 1, dtype=np.uint32) * np.uint32(keys.shape[1])
    arena = np.zeros(a.n_get * (VAL + 16), np.uint8)
    res = (pgs.GetResult * a.n_get)()

    def one_pass():
        t = time.perf_counter()
        st, _, _, _ = pgs.get_batch_multi(parts, flat, off, owner, NOW, arena, res)
        assert st == 0, st
        return (time.perf_counter() - t) * 1e3, eng.last_kernel_ms

    def set_phase(phase):
        for h in servers:
            pgs.detect_hotkey(h, pgs.HOTKEY_READ, pgs.HOTKEY_STOP, T0)
        if phase == "off":
            return 0
        for h in servers:
            pgs.detect_hotkey(h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)
        if phase == "fine":  # one coarse period: the partitions with a hot bucket move to FINE
            one_pass()
            for h in servers:
                pgs.hotkey_analyse(h, T0 + 10)
        return sum(pgs.hotkey_state(h, pgs.HOTKEY_READ) == pgs.HOTKEY_FINE_DETECTING for h in servers)

    phases = ["off", "coarse", "fine"]
    for ph in phases:  # warm-up of every shape
        set_phase(ph)
        one_pass()
    times = {ph: {"e2e_ms": [], "k_get_ms": []} for ph in phases}
    fine_slots = 0
    for r in range(a.rounds):
        for ph in (phases if r % 2 == 0 else phases[::-1]):
            n_fine = set_phase(ph)
            if ph == "fine":
                fine_slots = n_fine
            for _ in range(a.passes):
                e2e, kg = one_pass()
                times[ph]["e2e_ms"].append(e2e)
                times[ph]["k_get_ms"].append(kg)
    capture = {}
    import torch
    from torch.profiler import ProfilerActivity, profile
    for ph in ("coarse", "fine"):
        set_phase(ph)
        one_pass()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.passes):
                one_pass()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "k_hotkey_capture" in e.key]
        capture[ph] = round(ev[0].device_time_total / ev[0].count / 1e3, 4) if ev else None
    stat = lambda v: {"median": round(float(np.median(v)), 3), "min": round(float(np.min(v)), 3), "max": round(float(np.max(v)), 3)}
    out = {"card": card(), "n_get": a.n_get, "partitions": a.partitions, "rounds": a.rounds, "passes_per_round": a.passes,
           "fine_slots": int(fine_slots),
           "phases": {ph: {k: stat(v) for k, v in times[ph].items()} for ph in phases},
           "k_hotkey_capture_ms": capture}
    print(json.dumps(out))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "hotkey_bench.json"), "w") as f:
            json.dump(out, f, indent=1)
    for h in servers:
        L.pgs_rrdb_stop(h)
    eng.close()


if __name__ == "__main__":
    main()
