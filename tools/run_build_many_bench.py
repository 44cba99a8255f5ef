"""Measures what one pgs_run_build_many saves over one pgs_run_build per partition, and what one pgs_rrdb_flush_many saves
over one pgs_rrdb_flush per replica.

Records are config #2's (synth.compaction_runs defaults: 318 bytes per record), MB megabytes of them per partition, the same
records in every partition.
  build    N partitions built one pgs_run_build after another (seq) against one pgs_run_build_many (many).  Timed on device
           events (pgs_run_build_last_ms, summed over the sequence) and on the host wall clock, after warm-ups; the runs are
           dropped between repeats.
  flush    two sets of N replicas, twins of each other, whose memtables are filled with the same records (one
           pgs_rrdb_multi_put per hash key, the same decrees): one set flushed one pgs_rrdb_flush after another (seq), the other
           in one pgs_rrdb_flush_many (many), every round.  Timed on the host wall clock, and on device events
           (pgs_run_build_last_ms: summed over the sequence; for many only when the memtables fit one build call, 256 MB).
           The first round is the warm-up, after which the twins' runs, run info and last_flushed_decree are compared.
           Shapes of more than 1 GB of memtables per set are not run (the memtables are filled from Python).
Before timing, every partition's run built both ways is compared byte for byte, with its handles and run info.  A shape the
call refuses is reported with its error.

    python tools/run_build_many_bench.py [--n 1 16 64 256] [--mb 0.25 4 64] [--flush-mb 0.25 4 64] [--repeats 3]

Prints one JSON object.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import incubator_pegasus_b200 as pgs  # noqa: E402
from incubator_pegasus_b200 import synth  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from compact_many_bench import card  # noqa: E402

REC_BYTES = 318
NOW = 300_000_000
INFO = ("n_blocks", "n_records", "n_tombstones", "data_bytes", "raw_key_bytes", "raw_value_bytes", "max_ukey_len", "max_value_len",
        "max_block_size", "max_block_records", "smallest_seq", "largest_seq", "level")


def same_runs(pa, ia, pb, ib):
    """the runs ia of partition pa and ib of pb: the same blocks, handles and run info (all but the id)"""
    x, y = pa.download(ia), pb.download(ib)
    assert np.array_equal(x.data, y.data) and np.array_equal(x.blk_off, y.blk_off) and np.array_equal(x.blk_size, y.blk_size)
    u, v = pa.run_info(ia), pb.run_info(ib)
    assert all(getattr(u, f) == getattr(v, f) for f in INFO)


def records(mb):
    return synth.compaction_runs(k=1, n_per_run=max(1, int(mb * (1 << 20)) // REC_BYTES), seed=17)[0]


def bench_build(eng, n, recs, repeats):
    parts = [eng.partition(app_id=90, pidx=i) for i in range(n)]
    try:
        def seq():
            dev, ids = 0.0, []
            t = time.perf_counter()
            for p in parts:
                ids.append(p.build_records(recs))
                dev += sum(pgs.run_build_last_ms())
            return time.perf_counter() - t, dev, ids

        def many():
            t = time.perf_counter()
            ids = eng.build_many([(p, recs, 0) for p in parts])
            return time.perf_counter() - t, sum(pgs.run_build_last_ms()), ids

        def drop(ids):
            for p, i in zip(parts, ids):
                p.drop(i)

        _, _, a = seq()
        _, _, b = many()
        for p, i, j in zip(parts, a, b):
            same_runs(p, i, p, j)
        drop(a)
        drop(b)
        out = {}
        for name, fn in (("seq", seq), ("many", many)):
            walls, devs = [], []
            for _ in range(repeats):
                w, d, ids = fn()
                walls.append(w * 1e3)
                devs.append(d)
                drop(ids)
            launches0 = eng.launches
            drop(fn()[2])
            out[name] = {"wall_ms": float(np.median(walls)), "device_ms": float(np.median(devs)), "launches": eng.launches - launches0}
        gb = n * (int(recs.key_off[-1]) + int(recs.val_off[-1])) / 1e9
        for v in out.values():
            v["GB_per_s_wall"] = gb / (v["wall_ms"] / 1e3)
        out["speedup_wall"] = out["seq"]["wall_ms"] / out["many"]["wall_ms"]
        return out
    finally:
        for p in parts:
            p.close()


def bench_flush(eng, n, recs, repeats):
    L = pgs.lib()
    opts = pgs.ServerOptions()
    opts.memtable_bytes = 1 << 40  # no flush while filling, no compaction: the flushes alone are timed
    opts.l0_compaction_trigger = 1 << 30
    by_hk = {}
    for k, _s, _t, v in recs.to_list():
        hl = int.from_bytes(k[:2], "big")
        by_hk.setdefault(k[2:2 + hl], []).append((k[2 + hl:], v))
    keep, batches = [], []  # the blobs of every multi_put, made once

    def blob(b):
        keep.append(b)
        return pgs.Blob(C.cast(C.c_char_p(b), C.POINTER(C.c_uint8)), len(b))

    for hk, kvs in by_hk.items():
        batches.append((blob(hk), (pgs.Blob * len(kvs))(*[blob(sk) for sk, _ in kvs]), (pgs.Blob * len(kvs))(*[blob(v) for _, v in kvs]),
                        len(kvs)))
    sets = []
    for app in (92, 93):
        reps = []
        for i in range(n):
            h = C.c_void_p()
            assert L.pgs_rrdb_start(eng.h, app, i, C.byref(opts), None, 0, C.byref(h)) == 0
            reps.append(h)
        sets.append(reps)
    # flush_many stages a memtable as its bytes plus about 25 bytes per record (and the server's value headers)
    one_call = n * (int(recs.key_off[-1]) + int(recs.val_off[-1]) + 48 * recs.n) < (256 << 20)

    def fill(reps, decree):
        for h in reps:
            d = decree
            for hkb, sks, vs, m in batches:
                d += 1
                assert L.pgs_rrdb_multi_put(h, hkb, sks, vs, m, 0, d, 1, NOW) == 0

    try:
        walls = {"seq": [], "many": []}
        devs = {"seq": [], "many": []}
        for rnd in range(repeats + 1):
            for reps in sets:
                fill(reps, rnd * len(batches))
            t, dev = time.perf_counter(), 0.0
            for h in sets[0]:
                assert L.pgs_rrdb_flush(h, NOW) == 0
                dev += sum(pgs.run_build_last_ms())
            walls["seq"].append((time.perf_counter() - t) * 1e3)
            devs["seq"].append(dev)
            arr = (C.c_void_p * n)(*[h.value for h in sets[1]])
            t = time.perf_counter()
            assert L.pgs_rrdb_flush_many(arr, n, NOW) == 0
            walls["many"].append((time.perf_counter() - t) * 1e3)
            devs["many"].append(sum(pgs.run_build_last_ms()) if one_call else None)
            if rnd == 0:  # the twins hold the same runs and decrees
                for ha, hb in zip(*sets):
                    assert L.pgs_rrdb_last_flushed_decree(ha) == L.pgs_rrdb_last_flushed_decree(hb)
                    pa = pgs.Partition(eng, 0, 0, 0, handle=L.pgs_rrdb_partition(ha))
                    pb = pgs.Partition(eng, 0, 0, 0, handle=L.pgs_rrdb_partition(hb))
                    ra, rb = pa.runs(), pb.runs()
                    assert len(ra) == len(rb) == 1
                    same_runs(pa, ra[0], pb, rb[0])
        out = {}
        for name in ("seq", "many"):
            d = devs[name][1:]
            out[name] = {"wall_ms": float(np.median(walls[name][1:])), "device_ms": float(np.median(d)) if d[0] is not None else None}
        out["speedup_wall"] = out["seq"]["wall_ms"] / out["many"]["wall_ms"]
        return out
    finally:
        for reps in sets:
            for h in reps:
                L.pgs_rrdb_stop(h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--mb", type=float, nargs="*", default=[0.25, 4, 64])
    ap.add_argument("--flush-mb", type=float, nargs="*", default=[0.25, 4, 64])
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    eng = pgs.Engine()
    res = {"card": card(), "record_bytes": REC_BYTES, "build": {}, "flush": {}}
    try:
        for mb in a.mb:
            recs = records(mb)
            for n in a.n:
                key = f"{n}x{mb}MB"
                try:
                    res["build"][key] = bench_build(eng, n, recs, a.repeats)
                except pgs.PegasusError as e:
                    res["build"][key] = {"error": str(e)}
                print("build", key, json.dumps(res["build"][key]), file=sys.stderr, flush=True)
        for mb in a.flush_mb:
            recs = records(mb)
            for n in a.n:
                key = f"{n}x{mb}MB"
                res["flush"][key] = bench_flush(eng, n, recs, a.repeats) if n * mb <= 1024 else "not measured"
                print("flush", key, json.dumps(res["flush"][key]), file=sys.stderr, flush=True)
    finally:
        eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
