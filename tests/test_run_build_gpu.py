"""pgs_run_build on the device against the host path it replaces (pgs_run_builder_add_many + finish + pgs_run_upload) on the
same records: the downloaded run, its pgs_run_info (all but the run id), point lookups and forward and reverse batched scans are
identical, at several block geometries and for one config #2 run of 2.5 M records.  Refused inputs leave the run list as it was,
and every L0 run a replica's flush writes equals the host builder's encoding of its own records."""
import hashlib

import numpy as np
import pytest

import rrdb_harness as rh
from incubator_pegasus_b200 import synth
from test_run_build_sim import INFO_FIELDS, edge_items
from test_scan_kernels_gpu import run_scans

pytestmark = pytest.mark.gpu
NOW = synth.NOW


def _pair(pgs, eng, recs, bs, ri, level=0):
    """the host path in one partition, the device build in another -> (host part, host id, device part, device id)"""
    a, b = eng.partition(app_id=7, pidx=0), eng.partition(app_id=7, pidx=1)
    ia = a.upload(pgs.build_run(recs, bs, ri), level)
    ib = b.build_records(recs, level)
    return a, ia, b, ib


def _same_run(a, ia, b, ib):
    ra, rb = a.download(ia), b.download(ib)
    assert np.array_equal(ra.blk_off, rb.blk_off) and np.array_equal(ra.blk_size, rb.blk_size)
    assert np.array_equal(ra.data, rb.data)
    x, y = a.run_info(ia), b.run_info(ib)
    for f in INFO_FIELDS + ("level",):
        assert getattr(x, f) == getattr(y, f), f


def _gets(part, keys):
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    st, res, arena, _ = part.get_batch(np.frombuffer(b"".join(keys), np.uint8).copy(), off, NOW, arena_cap=64 << 20)
    assert st == 0
    return [(r.status, r.expire_ts, r.expired, arena[r.value_off:r.value_off + r.value_len].tobytes() if r.status == 0 else b"")
            for r in res[:len(keys)]]


def _scans(pgs, part, recs):
    full = dict(start=b"", stop=b"\xff" * 6, start_inclusive=True, stop_inclusive=True, key_mode=0, prefix=0, max_count=300,
                max_iter_count=100000, max_iter_size=0)
    keys = sorted({recs.key(i) for i in range(0, recs.n, max(1, recs.n // 20))})
    reqs = [full, dict(full, max_count=7)] + [dict(full, start=k) for k in keys] + [dict(full, stop=k, stop_inclusive=False) for k in keys]
    # (a reverse batch over blocks larger than k_scan stages is refused with kNotSupported; the status is compared too)
    return [run_scans(pgs, part, [dict(q, reverse=rev) for q in reqs], arena_stride=1 << 21, kv_stride=400) for rev in (False, True)]


@pytest.mark.parametrize("bs,ri", [(4096, 16), (512, 2), (16384, 1)])
def test_device_build_equals_host_upload(pgs, bs, ri):
    eng = pgs.Engine(block_size=bs, restart_interval=ri)
    try:
        for recs in [pgs.Records.from_list(edge_items(bs + ri)), synth.compaction_runs(k=1, n_per_run=20_000, seed=3)[0],
                     pgs.Records.from_list(edge_items(1)[:1])]:
            a, ia, b, ib = _pair(pgs, eng, recs, bs, ri)
            try:
                _same_run(a, ia, b, ib)
                keys = [recs.key(i) for i in range(0, recs.n, max(1, recs.n // 3000))] + [b"\x00\x01zz-missing", b"\x00"]
                assert _gets(a, keys) == _gets(b, keys)
                sa = _scans(pgs, a, recs)
                assert sa == _scans(pgs, b, recs)
                assert recs.n < 5000 or (sa[0][0] == 0 and sa[1][0] == 0)  # config #2 records: both directions answer
            finally:
                a.close()
                b.close()
    finally:
        eng.close()


def _digest(run):
    h = hashlib.sha256()
    for x in (run.data, run.blk_off, run.blk_size):
        h.update(x.tobytes())
    return h.hexdigest()


def test_config2_run_digest(pgs, engine):
    """config #2: one run of 2.5 M records of 318 bytes"""
    recs = synth.compaction_runs(k=1, n_per_run=2_500_000)[0]
    a, ia, b, ib = _pair(pgs, engine, recs, 4096, 16, level=1)
    try:
        assert _digest(a.download(ia)) == _digest(b.download(ib))
        x, y = a.run_info(ia), b.run_info(ib)
        assert all(getattr(x, f) == getattr(y, f) for f in INFO_FIELDS + ("level",))
        assert y.n_records == 2_500_000
        keys = [recs.key(i) for i in range(0, recs.n, 997)]
        assert _gets(a, keys) == _gets(b, keys)
    finally:
        a.close()
        b.close()


def test_refusals_leave_the_run_list(pgs, engine):
    part = engine.partition(app_id=8)
    try:
        base = part.build_records(synth.compaction_runs(k=1, n_per_run=500, seed=4)[0])
        before = part.runs()
        assert before == [base]
        ok = [(b"\x00\x01k%04d" % i, 5, 1, b"v") for i in range(300)]
        cases = [
            (ok[:100] + [(b"\x00\x01a", 5, 1, b"")] + ok[100:], pgs.INVALID_ARGUMENT),       # a descending user key
            (ok[:50] + [(ok[49][0], 5, 1, b"w")] + ok[50:], pgs.INVALID_ARGUMENT),            # equal trailer
            (ok[:20] + [(ok[19][0], 6, 0, b"")] + ok[20:], pgs.INVALID_ARGUMENT),             # ascending trailer
            (ok[:200] + [(ok[199][0] + bytes(4096), 5, 1, b"")] + ok[200:], pgs.NOT_SUPPORTED),  # a 4097+-byte user key
        ]
        for items, want in cases:
            with pytest.raises(pgs.PegasusError) as e:
                part.build_records(pgs.Records.from_list(items))
            assert e.value.code == want
            assert part.runs() == before
        assert part.build_records(pgs.Records.from_list([])) == 0
        assert part.runs() == before
    finally:
        part.close()


def test_replica_flush_runs_are_the_host_encoding(pgs, engine):
    """every L0 run a replica's flush writes (memtable -> pgs_run_build) equals pgs.build_run of its own records"""
    be = rh.Backend("gpu", engine, opts=dict(memtable_bytes=1 << 20, l0_compaction_trigger=100))
    try:
        L = pgs.lib()
        part = pgs.Partition(engine, 0, 0, 1, handle=L.pgs_rrdb_partition(be.h))
        rng = np.random.default_rng(5)
        seen = set()
        for rnd in range(4):
            for i in range(3000):
                hk = b"h%03d" % rng.integers(0, 200)
                sk = b"s%05d" % rng.integers(0, 3000)
                if rng.random() < 0.1:
                    be.remove(hk, sk, now=NOW)
                else:
                    be.put(hk, sk, rng.bytes(int(rng.integers(0, 600))), now=NOW)
            be.flush(now=NOW)
            for rid in part.runs():
                if rid in seen:
                    continue
                seen.add(rid)
                got = part.download(rid)
                want = pgs.build_run(pgs.decode_blocks(got), 4096, 16)
                assert np.array_equal(got.data, want.data)
                assert np.array_equal(got.blk_off, want.blk_off) and np.array_equal(got.blk_size, want.blk_size)
        assert len(seen) >= 4
    finally:
        be.close()
