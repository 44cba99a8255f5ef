"""Hot-key detection on the device (pgs_rrdb_detect_hotkey / pgs_rrdb_hotkey_analyse, k_hotkey_capture next to k_get):
a hot hash key of one partition is found through pgs_get_batch_multi and through 32 threads of pgs_batcher_get; a uniform
partition stays busy until the timeout; the rrdb handlers (memtable hits included) and the write operators capture what the
Python model of the collector (tests/hotkey_model.py) captures, step for step; and with no detection running a get launch is
byte- and launch-identical to one made before START and after STOP."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import hotkey_model as hm
from rrdb_harness import Backend, raw_key

pytestmark = pytest.mark.gpu

HOT = b"ThisisahotkeyThisisahotkey"
T0 = 1000


class Part:  # a server's partition handle, in the shape pgs.get_batch_multi / pgs.Batcher take
    def __init__(self, pgs, server):
        self.h = C.c_void_p(pgs.lib().pgs_rrdb_partition(server.h))


def flat(keys):
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    return np.frombuffer(b"".join(keys) + b"\0", np.uint8).copy(), off


def table(pgs, engine, n_parts=4, n_keys=400, app_id=31):
    srvs = [Backend("gpu", engine, app_id=app_id, pidx=p) for p in range(n_parts)]
    for p, s in enumerate(srvs):
        for i in range(n_keys):
            assert s.put(b"p%d_h%04d" % (p, i), b"s", b"v%d" % i) == 0
        assert s.put(HOT, b"s%d" % p, b"hot") == 0
        assert s.flush() == 0
    return srvs


def zipf_keys(rng, p, n, hot_share):
    return [raw_key(HOT, b"s%d" % p) if rng.random() < hot_share else raw_key(b"p%d_h%04d" % (p, rng.integers(0, 400)), b"s")
            for _ in range(n)]


def test_multi_partition_detection(pgs, engine):
    srvs = table(pgs, engine)
    try:
        parts = [Part(pgs, s) for s in srvs]
        for s in srvs[:2]:
            assert pgs.detect_hotkey(s.h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)[0] == pgs.HOTKEY_OK
        assert pgs.detect_hotkey(srvs[0].h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)[0] == pgs.HOTKEY_BUSY
        assert pgs.detect_hotkey(srvs[0].h, 7, pgs.HOTKEY_START, T0)[0] == pgs.HOTKEY_INVALID_PARAMETERS
        assert pgs.detect_hotkey(srvs[0].h, pgs.HOTKEY_READ, 9, T0)[0] == pgs.HOTKEY_INVALID_PARAMETERS
        rng = np.random.default_rng(3)
        found_at = None
        for step in range(1, 16):
            keys, kp = [], []
            for p in range(4):  # partition 0 has a hot hash key, partition 1 reads uniformly, 2 and 3 are not detecting
                ks = zipf_keys(rng, p, 3000, 0.3 if p == 0 else 0.0)
                keys += ks
                kp += [p] * len(ks)
            order = rng.permutation(len(keys))
            keys = [keys[i] for i in order]
            kp = np.array(kp, np.uint32)[order]
            k, off = flat(keys)
            st, res, _, _ = pgs.get_batch_multi(parts, k, off, kp, 0, np.zeros(1 << 22, np.uint8))
            assert st == 0 and all(res[i].status == pgs.OK for i in range(len(keys)))
            now = T0 + 10 * step
            for s in srvs:
                pgs.hotkey_analyse(s.h, now)
            if found_at is None and pgs.hotkey_state(srvs[0].h, pgs.HOTKEY_READ) == pgs.HOTKEY_FINISHED:
                found_at = step
            if now < T0 + 150:
                assert pgs.hotkey_state(srvs[1].h, pgs.HOTKEY_READ) == pgs.HOTKEY_COARSE_DETECTING, step
                assert pgs.detect_hotkey(srvs[1].h, pgs.HOTKEY_READ, pgs.HOTKEY_QUERY, now)[0] == pgs.HOTKEY_BUSY
            else:
                assert pgs.hotkey_state(srvs[1].h, pgs.HOTKEY_READ) == pgs.HOTKEY_STOPPED
        assert found_at == 2  # one coarse and one fine period
        assert pgs.detect_hotkey(srvs[0].h, pgs.HOTKEY_READ, pgs.HOTKEY_QUERY, T0 + 200) == (pgs.HOTKEY_OK, HOT)
        assert pgs.hotkey_state(srvs[2].h, pgs.HOTKEY_READ) == pgs.HOTKEY_STOPPED
        assert pgs.detect_hotkey(srvs[0].h, pgs.HOTKEY_READ, pgs.HOTKEY_STOP, T0 + 200)[0] == pgs.HOTKEY_OK
        assert pgs.hotkey_state(srvs[0].h, pgs.HOTKEY_READ) == pgs.HOTKEY_STOPPED
    finally:
        for s in srvs:
            s.close()


def test_batcher_threads_detect(pgs, engine):
    srvs = table(pgs, engine, app_id=32)
    try:
        parts = [Part(pgs, s) for s in srvs]
        assert pgs.detect_hotkey(srvs[2].h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)[0] == pgs.HOTKEY_OK
        b = pgs.Batcher(parts, max_batch=256, max_wait_us=500)
        try:
            rng = np.random.default_rng(8)
            for step in (1, 2):
                work = [(p, k) for p in range(4) for k in zipf_keys(rng, p, 1500, 0.3 if p == 2 else 0.0)]
                with ThreadPoolExecutor(max_workers=32) as pool:
                    got = list(pool.map(lambda w: b.get(w[0], w[1], 0)[:2], work))
                assert all(st == 0 and r.status == pgs.OK for st, r in got)
                pgs.hotkey_analyse(srvs[2].h, T0 + 10 * step)
            assert pgs.detect_hotkey(srvs[2].h, pgs.HOTKEY_READ, pgs.HOTKEY_QUERY, T0 + 30) == (pgs.HOTKEY_OK, HOT)
        finally:
            b.close()
    finally:
        for s in srvs:
            s.close()


def _step(pgs, s, model, now, kind):
    pgs.hotkey_analyse(s.h, now)
    model.analyse(now)
    assert pgs.hotkey_state(s.h, kind) == model.state, now
    out, text = pgs.detect_hotkey(s.h, kind, pgs.HOTKEY_QUERY, now)
    assert out == (hm.OK if model.state == hm.FINISHED else hm.BUSY)
    if out == hm.OK:
        assert text == model.result


def test_handlers_match_model(pgs, engine):
    s = Backend("gpu", engine, app_id=33, pidx=0)
    try:
        for i in range(300):
            s.put(b"h%03d" % i, b"s", b"v")
        s.put(HOT, b"s", b"v")
        s.flush()
        for i in range(0, 300, 7):  # memtable: these reads are answered on the host
            s.put(b"h%03d" % i, b"s", b"w")
        model = hm.Collector()
        assert pgs.detect_hotkey(s.h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)[0] == hm.OK and model.control(hm.START, T0) == hm.OK
        rng = np.random.default_rng(11)
        for step in range(1, 6):
            for _ in range(150):
                hk = HOT if rng.random() < 0.25 else b"h%03d" % rng.integers(0, 330)  # some keys are absent: counted too
                op = int(rng.integers(0, 5))
                if op == 0:
                    s.get(hk, b"s")
                    model.capture_hash_key(hk, 1)
                elif op == 1:
                    s.ttl(hk, b"s")
                    model.capture_hash_key(hk, 1)
                elif op == 2:
                    r = s.multi_get(hk, sort_keys=[b"s", b"t"])
                    model.capture_hash_key(hk, len(r["kvs"]))
                elif op == 3:
                    r = s.batch_get([(hk, b"s"), (b"h%03d" % rng.integers(0, 300), b"s")])
                    for kv in r["kvs"]:
                        model.capture_hash_key(kv[0][:kv[3]], 1)
                else:
                    s.sortkey_count(hk)
                    model.capture_hash_key(hk, 1)
            _step(pgs, s, model, T0 + 10 * step, pgs.HOTKEY_READ)
        assert model.state == hm.FINISHED and model.result == HOT
        # writes: put (raw key), multi_put (key count), check_and_mutate (mutation count) into the WRITE collector
        wm = hm.Collector()
        assert pgs.detect_hotkey(s.h, pgs.HOTKEY_WRITE, pgs.HOTKEY_START, T0)[0] == hm.OK and wm.control(hm.START, T0) == hm.OK
        for step in range(1, 5):
            for _ in range(120):
                hk = HOT if rng.random() < 0.2 else b"w%03d" % rng.integers(0, 200)
                op = int(rng.integers(0, 3))
                if op == 0:
                    s.put(hk, b"s", b"x")
                    wm.capture_hash_key(hk, 1)
                elif op == 1:
                    n = int(rng.integers(1, 4))
                    s.multi_put(hk, {b"m%d" % j: b"x" for j in range(n)})
                    wm.capture_hash_key(hk, n)
                else:
                    out = s.check_and_mutate(hk, b"s", 0, b"", [("put", b"c%d" % j, b"x") for j in range(3)])
                    assert out["error"] == 0
                    wm.capture_hash_key(hk, 3)
                    model.capture_hash_key(hk, 1)  # its read side
            _step(pgs, s, wm, T0 + 10 * step, pgs.HOTKEY_WRITE)
        assert wm.state == hm.FINISHED and wm.result == HOT
    finally:
        s.close()


def test_no_detection_is_identical(pgs, engine):
    srvs = table(pgs, engine, n_parts=3, app_id=34)
    try:
        parts = [Part(pgs, s) for s in srvs]
        rng = np.random.default_rng(5)
        keys = [k for p in range(3) for k in zipf_keys(rng, p, 2000, 0.2)]
        kp = np.repeat(np.arange(3, dtype=np.uint32), 2000)
        k, off = flat(keys)

        def call():
            arena = np.zeros(1 << 22, np.uint8)
            before = pgs.lib().pgs_engine_launches(engine.h)
            st, res, arena, used = pgs.get_batch_multi(parts, k, off, kp, 0, arena)
            assert st == 0
            # values are placed in the arena in the order the groups finish, so they are compared key by key
            ans = [(r.status, r.expire_ts, r.expired, arena[r.value_off:r.value_off + r.value_len].tobytes()) for r in res]
            return ans, used, pgs.lib().pgs_engine_launches(engine.h) - before

        base = call()
        for s in srvs:  # STARTed and STOPped again: back to the plain path
            assert pgs.detect_hotkey(s.h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)[0] == hm.OK
        on = call()
        assert on[:2] == base[:2] and on[2] == base[2] + 1  # the capture kernel, and nothing else changes
        for s in srvs:
            assert pgs.detect_hotkey(s.h, pgs.HOTKEY_READ, pgs.HOTKEY_STOP, T0)[0] == hm.OK
        assert call() == base
        # a WRITE detection does not touch the read path
        assert pgs.detect_hotkey(srvs[0].h, pgs.HOTKEY_WRITE, pgs.HOTKEY_START, T0)[0] == hm.OK
        assert call() == base
    finally:
        for s in srvs:
            s.close()


def test_bucket_count_is_validated(pgs, engine):
    for bad in (1, 2, 39):
        with pytest.raises(AssertionError):
            Backend("gpu", engine, app_id=35, opts={"hotkey_buckets_num": bad})
    s = Backend("gpu", engine, app_id=35, opts={"hotkey_buckets_num": 101, "max_seconds_to_detect_hotkey": 20})
    try:
        assert pgs.detect_hotkey(s.h, pgs.HOTKEY_READ, pgs.HOTKEY_START, T0)[0] == hm.OK
        pgs.hotkey_analyse(s.h, T0 + 10)
        assert pgs.hotkey_state(s.h, pgs.HOTKEY_READ) == hm.COARSE
        pgs.hotkey_analyse(s.h, T0 + 20)
        assert pgs.hotkey_state(s.h, pgs.HOTKEY_READ) == hm.STOPPED
    finally:
        s.close()
