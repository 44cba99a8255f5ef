"""Pins the scan model of tests/scan_model.py to the oracle's multi_get, whose forward and reverse loops are pinned to the
reference's own tables (tests/golden/multi_get_basic.json, test_oracle_golden.py): the same writes go into an oracle backend
and into the model's visible set; every multi_get is translated into the range request the server builds from it
(host/server.cpp do_multi_get) and run through model_scan.  kvs (reverse ones re-reversed), counters and the kIncomplete
status must agree."""
import random

from rrdb_harness import Backend
from scan_model import model_scan, next_key, raw_key, value

NOW = 200_000_000
INT_MAX = 2**31 - 1


def mget_request(hk, start=b"", stop=b"", start_inclusive=True, stop_inclusive=False, max_kv_count=0, max_kv_size=0, no_value=False,
                 reverse=False, filter_type=0, filter_pattern=b""):
    """on_multi_get's range mode as the server translates it (default limits: 3000 records, 30 MB); None = answered empty"""
    max_count = max_kv_count if 0 < max_kv_count < 3000 else 3000
    max_size = min(max_kv_size if max_kv_size > 0 else INT_MAX, 30 << 20)
    s = raw_key(hk, start)
    if stop:
        e, ei = raw_key(hk, stop), stop_inclusive
    else:
        e, ei = next_key(raw_key(hk, b"")), False
    si = start_inclusive
    if filter_type == 2 and filter_pattern:  # a sort-key prefix filter narrows the range (:558-578)
        ps = raw_key(hk, filter_pattern)
        pe = next_key(ps)
        if ps > s:
            s, si = ps, True
        if pe <= e:
            e, ei = pe, False
    if s > e or (s == e and not (si and ei)):
        return None
    return dict(start=s, stop=e, start_inclusive=si, stop_inclusive=ei, reverse=reverse, no_value=no_value, key_mode=1,
                prefix=not reverse, sft=filter_type, spat=filter_pattern, max_count=max_count, max_iter_count=3000, max_iter_size=max_size)


def test_model_matches_the_oracle_multi_get():
    rnd = random.Random(21)
    o = Backend("oracle", opts={"l0_compaction_trigger": 100})
    state = {}
    hks = [b"a", b"b", b""]
    try:
        for round_ in range(5):
            for _ in range(150):
                hk, sk = rnd.choice(hks), b"%03d" % rnd.randrange(60)
                if rnd.random() < 0.25:
                    o.remove(hk, sk, now=NOW)
                    state.pop(raw_key(hk, sk), None)
                else:
                    user = bytes(rnd.getrandbits(8) for _ in range(rnd.choice([0, 3, 40])))
                    ets = rnd.choice([0, 0, NOW + 50, NOW - 50])
                    o.put(hk, sk, user, expire_ts=ets, now=NOW)
                    state[raw_key(hk, sk)] = value(ets, user)
            o.flush(NOW)
        vis = sorted(state.items())
        cases = [dict(reverse=False), dict(reverse=True)]
        for _ in range(150):
            c = dict(reverse=rnd.random() < 0.5)
            if rnd.random() < 0.6:
                c["start"] = b"%03d" % rnd.randrange(70)
                c["start_inclusive"] = rnd.random() < 0.5
            if rnd.random() < 0.6:
                c["stop"] = b"%03d" % rnd.randrange(70)
                c["stop_inclusive"] = rnd.random() < 0.5
            if rnd.random() < 0.4:
                c["max_kv_count"] = rnd.randrange(1, 12)
            if rnd.random() < 0.3:
                c["max_kv_size"] = rnd.randrange(1, 200)
            if rnd.random() < 0.3:
                c["filter_type"], c["filter_pattern"] = rnd.randrange(1, 4), rnd.choice([b"1", b"0", b"05", b""])
            c["no_value"] = rnd.random() < 0.2
            cases.append(c)
        incomplete = 0
        for hk in hks:
            for c in cases:
                got = o.multi_get(hk, now=NOW, **c)
                q = mget_request(hk, **c)
                if q is None:
                    assert got["error"] == 0 and got["kvs"] == [], (hk, c)
                    continue
                want = model_scan(vis, q, NOW)
                kvs = want["kvs"][::-1] if c["reverse"] else want["kvs"]
                status = 7 if want["iter_valid"] and not want["complete"] else 0  # kIncomplete
                incomplete += status == 7
                assert got["kvs"] == kvs, (hk, c)
                assert len(got["kvs"]) == want["count"], (hk, c)
                assert (got["error"], got["iteration_count"], got["expire_count"], got["filter_count"]) == \
                    (status, want["iter_count"], want["expire_count"], want["filter_count"]), (hk, c, got["error"], want)
        assert incomplete > 20
    finally:
        o.close()
