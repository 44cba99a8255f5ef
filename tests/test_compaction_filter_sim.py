"""The fused compaction filter (dev_filter / dev_user_ops in csrc/compact_kernels.cuh) in the kernel simulator, against
tests/filter_model.py and the oracle: the reference's rule and operation tables, seeded random ops tables over records on the
filter's edges, data_version 0, long keys and patterns, values on the emit in-place path.  Every case runs at lane widths 1
and 8 (check), which also compares the new run's format and every statistic with the oracle."""
import numpy as np
import pytest

import filter_cases as fc
import filter_model as fm
from test_kernel_sim import STAT_FIELDS, check, sim, sim_compact  # noqa: F401  (sim is a fixture)


def run_filter_case(pgs, oracle, sim, runs, ops, *, bottommost, now=fc.NOW, data_version=1, seg_weight=8 * 1024, **kw):
    """the simulator against the oracle (check) and both against the model: records and the ten counters"""
    recs = [fc.to_records(pgs, r) for r in runs]
    x = check(pgs, oracle, sim, recs, bottommost=bottommost, ops_json=fm.to_json(ops) if ops else None, now=now,
              data_version=data_version, seg_weight=seg_weight, **kw)
    want, st = fm.compact(runs, bottommost, fc.model_params(ops, data_version=data_version, **kw), now)
    assert [x["stats"][i] for i in range(len(STAT_FIELDS))] == [st[f] for f in STAT_FIELDS]
    assert x["got"] == want
    return x, want, st


# ---- the model on its own ------------------------------------------------------------------------------------------------------
def test_model_agrees_with_the_golden_tables():
    """every row of the six tables through filter_model alone, as the reference's unit tests state them"""
    T = fc.T
    now = fc.NOW
    for v, pat, mt, want in T["hashkey_pattern_rule"]["rows"]:
        assert fm.rule_match(fm.Rule(fm.RULE_HASHKEY, mt, pat.encode()), v.encode(), b"", b"", now) == want
    for v, pat, mt, want in T["sortkey_pattern_rule"]["rows"]:
        assert fm.rule_match(fm.Rule(fm.RULE_SORTKEY, mt, pat.encode()), b"", v.encode(), b"", now) == want
    for start, stop, rel, want in T["ttl_range_rule"]["rows"]:
        r = fm.Rule(fm.RULE_TTL_RANGE, start_ttl=start, stop_ttl=stop)
        assert fm.rule_match(r, b"", b"", fc.value(now + rel), now) == want
    for want, hk, sk, rel, hp, hm, sp, sm, start, stop in T["all_rules_match"]["rows"]:
        op = fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_HASHKEY, hm, hp.encode()), fm.Rule(fm.RULE_SORTKEY, sm, sp.encode()),
                                  fm.Rule(fm.RULE_TTL_RANGE, start_ttl=start, stop_ttl=stop)])
        assert fm.op_filter(op, hk.encode(), sk.encode(), fc.value(now + rel), now)[0] == want
    assert fm.op_filter(fm.Op(fm.OP_DELETE, []), b"hash", b"sort", b"", now) == (T["all_rules_match"]["empty_rules_match"], None)
    for want, hk, pat, mt in T["delete_key_filter"]["rows"]:
        assert fm.op_filter(fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_HASHKEY, mt, pat.encode())]), hk.encode(), b"", b"", now)[0] == want
    eb = T["update_ttl_filter"]["epoch_begin"]
    assert eb == fm.EPOCH_BEGIN
    for changed, expect, hk, ets, pat, mt, ttl_type, ttl_value in T["update_ttl_filter"]["rows"]:
        op = fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_HASHKEY, mt, pat.encode())], ttl_type, ttl_value)
        delete, ts = fm.op_filter(op, hk.encode(), b"", fc.value(ets), now)
        assert not delete and (ts is not None) == changed
        if changed:
            assert ts == {fm.TTL_FROM_NOW: expect + now, fm.TTL_FROM_CURRENT: expect, fm.TTL_TIMESTAMP: expect - eb}[ttl_type]


def test_model_order_of_steps():
    """default_ttl first; every op sees the default_ttl value, a later update wins, a delete returns at once; the expiry check
    uses the default_ttl timestamp; the stale-split check comes last"""
    now = 1000
    key = fc.ukey(b"ab", b"cd")
    hk_a = fm.Rule(fm.RULE_HASHKEY, fm.MATCH_PREFIX, b"a")
    upd = lambda tt, v, *r: fm.Op(fm.OP_UPDATE_TTL, [hk_a, *r], tt, v)
    P = lambda **kw: fm.Params(**kw)
    # FROM_CURRENT on the default_ttl timestamp, not on the value's 0
    assert fm.filter(P(default_ttl=40, ops=[upd(fm.TTL_FROM_CURRENT, 5)]), key, fc.value(0), now)[2] == fc.value(1045)
    # the second op sees 1040 (default_ttl), not the first op's 2000, and its rewrite wins
    ops = [upd(fm.TTL_FROM_NOW, 1000), upd(fm.TTL_FROM_CURRENT, 1)]
    assert fm.filter(P(default_ttl=40, ops=ops), key, fc.value(0), now)[2] == fc.value(1041)
    # a range rule of a later op sees the entry's timestamp, not an earlier op's
    rng_1040 = fm.Rule(fm.RULE_TTL_RANGE, start_ttl=40, stop_ttl=40)
    assert fm.filter(P(default_ttl=40, ops=[upd(fm.TTL_FROM_NOW, 5), fm.Op(fm.OP_DELETE, [rng_1040])]), key, fc.value(0), now)[:2] == (True, fm.USER)
    # an update does not save an expired value, and expiry is decided on the value's own timestamp
    assert fm.filter(P(ops=[upd(fm.TTL_FROM_NOW, 50)]), key, fc.value(999), now)[:2] == (True, fm.EXPIRED)
    assert fm.filter(P(ops=[upd(fm.TTL_TIMESTAMP, 5)]), key, fc.value(2000), now) == (False, fm.KEEP, fc.value(5 - fm.EPOCH_BEGIN))
    # a delete op wins over expiry and over the stale-split check
    stale = P(validate_hash=True, pidx=1, partition_version=1, ops=[fm.Op(fm.OP_DELETE, [hk_a])])
    assert fm.filter(stale, key, fc.value(5), now)[:2] == (True, fm.USER)
    h = fm.key_hash(key) & 1
    assert fm.filter(P(validate_hash=True, pidx=1 - h, partition_version=1), key, fc.value(0), now)[:2] == (True, fm.STALE)
    assert fm.filter(P(validate_hash=True, pidx=1 - h, partition_version=1), key, fc.value(5), now)[:2] == (True, fm.EXPIRED)
    # u32 arithmetic: FROM_CURRENT wraps, a range whose sums wrap
    assert fm.filter(P(ops=[upd(fm.TTL_FROM_CURRENT, 2**32 - 1)]), key, fc.value(2000), now)[2] == fc.value(1999)
    assert fm.rule_match(fm.Rule(fm.RULE_TTL_RANGE, start_ttl=2**32 - 10, stop_ttl=2**32 - 1), b"", b"", fc.value(995), now)
    # never filtered: the empty write, a 1-byte key, a value shorter than its header
    for k, v in ((b"", fc.value(5)), (b"\x00", fc.value(5)), (key, b"\x00\x00\x05")):
        assert fm.filter(P(default_ttl=40, ops=[fm.Op(fm.OP_DELETE, [hk_a])]), k, v, now) == (False, fm.KEEP, None)


def test_model_crc64_and_key_hash(oracle):
    L = oracle.lib()
    for data in (b"", b"a", b"123456789", bytes(range(256)) * 3):
        assert fm.crc64(data) == L.orc_crc64(data, len(data), 0)
    for key in (fc.ukey(b"hash", b"sort"), fc.ukey(b"", b"sort"), fc.ukey(b"", b"")):
        assert fm.key_hash(key) == L.orc_key_hash(key, len(key))


# ---- the kernels -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table", fc.GOLDEN_TABLES)
def test_sim_golden_table_rows(pgs, oracle, sim, table):
    """every row of a golden table is one record and one op of a single compaction; each row's verdict is read back"""
    recs, ops, now, want = fc.golden_case(table)
    params = fc.model_params(ops)
    for (key, _, _, val), w in zip(recs, want):
        remove, why, nv = fm.filter(params, key, val, now)
        assert (why == fm.USER) == (w == "drop") and (why == fm.EXPIRED) == (w == "expired")
        assert (nv is not None) == isinstance(w, int) and (nv is None or fm.expire_ts(nv) == w)
    for bm in (False, True):
        x, out, st = run_filter_case(pgs, oracle, sim, [recs], ops, bottommost=bm, now=now)
        if not bm:
            assert fc.verdicts(out, recs) == ["drop" if w == "expired" else w for w in want]
        assert st["dropped_user"] == want.count("drop") and st["ttl_rewritten"] == sum(isinstance(w, int) for w in want)


@pytest.mark.parametrize("seed", range(6))
def test_sim_seeded_ops_tables(pgs, oracle, sim, seed):
    """a random table of 1-8 ops over records on the edges, crossed with default_ttl, validate_hash settings, a disabled
    filter and both output levels; odd seeds put now 40 s below 2^32, so that timestamps and range sums wrap"""
    rng = np.random.default_rng(1000 + seed)
    now = fc.NEAR_WRAP_NOW if seed % 2 else fc.NOW
    runs = fc.random_records(rng, now)
    ops = fc.random_ops(rng, now)
    settings = fc.filter_settings()
    seen = dict.fromkeys(STAT_FIELDS, 0)
    for i, kw in enumerate(settings):
        # every setting at one output level, the levels alternating (seed parity flips the pairing)
        x, out, st = run_filter_case(pgs, oracle, sim, runs, ops, bottommost=(i + seed) % 2 == 0, now=now, **kw)
        for f in STAT_FIELDS:
            seen[f] += st[f]
    assert seen["dropped_expired"] and seen["dropped_stale"] and seen["dropped_shadowed"]


def test_sim_seeded_tables_hit_every_verdict(pgs, oracle, sim):
    """the seeded tables are not vacuous: over the seeds, user deletes and rewrites both happen on the kernel"""
    tot_user = tot_rw = 0
    for seed in range(6):
        rng = np.random.default_rng(1000 + seed)
        now = fc.NEAR_WRAP_NOW if seed % 2 else fc.NOW
        runs = fc.random_records(rng, now)
        ops = fc.random_ops(rng, now)
        _, st = fm.compact(runs, True, fc.model_params(ops), now)
        tot_user += st["dropped_user"]
        tot_rw += st["ttl_rewritten"]
    assert tot_user > 20 and tot_rw > 20


def _edge_ops(now):
    """two updates that both fire, then a delete on a wrapping range; FROM_CURRENT on sums that overflow; TIMESTAMP below
    epoch_begin"""
    R = fm.Rule
    return [
        fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_HASHKEY, fm.MATCH_ANYWHERE, b"a")], fm.TTL_FROM_NOW, 10),
        fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_SORTKEY, fm.MATCH_PREFIX, b"a")], fm.TTL_FROM_CURRENT, 2**32 - 3),
        fm.Op(fm.OP_UPDATE_TTL, [R(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"b")], fm.TTL_TIMESTAMP, 7),
        fm.Op(fm.OP_DELETE, [R(fm.RULE_TTL_RANGE, start_ttl=2**32 - 100, stop_ttl=100), R(fm.RULE_HASHKEY, fm.MATCH_POSTFIX, b"b")]),
    ]


def test_sim_data_version_0(pgs, oracle, sim):
    """v0 values (BE32 expire_ts | data): TTL rules, every update kind and default_ttl on the 4-byte header"""
    rng = np.random.default_rng(77)
    runs = fc.random_records(rng, fc.NOW, data_version=0)
    for dt in (0, 40):
        for bm in (True, False):
            x, out, st = run_filter_case(pgs, oracle, sim, runs, _edge_ops(fc.NOW), bottommost=bm, data_version=0, default_ttl=dt)
            assert st["ttl_rewritten"] > 0 and st["dropped_user"] > 0


def test_sim_long_keys_and_patterns(pgs, oracle, sim):
    """4096-byte user keys, ANYWHERE and POSTFIX sort-key patterns of 1-2 KB that match, miss by one byte, or are longer
    than the field"""
    rng = np.random.default_rng(5)
    recs = []
    body = bytes(rng.integers(97, 100, 8000, dtype=np.uint8))
    for i in range(60):
        hk = b"h%03d" % i
        off = int(rng.integers(0, 3000))
        sk = body[off:off + 4096 - 2 - len(hk)]
        recs.append((fc.ukey(hk, sk), i + 1, 1, fc.value(0 if i % 3 else fc.NOW + 9, b"x" * (i % 7))))
    recs.sort(key=lambda r: r[0])
    sk0 = fm.restore_key(recs[7][0])[1]
    sk1 = fm.restore_key(recs[20][0])[1]
    ops = [
        fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, sk0[-1500:])]),
        fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_ANYWHERE, sk1[900:2900])], fm.TTL_FROM_NOW, 77),
        fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_ANYWHERE, sk1[1000:2000][:-1] + b"z")]),   # misses
        fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"a" + sk0)]),                   # longer than the field
        fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_ANYWHERE, body[4000:5024])], fm.TTL_FROM_CURRENT, 3),
    ]
    for bm in (True, False):
        x, out, st = run_filter_case(pgs, oracle, sim, [recs], ops, bottommost=bm, default_ttl=40, seg_weight=64 * 1024)
        assert st["dropped_user"] >= 1 and st["ttl_rewritten"] >= 1


def test_sim_rewrites_of_values_on_the_in_place_path(pgs, oracle, sim):
    """values just above the emit block buffer (k_emit copies them in place) rewritten by default_ttl and by an op, next to
    runs of tiny entries; older versions that would be rewritten but are shadowed do not count in ttl_rewritten"""
    rng = np.random.default_rng(9)
    new, old = [], []
    seq = 10_000
    for i in range(900):
        key = fc.ukey(b"k", b"%05d" % i)
        big = i % 97 == 50
        vl = int(rng.choice([4100, 4130, 4200, 8000])) if big else int(rng.integers(0, 6))
        ets = 0 if i % 2 else fc.NOW + 500
        new.append((key, seq + i, 1, fc.value(ets, bytes(rng.integers(0, 256, vl, dtype=np.uint8)))))
        if i % 5 == 0:  # an older version with no TTL: default_ttl would rewrite it, but it is shadowed
            old.append((key, 1 + i, 1, fc.value(0, b"old")))
    ops = [fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"0")], fm.TTL_FROM_NOW, 3600)]
    runs = [new, old]
    for ri in (1, 16):
        x, out, st = run_filter_case(pgs, oracle, sim, runs, ops, bottommost=True, default_ttl=40, restart_interval=ri,
                                     seg_weight=64 * 1024)
        newest_no_ttl = sum(1 for r in new if fm.expire_ts(r[3]) == 0)
        by_op = sum(1 for r in new if fm.expire_ts(r[3]) != 0 and r[0].endswith(b"0"))
        assert st["ttl_rewritten"] == newest_no_ttl + by_op and st["dropped_shadowed"] == len(old)
        assert any(len(r[3]) > 4096 and fm.expire_ts(r[3]) == fc.NOW + 3600 for r in out)
        assert any(len(r[3]) > 4096 and fm.expire_ts(r[3]) == fc.NOW + 40 for r in out)


# ---- the launch refuses a malformed ops table --------------------------------------------------------------------------------
def _table(*ops):
    """a binary ops table from (op_type, ttl_type, ttl_value, [(rule_type, match_type, pattern, start, stop, pattern_len)])"""
    out = bytearray(len(ops).to_bytes(4, "little"))
    for ot, tt, tv, rules in ops:
        out += bytes([ot, tt]) + len(rules).to_bytes(2, "little") + tv.to_bytes(4, "little")
        for rt, mt, pat, start, stop, pl in rules:
            out += bytes([rt, mt]) + pl.to_bytes(2, "little") + start.to_bytes(4, "little") + stop.to_bytes(4, "little")
            out += pat + bytes(-len(pat) % 4)
    return bytes(out)


GOOD_RULE = (fm.RULE_HASHKEY, fm.MATCH_PREFIX, b"abc", 0, 0, 3)
MALFORMED = {
    "short header": b"\x01\x00",
    "truncated op": _table((1, 3, 0, [GOOD_RULE]))[:10],
    "truncated pattern": _table((1, 3, 0, [GOOD_RULE]))[:-1],
    "trailing bytes": _table((1, 3, 0, [GOOD_RULE])) + bytes(4),
    "more ops than bytes": (2).to_bytes(4, "little") + _table((1, 3, 0, [GOOD_RULE]))[4:],
    "op type 2": _table((2, 3, 0, [GOOD_RULE])),
    "ttl type 4": _table((0, 4, 5, [GOOD_RULE])),
    "rule type 3": _table((1, 3, 0, [(3, 1, b"abc", 0, 0, 3)])),
    "match type 4": _table((1, 3, 0, [(0, 4, b"abc", 0, 0, 3)])),
    "pattern length past the end": _table((1, 3, 0, [(0, 1, b"abc", 0, 0, 200)])),
    # what the parser wrote for one 65 540-byte pattern before lengths were checked: the length field says 4
    "misframed long pattern": _table((1, 3, 0, [(0, 1, b"x" * 65540, 0, 0, 4)])),
}


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_sim_launch_refuses_a_malformed_ops_table(pgs, sim, name):
    runs = [pgs.Records.from_list([(fc.ukey(b"abc", b"d"), 1, 1, fc.value(0))])]
    table = np.frombuffer(MALFORMED[name], np.uint8).copy()
    assert sim_compact(pgs, sim, runs, bottommost=True, ops=table, status=pgs.INVALID_ARGUMENT) == (None, None)


def test_sim_launch_accepts_well_formed_tables(pgs, sim):
    runs = [pgs.Records.from_list([(fc.ukey(b"abc", b"d"), 1, 1, fc.value(0))])]
    for t in (_table(), _table((1, 3, 0, [GOOD_RULE])), _table((0, 1, 7, [GOOD_RULE, (2, 3, b"", 1, 2, 0)]), (1, 3, 0, []))):
        out, x = sim_compact(pgs, sim, runs, bottommost=True, ops=np.frombuffer(t, np.uint8).copy())
        assert x["stats"][0] == 1
