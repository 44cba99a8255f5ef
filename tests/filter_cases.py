"""Inputs for the compaction-filter tests (test_compaction_filter_sim.py, test_compaction_filter_gpu.py): the reference's rule
and operation tables (tests/golden/tables.json) turned into one compaction per table, and seeded random ops tables over
records drawn to sit on the filter's edges."""
import json
import os

import numpy as np

import filter_model as fm
from incubator_pegasus_b200 import synth

T = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tables.json")))
NOW = synth.NOW
GOLDEN_TABLES = ("hashkey_pattern_rule", "sortkey_pattern_rule", "ttl_range_rule", "all_rules_match", "delete_key_filter",
                 "update_ttl_filter")


def ukey(hk, sk):
    return len(hk).to_bytes(2, "big") + hk + sk


def value(ets, data=b"", data_version=1):
    return (ets & fm.M32).to_bytes(4, "big") + (bytes(8) if data_version == 1 else b"") + data


def _tag(i):
    return b"r%03d|" % i


def golden_case(name):
    """one compaction over every row of a golden table.  Row i becomes record i and op i, whose rules are the row's rules
    and one that selects record i alone (a PREFIX rule on "r%03d|", a field the row leaves free).  Returns (records, ops,
    now, want): want[i] is "drop" (a delete op fired), "keep" or the expire_ts an update wrote."""
    rows = T[name]["rows"]
    recs, ops, want = [], [], []
    now = NOW
    sel_sk = lambda i: fm.Rule(fm.RULE_SORTKEY, fm.MATCH_PREFIX, _tag(i))
    for i, row in enumerate(rows):
        if name == "hashkey_pattern_rule":
            v, pat, mt, match = row
            key, rules = ukey(v.encode(), _tag(i)), [fm.Rule(fm.RULE_HASHKEY, mt, pat.encode()), sel_sk(i)]
            ets, op, w = 0, fm.OP_DELETE, "drop" if match else "keep"
        elif name == "sortkey_pattern_rule":  # the sort key is the row's: record i is selected by its hash key
            v, pat, mt, match = row
            key = ukey(_tag(i), v.encode())
            rules = [fm.Rule(fm.RULE_SORTKEY, mt, pat.encode()), fm.Rule(fm.RULE_HASHKEY, fm.MATCH_PREFIX, _tag(i))]
            ets, op, w = 0, fm.OP_DELETE, "drop" if match else "keep"
        elif name == "ttl_range_rule":
            start, stop, rel, match = row
            key, rules = ukey(b"h", _tag(i)), [fm.Rule(fm.RULE_TTL_RANGE, start_ttl=start, stop_ttl=stop), sel_sk(i)]
            ets, op = (NOW + rel) & fm.M32, fm.OP_DELETE
            w = "drop" if match else ("keep" if ets > now else "expired")
        elif name == "all_rules_match":  # ANYWHERE patterns: the "r%03d|" in front of the sort key changes no verdict
            match, hk, sk, rel, hp, hm, sp, sm, start, stop = row
            assert hm == sm == fm.MATCH_ANYWHERE and "|" not in sp
            key = ukey(hk.encode(), _tag(i) + sk.encode())
            rules = [fm.Rule(fm.RULE_HASHKEY, hm, hp.encode()), fm.Rule(fm.RULE_SORTKEY, sm, sp.encode()),
                     fm.Rule(fm.RULE_TTL_RANGE, start_ttl=start, stop_ttl=stop), sel_sk(i)]
            ets, op, w = NOW + rel, fm.OP_DELETE, "drop" if match else "keep"
        elif name == "delete_key_filter":
            match, hk, pat, mt = row
            key, rules = ukey(hk.encode(), _tag(i)), [fm.Rule(fm.RULE_HASHKEY, mt, pat.encode()), sel_sk(i)]
            ets, op, w = 0, fm.OP_DELETE, "drop" if match else "keep"
        else:  # update_ttl_filter: the row's expire_ts and FROM_NOW / FROM_CURRENT results are relative to now
            changed, expect, hk, ets0, pat, mt, ttl_type, ttl_value = row
            key, rules = ukey(hk.encode(), _tag(i)), [fm.Rule(fm.RULE_HASHKEY, mt, pat.encode()), sel_sk(i)]
            ets = NOW + ets0 if ets0 else 0
            w = "keep"
            if changed:
                w = expect - T[name]["epoch_begin"] if ttl_type == fm.TTL_TIMESTAMP else NOW + expect
            recs.append((key, i + 1, 1, value(ets, b"v%d" % i)))
            ops.append(fm.Op(fm.OP_UPDATE_TTL, rules, ttl_type, ttl_value))
            want.append(w)
            continue
        recs.append((key, i + 1, 1, value(ets, b"v%d" % i)))
        ops.append(fm.Op(op, rules))
        want.append(w)
    order = sorted(range(len(recs)), key=lambda i: recs[i][0])
    return [recs[i] for i in order], ops, now, [want[i] for i in order]


# ---- seeded random ops tables ------------------------------------------------------------------------------------------------
HASH_KEYS = [b"", b"a", b"ab", b"abc", b"ba", b"b\xff", b"\x01a", b"x" * 20]
SORT_KEYS = [b"", b"a", b"b", b"ab", b"ba", b"abab", b"xyz", b"0", b"10", b"s\xff"]
NEAR_WRAP_NOW = 0xFFFFFFFF - 40


def _ets_choices(now):
    return [0, 0, (now - 1) & fm.M32, now, (now + 1) & fm.M32, (now + 30) & fm.M32, 0xFFFFFFFF, 1, (now + 100000) & fm.M32]


def random_records(rng, now, n_runs=3, per_run=150, data_version=1):
    """runs of (key, seq, type, value), newest run first: keys repeat across runs (shadowed versions); empty writes and
    1-byte keys; values of 4 and 12 bytes, a few shorter than their header; expire_ts on and around now"""
    runs, seq = [], 1
    ets_c = _ets_choices(now)
    for _ in range(n_runs):
        items = {}
        for _ in range(per_run):
            u = rng.random()
            if u < 0.03:
                key = b""
            elif u < 0.06:
                key = bytes([int(rng.integers(0, 256))])
            else:
                key = ukey(HASH_KEYS[rng.integers(len(HASH_KEYS))], SORT_KEYS[rng.integers(len(SORT_KEYS))])
            typ = 0 if rng.random() < 0.08 else 1
            ets = int(ets_c[rng.integers(len(ets_c))])
            u = rng.random()
            if typ == 0:
                val = b""
            elif u < 0.03:
                val = bytes(int(rng.integers(0, 4)))  # shorter than the expire_ts header: kept as it is
            elif u < 0.25:
                val = ets.to_bytes(4, "big")  # the header alone
            elif u < 0.45 and data_version == 1:
                val = value(ets)  # 12 bytes: the v1 header alone
            else:
                val = value(ets, bytes(rng.integers(0, 256, int(rng.integers(0, 20)), dtype=np.uint8)), data_version)
            items[key] = (key, seq, typ, val)
            seq += 1
        runs.append(sorted(items.values(), key=lambda r: r[0]))
    return runs[::-1]


def _pattern(rng):
    choices = [b"", b"a", b"a", b"b", b"b", b"ab", b"ba", b"abc", b"abab", b"x" * 20, b"x" * 21, b"xyz", b"0", b"\x01", b"zz",
               b"aba", b"\xc3\xa9", b"s"]
    return choices[rng.integers(len(choices))]


def random_ops(rng, now):
    """1-8 ops of 0-4 rules: every match type, TTL ranges whose sums wrap, updates of every kind with values that overflow"""
    # (start_ttl, stop_ttl): windows around now, windows whose sums wrap, the (0, 0) rule of TTL-less values, empty windows
    ranges = [(0, 0), (0, 100000), (2**32 - 1, 1), (2**32 - 100, 31), (1, 2**32 - 1), (2**32 - 1, 2**32 - 1), (0, 30),
              ((2**32 - now) & fm.M32, 2**32 - 1), (50, 40), (2**31, 2**32 - 1)]
    ops = []
    for _ in range(int(rng.integers(1, 9))):
        rules = []
        for _ in range(int(rng.choice([0, 1, 1, 1, 2, 2, 3, 4]))):
            t = int(rng.integers(0, 3))
            if t == fm.RULE_TTL_RANGE:
                start, stop = ranges[rng.integers(len(ranges))]
                rules.append(fm.Rule(t, start_ttl=start, stop_ttl=stop))
            else:
                rules.append(fm.Rule(t, int(rng.choice([0, 0, 1, 1, 2, 2, 3])), _pattern(rng)))
        if rng.random() < 0.35:
            ops.append(fm.Op(fm.OP_DELETE, rules))
        else:
            tt = int(rng.integers(0, 3))
            vals = {fm.TTL_FROM_NOW: [0, 10, 2**32 - 5, 3600],
                    fm.TTL_FROM_CURRENT: [0, 7, 2**32 - 1, 2**31],
                    fm.TTL_TIMESTAMP: [5, fm.EPOCH_BEGIN - 1, fm.EPOCH_BEGIN + now + 30, 2**32 - 1, fm.EPOCH_BEGIN]}[tt]
            ops.append(fm.Op(fm.OP_UPDATE_TTL, rules, tt, int(vals[rng.integers(len(vals))])))
    return ops


# (pidx, partition_version) of validate_hash; None: no hash check
HASH_SETTINGS = [None, (1, 3), (5, 3), (0, 0), (200, 255), (0, -1)]


def filter_settings():
    """the filter settings one seeded table is crossed with"""
    out = []
    for dt in (0, 40):
        for hs in HASH_SETTINGS:
            kw = {"default_ttl": dt}
            if hs:
                kw.update(validate_hash=True, pidx=hs[0], partition_version=hs[1])
            out.append(kw)
    out.append({"enabled": False, "default_ttl": 40})
    return out


def to_records(pgs, run):
    return pgs.Records.from_list(run)


def model_params(ops, **kw):
    kw = {k: v for k, v in kw.items() if k in ("enabled", "default_ttl", "validate_hash", "pidx", "partition_version", "data_version")}
    return fm.Params(ops=list(ops), **kw)


def verdicts(out_records, recs):
    """what became of each of recs in a non-bottommost output: "drop" (a tombstone), "keep" or the expire_ts written"""
    got = {r[0]: r for r in out_records}
    res = []
    for key, _, _, val in recs:
        k, _, typ, v = got[key]
        res.append("drop" if typ == 0 else ("keep" if v == val else fm.expire_ts(v)))
    return res
