"""Plain-Python restatement of the compaction filter (KeyWithTTLCompactionFilter) and of the merge that runs it, written
from the reference sources, not from the oracle or the kernels:

- key_ttl_compaction_filter.h:55-121       Filter, user_specified_operation_filter, check_if_stale_split_data
- compaction_operation.cpp:33-113          all_rules_match, delete_key::filter, update_ttl::filter
- compaction_filter_rule.cpp:31-90         string_pattern_match and the three rules
- pegasus_value_schema.h                   v0 / v1 values: a BE32 expire_ts first (v1 then a BE64 timetag)
- pegasus_key_schema.h                     pegasus_restore_key, pegasus_key_hash

All arithmetic on timestamps is u32, as in the reference.  One pinned deviation (DESIGN §8): a value shorter than its 4-byte
header is kept as it stands; the reference reads past it.

decode_ops(table) walks the binary ops table the way dev_user_ops does (csrc/format.h), so a test can compare what the
parser wrote with what it meant."""
import json
from dataclasses import dataclass, field

EPOCH_BEGIN = 1451606400  # pegasus::utils::epoch_begin
M32 = 0xFFFFFFFF

OP_UPDATE_TTL, OP_DELETE = 0, 1
RULE_HASHKEY, RULE_SORTKEY, RULE_TTL_RANGE = 0, 1, 2
MATCH_ANYWHERE, MATCH_PREFIX, MATCH_POSTFIX, MATCH_INVALID = 0, 1, 2, 3
TTL_FROM_NOW, TTL_FROM_CURRENT, TTL_TIMESTAMP, TTL_INVALID = 0, 1, 2, 3

KEEP, EXPIRED, USER, STALE = 0, 1, 2, 3  # why a value was removed (dev_filter's codes)

STAT_FIELDS = ("in_records", "out_records", "in_bytes", "out_bytes", "dropped_shadowed", "dropped_tombstone", "dropped_expired",
               "dropped_user", "dropped_stale", "ttl_rewritten")

_OP_NAMES = ("COT_UPDATE_TTL", "COT_DELETE")
_RULE_NAMES = ("FRT_HASHKEY_PATTERN", "FRT_SORTKEY_PATTERN", "FRT_TTL_RANGE")
_MATCH_NAMES = ("SMT_MATCH_ANYWHERE", "SMT_MATCH_PREFIX", "SMT_MATCH_POSTFIX", "SMT_INVALID")
_TTL_NAMES = ("UTOT_FROM_NOW", "UTOT_FROM_CURRENT", "UTOT_TIMESTAMP", "UTOT_INVALID")


@dataclass
class Rule:
    type: int
    match: int = MATCH_INVALID
    pattern: bytes = b""
    start_ttl: int = 0
    stop_ttl: int = 0


@dataclass
class Op:
    type: int
    rules: list
    ttl_type: int = TTL_INVALID
    ttl_value: int = 0


@dataclass
class Params:
    enabled: bool = True
    default_ttl: int = 0
    validate_hash: bool = False
    pidx: int = 0
    partition_version: int = -1
    ops: list = field(default_factory=list)
    data_version: int = 1


def to_json(ops, ensure_ascii=True):
    """the `user_specified_compaction` env that create_compaction_operations turns into `ops` (patterns must be UTF-8);
    ensure_ascii: every non-ASCII character of a pattern as a \\u escape, otherwise as UTF-8 text"""
    out = []
    for op in ops:
        rules = []
        for r in op.rules:
            if r.type == RULE_TTL_RANGE:
                p = {"start_ttl": r.start_ttl, "stop_ttl": r.stop_ttl}
            else:
                p = {"pattern": r.pattern.decode("utf-8"), "match_type": _MATCH_NAMES[r.match]}
            rules.append({"type": _RULE_NAMES[r.type], "params": json.dumps(p, ensure_ascii=ensure_ascii)})
        params = json.dumps({"type": _TTL_NAMES[op.ttl_type], "value": op.ttl_value}) if op.type == OP_UPDATE_TTL else ""
        out.append({"type": _OP_NAMES[op.type], "params": params, "rules": rules})
    return json.dumps({"ops": out}, ensure_ascii=ensure_ascii)


def decode_ops(table):
    """the binary ops table as dev_user_ops walks it: u32 n_ops; per op u8 op_type, u8 ttl_type, u16 n_rules, u32 ttl_value;
    per rule u8 rule_type, u8 match_type, u16 pattern_len, u32 start_ttl, u32 stop_ttl, the pattern zero-padded to 4 bytes.
    Also returns where the walk ended."""
    t = bytes(table)
    le = lambda a, n: int.from_bytes(t[a:a + n], "little")
    ops, p = [], 4
    for _ in range(le(0, 4)):
        op = Op(type=t[p], ttl_type=t[p + 1], ttl_value=le(p + 4, 4), rules=[])
        n_rules = le(p + 2, 2)
        p += 8
        for _ in range(n_rules):
            pl = le(p + 2, 2)
            op.rules.append(Rule(type=t[p], match=t[p + 1], pattern=t[p + 12:p + 12 + pl], start_ttl=le(p + 4, 4), stop_ttl=le(p + 8, 4)))
            p += 12 + ((pl + 3) & ~3)
        ops.append(op)
    return ops, p


# ---- schemas -------------------------------------------------------------------------------------------------------------
def expire_ts(value):
    return int.from_bytes(value[:4], "big")


def with_expire_ts(value, ts):
    return (ts & M32).to_bytes(4, "big") + value[4:]


def restore_key(key):
    """pegasus_restore_key: (hash key, sort key) of a user key of >= 2 bytes"""
    hkl = int.from_bytes(key[:2], "big")
    return key[2:2 + hkl], key[2 + hkl:]


def _crc64_table():
    bits = (63, 61, 59, 58, 56, 55, 52, 49, 48, 47, 46, 44, 41, 37, 36, 34, 32, 31, 28, 26, 23, 22, 19, 16, 13, 12, 10, 9, 6, 4,
            3, 0)  # utils/crc.cpp: the polynomial's bit list
    poly = sum(1 << (63 - b) for b in bits)
    tab = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ poly if c & 1 else c >> 1
        tab.append(c)
    return tab


_CRC = _crc64_table()


def crc64(data, init=0):
    c = ~init & 0xFFFFFFFFFFFFFFFF
    for b in data:
        c = _CRC[(c ^ b) & 0xFF] ^ (c >> 8)
    return ~c & 0xFFFFFFFFFFFFFFFF


def key_hash(key):
    """pegasus_key_hash: crc64 of the hash key, or of the sort key when the hash key is empty"""
    hkl = int.from_bytes(key[:2], "big")
    return crc64(key[2:2 + hkl]) if hkl > 0 else crc64(key[2:])


# ---- rules and operations ------------------------------------------------------------------------------------------------
def string_pattern_match(value, match, pattern):
    if not pattern or len(value) < len(pattern):
        return False
    if match == MATCH_ANYWHERE:
        return pattern in value
    if match == MATCH_PREFIX:
        return value.startswith(pattern)
    if match == MATCH_POSTFIX:
        return value.endswith(pattern)
    return False


def rule_match(rule, hk, sk, value, now):
    if rule.type == RULE_HASHKEY:
        return string_pattern_match(hk, rule.match, rule.pattern)
    if rule.type == RULE_SORTKEY:
        return string_pattern_match(sk, rule.match, rule.pattern)
    if rule.type == RULE_TTL_RANGE:
        ets = expire_ts(value)
        if ets == 0 and rule.start_ttl == 0 and rule.stop_ttl == 0:
            return True
        return (rule.start_ttl + now) & M32 <= ets and (rule.stop_ttl + now) & M32 >= ets
    return False


def op_filter(op, hk, sk, value, now):
    """(delete, the expire_ts the op writes or None)"""
    if not op.rules or not all(rule_match(r, hk, sk, value, now) for r in op.rules):
        return False, None
    if op.type == OP_DELETE:
        return True, None
    if op.ttl_type == TTL_FROM_NOW:
        return False, (now + op.ttl_value) & M32
    if op.ttl_type == TTL_FROM_CURRENT:
        ets = expire_ts(value)
        return False, None if ets == 0 else (op.ttl_value + ets) & M32
    if op.ttl_type == TTL_TIMESTAMP:
        return False, (op.ttl_value - EPOCH_BEGIN) & M32
    return False, None


def filter(params, key, value, now):
    """KeyWithTTLCompactionFilter::Filter on one value: (remove, reason, new value or None when unchanged)"""
    if not params.enabled or len(key) < 2 or len(value) < 4:
        return False, KEEP, None
    ets = expire_ts(value)
    new_value = None
    if params.default_ttl != 0 and ets == 0:  # the default_ttl rewrite comes first
        ets = (now + params.default_ttl) & M32
        new_value = with_expire_ts(value, ets)
    if params.ops:
        entry = value if new_value is None else new_value  # every op sees this value, never another op's rewrite
        hk, sk = restore_key(key)
        for op in params.ops:
            delete, ts = op_filter(op, hk, sk, entry, now)
            if delete:
                return True, USER, None
            if ts is not None:  # a later rewrite replaces an earlier one
                new_value = with_expire_ts(entry, ts)
    if 0 < ets <= now:  # check_if_ts_expired on the default_ttl timestamp, whatever an op wrote
        return True, EXPIRED, None
    if params.validate_hash and params.partition_version >= 0 and params.pidx <= params.partition_version:
        if key_hash(key) & params.partition_version != params.pidx & 0xFFFFFFFFFFFFFFFF:
            return True, STALE, None
    return False, KEEP, new_value


# ---- the merge -------------------------------------------------------------------------------------------------------------
def compact(runs, bottommost, params, now):
    """RocksDB's compaction iterator without snapshots over runs of (user key, seq, type, value) records (type 1 value,
    0 deletion): the newest version of each user key wins and only it is filtered, and only when it is a value.  A removed
    value becomes a deletion with the same seq and an empty value, except at the bottommost level, where deletions are
    dropped and survivors' seqs are zeroed.  Returns (records in internal-key order, the ten CompactResult counters)."""
    st = dict.fromkeys(STAT_FIELDS, 0)
    recs = [r for run in runs for r in run]
    for k, _, _, v in recs:
        st["in_records"] += 1
        st["in_bytes"] += len(k) + len(v)
    recs.sort(key=lambda r: (r[0], -r[1]))
    out, prev = [], None
    for key, seq, typ, value in recs:
        if key == prev:
            st["dropped_shadowed"] += 1
            continue
        prev = key
        if typ == 1:
            remove, why, nv = filter(params, key, value, now)
            if remove:
                st[("", "dropped_expired", "dropped_user", "dropped_stale")[why]] += 1
                if not bottommost:
                    out.append((key, seq, 0, b""))
                continue
            if nv is not None:
                st["ttl_rewritten"] += 1
                value = nv
            out.append((key, 0 if bottommost else seq, 1, value))
        elif bottommost:
            st["dropped_tombstone"] += 1
        else:
            out.append((key, seq, typ, value))
    for k, _, _, v in out:
        st["out_records"] += 1
        st["out_bytes"] += len(k) + len(v)
    return out, st
