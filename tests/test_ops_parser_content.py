"""What the `user_specified_compaction` parser writes (pgs_compaction_ops_parse, host/host_util.cpp), field by field: the binary
table, walked the way the compaction kernel walks it (filter_model.decode_ops), must hold the operations and rules the
oracle's create_compaction_operations keeps (orc_ops_describe / orc_ops_describe_rule), for patterns with \\u escapes and
non-ASCII text and for patterns too long for the table's 16-bit length field."""
import ctypes as C
import json

import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import filter_model as fm

MAX_PATTERN = 0xFFFF


def oracle_ops(oracle, text):
    L = oracle.lib()
    L.orc_ops_describe.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
    L.orc_ops_describe_rule.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_char_p, C.c_uint32,
                                        C.c_void_p, C.c_void_p]
    ops = oracle.Ops(text)
    out = []
    for i in range(len(ops)):
        ot, tt, tv, nr = C.c_int32(), C.c_int32(), C.c_uint32(), C.c_uint32()
        assert L.orc_ops_describe(ops.h, i, C.byref(ot), C.byref(tt), C.byref(tv), C.byref(nr)) == 0
        op = fm.Op(ot.value, [], tt.value if ot.value == fm.OP_UPDATE_TTL else fm.TTL_INVALID,
                   tv.value if ot.value == fm.OP_UPDATE_TTL else 0)
        for r in range(nr.value):
            rt, mt, s, e = C.c_int32(), C.c_int32(), C.c_uint32(), C.c_uint32()
            buf = C.create_string_buffer(80_000)
            L.orc_ops_describe_rule(ops.h, i, r, C.byref(rt), C.byref(mt), buf, len(buf), C.byref(s), C.byref(e))
            if rt.value == fm.RULE_TTL_RANGE:
                op.rules.append(fm.Rule(rt.value, fm.MATCH_INVALID, b"", s.value, e.value))
            else:
                op.rules.append(fm.Rule(rt.value, mt.value, buf.value))  # patterns here hold no NUL byte
        out.append(op)
    return out


def expected_table(ops):
    """the table the kernel should see: the oracle's ops, with a pattern longer than 65 535 bytes (it can match no key)
    stored as the empty pattern, which never matches either"""
    for op in ops:
        for r in op.rules:
            if len(r.pattern) > MAX_PATTERN:
                r.pattern = b""
    return ops


def check_parse(pgs, oracle, text):
    table = pgs.parse_ops(text)
    got, end = fm.decode_ops(table)
    assert end == len(table)  # the walk ends exactly at the table's end
    want = expected_table(oracle_ops(oracle, text))
    assert got == want
    return got


# ---- hypothesis: well-formed tables of every field ---------------------------------------------------------------------------
pattern_text = st.text(alphabet=st.characters(min_codepoint=1, max_codepoint=0x2FFFF, blacklist_categories=("Cs",)), max_size=12)
u32 = st.one_of(st.sampled_from([0, 1, 2**31, 2**32 - 1, fm.EPOCH_BEGIN, fm.EPOCH_BEGIN - 1]), st.integers(0, 2**32 - 1))


@st.composite
def rule(draw):
    t = draw(st.integers(0, 2))
    if t == fm.RULE_TTL_RANGE:
        return fm.Rule(t, start_ttl=draw(u32), stop_ttl=draw(u32))
    return fm.Rule(t, draw(st.integers(0, 3)), draw(pattern_text).encode("utf-8"))


@st.composite
def op(draw):
    rules = draw(st.lists(rule(), min_size=1, max_size=4))
    if draw(st.booleans()):
        return fm.Op(fm.OP_DELETE, rules)
    return fm.Op(fm.OP_UPDATE_TTL, rules, draw(st.integers(0, 3)), draw(u32))


@settings(max_examples=300, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(ops=st.lists(op(), max_size=5), ascii_only=st.booleans())
def test_parsed_table_matches_the_oracle_field_by_field(pgs, oracle, ops, ascii_only):
    text = fm.to_json(ops, ensure_ascii=ascii_only)
    got = check_parse(pgs, oracle, text)
    assert got == ops  # fm.to_json writes nothing the reference drops


def test_escapes_and_non_ascii_patterns(pgs, oracle):
    raw = ('{"ops":[{"type":"COT_DELETE","params":"","rules":['
           '{"type":"FRT_HASHKEY_PATTERN","params":"{\\"pattern\\":\\"\\\\u00e9\\\\u4e2d\\\\ud83d\\\\ude00\\\\\\"\\\\\\\\\\\\/\\\\t\\",\\"match_type\\":\\"SMT_MATCH_PREFIX\\"}"},'
           '{"type":"FRT_SORTKEY_PATTERN","params":"{\\"pattern\\":\\"é中\\",\\"match_type\\":\\"SMT_MATCH_POSTFIX\\"}"}]}]}')
    got = check_parse(pgs, oracle, raw)
    assert got[0].rules[0].pattern == "é中😀\"\\/\t".encode()
    assert got[0].rules[1].pattern == "é中".encode()


@pytest.mark.parametrize("n", [65_535, 65_536, 70_000])
def test_patterns_longer_than_the_length_field(pgs, oracle, n):
    """a pattern of n bytes between two ordinary rules and before another op: the table stays framed; up to 65 535 bytes the
    pattern is kept, longer ones become the empty pattern (no key is that long, so neither ever matches)"""
    big = ("ab" * n)[:n]
    ops = [fm.Op(fm.OP_DELETE, [fm.Rule(fm.RULE_SORTKEY, fm.MATCH_PREFIX, b"s"), fm.Rule(fm.RULE_HASHKEY, fm.MATCH_PREFIX, big.encode()),
                                fm.Rule(fm.RULE_SORTKEY, fm.MATCH_POSTFIX, b"xy")]),
           fm.Op(fm.OP_UPDATE_TTL, [fm.Rule(fm.RULE_TTL_RANGE, start_ttl=3, stop_ttl=9)], fm.TTL_FROM_NOW, 77)]
    got = check_parse(pgs, oracle, fm.to_json(ops))
    assert len(got) == 2 and len(got[0].rules) == 3
    assert got[0].rules[1].pattern == (big.encode() if n <= MAX_PATTERN else b"")
    assert got[0].rules[2] == ops[0].rules[2] and got[1] == ops[1]


def test_more_rules_than_the_count_field_is_refused(pgs, oracle):
    rule_ = {"type": "FRT_TTL_RANGE", "params": json.dumps({"start_ttl": 0, "stop_ttl": 1})}
    for n, ok in ((65_535, True), (65_536, False)):
        text = json.dumps({"ops": [{"type": "COT_DELETE", "params": "", "rules": [rule_] * n}]})
        if ok:
            got, end = fm.decode_ops(pgs.parse_ops(text))
            assert len(got) == 1 and len(got[0].rules) == n and len(oracle.Ops(text)) == 1
        else:
            with pytest.raises(pgs.PegasusError) as e:
                pgs.parse_ops(text)
            assert e.value.code == pgs.INVALID_ARGUMENT
