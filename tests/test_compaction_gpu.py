"""GPU parity: pgs_compact (CUDA k-way merge + fused KeyWithTTLCompactionFilter) against the CPU
oracle on the same seeded inputs, through the C ABI.  Bit-exact on (user key, seq, type, value)."""
import numpy as np
import pytest

from incubator_pegasus_b200 import synth

pytestmark = pytest.mark.gpu

OPS_JSON = (
    '{"ops":[{"type":"COT_DELETE","params":"","rules":[{"type":"FRT_HASHKEY_PATTERN","params":'
    '"{\\"pattern\\":\\"\\\\u0001\\",\\"match_type\\":\\"SMT_MATCH_PREFIX\\"}"}]},'
    '{"type":"COT_UPDATE_TTL","params":"{\\"type\\":\\"UTOT_FROM_NOW\\",\\"value\\":10000}","rules":['
    '{"type":"FRT_SORTKEY_PATTERN","params":"{\\"pattern\\":\\"7\\",\\"match_type\\":\\"SMT_MATCH_POSTFIX\\"}"},'
    '{"type":"FRT_TTL_RANGE","params":"{\\"start_ttl\\":0,\\"stop_ttl\\":50000}"}]}]}'
)


def run_case(pgs, oracle, engine, runs, *, bottommost, now=synth.NOW, default_ttl=0, validate_hash=False, pidx=0,
             partition_version=-1, ops_json=None, enabled=True):
    part = engine.partition()
    try:
        ids = [part.upload_records(r) for r in runs]  # later upload = newer L0 run
        ops_bin = pgs.parse_ops(ops_json) if ops_json else None
        res = part.compact(ids, out_level=1, bottommost=1 if bottommost else 0, now=now, enabled=enabled,
                           default_ttl=default_ttl, validate_hash=validate_hash, pidx=pidx,
                           partition_version=partition_version, ops=ops_bin)
        oruns = [oracle.Run.from_records(r) for r in runs]
        oops = oracle.Ops(ops_json) if ops_json else None
        fp = oracle.filter_params(enabled=enabled, default_ttl=default_ttl, validate_hash=validate_hash, pidx=pidx,
                                  partition_version=partition_version, ops=oops)
        want_run, st = oracle.compact(oruns, bottommost, fp, now)
        want = want_run.records()
        if want.n == 0:
            assert res.new_run_id == 0
            got = None
        else:
            raw = part.download(res.new_run_id)
            got = pgs.decode_blocks(raw)                      # product's host decoder
            got2 = oracle.Run.from_blocks(raw).records()      # independent decoder of the raw blocks
            assert got.same_as(got2)
            assert got.n == want.n, (got.n, want.n)
            assert got.same_as(want)
            info = part.run_info(res.new_run_id)
            assert info.n_records == want.n
            assert info.raw_key_bytes == want.keys.shape[0]
            assert info.raw_value_bytes == want.vals.shape[0]
            assert part.runs() == [res.new_run_id]
        for f in ("in_records", "out_records", "in_bytes", "out_bytes", "dropped_shadowed", "dropped_tombstone",
                  "dropped_expired", "dropped_user", "dropped_stale", "ttl_rewritten"):
            assert getattr(res, f) == getattr(st, f), f
        return res, got
    finally:
        part.close()


@pytest.mark.parametrize("bottommost", [True, False])
def test_l0_to_l1_small(pgs, oracle, engine, bottommost):
    runs = synth.compaction_runs(k=4, n_per_run=2_000)
    run_case(pgs, oracle, engine, runs, bottommost=bottommost)


def test_l0_to_l1_medium(pgs, oracle, engine):
    runs = synth.compaction_runs(k=4, n_per_run=25_000)
    res, _ = run_case(pgs, oracle, engine, runs, bottommost=True)
    assert res.n_tiles > 1


def test_default_ttl_rewrite(pgs, oracle, engine):
    runs = synth.compaction_runs(k=3, n_per_run=5_000, seed=7)
    res, _ = run_case(pgs, oracle, engine, runs, bottommost=True, default_ttl=3600)
    assert res.ttl_rewritten > 0


def test_validate_partition_hash(pgs, oracle, engine):
    runs = synth.compaction_runs(k=2, n_per_run=4_000, seed=11)
    res, _ = run_case(pgs, oracle, engine, runs, bottommost=True, validate_hash=True, pidx=1, partition_version=3)
    assert res.dropped_stale > 0


def test_user_specified_ops(pgs, oracle, engine):
    runs = synth.compaction_runs(k=3, n_per_run=6_000, seed=13)
    res, _ = run_case(pgs, oracle, engine, runs, bottommost=False, ops_json=OPS_JSON)
    assert res.ttl_rewritten > 0


def test_filter_disabled(pgs, oracle, engine):
    runs = synth.compaction_runs(k=2, n_per_run=3_000, seed=17)
    res, _ = run_case(pgs, oracle, engine, runs, bottommost=True, enabled=False)
    assert res.dropped_expired == 0


def test_ragged_small_values_and_long_keys(pgs, oracle, engine):
    # many small records per block, several restart intervals per block, ragged key lengths
    rng = np.random.default_rng(5)
    runs = []
    seq = 1
    for i in range(3):
        items = {}
        for _ in range(4000):
            hk = bytes(rng.integers(97, 100, rng.integers(0, 5)).astype(np.uint8))
            sk = bytes(rng.integers(97, 123, rng.integers(0, 40)).astype(np.uint8))
            key = len(hk).to_bytes(2, "big") + hk + sk
            typ = 0 if rng.random() < 0.05 else 1
            val = b"" if typ == 0 else (int(rng.choice([0, synth.NOW + 50, synth.NOW - 50])).to_bytes(4, "big")
                                        + bytes(8) + bytes(rng.integers(0, 256, rng.integers(0, 30)).astype(np.uint8)))
            items[key] = (key, seq, typ, val)
            seq += 1
        runs.append(pgs.Records.from_list(sorted(items.values(), key=lambda t: t[0])))
    run_case(pgs, oracle, engine, runs, bottommost=True)
    run_case(pgs, oracle, engine, runs, bottommost=False, default_ttl=100)


def test_single_run_and_empty_output(pgs, oracle, engine):
    runs = synth.compaction_runs(k=1, n_per_run=1_000, seed=3)
    run_case(pgs, oracle, engine, runs, bottommost=True)
    # everything expired -> empty output
    items = [((2).to_bytes(2, "big") + b"hk" + b"%04d" % i, i + 1, 1, (5).to_bytes(4, "big") + bytes(8) + b"v")
             for i in range(100)]
    run_case(pgs, oracle, engine, [pgs.Records.from_list(items)], bottommost=True, now=1000)


def test_compact_gpu_built_runs_again(pgs, oracle, engine):
    """L0->L1 then (L0 + L1)->L1: the second merge reads blocks the GPU itself wrote."""
    runs = synth.compaction_runs(k=4, n_per_run=8_000, seed=23)
    part = engine.partition()
    try:
        ids = [part.upload_records(r) for r in runs[:2]]
        r1 = part.compact(ids, out_level=1, bottommost=0, now=synth.NOW)
        ids2 = [part.upload_records(r) for r in runs[2:]]
        r2 = part.compact(ids2 + [r1.new_run_id], out_level=1, bottommost=1, now=synth.NOW)
        got = pgs.decode_blocks(part.download(r2.new_run_id))
        o = [oracle.Run.from_records(r) for r in runs]
        fp = oracle.filter_params()
        mid, _ = oracle.compact(o[:2], False, fp, synth.NOW)
        want, _ = oracle.compact(o[2:] + [mid], True, fp, synth.NOW)
        assert got.same_as(want.records())
    finally:
        part.close()


def test_large_partition_properties(pgs, oracle, engine):
    """4 x 1 M records (1.27 GB merged, same shape as BASELINE configs[1]): full comparison with the oracle's
    threaded block-level compaction, plus size-independent properties: sorted, one version per key, idempotent."""
    runs = synth.compaction_runs(k=4, n_per_run=1_000_000, seed=77)
    part = engine.partition()
    try:
        ids = [part.upload_records(r) for r in runs]
        res = part.compact(ids, out_level=1, bottommost=1, now=synth.NOW)
        raw = part.download(res.new_run_id)
        got = pgs.decode_blocks(raw)
        bruns = [oracle.BlockRunCPU.from_run(oracle.Run.from_records(r)) for r in runs]
        want_b, st, _ = oracle.compact_blocks(bruns, True, oracle.filter_params(), synth.NOW, threads=8)
        want = want_b.decode().records()
        assert got.n == want.n == res.out_records
        assert got.same_as(want)
        assert (res.in_records, res.dropped_expired, res.dropped_shadowed, res.dropped_tombstone) == \
               (st.in_records, st.dropped_expired, st.dropped_shadowed, st.dropped_tombstone)
        keys = got.keys.reshape(got.n, 50)
        k64 = np.concatenate([keys, np.zeros((got.n, 6), np.uint8)], axis=1).reshape(got.n, 7, 8).view(">u8").reshape(got.n, 7)
        order_ok = np.ones(got.n - 1, bool)
        undecided = np.ones(got.n - 1, bool)
        for c in range(7):  # strictly increasing user keys
            lt, gt = k64[:-1, c] < k64[1:, c], k64[:-1, c] > k64[1:, c]
            order_ok &= ~(undecided & gt)
            undecided &= ~(lt | gt)
        assert order_ok.all() and not undecided.any()
        assert (got.seq == 0).all() and (got.type == 1).all()  # bottommost: seqnos zeroed, no tombstones
        # idempotence: compacting the result again (same `now`) changes nothing
        res2 = part.compact([res.new_run_id], out_level=1, bottommost=1, now=synth.NOW)
        assert res2.out_records == res.out_records and res2.dropped_expired == 0
        assert pgs.decode_blocks(part.download(res2.new_run_id)).same_as(got)
        # blocks stay within the format the engine itself reads back
        info = part.run_info(res2.new_run_id)
        assert info.max_block_size < 2 * 4096 + 512 and info.n_records == got.n
    finally:
        part.close()


def test_bench_size_digest(pgs, oracle, engine):
    """BASELINE configs[1] at full size, the data set bench.py times (4 x 2.5 M records, seed 1000): the decoded output and
    every statistic equal the oracle's; compared through a digest of the flat arrays and the arrays themselves."""
    import hashlib
    runs = synth.compaction_runs(k=4, n_per_run=2_500_000, hk_len=16, sk_len=32, user_len=256, now=300_000_000, seed=1000)
    part = engine.partition()
    try:
        ids = part.upload_many([pgs.build_run(r) for r in runs])
        res = part.compact(ids, out_level=1, bottommost=1, now=300_000_000, enabled=True)
        got = pgs.decode_blocks(part.download(res.new_run_id))
        bruns = [oracle.BlockRunCPU.from_run(oracle.Run.from_records(r)) for r in runs]
        want_b, st, _ = oracle.compact_blocks(bruns, True, oracle.filter_params(enabled=True), 300_000_000, threads=16)
        want = want_b.decode().records()
        for f in ("in_records", "out_records", "in_bytes", "out_bytes", "dropped_shadowed", "dropped_tombstone", "dropped_expired",
                  "dropped_user", "dropped_stale", "ttl_rewritten"):
            assert getattr(res, f) == getattr(st, f), f

        def digest(r):
            h = hashlib.blake2b(digest_size=16)
            for a in (r.key_off, r.keys, r.val_off, r.vals, r.seq, r.type):
                h.update(np.ascontiguousarray(a).view(np.uint8).data)
            return h.hexdigest()
        assert got.n == want.n == res.out_records == 8_240_347  # the survivor count of this seed (bench.py's compaction step)
        assert digest(got) == digest(want)
    finally:
        part.close()


def test_value_schema_v0(pgs, oracle, engine):
    """data_version 0 (src/base/pegasus_value_schema.h:133-170: BE32 expire_ts | data, no timetag): the filter's expiry check and
    default-TTL rewrite and the 4-byte header strip of point reads on the device, against the oracle"""
    rng = np.random.default_rng(31)
    runs, seq = [], 1
    for i in range(3):
        items = {}
        for j in range(3000):
            key = (3).to_bytes(2, "big") + b"h%02d" % rng.integers(0, 60) + b"s%03d" % rng.integers(0, 400)
            ets = int(rng.choice([0, 0, synth.NOW + 500, synth.NOW - 7]))
            items[key] = (key, seq, 1, ets.to_bytes(4, "big") + bytes(rng.integers(0, 256, int(rng.integers(0, 90)), dtype=np.uint8)))
            seq += 1
        runs.append(pgs.Records.from_list([items[k] for k in sorted(items)]))
    part = engine.partition(data_version=0)
    try:
        ids = [part.upload_records(r) for r in runs]
        res = part.compact(ids, out_level=1, bottommost=1, now=synth.NOW, default_ttl=900, data_version=0)
        want_run, st = oracle.compact([oracle.Run.from_records(r) for r in runs], True, oracle.filter_params(default_ttl=900, data_version=0), synth.NOW)
        want = want_run.records()
        got = pgs.decode_blocks(part.download(res.new_run_id))
        assert got.same_as(want) and res.ttl_rewritten == st.ttl_rewritten > 0 and res.dropped_expired == st.dropped_expired > 0
        pick = np.arange(0, want.n, 37)
        keys = b"".join(want.key(int(i)) for i in pick)
        off = np.zeros(len(pick) + 1, np.uint32)
        off[1:] = np.cumsum([len(want.key(int(i))) for i in pick])
        st_, results, arena, _ = part.get_batch(np.frombuffer(keys, np.uint8), off, synth.NOW)
        assert st_ == 0
        for j, i in enumerate(pick):
            v = want.value(int(i))
            assert results[j].status == pgs.OK and results[j].expire_ts == int.from_bytes(v[:4], "big")
            o, l = results[j].value_off, results[j].value_len
            assert arena[o:o + l].tobytes() == v[4:]   # v0: the user data starts right after the expire_ts
    finally:
        part.close()
