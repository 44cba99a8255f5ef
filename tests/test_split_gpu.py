"""GPU: pgs_partition_split against tests/split_model.py.  A parent of several levels (three L0 runs, L1 and L2, with
versions, tombstones and expired values) is split into 2, 4 and 8 children: every child run equals the model's share of the
parent run at the same level, the parent is unchanged, every key's get answers alike on the parent and on its child, and a
child run that is downloaded and uploaded again is accepted with the same info.  The refusals leave parent and children as
they were."""
import numpy as np
import pytest

import split_model as sm
from incubator_pegasus_b200 import synth

pytestmark = pytest.mark.gpu

NOW = synth.NOW


def _parent(pgs, engine, pidx, src_count, n_per_run=6000, seed=7):
    """runs 0..4 of synth (run 0 oldest): 0 -> L2, 1 -> L1, 2..4 -> L0 (4 newest)"""
    runs = synth.compaction_runs(k=5, n_per_run=n_per_run, seed=seed)
    part = engine.partition(app_id=3, pidx=pidx)
    for i, lvl in enumerate((2, 1, 0, 0, 0)):
        part.upload_records(runs[i], lvl)
    return part


def _children(engine, pidx, src_count, dst_count, app_id=3):
    return [engine.partition(app_id=app_id, pidx=pidx + i * src_count) for i in range(dst_count // src_count)]


def _snapshot(part):
    return [(rid, part.run_info(rid).level, part.download(rid)) for rid in part.runs()]


def _gets(pgs, part, keys):
    ko = np.zeros(len(keys) + 1, np.uint32)
    ko[1:] = np.cumsum([len(k) for k in keys])
    st, res, arena, _used = part.get_batch(np.frombuffer(b"".join(keys), np.uint8).copy(), ko, NOW, arena_cap=len(keys) * 400 + (1 << 16))
    assert st == pgs.OK
    return [(r.status, r.expire_ts, arena[r.value_off:r.value_off + r.value_len].tobytes() if r.status == 0 else b"") for r in res[:len(keys)]]


@pytest.mark.parametrize("src,dst", [(1, 2), (2, 8), (1, 8)])
def test_split_a_partition_of_several_levels(pgs, engine, src, dst):
    pidx = src - 1
    parent = _parent(pgs, engine, pidx, src)
    kids = _children(engine, pidx, src, dst, app_id=8)  # the offline split writes the children into another table
    before = _snapshot(parent)
    try:
        res = parent.split(src, dst, kids)
        after = _snapshot(parent)
        assert [(a, b) for a, b, _ in after] == [(a, b) for a, b, _ in before]
        for (_, _, x), (_, _, y) in zip(before, after):
            assert np.array_equal(x.data, y.data) and np.array_equal(x.blk_off, y.blk_off)
        S = dst // src
        want = [[] for _ in range(S)]  # per child: (level, items) of each parent run, in the parent's order
        n_in = 0
        for _rid, lvl, br in before:
            items = pgs.decode_blocks(br).to_list()
            n_in += len(items)
            parts, dropped = sm.split_items(items, src, dst)
            assert dropped == 0
            for c in range(S):
                if parts[c]:
                    want[c].append((lvl, parts[c]))
        assert res.in_records == n_in and res.dropped_empty == 0 and res.kernel_ms > 0
        all_keys = sorted({k for _rid, _l, br in before for k, *_ in pgs.decode_blocks(br).to_list()})
        parent_answers = dict(zip(all_keys, _gets(pgs, parent, all_keys)))
        for c, kid in enumerate(kids):
            ids = kid.runs()
            assert [kid.run_info(r).level for r in ids] == [lvl for lvl, _ in want[c]]
            assert res.child[c].runs == len(ids) and res.child[c].records == sum(len(it) for _, it in want[c])
            for rid, (_lvl, items) in zip(ids, want[c]):
                raw = kid.download(rid)
                assert pgs.decode_blocks(raw).to_list() == items
                info = kid.run_info(rid)
                assert info.n_records == len(items) and info.n_tombstones == sum(1 for it in items if it[2] == 0)
                again = engine.partition(app_id=9)
                try:  # a child run is an ordinary run: it uploads again with the same info
                    info2 = again.run_info(again.upload(raw, info.level))
                    for f in ("n_blocks", "n_records", "n_tombstones", "data_bytes", "raw_key_bytes", "raw_value_bytes", "max_ukey_len",
                              "max_block_size", "smallest_seq", "largest_seq"):
                        assert getattr(info2, f) == getattr(info, f), f
                finally:
                    again.close()
            mine = [k for k in all_keys if sm.child_of(k, src, dst) == c]
            assert _gets(pgs, kid, mine) == [parent_answers[k] for k in mine]
            # prefix scans of the child's hash keys answer as the parent's
            hks = sorted({k[2:2 + int.from_bytes(k[:2], "big")] for k in mine})
            pb, kb = parent.prefix_scan_batch(hks, max_records=200), kid.prefix_scan_batch(hks, max_records=200)
            assert pb.run(NOW) == pgs.OK and kb.run(NOW) == pgs.OK
            for i in range(len(hks)):
                assert kb.records(i) == pb.records(i)
                assert (kb.results[i].count, kb.results[i].status) == (pb.results[i].count, pb.results[i].status)
    finally:
        for k in kids:
            k.close()
        parent.close()


def test_split_scale_digest(pgs, engine):
    """config #2 at scale, four runs of 2.5 M records, into 2 and into 8: every child run holds the model's records of its
    parent run, in order, with their keys, sequence numbers and types"""
    runs = synth.compaction_runs(k=4, n_per_run=2_500_000)
    parent = engine.partition(app_id=4, pidx=0)
    try:
        for r in runs:
            parent.upload_records(r, 0)
        order = runs[::-1]  # read order: the newest L0 run first
        routes = []  # per run: the child of every record at dst = 8 (dst = 2 is its value mod 2)
        for r in order:
            keys = r.keys.reshape(r.n, -1)  # fixed 50-byte keys: 2 + 16-byte hash key + 32-byte sort key
            hk, inv = np.unique(np.ascontiguousarray(keys[:, :18]).view(np.dtype((np.void, 18))).ravel(), return_inverse=True)
            h = np.array([sm.key_hash(bytes(x)) % 8 for x in hk], np.int64)
            routes.append(h[inv.ravel()])
        for dst in (2, 8):
            kids = _children(engine, 0, 1, dst, app_id=4)
            try:
                res = parent.split(1, dst, kids)
                assert res.in_records == 4 * 2_500_000 and sum(res.child[c].records for c in range(dst)) == res.in_records
                for c, kid in enumerate(kids):
                    ids = kid.runs()
                    assert len(ids) == len(order)
                    for rid, r, route in zip(ids, order, routes):
                        got = pgs.decode_blocks(kid.download(rid))
                        sel = np.nonzero(route % dst == c)[0]
                        assert got.n == sel.shape[0]
                        assert np.array_equal(got.seq, r.seq[sel]) and np.array_equal(got.type, r.type[sel])
                        assert np.array_equal(got.keys.reshape(got.n, -1), r.keys.reshape(r.n, -1)[sel])
                        del got
            finally:
                for k in kids:
                    k.close()
    finally:
        parent.close()


def test_split_refusals(pgs, engine):
    parent = _parent(pgs, engine, 1, 2, n_per_run=500)
    before = _snapshot(parent)
    other = pgs.Engine()
    try:
        def refused(code, src, dst, kids):
            held = [k.runs() if k is not None else None for k in kids]
            with pytest.raises(pgs.PegasusError) as e:
                parent.split(src, dst, kids)
            assert e.value.code == code
            assert [k.runs() if k is not None else None for k in kids] == held
            assert [(a, b) for a, b, _ in _snapshot(parent)] == [(a, b) for a, b, _ in before]
        good = _children(engine, 1, 2, 4)
        assert len(good) == 2  # partitions 1 and 3: the right count for 2 -> 4 and for 1 -> 2
        refused(pgs.INVALID_ARGUMENT, 2, 6, good + [None])        # not src_count * 2^n
        refused(pgs.INVALID_ARGUMENT, 2, 2, good[:1])             # n = 0
        refused(pgs.INVALID_ARGUMENT, 2, 8, good)                 # n_dst != S
        refused(pgs.INVALID_ARGUMENT, 1, 2, good)                 # pidx >= src_count
        wrong = engine.partition(app_id=3, pidx=2)
        refused(pgs.INVALID_ARGUMENT, 2, 4, [good[0], wrong])     # child with the wrong pidx
        full = engine.partition(app_id=3, pidx=3)
        full.upload_records(synth.compaction_runs(k=1, n_per_run=50)[0])
        refused(pgs.INVALID_ARGUMENT, 2, 4, [good[0], full])      # a child that holds runs
        far = other.partition(app_id=3, pidx=3)
        refused(pgs.INVALID_ARGUMENT, 2, 4, [good[0], far])       # a child on another engine
        v2 = engine.partition(app_id=3, pidx=3, data_version=0)
        refused(pgs.NOT_SUPPORTED, 2, 4, [good[0], v2])           # another data_version
        many = [engine.partition(app_id=3, pidx=1 + 2 * i) for i in range(64)]
        refused(pgs.NOT_SUPPORTED, 2, 128, many)                  # beyond PGS_SPLIT_MAX_CHILDREN
        for p in [wrong, full, far, v2] + many + good:
            p.close()
    finally:
        other.close()
        parent.close()
