"""Data blocks the library's own builder never writes, and a reference model of what the upload does with them.

pgs_run_builder and k_emit write one canonical encoding of RocksDB's data-block format: exact shared prefixes, minimal
varints, a restart point every N entries, blocks back to back.  Runs that arrive through pgs_run_upload, pgs_sst_ingest or
a checkpoint may use any legal encoding, and four device decoders read them (k_index_walk at upload, cur_decode in k_get /
k_scan_fwd, cur_decode with the head window in k_walk, the staging decoder of k_scan).  This module is plain Python and
calls nothing of the library:

  encode_run()   writes Records as blocks with legal, non-canonical choices, every policy selectable and seeded
  classify()     the status pgs_run_upload answers: the handle rule on the host, then k_index_walk's rule per block
  decode()       the records of a run the model accepts
  model_index()  what the upload leaves behind: blk_rec, ikey_off, ikeys, rec_off, the pgs_run_info fields
  mutants()      named and seeded damaged copies of a run, each with the verdict it must get

The restart array's offsets are written correctly but no device decoder reads them (every block is walked from its first
entry, or through rec_off); only the restart COUNT bounds the entries."""
from dataclasses import dataclass

import numpy as np

from incubator_pegasus_b200 import BlockRun, Records

OK, CORRUPTION, NOT_SUPPORTED, INVALID_ARGUMENT = 0, 2, 3, 4
M32 = 0xFFFFFFFF
MAX_UKEY = 4096   # kMaxUkeyLen (format.h)
IDX_WARPS = 8     # kIdxWarps (index_kernel.cuh): blocks per CTA of k_index_walk
FILL = 0xEE       # what lies between and behind the blocks


# ---- varints ------------------------------------------------------------------------------------------------------------
def put_varint(v, extra=0):
    """RocksDB's varint32; extra = redundant continuation bytes (0x85 0x80 0x00 for 5), never more than five bytes in all"""
    out = bytearray()
    while v >= 128:
        out.append((v & 127) | 128)
        v >>= 7
    out.append(v)
    extra = min(extra, 5 - len(out))
    if extra > 0:
        out[-1] |= 128
        out += bytes([128] * (extra - 1)) + b"\0"
    return bytes(out)


def get_varint32(buf, p, avail):
    """device_util.cuh get_varint32: at most five bytes and at most `avail`; the value is cut to 32 bits.  -> (value,
    bytes consumed), consumed = 0 for a malformed or cut varint"""
    r = 0
    for i in range(5):
        if i >= avail:
            return 0, 0
        b = buf[p + i]
        r |= (b & 127) << (7 * i)
        if b < 128:
            return r & M32, i + 1
    return 0, 0


def ikey(k, seq, typ):
    return k + ((seq << 8) | typ).to_bytes(8, "little")


def _lcp(a, b):
    n = min(len(a), len(b))
    for i in range(n):
        if a[i] != b[i]:
            return i
    return n


# ---- the writer ---------------------------------------------------------------------------------------------------------
def _shared(policy, exact, rng):
    if policy == "exact":
        return exact
    if policy == "zero":
        return 0
    if policy == "random":
        return int(rng.integers(0, exact + 1))
    if policy == "exact_minus_one":
        return max(exact - 1, 0)
    kind, n = policy
    assert kind == "cap"
    return min(exact, n)


def _cut(block_cut, rng):
    """-> (bytes, entries): a block is closed once it holds that many bytes or entries"""
    if block_cut != "irregular":
        return int(block_cut), 1 << 30
    u = rng.random()
    if u < 0.3:
        return 1 << 30, 1                          # a block of one entry
    if u < 0.4:
        return 60_000, 1500                        # as many tiny entries as there are, up to 1500
    return int(rng.integers(64, 1500)), 1 << 30    # ragged sizes: every residue mod 16 turns up


def encode_block(items, *, rng, restart=16, shared="exact", varints="minimal"):
    """one block of (user key, seq, type, value) entries -> bytes"""
    buf, restarts, prev, to_restart = bytearray(), [], b"", 0
    for k, s, t, v in items:
        ik = ikey(k, s, t)
        if to_restart == 0:
            restarts.append(len(buf))
            sh = 0
            to_restart = (1 << 30) if restart == "single" else int(rng.integers(1, 41)) if restart == "irregular" else int(restart)
        else:
            sh = _shared(shared, _lcp(prev, ik), rng)
        to_restart -= 1
        pad = (lambda: int(rng.integers(0, 3))) if varints == "padded" else (lambda: 0)
        buf += put_varint(sh, pad()) + put_varint(len(ik) - sh, pad()) + put_varint(len(v), pad()) + ik[sh:] + v
        prev = ik
    return bytes(buf) + b"".join(r.to_bytes(4, "little") for r in restarts) + len(restarts).to_bytes(4, "little")


def assemble(blocks, *, rng=None, gaps=0, tail=0):
    """blocks (bytes) -> BlockRun: every block on a multiple of 16; gaps > 0: up to `gaps` x 16 further bytes in front of a
    block (seeded); tail: bytes behind the last block.  All filler is 0xEE."""
    data, off, size = bytearray(), [], []
    for i, b in enumerate(blocks):
        data += bytes([FILL]) * (-len(data) % 16)
        if gaps and i:
            data += bytes([FILL]) * (16 * int(rng.integers(0, gaps + 1)))
        off.append(len(data))
        size.append(len(b))
        data += b
    data += bytes([FILL]) * tail
    return BlockRun(np.frombuffer(bytes(data), np.uint8).copy() if data else np.zeros(0, np.uint8), np.array(off, np.uint64),
                    np.array(size, np.uint32))


def encode_run(records, *, seed=0, block_cut=4096, restart=16, shared="exact", varints="minimal", gaps=0, tail=0):
    """Records (internal-key order) -> BlockRun.
    block_cut  bytes at which a block is closed, "irregular" (blocks of one entry, of up to 1500 entries, ragged sizes), or a
               list of entry counts, one per block (the block boundaries of another run of the same records)
    restart    entries per restart point, "irregular" (1..40, seeded) or "single" (one restart point per block)
    shared     "exact" | "zero" | ("cap", n) | "random" (uniform in [0, exact]) | "exact_minus_one"
    varints    "minimal" | "padded" (0..2 redundant continuation bytes per field)
    gaps       0, or the largest gap between blocks in units of 16 bytes;  tail: bytes behind the last block"""
    rng = np.random.default_rng(seed)
    items = records.to_list()
    blocks, i = [], 0
    counts = iter(block_cut) if isinstance(block_cut, (list, tuple)) else None
    while i < len(items):
        max_bytes, max_entries = (1 << 30, next(counts)) if counts else _cut(block_cut, rng)
        j, est = i, 0
        while j < len(items) and (j == i or (est < max_bytes and j - i < max_entries)):
            est += 3 + 8 + len(items[j][0]) // 2 + len(items[j][3])  # about what the entry takes
            j += 1
        blocks.append(encode_block(items[i:j], rng=rng, restart=restart, shared=shared, varints=varints))
        i = j
    return assemble(blocks, rng=rng, gaps=gaps, tail=tail)


# ---- the validator (k_index_walk pass 1) and the decoder ----------------------------------------------------------------
@dataclass
class Entry:
    p: int        # offset of the entry inside its block
    fields: list  # (offset, length) of the three header varints
    sh: int
    ns: int
    vl: int
    key: bytes    # the internal key
    value: bytes


def walk_block(blk):
    """k_index_walk over one block -> (status, entries decoded before the walk stopped)"""
    size = len(blk)
    if size < 8:
        return CORRUPTION, []
    nr = int.from_bytes(blk[-4:], "little")
    if nr == 0 or nr * 4 + 4 > size:
        return CORRUPTION, []
    limit, p, prev, ents = size - 4 - 4 * nr, 0, b"", []
    while p < limit:
        h, vals, fields = 0, [], []
        for _ in range(3):
            v, c = get_varint32(blk, p + h, limit - p - h)
            if not c:
                return CORRUPTION, ents
            fields.append((p + h, c))
            vals.append(v)
            h += c
        sh, ns, vl = vals
        klen = (sh + ns) & M32   # the kernel adds in 32 bits; the entry's end is checked in 64
        if sh > len(prev) or klen < 8 or p + h + ns + vl > limit:
            return CORRUPTION, ents
        if klen > MAX_UKEY + 8:
            return NOT_SUPPORTED, ents
        key = prev[:sh] + blk[p + h:p + h + ns]
        ents.append(Entry(p, fields, sh, ns, vl, key, blk[p + h + ns:p + h + ns + vl]))
        prev = key
        p += h + ns + vl
    return (OK, ents) if ents else (CORRUPTION, ents)


def run_blocks(run):
    data = run.data.tobytes()
    return [data[o:o + s] for o, s in zip(run.blk_off.tolist(), run.blk_size.tolist())]


def handles_ok(run):
    """the handle rule of pgs_run_upload, checked on the host before anything else: 16-aligned, ordered, not overlapping,
    inside the data"""
    end, nbytes = 0, int(run.data.shape[0])
    for o, s in zip(run.blk_off.tolist(), run.blk_size.tolist()):
        if o % 16 or o < end or o + s > nbytes:
            return False
        end = o + s
    return True


def classify(run):
    """the status of pgs_run_upload(run): kInvalidArgument for a bad handle; else the largest block verdict (the kernel's
    atomicMax: kNotSupported = 3 wins over kCorruption = 2)"""
    if not handles_ok(run):
        return INVALID_ARGUMENT
    return max([walk_block(b)[0] for b in run_blocks(run)] + [OK])


def decode(run):
    """the records of an accepted run"""
    items = []
    for b in run_blocks(run):
        st, ents = walk_block(b)
        assert st == OK, st
        for e in ents:
            tr = int.from_bytes(e.key[-8:], "little")
            items.append((e.key[:-8], tr >> 8, tr & 0xFF, e.value))
    return Records.from_list(items)


def readable(recs):
    """user key ascending, sequence number descending, every type a deletion (0) or a value (1): what every reader assumes
    and no upload checks"""
    it = [(k, -s) for k, s, _t, _v in recs.to_list()]
    return all(a < b for a, b in zip(it, it[1:])) and set(recs.type.tolist()) <= {0, 1}


def model_index(run):
    """what the upload of an accepted run leaves on the device, and its pgs_run_info"""
    blk_rec, ikey_off, ikeys, rec_off = [0], [0], b"", []
    info = dict(n_blocks=run.n_blocks, n_records=0, n_tombstones=0, raw_key_bytes=0, raw_value_bytes=0, max_ukey_len=0, max_value_len=0,
                max_block_size=int(run.blk_size.max(initial=0)), max_block_records=0, smallest_seq=(1 << 64) - 1, largest_seq=0,
                data_bytes=(int(run.blk_off[-1]) + int(run.blk_size[-1]) + 15) & ~15)
    for b in run_blocks(run):
        st, ents = walk_block(b)
        assert st == OK, st
        rec_off += [e.p for e in ents]
        blk_rec.append(blk_rec[-1] + len(ents))
        ikeys += ents[-1].key[:-8]
        ikey_off.append(len(ikeys))
        info["max_block_records"] = max(info["max_block_records"], len(ents))
        for e in ents:
            tr = int.from_bytes(e.key[-8:], "little")
            info["n_records"] += 1
            info["n_tombstones"] += (tr & 0xFF) == 0
            info["raw_key_bytes"] += len(e.key) - 8
            info["raw_value_bytes"] += e.vl
            info["max_ukey_len"] = max(info["max_ukey_len"], len(e.key) - 8)
            info["max_value_len"] = max(info["max_value_len"], e.vl)
            info["smallest_seq"] = min(info["smallest_seq"], tr >> 8)
            info["largest_seq"] = max(info["largest_seq"], tr >> 8)
    return dict(blk_rec=blk_rec, ikey_off=ikey_off, ikeys=ikeys, rec_off=rec_off, info=info)


# ---- record sets ------------------------------------------------------------------------------------------------------
def _val(rng, n):
    return bytes(4) + bytes(rng.integers(0, 256, n - 4, dtype=np.uint8)) if n >= 4 else bytes(n)


def edge_records(seed, big_value=0):
    """the empty user key; user keys of exactly 4 096 bytes; keys that share 128..300 bytes (a two-byte `shared` that is
    legitimate); twelve versions of one key (they cross a block boundary at small blocks) and of a 200-byte key (shared
    lengths inside its trailer need two bytes); short keys in between; big_value: one value of that many bytes (2 MiB and
    more take a four-byte length varint)"""
    rng = np.random.default_rng(seed)
    items, seq = [], 0
    def add(k, n=1, vl=None, tomb=False):
        nonlocal seq
        for _ in range(n):
            seq += 1
            t = 0 if tomb or rng.random() < 0.1 else 1
            items.append((k, seq, t, _val(rng, int(rng.integers(4, 30)) if vl is None else vl) if t else b""))
    add(b"")
    add(b"\x00\x03abc", 12)
    for i in range(40):
        add(b"\x00\x02hk" + b"s%03d" % i, 1 + i % 3)
    for i in range(12):
        add(b"\x00\x04long" + b"Q" * (124 + 16 * i) + b"%02d" % i, 1 + i % 2)
    add(b"\x00\x01v" + b"V" * 197, 12)
    for c in (b"a", b"b"):
        add(b"\x00\x01L" + b"q" * 4092 + c)
    if big_value:
        add(b"\x00\x03big", vl=big_value)
    add(b"\xff\xff", tomb=True)
    return Records.from_list(sorted(items, key=lambda r: (r[0], -r[1])))


def tiny_records(seed, n=1300):
    """n entries of a few bytes each: one block can hold more than a thousand of them"""
    rng = np.random.default_rng(seed)
    return Records.from_list([(b"t%05d" % i, i + 1, 1, _val(rng, 4)) for i in range(n)])


# ---- the policy rows and record sets of the tests (simulator and device) -------------------------------------------------
# A pairwise cover of the writer's policies: every value of every policy meets every value of every other one at least
# once over these rows or the ones the single tests add.
GRID = {
    "zero-min-r16-512": dict(shared="zero", varints="minimal", restart=16, block_cut=512, gaps=0, tail=0),
    "random-pad-rirr-irr-gaps": dict(shared="random", varints="padded", restart="irregular", block_cut="irregular", gaps=3, tail=7),
    "cap3-pad-r1-256-gaps": dict(shared=("cap", 3), varints="padded", restart=1, block_cut=256, gaps=2, tail=0),
    "minus1-min-r128-4096-tail": dict(shared="exact_minus_one", varints="minimal", restart=128, block_cut=4096, gaps=0, tail=33),
    "exact-pad-single-1024-gaps": dict(shared="exact", varints="padded", restart="single", block_cut=1024, gaps=1, tail=0),
    "random-min-single-64-tail": dict(shared="random", varints="minimal", restart="single", block_cut=64, gaps=0, tail=1),
    "cap9-min-rirr-64k-gaps": dict(shared=("cap", 9), varints="minimal", restart="irregular", block_cut=65536, gaps=4, tail=0),
    "minus1-pad-r16-irr": dict(shared="exact_minus_one", varints="padded", restart=16, block_cut="irregular", gaps=0, tail=0),
    "zero-pad-r128-irr-gaps": dict(shared="zero", varints="padded", restart=128, block_cut="irregular", gaps=2, tail=16),
    "exact-min-r1-irr": dict(shared="exact", varints="minimal", restart=1, block_cut="irregular", gaps=0, tail=0),
}
POLICIES = list(GRID.values())


def record_sets():
    """name -> Records: the edge inputs of the merge tests (first run of each) and the edge set of foreign_blocks"""
    import merge_inputs
    return {"edge": edge_records(1), "ragged": merge_inputs.ragged_records(11)[0], "window_keys": merge_inputs.window_key_lengths(3)[0],
            "crossings": merge_inputs.window_block_crossings(4)[0], "empty_hash_keys": merge_inputs.empty_hash_keys(21)[0],
            "long_keys": merge_inputs.long_keys(3)[0]}


# ---- damaged copies -----------------------------------------------------------------------------------------------------
def _split(blk):
    """an intact block -> (raw bytes of each entry, entries, restart array bytes without the count)"""
    st, ents = walk_block(blk)
    assert st == OK
    nr = int.from_bytes(blk[-4:], "little")
    limit = len(blk) - 4 - 4 * nr
    ends = [e.p for e in ents[1:]] + [limit]
    return [blk[e.p:end] for e, end in zip(ents, ends)], ents, blk[limit:-4]


def _join(raw, restarts, nr=None, stray=b""):
    return b"".join(raw) + stray + restarts + (len(restarts) // 4 if nr is None else nr).to_bytes(4, "little")


def _entry(sh, ns, vl, payload):
    return put_varint(sh) + put_varint(ns) + put_varint(vl) + payload


def _block_mutants(blk):
    """(name, damaged block, verdict of the block) for a block of at least three entries whose keys have 24 bytes or more"""
    raw, ents, rst = _split(blk)
    assert len(ents) >= 3 and all(len(e.key) >= 24 for e in ents[:2])
    e0, e1, last = ents[0], ents[1], ents[-1]
    body = lambda e: e.key[e.sh:] + e.value
    yield "size_7", blk[:7], CORRUPTION
    yield "size_8_no_entries", bytes(4) + (1).to_bytes(4, "little"), CORRUPTION
    for nr in (0, len(blk) // 4, 0x40000000, M32):
        yield "restart_count_%#x" % nr, _join(raw, rst, nr=nr), CORRUPTION
    yield "varint_cut_by_the_bound", _join(raw, rst, stray=b"\x00\x90"), CORRUPTION
    yield "five_continuation_bytes", _join([b"\x80" * 5 + b"\x00" + raw[0][1:]] + raw[1:], rst), CORRUPTION
    yield "first_entry_shared_1", _join([_entry(1, e0.ns, e0.vl, body(e0))] + raw[1:], rst), CORRUPTION
    yield "shared_prev_klen_plus_1", _join([raw[0], _entry(len(e0.key) + 1, e1.ns, e1.vl, body(e1))] + raw[2:], rst), CORRUPTION
    yield "klen_7", _join(raw + [_entry(0, 7, 0, b"k" * 7)], rst), CORRUPTION
    yield "non_shared_wraps_klen", _join([raw[0], _entry(0x18, 0xFFFFFFF0, e1.vl, body(e1))] + raw[2:], rst), CORRUPTION
    yield "value_len_ffffffff", _join(raw[:-1] + [_entry(last.sh, last.ns, M32, body(last))], rst), CORRUPTION
    yield "entry_ends_inside_restart_array", _join(raw[:-1] + [_entry(last.sh, last.ns, last.vl + 1, body(last))], rst), CORRUPTION
    for n in (1, 2, 3):
        yield "stray_%d" % n, _join(raw, rst, stray=bytes(n)), CORRUPTION
    k96 = b"\x00\x01Z" + b"z" * 4093
    yield "ukey_4096", _join(raw + [_entry(0, 4096 + 8, 4, ikey(k96, 7, 1) + bytes(4))], rst), OK
    yield "ukey_4097", _join(raw + [_entry(0, 4096 + 8, 4, ikey(k96, 7, 1) + bytes(4)), _entry(4096 + 8, 1, 4, b"z" + bytes(4))], rst), NOT_SUPPORTED


def _with_block(run, b, blk):
    blocks = run_blocks(run)
    blocks[b] = blk
    return assemble(blocks)


def _with_handles(run, off=None, size=None):
    return BlockRun(run.data.copy(), run.blk_off.copy() if off is None else np.array(off, np.uint64),
                    run.blk_size.copy() if size is None else np.array(size, np.uint32))


N_RANDOM = 300


def mutant_base(seed):
    """the run the damaged copies are made of: 16-byte user keys and more, a few entries per block, 8 gaps; its block count
    leaves the last CTA of k_index_walk partly filled"""
    rng = np.random.default_rng(seed)
    items = [(b"\x00\x06mutant%08d" % (i - (i % 4 == 3)), 1000 - i, 1 if i % 7 else 0, _val(rng, 4 + i % 23) if i % 7 else b"") for i in range(150)]
    return encode_run(Records.from_list(items), seed=seed, block_cut=160, restart=3, gaps=2, tail=5)


def mutants(run, seed):
    """(name, BlockRun, status) of damaged copies of an accepted run of 2 * IDX_WARPS + 2 blocks or more, deterministic.
    The named ones carry the verdict their construction intends (test_foreign_blocks_sim.py checks that classify agrees);
    the random ones, single-byte changes confined to entry headers and to block tails (restart array and count), carry
    classify's."""
    nb = run.n_blocks
    assert classify(run) == OK and nb >= 2 * IDX_WARPS + 2 and nb % IDX_WARPS != 0
    blocks = run_blocks(run)
    mid = IDX_WARPS + 2
    named = {n: (b, st) for n, b, st in _block_mutants(blocks[mid])}
    for n, (b, st) in named.items():
        yield n, _with_block(run, mid, b), st
    # where the damage lies: block 0, the last block, warp 7 of the first CTA, the first block of the last, partly filled CTA
    for where, b in (("block_0", 0), ("last_block", nb - 1), ("warp_7", IDX_WARPS - 1), ("last_cta", nb - nb % IDX_WARPS)):
        dmg = [m for n, m, _ in _block_mutants(blocks[b]) if n == "entry_ends_inside_restart_array"][0]
        yield "damage_in_" + where, _with_block(run, b, dmg), CORRUPTION
    both = run_blocks(_with_block(run, 1, named["klen_7"][0]))
    both[nb - 2] = [m for n, m, _ in _block_mutants(blocks[nb - 2]) if n == "ukey_4097"][0]
    yield "not_supported_and_corruption", assemble(both), NOT_SUPPORTED
    off, size = run.blk_off.tolist(), run.blk_size.tolist()
    yield "handle_misaligned", _with_handles(run, off[:3] + [off[3] + 8] + off[4:]), INVALID_ARGUMENT
    yield "handle_overlaps", _with_handles(run, off[:3] + [off[2]] + off[4:]), INVALID_ARGUMENT
    yield "handle_out_of_order", _with_handles(run, off[:2] + [off[3], off[2]] + off[4:], size[:2] + [size[3], size[2]] + size[4:]), INVALID_ARGUMENT
    yield "handle_past_the_data", _with_handles(run, size=size[:-1] + [size[-1] + 17]), INVALID_ARGUMENT
    yield "handle_offset_wraps", _with_handles(run, off[:-1] + [(1 << 64) - 16]), INVALID_ARGUMENT
    bad = _with_block(run, 0, named["klen_7"][0])
    yield "bad_handle_and_corrupt_block", _with_handles(bad, size=bad.blk_size.tolist()[:-1] + [M32]), INVALID_ARGUMENT
    rng = np.random.default_rng(seed)
    for i in range(N_RANDOM):
        b = int(rng.integers(0, nb))
        _st, ents = walk_block(blocks[b])
        nr = int.from_bytes(blocks[b][-4:], "little")
        spots = [o + d for e in ents for o, n in e.fields for d in range(n)] + list(range(len(blocks[b]) - 4 - 4 * nr, len(blocks[b])))
        at = spots[int(rng.integers(0, len(spots)))]
        old = blocks[b][at]
        new = int(rng.choice([old ^ (1 << int(rng.integers(0, 8))), old | 0x80, 0, 0xFF, int(rng.integers(0, 256))]))
        if new == old:
            new = old ^ 1
        m = run.data.copy()
        m[int(run.blk_off[b]) + at] = new
        mr = BlockRun(m, run.blk_off.copy(), run.blk_size.copy())
        yield "byte_%03d_block_%d_at_%d_%02x_to_%02x" % (i, b, at, old, new), mr, classify(mr)
