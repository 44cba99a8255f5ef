"""The edge inputs of the merge tests, shared by the kernel simulator (test_kernel_sim.py, test_walk_window_sim.py,
test_emit_geometry_sim.py) and the device (test_merge_geometry_gpu.py).  Every function takes a seed and returns the input
runs as Records, in the order the tests hand them to the merge; the simulator tests call them with the seeds they always
used, so they check what they checked before."""
import numpy as np

from incubator_pegasus_b200 import Records
from scan_model import make_db


def _records(items):
    return Records.from_list(sorted(items, key=lambda r: (r[0], -r[1])))


def _value(rng, vl):
    """a value of vl >= 4 bytes: the 4-byte expire_ts header (0, no TTL), then random bytes"""
    return bytes(4) + bytes(rng.integers(0, 256, vl - 4, dtype=np.uint8))


def ragged_records(seed):
    """keys of 0..300 bytes, values of 0..9000 bytes (blocks of one entry, entries larger than the block buffer), several
    versions of a key inside one run, tombstones; three runs, the oldest first"""
    rng = np.random.default_rng(seed)
    def mk(seq0, n):
        items = {}
        for i in range(n):
            kl = int(rng.integers(0, 12)) if rng.random() < 0.8 else int(rng.integers(12, 300))
            key = bytes(rng.integers(0, 3, kl, dtype=np.uint8) + (0 if rng.random() < 0.5 else 0xfe)) if kl else b""
            for _ in range(int(rng.integers(1, 4))):
                seq0 += 1
                t = 0 if rng.random() < 0.15 else 1
                vl = 0 if t == 0 else (int(rng.integers(4, 40)) if rng.random() < 0.9 else int(rng.integers(3000, 9000)))  # a value always carries its 4-byte header
                val = bytes(rng.integers(0, 256, vl, dtype=np.uint8))
                if t == 1 and vl >= 4 and rng.random() < 0.5:
                    val = (0).to_bytes(4, "big") + val[4:]
                items[(key, -seq0)] = (key, seq0, t, val)
        return seq0, Records.from_list([items[k] for k in sorted(items)])
    seq = 0
    runs = []
    for n in (150, 120, 90):
        seq, r = mk(seq, n)
        runs.append(r)
    return runs[::-1]  # newest first is not required: the merge orders by (key, seq)


def long_restart_arrays(seed):
    """tiny entries (at restart interval 1 a 4 KB block holds ~270 of them and spans many emit batches), and values just
    below / above the 4 KB block buffer right after such a block"""
    rng = np.random.default_rng(seed)
    def mk(seq0, n, big_every):
        recs = []
        for i in range(n):
            key = b"k%05d" % (i * 3 + seq0 % 3)
            seq0 += 1
            if big_every and i % big_every == big_every - 1:
                vl = int(rng.choice([4050, 4090, 4100, 4130, 4200, 8000]))
            else:
                vl = 4
            recs.append((key, seq0, 1, bytes(rng.integers(0, 256, vl, dtype=np.uint8))))
        return seq0, Records.from_list(sorted(recs, key=lambda r: (r[0], -r[1])))
    seq, a = mk(0, 2000, 0)
    seq, b = mk(seq, 1500, 301)
    return [b, a]


def long_keys(seed):
    """2 KB user keys: a narrow merge group's key rows no longer fit shared memory"""
    rng = np.random.default_rng(seed)
    runs, seq = [], 1
    for i in range(3):
        items = {}
        for j in range(120):
            hk = b"h%03d" % rng.integers(0, 20)
            sk = bytes(rng.integers(97, 100, int(rng.integers(1500, 2000))).astype(np.uint8))
            key = len(hk).to_bytes(2, "big") + hk + sk
            items[key] = (key, seq, 1, (0).to_bytes(4, "big") + bytes(8) + b"v%d" % j)
            seq += 1
        runs.append(Records.from_list([items[k] for k in sorted(items)]))
    return runs


def empty_hash_keys(seed):
    """hash keys "", "h1", "a01b", "h22" with sort keys s0000..s0059: an empty hash key, and "01" inside sort keys"""
    import incubator_pegasus_b200 as pgs
    runs, _ = make_db(pgs, np.random.default_rng(seed), 3, [b"", b"h1", b"a01b", b"h22"], 60)
    return runs


def window_key_lengths(seed):
    """user keys of 40..100 bytes around the walker's head window (a restart point's head fits up to ~60 bytes of key),
    sharing long prefixes so that non-restart entries carry short deltas; values of 4..7 bytes and tombstones"""
    rng = np.random.default_rng(seed)
    runs, seq = [], 0
    for r in range(3):
        items = []
        for i in range(160):
            kl = 40 + (i * 7 + r * 3) % 61
            key = (b"P" * (kl - 6) + b"%06d" % (i * 3 + r))[:kl]
            seq += 1
            t = 0 if i % 11 == 5 else 1
            items.append((key, seq, t, _value(rng, int(rng.integers(4, 8))) if t else b""))
        runs.append(_records(items))
    return runs


def window_block_crossings(seed):
    """values just under and over 256 / 384-byte blocks cut blocks of one entry, runs of short ones fill blocks of a few"""
    rng = np.random.default_rng(seed)
    runs, seq = [], 0
    for r in range(3):
        items = []
        pattern = [300, 5, 300, 5, 5, 300, 5, 5, 5, 300, 40, 40, 40, 40, 600, 4, 0]
        for i in range(200):
            key = b"blk%05d" % (i * 3 + r)
            seq += 1
            vl = pattern[(i + r) % len(pattern)]
            items.append((key, seq, 1, _value(rng, vl)) if vl else (key, seq, 0, b""))
        runs.append(_records(items))
    return runs


def window_end_of_buffer(seed):
    """runs that end in tiny entries (4-byte values, a tombstone of a one- or two-byte key)"""
    rng = np.random.default_rng(seed)
    runs, seq = [], 0
    for r in range(2):
        items = []
        for i in range(120):
            key = b"e%04d" % (i * 2 + r)
            seq += 1
            items.append((key, seq, 1, _value(rng, int(rng.integers(4, 30)) if i < 110 else 4)))
        items.append((b"\xff" * (1 + r), seq + 1, 0, b""))
        seq += 1
        runs.append(_records(items))
    return runs


def huge_blocks(seed):
    """tiny entries (a block cut to ~74 KB spans many emit batches) and values of 30..90 KB on both sides of the cut block
    buffer"""
    rng = np.random.default_rng(seed)
    def mk(seq0, n, big_every):
        recs = []
        for i in range(n):
            key = b"h%06d" % (i * 2 + seq0 % 2)
            seq0 += 1
            vl = int(rng.integers(30_000, 90_000)) if big_every and i % big_every == big_every - 1 else int(rng.integers(4, 24))
            recs.append((key, seq0, 1, (0).to_bytes(4, "big") + bytes(rng.integers(0, 256, vl - 4, dtype=np.uint8))))
        return seq0, Records.from_list(sorted(recs, key=lambda r: (r[0], -r[1])))
    seq, a = mk(0, 6000, 0)
    seq, b = mk(seq, 3000, 250)
    return [b, a]


def _varint_len(v):
    n = 1
    while v >= 128:
        v >>= 7
        n += 1
    return n


def restart_entry_bytes(ulen, vlen):
    """the bytes of an entry that shares nothing with the one before (a restart point): shared = 0 | non-shared length |
    value length varints, the user key, the 8-byte trailer, the value"""
    return 1 + _varint_len(ulen + 8) + _varint_len(vlen) + ulen + 8 + vlen


def df_big_threshold(seed, blk_buf):
    """k_walk sends an entry to k_emit's in-place path (DF_BIG) when its bytes e + 8 exceed k_emit's block buffer blk_buf.
    Entries of 7-byte keys whose restart-point size e is exactly blk_buf - 9, blk_buf - 8 (the largest that still goes
    through a batch) and blk_buf - 7 (the smallest in-place one), between runs of 1..40 tiny entries, so that the batch
    path, the value stage (a value's 16-byte span is up to vlen + 30 bytes) and the in-place path meet at the boundary at
    every position of a batch.  Two runs, the newer first; the older one interleaves tiny entries and holds older versions
    of some threshold keys (shadowed)."""
    rng = np.random.default_rng(seed)
    def vlen_for(e):
        for vv in range(1, 5):
            vl = e - restart_entry_bytes(7, 0) + 1 - vv
            if vl >= 4 and _varint_len(vl) == vv:
                assert restart_entry_bytes(7, vl) == e
                return vl
        raise ValueError(e)
    sizes = [vlen_for(blk_buf - d) for d in (9, 8, 7)]
    new, old, seq, i = [], [], 0, 0
    for rep in range(4):
        for vl in sizes + sizes[::-1]:
            for _ in range(int(rng.integers(1, 41)) if rep % 2 else 1 + (i % 3)):  # runs of tiny entries, or of one to three
                seq += 1
                new.append((b"t%06d" % (2 * i), seq, 1, _value(rng, int(rng.integers(4, 12)))))
                old.append((b"t%06d" % (2 * i + 1), seq, 1, _value(rng, int(rng.integers(4, 12)))))
                i += 1
            key = b"t%06d" % (2 * i)
            old.append((key, seq + 1, 1, _value(rng, int(rng.integers(4, 40)))))  # shadowed by the newer threshold entry
            seq += 2
            new.append((key, seq, 1, _value(rng, vl)))
            i += 1
    return [_records(new), _records(old)]


def carried_restart_arrays(seed):
    """one run of tiny entries of ragged sizes: a block of 1 KB spans two or three emit batches, and in the batch that
    closes it the next block records restart points of its own (at other offsets) while the closed block's earlier ones
    are still to be written"""
    rng = np.random.default_rng(seed)
    return [_records([(b"c%05d" % i, i + 1, 1, _value(rng, int(rng.integers(4, 10)))) for i in range(400)])]
