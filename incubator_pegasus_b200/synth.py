"""Synthetic YCSB-shaped inputs (SURVEY.md §8d, BASELINE.md §2): fixed seed, fixed `now`.

Config #2 shape: 16 B hashkey / 32 B sortkey / 256 B user value -> 50 B raw key, 268 B raw value
(schema v1: BE32 expire_ts | BE64 timetag | user data), 64 sortkeys per hashkey with a zero padded
decimal counter as sort key, expire_ts 70 % none / 20 % future / 10 % already expired, 10 % of the
keys of a run are newer versions of keys in older runs, 1 % tombstones.
"""
from __future__ import annotations

import numpy as np

from . import Records, TYPE_DELETION, TYPE_VALUE

NOW = 300_000_000  # fixed epoch_now() for reproducible parity
SEED = 1000


def _sort_fixed(keys: np.ndarray) -> np.ndarray:
    """argsort rows of an (n, L) uint8 matrix bytewise-lexicographically."""
    n, L = keys.shape
    pad = (-L) % 8
    k = np.concatenate([keys, np.zeros((n, pad), np.uint8)], axis=1) if pad else keys
    cols = k.reshape(n, -1, 8).view(">u8").reshape(n, -1)
    return np.lexsort(tuple(cols[:, c] for c in range(cols.shape[1] - 1, -1, -1)))


def make_keys(hash_ids: np.ndarray, sort_ids: np.ndarray, hk_len: int = 16, sk_len: int = 32,
              seed: int = SEED) -> np.ndarray:
    """raw keys (n, 2+hk_len+sk_len): hashkey = hk_len pseudo-random bytes derived from hash_ids,
    sortkey = zero padded decimal sort_ids."""
    n = hash_ids.shape[0]
    out = np.zeros((n, 2 + hk_len + sk_len), np.uint8)
    out[:, 0] = hk_len >> 8
    out[:, 1] = hk_len & 0xFF
    # splitmix64 of (id, word) -> bytes
    words = (hk_len + 7) // 8
    hk = np.zeros((n, words), np.uint64)
    with np.errstate(over="ignore"):
        for w in range(words):
            z = hash_ids.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed * 1315423911 + w * 0xBF58476D1CE4E5B9 & 0xFFFFFFFFFFFFFFFF)
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            hk[:, w] = z ^ (z >> np.uint64(31))
    out[:, 2:2 + hk_len] = hk.view(np.uint8).reshape(n, words * 8)[:, :hk_len]
    s = sort_ids.astype(np.uint64).copy()
    for d in range(sk_len - 1, -1, -1):
        out[:, 2 + hk_len + d] = (s % np.uint64(10)).astype(np.uint8) + ord("0")
        s //= np.uint64(10)
    return out


def make_values(rng: np.random.Generator, n: int, user_len: int, now: int, ts_us: int) -> np.ndarray:
    """raw v1 values (n, 12+user_len)."""
    v = np.zeros((n, 12 + user_len), np.uint8)
    u = rng.random(n)
    delta = rng.integers(1, 86401, n, dtype=np.int64)
    ets = np.where(u < 0.7, 0, np.where(u < 0.9, now + delta, now - delta)).astype(np.uint32)
    v[:, 0:4] = ets.astype(">u4").view(np.uint8).reshape(n, 4)
    timetag = np.uint64(((ts_us << 8) | (1 << 1)) & 0xFFFFFFFFFFFFFFFF)
    v[:, 4:12] = np.full(n, timetag, ">u8").view(np.uint8).reshape(n, 8)
    if user_len:
        v[:, 12:] = rng.integers(0, 256, (n, user_len), dtype=np.uint8)
    return v


def fixed_records(keys: np.ndarray, vals: np.ndarray, seq: np.ndarray, typ: np.ndarray) -> Records:
    """Records from fixed-width key/value matrices; tombstones get an empty value."""
    n, kl = keys.shape
    vl = vals.shape[1]
    is_val = typ == TYPE_VALUE
    val_len = np.where(is_val, vl, 0).astype(np.uint64)
    val_off = np.zeros(n + 1, np.uint64)
    np.cumsum(val_len, out=val_off[1:])
    flat_vals = vals[is_val].reshape(-1)
    key_off = (np.arange(n + 1, dtype=np.uint64) * np.uint64(kl))
    return Records(np.ascontiguousarray(keys.reshape(-1)), key_off, np.ascontiguousarray(flat_vals), val_off,
                   seq.astype(np.uint64), typ.astype(np.uint8))


def compaction_runs(k: int = 4, n_per_run: int = 25_000, hk_len: int = 16, sk_len: int = 32, user_len: int = 256,
                    sortkeys_per_hash: int = 64, dup_frac: float = 0.10, tomb_frac: float = 0.01,
                    now: int = NOW, seed: int = SEED):
    """k overlapping L0-style runs; run 0 is the oldest (lowest seqnos), run k-1 the newest.
    Returns a list of Records, each sorted in internal-key order."""
    rng = np.random.default_rng(seed)
    runs = []
    older_hash = []  # (hash_ids, sort_ids) of earlier runs, for duplicates
    next_hash = 0
    for i in range(k):
        n_dup = int(n_per_run * dup_frac) if i > 0 else 0
        n_own = n_per_run - n_dup
        n_hash = (n_own + sortkeys_per_hash - 1) // sortkeys_per_hash
        own_h = np.repeat(np.arange(next_hash, next_hash + n_hash, dtype=np.uint64), sortkeys_per_hash)[:n_own]
        own_s = np.tile(np.arange(sortkeys_per_hash, dtype=np.uint64), n_hash)[:n_own]
        next_hash += n_hash
        if n_dup:
            oh = np.concatenate([h for h, _ in older_hash])
            os_ = np.concatenate([s for _, s in older_hash])
            pick = rng.choice(oh.shape[0], n_dup, replace=False)
            h = np.concatenate([own_h, oh[pick]])
            s = np.concatenate([own_s, os_[pick]])
        else:
            h, s = own_h, own_s
        older_hash.append((own_h, own_s))
        keys = make_keys(h, s, hk_len, sk_len, seed)
        vals = make_values(rng, n_per_run, user_len, now, ts_us=1_700_000_000_000_000 + i)
        typ = np.full(n_per_run, TYPE_VALUE, np.uint8)
        n_tomb = int(n_per_run * tomb_frac)
        if n_tomb:
            typ[rng.choice(n_per_run, n_tomb, replace=False)] = TYPE_DELETION
        seq = (np.uint64(i * n_per_run + 1) + rng.permutation(n_per_run).astype(np.uint64))
        order = _sort_fixed(keys)
        runs.append(fixed_records(keys[order], vals[order], seq[order], typ[order]))
    return runs


def total_bytes(runs) -> int:
    return int(sum(r.keys.shape[0] + r.vals.shape[0] for r in runs))


def shuffled(recs: Records, seed: int = 1) -> Records:
    """the records of `recs` (fixed-width keys) in a seeded random order"""
    n = recs.n
    perm = np.random.default_rng(seed).permutation(n)
    klen, vlen = np.diff(recs.key_off.astype(np.int64)), np.diff(recs.val_off.astype(np.int64))
    kw = int(klen[0]) if n else 0
    assert (klen == kw).all(), "fixed-width keys only"
    keys = recs.keys[int(recs.key_off[0]):int(recs.key_off[0]) + n * kw].reshape(n, kw)[perm].reshape(-1)
    voff = np.zeros(n + 1, np.uint64)
    voff[1:] = np.cumsum(vlen[perm])
    src = np.repeat(recs.val_off[:-1].astype(np.int64)[perm] - voff[:-1].astype(np.int64), vlen[perm]) + np.arange(int(voff[-1]))
    return Records(np.ascontiguousarray(keys), np.arange(n + 1, dtype=np.uint64) * np.uint64(kw), recs.vals[src], voff,
                   recs.seq[perm].copy(), recs.type[perm].copy())
