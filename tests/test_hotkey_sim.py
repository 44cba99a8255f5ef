"""CPU check of k_hotkey_capture (incubator_pegasus_b200/csrc/hotkey_kernels.cuh) inside the host SIMT interpreter
(tools/simt): several partition slots in mixed phases (off, coarse, fine), zipfian batches with heavy duplication inside
warps, empty, short and long hash keys, and fine queues that fill in the middle of the launch.  The coarse counters must
equal a Python model exactly, and every fine slot must admit exactly min(room, in-bucket keys) distinct keys of its target
bucket.  The same check runs in the plain build and, in a subprocess, in the AddressSanitizer build (tools/simt/build.sh asan),
which checks every access of the kernel against the exact bounds of its buffers."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import hotkey_model as hm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM_DIR = os.path.join(ROOT, "tools", "simt")
SRCS = [os.path.join(SIM_DIR, f) for f in ("sim_compact.cpp", "simt.h")] + [
    os.path.join(ROOT, "incubator_pegasus_b200", "csrc", f)
    for f in ("hotkey_kernels.cuh", "compact_kernels.cuh", "index_kernel.cuh", "read_kernels.cuh", "scan_kernel.cuh", "group.cuh",
              "device_util.cuh", "format.h")]
NB = 37


def build_sim(so, asan=False):
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in SRCS):
        extra = ["-fsanitize=address", "-fno-omit-frame-pointer"] if asan else []
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wno-unknown-pragmas", *extra,
                               os.path.join(SIM_DIR, "sim_compact.cpp"), "-o", so])
    return so


def load_sim(so):
    lib = C.CDLL(so)
    lib.sim_hotkey_capture.restype = C.c_uint32
    lib.sim_hotkey_capture.argtypes = [C.c_void_p] * 3 + [C.c_uint32] * 3 + [C.c_void_p] * 6 + [C.c_uint32]
    lib.sim_hotkey_hash.restype = C.c_uint64
    lib.sim_hotkey_hash.argtypes = [C.c_char_p, C.c_uint32]
    return lib


def raw_key(hk: bytes, sk: bytes) -> bytes:
    return len(hk).to_bytes(2, "big") + hk + sk


def make_batch(rng, n, n_slots):
    """zipfian hash keys (a few very hot ones, so that whole warps repeat a key), plus empty, long and malformed keys"""
    pool = [b"hot%d" % i for i in range(4)] + [bytes(rng.integers(0, 256, int(rng.integers(1, 24)), dtype=np.uint8)) for _ in range(300)]
    pool += [b"L" * 65, bytes(rng.integers(0, 256, 300, dtype=np.uint8)), b"", b"x" * 64, b"y" * 1000]
    ranks = np.minimum(rng.zipf(1.3, n) - 1, len(pool) - 1)
    keys = []
    for i, r in enumerate(ranks):
        if i % 97 == 5:
            keys.append(b"\x00")                        # shorter than a hash-key length: an empty hash key
        elif i % 89 == 7:
            keys.append(b"\x7f\xff" + b"clamped")       # a hash-key length past the key: clamped to it
        else:
            keys.append(raw_key(pool[int(r)], b"s%d" % int(rng.integers(0, 9))))
    part = rng.integers(0, n_slots, n).astype(np.uint32)
    part[:64] = 0                                       # whole warps of one slot and one hot key
    for i in range(64):
        keys[i] = raw_key(b"hot0", b"s")
    return keys, part


def run_case(lib, seed, grid):
    rng = np.random.default_rng(seed)
    n_slots = 6
    keys, part = make_batch(rng, 3000, n_slots)
    hot_bucket = hm.bucket(b"hot0", NB)
    state = np.array([1, 0, 2, 1, 2, 2], np.uint32)
    target = np.array([0, 0, hot_bucket, 0, hm.bucket(b"y" * 1000, NB), hm.bucket(b"hot1", NB)], np.uint32)
    room = np.array([0, 0, 7, 0, 1000, 0], np.uint32)  # slot 2 fills mid-launch, slot 4 has room for all, slot 5 none
    flat = np.frombuffer(b"".join(keys) + b"\0", np.uint8).copy()
    off = np.zeros(len(keys) + 1, np.uint32)
    off[1:] = np.cumsum([len(k) for k in keys])
    buckets = rng.integers(0, 1000, (n_slots, NB)).astype(np.uint64)  # counters accumulate across launches
    want = buckets.copy()
    inb = {s: [] for s in range(n_slots)}
    for i, k in enumerate(keys):
        s = int(part[i])
        hk = hm.hash_key_of(k)
        b = hm.bucket(hk, NB)
        if state[s] == 1:
            want[s, b] += 1
        elif state[s] == 2 and b == target[s]:
            inb[s].append(i)
    tickets = np.zeros(n_slots, np.uint32)
    idx = np.zeros(int(room[state == 2].sum()) + 1, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    total = lib.sim_hotkey_capture(p(flat), p(off), p(part), len(keys), NB, n_slots, p(state), p(target), p(room), p(buckets),
                                   p(tickets), p(idx), grid)
    assert total == int(room[state == 2].sum())
    assert (buckets[state == 1] == want[state == 1]).all(), "coarse counters differ from the model"
    assert (buckets[state != 1] == want[state != 1]).all(), "a slot that is not coarse was counted"
    base = 0
    for s in range(n_slots):
        if state[s] != 2:
            assert tickets[s] == 0
            continue
        assert tickets[s] == len(inb[s]), (s, tickets[s], len(inb[s]))
        got = idx[base:base + min(int(room[s]), len(inb[s]))]
        assert len(set(got.tolist())) == len(got) == min(int(room[s]), len(inb[s]))
        assert set(got.tolist()) <= set(inb[s]), "a fine index outside the target bucket"
        base += int(room[s])
    assert len(inb[2]) > room[2] and 0 < len(inb[4]) < room[4] and len(inb[5]) > 0
    # single-slot launch (pgs_get_batch): no key_part
    one = np.zeros(NB, np.uint64)
    lib.sim_hotkey_capture(p(flat), p(off), None, len(keys), NB, 1, p(state[:1]), p(target[:1]), p(room[:1]), p(one), p(tickets),
                           p(idx), grid)
    ref = np.zeros(NB, np.uint64)
    for k in keys:
        ref[hm.bucket(hm.hash_key_of(k), NB)] += 1
    assert (one == ref).all()


def check_all(lib):
    for b in [b"", b"a", b"abcd", b"abcde", bytes(range(256)) * 3]:
        assert lib.sim_hotkey_hash(b, len(b)) == hm.hotkey_hash(b)
    run_case(lib, 1, 3)
    run_case(lib, 2, 1)


@pytest.fixture(scope="module")
def hsim():
    return load_sim(build_sim(os.path.join(SIM_DIR, "libpgs_sim.so")))


def test_sim_hotkey_capture(hsim):
    check_all(hsim)


def test_sim_hotkey_capture_asan(tmp_path):
    cxx = shutil.which("g++")
    asan = subprocess.run([cxx, "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("no libasan in this toolchain")
    so = build_sim(str(tmp_path / "libpgs_sim_asan.so"), asan=True)  # loaded only by the child, behind the ASan runtime
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0")
    code = ("import sys; sys.path[:0] = [%r]; import test_hotkey_sim as t; t.check_all(t.load_sim(%r)); print('OK')"
            % (os.path.dirname(os.path.abspath(__file__)), so))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-3000:] + out.stderr[-3000:]
