"""incubator_pegasus_b200 — thin ctypes binding of libpegasus_b200.so (the C ABI in
include/pegasus_b200.h).  The product is the shared library; this module only marshals numpy
buffers into it for tests, the smoke run and bench.py.  There is no CPU fallback: if the library
or a CUDA device is missing, calls fail loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpegasus_b200.so")

OK, NOT_FOUND, CORRUPTION, NOT_SUPPORTED, INVALID_ARGUMENT, IO_ERROR = 0, 1, 2, 3, 4, 5
INCOMPLETE, ABORTED = 7, 10
TYPE_DELETION, TYPE_VALUE = 0, 1
FT_NO_FILTER, FT_MATCH_ANYWHERE, FT_MATCH_PREFIX, FT_MATCH_POSTFIX = 0, 1, 2, 3

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)


def build(force: bool = False) -> str:
    """Compile the library in-tree with nvcc for sm_90a (no GPU needed)."""
    env = dict(os.environ)
    if force:
        env["FORCE"] = "1"
    subprocess.check_call(["bash", os.path.join(_HERE, "build.sh")], env=env)
    return LIB_PATH


class Blob(C.Structure):
    _fields_ = [("data", u8p), ("len", C.c_uint32)]


class EngineConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("block_size", C.c_uint32), ("restart_interval", C.c_uint32),
                ("ctas_per_sm", C.c_uint32), ("flags", C.c_uint32)]


class RunInfo(C.Structure):
    _fields_ = [("run_id", C.c_uint64), ("level", C.c_int32), ("n_blocks", C.c_uint32),
                ("n_records", C.c_uint64), ("n_tombstones", C.c_uint64), ("data_bytes", C.c_uint64),
                ("raw_key_bytes", C.c_uint64), ("raw_value_bytes", C.c_uint64),
                ("max_ukey_len", C.c_uint32), ("max_value_len", C.c_uint32),
                ("max_block_size", C.c_uint32), ("max_block_records", C.c_uint32),
                ("smallest_seq", C.c_uint64), ("largest_seq", C.c_uint64)]


class RunSrc(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_bytes", C.c_uint64), ("blk_off", C.c_void_p), ("blk_size", C.c_void_p),
                ("n_blocks", C.c_uint32), ("level", C.c_int32)]


class FilterParams(C.Structure):
    _fields_ = [("enabled", C.c_uint8), ("validate_hash", C.c_uint8), ("reserved", C.c_uint8 * 2),
                ("data_version", C.c_uint32), ("default_ttl", C.c_uint32), ("pidx", C.c_int32),
                ("partition_version", C.c_int32), ("ops", u8p), ("ops_len", C.c_uint32)]


class CompactResult(C.Structure):
    _fields_ = [("new_run_id", C.c_uint64), ("in_records", C.c_uint64), ("out_records", C.c_uint64),
                ("in_bytes", C.c_uint64), ("out_bytes", C.c_uint64), ("in_block_bytes", C.c_uint64),
                ("out_block_bytes", C.c_uint64), ("dropped_shadowed", C.c_uint64),
                ("dropped_tombstone", C.c_uint64), ("dropped_expired", C.c_uint64),
                ("dropped_user", C.c_uint64), ("dropped_stale", C.c_uint64), ("ttl_rewritten", C.c_uint64),
                ("n_tiles", C.c_uint32), ("n_launches", C.c_uint32), ("device_ms", C.c_float),
                ("merge_kernel_ms", C.c_float), ("walk_ms", C.c_float), ("emit_ms", C.c_float),
                ("reserved", C.c_uint32)]


class CompactJob(C.Structure):
    _fields_ = [("part", C.c_void_p), ("run_ids", C.POINTER(C.c_uint64)), ("k", C.c_uint32), ("out_level", C.c_int32),
                ("bottommost", C.c_int32), ("fp", C.POINTER(FilterParams))]


class RunBuildJob(C.Structure):
    _fields_ = [("part", C.c_void_p), ("level", C.c_int32), ("n", C.c_uint64), ("keys", C.c_void_p), ("key_off", C.c_void_p),
                ("vals", C.c_void_p), ("val_off", C.c_void_p), ("seq", C.c_void_p), ("type", C.c_void_p)]

    @staticmethod
    def of(part, recs: "Records", level: int = 0) -> "RunBuildJob":
        """the job of `recs` for `part` (a Partition or None); the arrays of recs must outlive the call"""
        return RunBuildJob(part.h.value if part is not None else None, level, recs.n, recs.keys.ctypes.data, recs.key_off.ctypes.data,
                           recs.vals.ctypes.data, recs.val_off.ctypes.data, recs.seq.ctypes.data, recs.type.ctypes.data)


SPLIT_MAX_CHILDREN = 32


class SplitChildResult(C.Structure):
    _fields_ = [("records", C.c_uint64), ("tombstones", C.c_uint64), ("raw_bytes", C.c_uint64), ("block_bytes", C.c_uint64),
                ("runs", C.c_uint32), ("reserved", C.c_uint32)]


class SplitResult(C.Structure):
    _fields_ = [("child", SplitChildResult * SPLIT_MAX_CHILDREN), ("in_records", C.c_uint64), ("in_bytes", C.c_uint64),
                ("dropped_empty", C.c_uint64), ("device_ms", C.c_float), ("kernel_ms", C.c_float), ("count_ms", C.c_float),
                ("walk_ms", C.c_float), ("emit_ms", C.c_float), ("n_launches", C.c_uint32)]


class SplitJob(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.POINTER(C.c_void_p))]


SPLIT_MANY_MAX_JOBS = 4096
SPLIT_MANY_LAUNCHES = 7


class GetResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("expire_ts", C.c_uint32), ("value_off", C.c_uint32),
                ("value_len", C.c_uint32), ("expired", C.c_uint8), ("reserved", C.c_uint8 * 3)]


class DecodeSizes(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("key_bytes", C.c_uint64), ("value_bytes", C.c_uint64)]


class KV(C.Structure):
    _fields_ = [("key_off", C.c_uint32), ("key_len", C.c_uint32), ("value_off", C.c_uint32),
                ("value_len", C.c_uint32), ("expire_ts", C.c_uint32)]


class ScanRequest(C.Structure):
    _fields_ = [("start", Blob), ("stop", Blob), ("start_inclusive", C.c_uint8), ("stop_inclusive", C.c_uint8),
                ("reverse", C.c_uint8), ("no_value", C.c_uint8), ("key_mode", C.c_uint8),
                ("return_expire_ts", C.c_uint8), ("count_only", C.c_uint8), ("validate_hash", C.c_uint8),
                ("prefix_same_as_start", C.c_uint8), ("skip_first_exclusive", C.c_uint8),
                ("reserved", C.c_uint8 * 2), ("hash_filter_type", C.c_int32), ("sort_filter_type", C.c_int32),
                ("hash_filter", Blob), ("sort_filter", Blob), ("max_count", C.c_uint32),
                ("max_iter_count", C.c_uint32), ("max_iter_size", C.c_uint64), ("pidx", C.c_int32),
                ("partition_version", C.c_int32)]


class ScanResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("n_kvs", C.c_uint32), ("count", C.c_uint32), ("iter_count", C.c_uint32),
                ("expire_count", C.c_uint32), ("filter_count", C.c_uint32), ("size", C.c_uint64),
                ("complete", C.c_uint8), ("iter_valid", C.c_uint8), ("reserved", C.c_uint8 * 2),
                ("resume_len", C.c_uint32), ("arena_used", C.c_uint64)]


class ServerOptions(C.Structure):
    _fields_ = [("rocksdb_max_iteration_count", C.c_uint32),
                ("rocksdb_multi_get_max_iteration_count", C.c_uint32),
                ("rocksdb_multi_get_max_iteration_size", C.c_uint64), ("l0_compaction_trigger", C.c_uint32),
                ("memtable_bytes", C.c_uint64), ("prefix_filter", C.c_uint8), ("cluster_id", C.c_uint8),
                ("reserved", C.c_uint8 * 6), ("hotkey_buckets_num", C.c_uint32), ("hot_bucket_variance_threshold", C.c_uint32),
                ("hot_key_variance_threshold", C.c_uint32), ("max_seconds_to_detect_hotkey", C.c_uint32)]


class Response(C.Structure):
    _fields_ = [("error", C.c_int32), ("app_id", C.c_int32), ("partition_index", C.c_int32),
                ("ttl_seconds", C.c_int32), ("count", C.c_int64), ("context_id", C.c_int64),
                ("kv_count", C.c_int32), ("n_kvs", C.c_uint32), ("kvs", C.POINTER(KV)), ("hk_len", u32p),
                ("arena", u8p), ("arena_len", C.c_uint64), ("iteration_count", C.c_uint32),
                ("expire_count", C.c_uint32), ("filter_count", C.c_uint32)]


class MultiGetRequest(C.Structure):
    _fields_ = [("hash_key", Blob), ("sort_keys", C.POINTER(Blob)), ("n_sort_keys", C.c_uint32),
                ("max_kv_count", C.c_int32), ("max_kv_size", C.c_int32), ("no_value", C.c_uint8),
                ("start_inclusive", C.c_uint8), ("stop_inclusive", C.c_uint8), ("reverse", C.c_uint8),
                ("start_sortkey", Blob), ("stop_sortkey", Blob), ("sort_key_filter_type", C.c_int32),
                ("sort_key_filter_pattern", Blob)]


class GetScannerRequest(C.Structure):
    _fields_ = [("start_key", Blob), ("stop_key", Blob), ("start_inclusive", C.c_uint8),
                ("stop_inclusive", C.c_uint8), ("no_value", C.c_uint8), ("validate_partition_hash", C.c_uint8),
                ("return_expire_ts", C.c_uint8), ("full_scan", C.c_uint8), ("only_return_count", C.c_uint8),
                ("reserved", C.c_uint8), ("batch_size", C.c_int32), ("hash_key_filter_type", C.c_int32),
                ("hash_key_filter_pattern", Blob), ("sort_key_filter_type", C.c_int32),
                ("sort_key_filter_pattern", Blob)]


class FullKey(C.Structure):
    _fields_ = [("hash_key", Blob), ("sort_key", Blob)]


_lib = None


def lib() -> C.CDLL:
    """Load libpegasus_b200.so; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run incubator_pegasus_b200/build.sh (nvcc, sm_90a)")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.pgs_last_error.restype = C.c_char_p
    L.pgs_engine_open.argtypes = [C.POINTER(EngineConfig), C.POINTER(vp)]
    L.pgs_engine_close.argtypes = [vp]
    L.pgs_engine_close.restype = None
    L.pgs_engine_stream.argtypes = [vp]
    L.pgs_engine_stream.restype = vp
    L.pgs_engine_sync.argtypes = [vp]
    L.pgs_engine_launches.argtypes = [vp]
    L.pgs_engine_launches.restype = C.c_uint64
    L.pgs_engine_last_kernel_ms.argtypes = [vp]
    L.pgs_engine_last_kernel_ms.restype = C.c_float
    L.pgs_engine_last_blocks_probed.argtypes = [vp]
    L.pgs_engine_last_blocks_probed.restype = C.c_uint64
    L.pgs_router_open.argtypes = [C.POINTER(EngineConfig), C.c_int32, C.POINTER(vp)]
    L.pgs_router_close.argtypes = [vp]
    L.pgs_router_close.restype = None
    L.pgs_router_device_count.argtypes = [vp]
    L.pgs_router_device_for.argtypes = [vp, C.c_int32, C.c_int32]
    L.pgs_router_engine_for.argtypes = [vp, C.c_int32, C.c_int32]
    L.pgs_router_engine_for.restype = vp
    L.pgs_partition_index.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32]
    L.pgs_partition_index.restype = C.c_uint32
    L.pgs_engine_last_runs_skipped.argtypes = [vp]
    L.pgs_engine_last_runs_skipped.restype = C.c_uint64
    L.pgs_range_scan_many.argtypes = [vp, C.POINTER(ScanRequest), C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, vp, C.c_uint64,
                                      vp, C.c_uint64, vp, C.c_uint32, vp, vp, vp]
    L.pgs_range_scan_many_multi.argtypes = [C.POINTER(vp), C.c_uint32, C.POINTER(ScanRequest), vp, C.c_uint32, C.c_uint32, C.c_uint64,
                                            C.c_uint32, vp, C.c_uint64, vp, C.c_uint64, vp, C.c_uint32, vp, vp, vp]
    L.pgs_partition_create.argtypes = [vp, C.c_int32, C.c_int32, C.c_uint32, C.POINTER(vp)]
    L.pgs_partition_destroy.argtypes = [vp]
    L.pgs_partition_destroy.restype = None
    L.pgs_run_upload.argtypes = [vp, C.c_int32, vp, C.c_uint64, vp, vp, C.c_uint32, u64p]
    L.pgs_get_batch_multi.argtypes = [C.POINTER(vp), C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, vp, C.c_uint64, vp, u64p]
    L.pgs_run_upload_many.argtypes = [vp, C.POINTER(RunSrc), C.c_uint32, u64p]
    L.pgs_run_build.argtypes = [vp, C.c_int32, C.c_uint64, vp, vp, vp, vp, vp, vp, u64p]
    L.pgs_run_build_last_ms.argtypes = [C.POINTER(C.c_float)]
    L.pgs_run_build_last_ms.restype = None
    L.pgs_run_build_unsorted.argtypes = [vp, C.c_int32, C.c_uint64, vp, vp, vp, vp, vp, vp, u64p]
    L.pgs_run_build_last_sort_ms.argtypes = []
    L.pgs_run_build_last_sort_ms.restype = C.c_float
    L.pgs_run_drop.argtypes = [vp, C.c_uint64]
    L.pgs_run_info_get.argtypes = [vp, C.c_uint64, C.POINTER(RunInfo)]
    L.pgs_run_list.argtypes = [vp, u64p, C.c_uint32, u32p]
    L.pgs_run_download.argtypes = [vp, C.c_uint64, vp, C.c_uint64, vp, vp, C.c_uint32]
    L.pgs_compact.argtypes = [vp, u64p, C.c_uint32, C.c_int32, C.c_int32, C.POINTER(FilterParams), C.c_uint32,
                              C.POINTER(CompactResult)]
    L.pgs_compact_ex.argtypes = [vp, u64p, C.c_uint32, C.c_int32, C.c_int32, C.POINTER(FilterParams), C.c_uint32,
                                 C.c_uint32, C.POINTER(CompactResult)]
    L.pgs_compaction_ops_parse.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, vp, C.c_uint32, u32p]
    L.pgs_compaction_ops_parse.restype = C.c_int64
    L.pgs_generate_key.argtypes = [vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32]
    L.pgs_generate_next_blob.argtypes = [vp, C.c_uint32, vp, C.c_uint32, C.c_int32, vp, C.c_uint32]
    L.pgs_key_hash.argtypes = [vp, C.c_uint32]
    L.pgs_key_hash.restype = C.c_uint64
    L.pgs_crc64.argtypes = [vp, C.c_uint64, C.c_uint64]
    L.pgs_crc64.restype = C.c_uint64
    L.pgs_run_builder_new.argtypes = [C.c_uint32, C.c_uint32]
    L.pgs_run_builder_new.restype = vp
    L.pgs_run_builder_add.argtypes = [vp, vp, C.c_uint32, C.c_uint64, C.c_uint8, vp, C.c_uint32]
    L.pgs_run_builder_add_many.argtypes = [vp, C.c_uint64, vp, vp, vp, vp, vp, vp]
    L.pgs_run_builder_finish.argtypes = [vp, C.POINTER(vp), u64p, C.POINTER(vp), C.POINTER(vp), u32p]
    L.pgs_run_builder_free.argtypes = [vp]
    L.pgs_run_builder_free.restype = None
    L.pgs_blocks_decode.argtypes = [vp, vp, vp, C.c_uint32, C.POINTER(DecodeSizes), vp, vp, vp, vp, vp, vp]
    for name, args in {
        "pgs_get_batch": [vp, vp, vp, C.c_uint32, C.c_uint32, vp, C.c_uint64, vp, u64p],
        "pgs_partition_split": [vp, C.c_uint32, C.c_uint32, C.POINTER(vp), C.c_uint32, C.POINTER(SplitResult)],
        "pgs_rrdb_split": [vp, C.c_uint32, C.c_uint32, C.POINTER(vp), C.c_uint32, C.POINTER(C.c_int64)],
        "pgs_partition_split_many": [C.POINTER(SplitJob), C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(SplitResult)],
        "pgs_rrdb_split_many": [C.POINTER(vp), C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(vp), C.POINTER(C.c_int64)],
        "pgs_range_scan": [vp, C.POINTER(ScanRequest), C.c_uint32, vp, C.c_uint64, vp, C.c_uint32, vp, C.c_uint32,
                           C.POINTER(ScanResult)],
        "pgs_rrdb_start": [vp, C.c_int32, C.c_int32, C.POINTER(ServerOptions), C.c_char_p, C.c_uint32, C.POINTER(vp)],
        "pgs_rrdb_update_app_envs": [vp, C.c_char_p, C.c_uint32, C.c_uint32],
        "pgs_rrdb_get": [vp, Blob, C.c_uint32, vp],
        "pgs_rrdb_ttl": [vp, Blob, C.c_uint32, vp],
        "pgs_rrdb_multi_get": [vp, C.POINTER(MultiGetRequest), C.c_uint32, vp],
        "pgs_rrdb_batch_get": [vp, C.POINTER(FullKey), C.c_uint32, C.c_uint32, vp],
        "pgs_rrdb_sortkey_count": [vp, Blob, C.c_uint32, vp],
        "pgs_rrdb_get_scanner": [vp, C.POINTER(GetScannerRequest), C.c_uint32, vp],
        "pgs_rrdb_scan": [vp, C.c_int64, C.c_uint32, vp],
        "pgs_rrdb_get_many": [vp, vp, vp, C.c_uint32, C.c_uint32, vp, C.c_uint64, vp, u64p],
        "pgs_rrdb_put": [vp, Blob, Blob, C.c_uint32, C.c_int64, C.c_uint64, C.c_uint32],
        "pgs_rrdb_remove": [vp, Blob, C.c_int64, C.c_uint32],
        "pgs_rrdb_multi_put": [vp, Blob, C.POINTER(Blob), C.POINTER(Blob), C.c_uint32, C.c_uint32, C.c_int64,
                               C.c_uint64, C.c_uint32],
        "pgs_rrdb_multi_remove": [vp, Blob, C.POINTER(Blob), C.c_uint32, C.c_int64, C.POINTER(C.c_int64), C.c_uint32],
        "pgs_rrdb_flush": [vp, C.c_uint32],
        "pgs_rrdb_flush_many": [C.POINTER(vp), C.c_uint32, C.c_uint32],
        "pgs_run_build_many": [C.POINTER(RunBuildJob), C.c_uint32, u64p],
        "pgs_rrdb_manual_compact": [vp, C.c_uint32, C.POINTER(CompactResult)],
        "pgs_rrdb_manual_compact_many": [C.POINTER(vp), C.c_uint32, C.c_uint32, C.POINTER(CompactResult)],
        "pgs_compact_many": [C.POINTER(CompactJob), C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(CompactResult)],
        "pgs_rrdb_detect_hotkey": [vp, C.c_int32, C.c_int32, C.c_uint32, C.c_char_p, C.c_uint32, u32p],
        "pgs_rrdb_hotkey_analyse": [vp, C.c_uint32],
        "pgs_rrdb_hotkey_state": [vp, C.c_int32],
    }.items():
        if hasattr(L, name):
            getattr(L, name).argtypes = args
    for name, res, args in [("pgs_rrdb_stop", None, [vp]), ("pgs_rrdb_partition", vp, [vp]),
                            ("pgs_rrdb_set_partition_version", None, [vp, C.c_int32]),
                            ("pgs_rrdb_clear_scanner", None, [vp, C.c_int64]),
                            ("pgs_rrdb_last_flushed_decree", C.c_int64, [vp]),
                            ("pgs_response_new", vp, []), ("pgs_response_free", None, [vp]),
                            ("pgs_response_view", C.POINTER(Response), [vp])]:
        if hasattr(L, name):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
    _lib = L
    return L


class PegasusError(RuntimeError):
    def __init__(self, code: int, what: str):
        super().__init__(f"{what}: status {code}: {lib().pgs_last_error().decode(errors='replace')}")
        self.code = code


def _check(code: int, what: str) -> None:
    if code != OK:
        raise PegasusError(code, what)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


@dataclass
class Records:
    """Flat record set: record i has user key keys[key_off[i]:key_off[i+1]] etc."""
    keys: np.ndarray      # uint8
    key_off: np.ndarray   # uint64 [n+1]
    vals: np.ndarray      # uint8
    val_off: np.ndarray   # uint64 [n+1]
    seq: np.ndarray       # uint64 [n]
    type: np.ndarray      # uint8 [n]

    @property
    def n(self) -> int:
        return int(self.seq.shape[0])

    def key(self, i: int) -> bytes:
        return self.keys[int(self.key_off[i]):int(self.key_off[i + 1])].tobytes()

    def value(self, i: int) -> bytes:
        return self.vals[int(self.val_off[i]):int(self.val_off[i + 1])].tobytes()

    def same_as(self, other: "Records") -> bool:
        return (self.n == other.n and np.array_equal(self.key_off, other.key_off)
                and np.array_equal(self.val_off, other.val_off) and np.array_equal(self.seq, other.seq)
                and np.array_equal(self.type, other.type) and np.array_equal(self.keys, other.keys)
                and np.array_equal(self.vals, other.vals))

    @staticmethod
    def from_list(items) -> "Records":
        """items: iterable of (ukey bytes, seq, type, value bytes), already in internal-key order."""
        items = list(items)
        ko = np.zeros(len(items) + 1, np.uint64)
        vo = np.zeros(len(items) + 1, np.uint64)
        for i, (k, _s, _t, v) in enumerate(items):
            ko[i + 1] = ko[i] + len(k)
            vo[i + 1] = vo[i] + len(v)
        keys = np.frombuffer(b"".join(k for k, _, _, _ in items), np.uint8).copy() if items else np.zeros(0, np.uint8)
        vals = np.frombuffer(b"".join(v for _, _, _, v in items), np.uint8).copy() if items else np.zeros(0, np.uint8)
        return Records(keys, ko, vals, vo, np.array([s for _, s, _, _ in items], np.uint64),
                       np.array([t for _, _, t, _ in items], np.uint8))

    def to_list(self):
        return [(self.key(i), int(self.seq[i]), int(self.type[i]), self.value(i)) for i in range(self.n)]


@dataclass
class BlockRun:
    """Host copy of a run in upload layout."""
    data: np.ndarray
    blk_off: np.ndarray
    blk_size: np.ndarray

    @property
    def n_blocks(self) -> int:
        return int(self.blk_off.shape[0])


def build_run(recs: Records, block_size: int = 4096, restart_interval: int = 16) -> BlockRun:
    """memtable -> data blocks (the flush side), through the product's host run builder."""
    L = lib()
    b = L.pgs_run_builder_new(block_size, restart_interval)
    try:
        _check(L.pgs_run_builder_add_many(b, recs.n, _ptr(recs.keys), _ptr(recs.key_off), _ptr(recs.vals),
                                          _ptr(recs.val_off), _ptr(recs.seq), _ptr(recs.type)), "run_builder_add_many")
        data, off, size = C.c_void_p(), C.c_void_p(), C.c_void_p()
        nbytes, nb = C.c_uint64(), C.c_uint32()
        _check(L.pgs_run_builder_finish(b, C.byref(data), C.byref(nbytes), C.byref(off), C.byref(size), C.byref(nb)),
               "run_builder_finish")
        n = nb.value
        d = np.ctypeslib.as_array(C.cast(data, u8p), (nbytes.value,)).copy() if nbytes.value else np.zeros(0, np.uint8)
        o = np.ctypeslib.as_array(C.cast(off, u64p), (n,)).copy() if n else np.zeros(0, np.uint64)
        s = np.ctypeslib.as_array(C.cast(size, u32p), (n,)).copy() if n else np.zeros(0, np.uint32)
        return BlockRun(d, o, s)
    finally:
        L.pgs_run_builder_free(b)


def decode_blocks(run: BlockRun) -> Records:
    L = lib()
    sz = DecodeSizes()
    _check(L.pgs_blocks_decode(_ptr(run.data), _ptr(run.blk_off), _ptr(run.blk_size), run.n_blocks, C.byref(sz),
                               None, None, None, None, None, None), "blocks_decode(sizes)")
    n = sz.n_records
    r = Records(np.zeros(sz.key_bytes, np.uint8), np.zeros(n + 1, np.uint64), np.zeros(sz.value_bytes, np.uint8),
                np.zeros(n + 1, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.uint8))
    _check(L.pgs_blocks_decode(_ptr(run.data), _ptr(run.blk_off), _ptr(run.blk_size), run.n_blocks, C.byref(sz),
                               _ptr(r.keys), _ptr(r.key_off), _ptr(r.vals), _ptr(r.val_off), _ptr(r.seq),
                               _ptr(r.type)), "blocks_decode")
    return r


def parse_ops(json_text: str, data_version: int = 1) -> np.ndarray:
    L = lib()
    buf = np.zeros(max(64, 4 * len(json_text) + 64), np.uint8)
    n_ops = C.c_uint32()
    raw = json_text.encode()
    n = L.pgs_compaction_ops_parse(raw, len(raw), data_version, _ptr(buf), buf.shape[0], C.byref(n_ops))
    if n < 0:
        raise PegasusError(int(-n), "compaction_ops_parse")
    return buf[:n].copy()


def _filter_params(enabled: bool = True, default_ttl: int = 0, validate_hash: bool = False, pidx: int = 0,
                   partition_version: int = -1, ops: np.ndarray | None = None, data_version: int = 1) -> FilterParams:
    """the FilterParams of Engine.compact_many's filter kwargs; the struct keeps its ops table alive (fp._ops)"""
    fp = FilterParams()
    fp.enabled = 1 if enabled else 0
    fp.validate_hash = 1 if validate_hash else 0
    fp.data_version = data_version
    fp.default_ttl = default_ttl
    fp.pidx = pidx
    fp.partition_version = partition_version
    if ops is not None and ops.shape[0] >= 4:
        fp._ops = np.ascontiguousarray(ops)
        fp.ops = fp._ops.ctypes.data_as(u8p)
        fp.ops_len = fp._ops.shape[0]
    return fp


class Engine:
    def __init__(self, device: int = -1, ctas_per_sm: int = 0, block_size: int = 0, restart_interval: int = 0):
        cfg = EngineConfig(device, block_size, restart_interval, ctas_per_sm, 0)
        self.h = C.c_void_p()
        _check(lib().pgs_engine_open(C.byref(cfg), C.byref(self.h)), "engine_open")

    def close(self):
        if self.h:
            lib().pgs_engine_close(self.h)
            self.h = None

    def sync(self):
        _check(lib().pgs_engine_sync(self.h), "engine_sync")

    @property
    def stream(self) -> int:
        return int(lib().pgs_engine_stream(self.h) or 0)

    @property
    def launches(self) -> int:
        return int(lib().pgs_engine_launches(self.h))

    @property
    def last_kernel_ms(self) -> float:
        return float(lib().pgs_engine_last_kernel_ms(self.h))

    @property
    def last_blocks_probed(self) -> int:
        return int(lib().pgs_engine_last_blocks_probed(self.h))

    @property
    def last_runs_skipped(self) -> int:
        return int(lib().pgs_engine_last_runs_skipped(self.h))

    def partition(self, app_id: int = 1, pidx: int = 0, data_version: int = 1) -> "Partition":
        return Partition(self, app_id, pidx, data_version)

    def compact_many(self, jobs, now: int, flags: int = 0) -> list[CompactResult]:
        """pgs_compact_many: the compactions of many partitions of this engine in one launch.  A job is (partition, run_ids,
        out_level, bottommost, filter kwargs as Partition.compact takes them -- enabled, default_ttl, validate_hash, pidx,
        partition_version, ops, data_version); returns one CompactResult per job."""
        n = len(jobs)
        arr = (CompactJob * max(1, n))()
        keep = []  # the id arrays, filter params and ops tables must outlive the call
        for i, (part, run_ids, out_level, bottommost, kw) in enumerate(jobs):
            ids = np.array(list(run_ids), np.uint64)
            fp = _filter_params(**(kw or {}))
            keep += [ids, fp]
            arr[i] = CompactJob(part.h.value if part is not None else None, ids.ctypes.data_as(u64p), ids.shape[0], out_level,
                                bottommost, C.pointer(fp))
        res = (CompactResult * max(1, n))()
        _check(lib().pgs_compact_many(arr if n else None, n, now, flags, res), "compact_many")
        return [res[i] for i in range(n)]

    def build_many(self, jobs) -> list[int]:
        """pgs_run_build_many: the runs of many partitions of this engine built in one set of launches.  A job is (partition,
        records in internal-key order, level); returns one run id per job (0 for a job without records)."""
        n = len(jobs)
        arr = (RunBuildJob * max(1, n))()
        for i, (part, recs, level) in enumerate(jobs):
            arr[i] = RunBuildJob.of(part, recs, level)
        ids = np.zeros(max(1, n), np.uint64)
        _check(lib().pgs_run_build_many(arr if n else None, n, ids.ctypes.data_as(u64p)), "run_build_many")
        return [int(x) for x in ids[:n]]

    def split_many(self, jobs, src_count: int, dst_count: int) -> list[SplitResult]:
        """pgs_partition_split_many: the splits of many parent partitions of this engine in one set of launches.  A job is
        (parent Partition, its children as Partition.split takes them); returns one SplitResult per job."""
        n = len(jobs)
        arr = (SplitJob * max(1, n))()
        keep = []  # the child arrays must outlive the call
        for i, (parent, children) in enumerate(jobs):
            hs = (C.c_void_p * max(1, len(children)))(*[c.h.value if c is not None else None for c in children])
            keep.append(hs)
            arr[i] = SplitJob(parent.h.value if parent is not None else None, C.cast(hs, C.POINTER(C.c_void_p)))
        res = (SplitResult * max(1, n))()
        _check(lib().pgs_partition_split_many(arr if n else None, n, src_count, dst_count, res), "partition_split_many")
        return [res[i] for i in range(n)]

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Router:
    """One engine per visible GPU; replica (app_id, pidx) lives on GPU pidx % n (pgs_router_*, include/pegasus_b200.h §7)."""

    def __init__(self, n_devices: int = 0, ctas_per_sm: int = 0, block_size: int = 0, restart_interval: int = 0):
        cfg = EngineConfig(-1, block_size, restart_interval, ctas_per_sm, 0)
        self.h = C.c_void_p()
        _check(lib().pgs_router_open(C.byref(cfg), n_devices, C.byref(self.h)), "router_open")

    @property
    def device_count(self) -> int:
        return int(lib().pgs_router_device_count(self.h))

    def device_for(self, app_id: int, pidx: int) -> int:
        return int(lib().pgs_router_device_for(self.h, app_id, pidx))

    def engine_for(self, app_id: int, pidx: int) -> Engine:
        h = lib().pgs_router_engine_for(self.h, app_id, pidx)
        if not h:
            raise PegasusError(INVALID_ARGUMENT, "router_engine_for")
        e = Engine.__new__(Engine)  # borrowed: the router owns and closes it
        e.h = C.c_void_p(h)
        e.close = lambda: None
        return e

    def close(self):
        if self.h:
            lib().pgs_router_close(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def get_batch_multi(parts, keys: np.ndarray, key_off: np.ndarray, key_part: np.ndarray, now: int, arena: np.ndarray, results=None):
    """keys of several partitions of one engine in one launch (pgs_get_batch_multi); key i goes to parts[key_part[i]]"""
    n = key_off.shape[0] - 1
    results = (GetResult * n)() if results is None else results
    handles = (C.c_void_p * len(parts))(*[p.h for p in parts])
    used = C.c_uint64()
    st = lib().pgs_get_batch_multi(handles, len(parts), _ptr(keys), _ptr(key_off), _ptr(key_part), n, now, _ptr(arena), arena.shape[0],
                                   results, C.byref(used))
    return st, results, arena, used.value


class Batcher:
    """pgs_batcher_*: blocking point reads of many host threads share pgs_get_batch_multi launches"""

    def __init__(self, parts, max_batch: int = 0, max_wait_us: int = 200):
        L = lib()
        L.pgs_batcher_open.argtypes = [C.POINTER(C.c_void_p), C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
        L.pgs_batcher_close.argtypes = [C.c_void_p]
        L.pgs_batcher_close.restype = None
        L.pgs_batcher_get.argtypes = [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(GetResult)]
        L.pgs_batcher_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.pgs_batcher_stats.restype = None
        self._parts = list(parts)
        handles = (C.c_void_p * len(self._parts))(*[p.h for p in self._parts])
        self.h = C.c_void_p()
        _check(L.pgs_batcher_open(handles, len(self._parts), max_batch, max_wait_us, C.byref(self.h)), "batcher_open")

    def get(self, slot: int, key: bytes, now: int, cap: int = 4096):
        """-> (launch status, GetResult, value bytes or None)"""
        buf = C.create_string_buffer(max(1, cap))
        r = GetResult()
        st = lib().pgs_batcher_get(self.h, slot, key, len(key), now, buf, cap, C.byref(r))
        return st, r, (buf.raw[:r.value_len] if st == 0 and r.status == OK else None)

    def stats(self):
        rq, ln = C.c_uint64(), C.c_uint64()
        lib().pgs_batcher_stats(self.h, C.byref(rq), C.byref(ln))
        return rq.value, ln.value

    def close(self):
        if self.h:
            lib().pgs_batcher_close(self.h)
            self.h = None


class ManualCompactDecision(C.Structure):
    _fields_ = [("rule", C.c_int32), ("disabled", C.c_int32), ("max_concurrent_running_count", C.c_int32),
                ("target_level", C.c_int32), ("bottommost_force", C.c_int32), ("reserved", C.c_int32)]


def manual_compact_decide(envs: dict, now_ms: int, last_finish_ms: int, today_midnight_s: int = -1, num_levels: int = 7):
    """pgs_manual_compact_decide: which manual-compaction rule of the env map fires at now_ms (host logic only)"""
    blob = b"".join(k.encode() + b"\0" + v.encode() + b"\0" for k, v in envs.items())
    out = ManualCompactDecision()
    f = lib().pgs_manual_compact_decide
    f.argtypes = [C.c_char_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_int64, C.c_int32, C.POINTER(ManualCompactDecision)]
    _check(f(blob if blob else None, len(envs), now_ms, last_finish_ms, today_midnight_s, num_levels, C.byref(out)), "manual_compact_decide")
    return out


def manual_compact_state_check(now_ms: int, last_finish_ms: int, min_interval_s: int, enqueue_ms: int):
    """pgs_manual_compact_state_check -> (allowed, new enqueue_ms)"""
    e = C.c_uint64(enqueue_ms)
    f = lib().pgs_manual_compact_state_check
    f.argtypes = [C.c_uint64, C.c_uint64, C.c_int32, C.POINTER(C.c_uint64)]
    ok = f(now_ms, last_finish_ms, min_interval_s, C.byref(e))
    return bool(ok), e.value


HOTKEY_READ, HOTKEY_WRITE = 0, 1
HOTKEY_START, HOTKEY_STOP, HOTKEY_QUERY = 0, 1, 2
HOTKEY_OK, HOTKEY_BUSY, HOTKEY_INVALID_STATE, HOTKEY_INVALID_PARAMETERS = 0, 1, 2, 3
HOTKEY_STOPPED, HOTKEY_COARSE_DETECTING, HOTKEY_FINE_DETECTING, HOTKEY_FINISHED = 0, 1, 2, 3


def detect_hotkey(server, hotkey_type: int, action: int, now_s: int):
    """pgs_rrdb_detect_hotkey on a pgs_server handle -> (outcome, hint or hot hash key as bytes)"""
    L = lib()
    n = C.c_uint32(0)
    buf = C.create_string_buffer(4096)
    out = L.pgs_rrdb_detect_hotkey(server, hotkey_type, action, now_s, buf, len(buf), C.byref(n))
    if n.value > len(buf):
        buf = C.create_string_buffer(n.value)
        out = L.pgs_rrdb_detect_hotkey(server, hotkey_type, HOTKEY_QUERY, now_s, buf, len(buf), C.byref(n)) if action == HOTKEY_QUERY else out
    return int(out), buf.raw[:n.value]


def hotkey_analyse(server, now_s: int) -> None:
    """pgs_rrdb_hotkey_analyse: one analysis step of both collectors of a pgs_server handle (the binding's 10 s timer)"""
    _check(lib().pgs_rrdb_hotkey_analyse(server, now_s), "rrdb_hotkey_analyse")


def hotkey_state(server, hotkey_type: int) -> int:
    return int(lib().pgs_rrdb_hotkey_state(server, hotkey_type))


def rrdb_split(parent, src_count: int, dst_count: int, children) -> int:
    """pgs_rrdb_split: the pgs_server handle `parent` into its children (server handles, or None: not built); returns the
    split's decree"""
    handles = (C.c_void_p * max(1, len(children)))(*[c if c is not None else None for c in children])
    decree = C.c_int64()
    _check(lib().pgs_rrdb_split(parent, src_count, dst_count, handles, len(children), C.byref(decree)), "rrdb_split")
    return decree.value


def rrdb_split_many(parents, src_count: int, dst_count: int, children) -> list[int]:
    """pgs_rrdb_split_many: the pgs_server handles `parents` split together; children[i] is parent i's row of dst_count /
    src_count child handles (None: not built); returns every parent's split decree"""
    n = len(parents)
    flat = [c for row in children for c in row]
    ph = (C.c_void_p * max(1, n))(*parents)
    ch = (C.c_void_p * max(1, len(flat)))(*flat)
    decrees = (C.c_int64 * max(1, n))()
    _check(lib().pgs_rrdb_split_many(ph, n, src_count, dst_count, ch, decrees), "rrdb_split_many")
    return [decrees[i] for i in range(n)]


def run_build_last_ms() -> list[float]:
    """device times (ms) of this thread's last Partition.build_records: input copy, block plan, block writing, index"""
    ms = (C.c_float * 4)()
    lib().pgs_run_build_last_ms(ms)
    return list(ms)


def run_build_last_sort_ms() -> float:
    """device time (ms) of the sort and the gather of this thread's last Partition.build_records_unsorted"""
    return float(lib().pgs_run_build_last_sort_ms())


def partition_index(hash_key: bytes, sort_key: bytes, partition_count: int) -> int:
    return int(lib().pgs_partition_index(hash_key, len(hash_key), sort_key, len(sort_key), partition_count))


class Partition:
    def __init__(self, eng: Engine, app_id: int, pidx: int, data_version: int, handle=None):
        self.eng = eng
        self.owned = handle is None
        self.h = C.c_void_p()
        if handle is None:
            _check(lib().pgs_partition_create(eng.h, app_id, pidx, data_version, C.byref(self.h)), "partition_create")
        else:
            self.h = C.c_void_p(handle)

    def close(self):
        if self.h and self.owned:
            lib().pgs_partition_destroy(self.h)
        self.h = None

    def upload(self, run: BlockRun, level: int = 0) -> int:
        rid = C.c_uint64()
        _check(lib().pgs_run_upload(self.h, level, _ptr(run.data), run.data.shape[0], _ptr(run.blk_off),
                                    _ptr(run.blk_size), run.n_blocks, C.byref(rid)), "run_upload")
        return rid.value

    def upload_many(self, runs, levels=None) -> list[int]:
        """several runs in one pipelined call (pgs_run_upload_many); runs[0] is installed first"""
        n = len(runs)
        src = (RunSrc * max(1, n))()
        for i, r in enumerate(runs):
            src[i] = RunSrc(r.data.ctypes.data, r.data.shape[0], r.blk_off.ctypes.data, r.blk_size.ctypes.data, r.n_blocks,
                            0 if levels is None else levels[i])
        ids = np.zeros(max(1, n), np.uint64)
        _check(lib().pgs_run_upload_many(self.h, src, n, ids.ctypes.data_as(u64p)), "run_upload_many")
        return [int(x) for x in ids[:n]]

    def upload_records(self, recs: Records, level: int = 0) -> int:
        return self.upload(build_run(recs), level)

    def build_records(self, recs: Records, level: int = 0) -> int:
        """the run of `recs` (in internal-key order) built on the device at the engine's block geometry (pgs_run_build): the
        same blocks and run info as upload(build_run(recs)) at that geometry; 0 for no records"""
        rid = C.c_uint64()
        _check(lib().pgs_run_build(self.h, level, recs.n, _ptr(recs.keys), _ptr(recs.key_off), _ptr(recs.vals), _ptr(recs.val_off),
                                   _ptr(recs.seq), _ptr(recs.type), C.byref(rid)), "run_build")
        return rid.value

    def build_records_unsorted(self, recs: Records, level: int = 0) -> int:
        """the run of `recs` in any order, sorted into internal-key order and built on the device (pgs_run_build_unsorted): the
        same blocks and run info as build_records of the records sorted first; 0 for no records"""
        rid = C.c_uint64()
        _check(lib().pgs_run_build_unsorted(self.h, level, recs.n, _ptr(recs.keys), _ptr(recs.key_off), _ptr(recs.vals),
                                            _ptr(recs.val_off), _ptr(recs.seq), _ptr(recs.type), C.byref(rid)), "run_build_unsorted")
        return rid.value

    def run_info(self, run_id: int) -> RunInfo:
        info = RunInfo()
        _check(lib().pgs_run_info_get(self.h, run_id, C.byref(info)), "run_info")
        return info

    def runs(self):
        ids = np.zeros(1024, np.uint64)
        n = C.c_uint32()
        _check(lib().pgs_run_list(self.h, ids.ctypes.data_as(u64p), 1024, C.byref(n)), "run_list")
        return [int(x) for x in ids[:n.value]]

    def drop(self, run_id: int):
        _check(lib().pgs_run_drop(self.h, run_id), "run_drop")

    def download(self, run_id: int) -> BlockRun:
        info = self.run_info(run_id)
        data = np.zeros(info.data_bytes, np.uint8)
        off = np.zeros(info.n_blocks, np.uint64)
        size = np.zeros(info.n_blocks, np.uint32)
        _check(lib().pgs_run_download(self.h, run_id, _ptr(data), data.shape[0], _ptr(off), _ptr(size),
                                      info.n_blocks), "run_download")
        return BlockRun(data, off, size)

    def compact(self, run_ids, out_level: int = 1, bottommost: int = -1, now: int = 0, enabled: bool = True,
                default_ttl: int = 0, validate_hash: bool = False, pidx: int = 0, partition_version: int = -1,
                ops: np.ndarray | None = None, data_version: int = 1, flags: int = 0) -> CompactResult:
        ids = np.array(list(run_ids), np.uint64)
        fp = FilterParams()
        fp.enabled = 1 if enabled else 0
        fp.validate_hash = 1 if validate_hash else 0
        fp.data_version = data_version
        fp.default_ttl = default_ttl
        fp.pidx = pidx
        fp.partition_version = partition_version
        if ops is not None and ops.shape[0] >= 4:
            self._ops_keepalive = np.ascontiguousarray(ops)
            fp.ops = self._ops_keepalive.ctypes.data_as(u8p)
            fp.ops_len = self._ops_keepalive.shape[0]
        res = CompactResult()
        _check(lib().pgs_compact_ex(self.h, ids.ctypes.data_as(u64p), ids.shape[0], out_level, bottommost,
                                    C.byref(fp), now, flags, C.byref(res)), "compact")
        return res

    def split(self, src_count: int, dst_count: int, children) -> SplitResult:
        """pgs_partition_split: this partition (index pidx of src_count) into dst_count / src_count children; children[i]
        is the empty Partition pidx + i * src_count of the same engine, or None (child i is not built)"""
        handles = (C.c_void_p * max(1, len(children)))(*[c.h.value if c is not None else None for c in children])
        res = SplitResult()
        _check(lib().pgs_partition_split(self.h, src_count, dst_count, handles, len(children), C.byref(res)), "partition_split")
        return res

    def prefix_scan_batch(self, hashkeys, max_records: int = 1000, arena_stride: int = 32768, alloc=None) -> "ScanBatch":
        """multi_get(hash_key, all sort keys) for many hash keys: the request structs are marshalled once, run() is
        the C-ABI call (pgs_range_scan_many) from host buffers."""
        return ScanBatch(self, hashkeys, max_records, arena_stride, alloc)

    def get_batch(self, keys: np.ndarray, key_off: np.ndarray, now: int, arena_cap: int | None = None, arena=None, results=None):
        n = key_off.shape[0] - 1
        results = (GetResult * n)() if results is None else results
        cap = arena_cap if arena_cap is not None else max(1 << 16, n * 1024)
        arena = np.zeros(cap, np.uint8) if arena is None else arena
        cap = min(cap, arena.shape[0])
        used = C.c_uint64()
        st = lib().pgs_get_batch(self.h, _ptr(keys), _ptr(key_off), n, now, _ptr(arena), cap, results, C.byref(used))
        return st, results, arena, used.value


class ScanBatch:
    def __init__(self, part, hashkeys, max_records: int, arena_stride: int, alloc=None, parts=None, req_part=None):
        """part: one Partition; or parts = a list of partitions of one engine and req_part[i] = the slot of request i
        (pgs_range_scan_many_multi: one launch over all of them)"""
        alloc = alloc or (lambda n, dt: np.zeros(n, dt))  # bench.py passes a pinned-memory allocator
        self.part = part
        self.parts = parts
        if parts is not None:
            self.handles = (C.c_void_p * len(parts))(*[p.h for p in parts])
            self.req_part = np.ascontiguousarray(req_part, np.uint32)
            assert self.req_part.shape[0] == len(hashkeys)
        n = len(hashkeys)
        self.n = n
        self.reqs = (ScanRequest * n)()
        self._keep = []
        for i, hk in enumerate(hashkeys):
            start = len(hk).to_bytes(2, "big") + hk
            stop = bytearray(start)
            while stop[-1] == 0xFF:
                stop.pop()
            stop[-1] += 1
            for name, b in (("start", start), ("stop", bytes(stop))):
                buf = (C.c_uint8 * len(b)).from_buffer_copy(b)
                self._keep.append(buf)
                setattr(self.reqs[i], name, Blob(C.cast(buf, u8p), len(b)))
            q = self.reqs[i]
            q.start_inclusive, q.stop_inclusive, q.key_mode, q.prefix_same_as_start = 1, 0, 1, 1
            q.max_count, q.max_iter_count = max_records, 3000
        self.max_records, self.arena_stride = max_records, arena_stride
        self.arena = alloc(n * arena_stride, np.uint8)
        self.kvs = alloc(n * max_records * 5, np.uint32)
        self.results = (ScanResult * n)()
        self.abase = np.zeros(n + 1, np.uint64)
        self.kbase = np.zeros(n + 1, np.uint32)

    def run(self, now: int) -> int:
        if self.parts is not None:
            return lib().pgs_range_scan_many_multi(self.handles, len(self.parts), self.reqs, _ptr(self.req_part), self.n, now,
                                                   self.arena_stride, self.max_records, _ptr(self.arena), self.arena.shape[0],
                                                   _ptr(self.kvs), self.kvs.shape[0] // 5, None, 0, self.results, _ptr(self.abase),
                                                   _ptr(self.kbase))
        return lib().pgs_range_scan_many(self.part.h, self.reqs, self.n, now, self.arena_stride, self.max_records,
                                         _ptr(self.arena), self.arena.shape[0], _ptr(self.kvs), self.kvs.shape[0] // 5, None, 0,
                                         self.results, _ptr(self.abase), _ptr(self.kbase))

    def records(self, i: int):
        """(sort key, user value) pairs of request i"""
        kv = self.kvs.reshape(-1, 5)
        base = int(self.abase[i])
        out = []
        for j in range(int(self.kbase[i]), int(self.kbase[i + 1])):
            ko, kl, vo, vl, _ = (int(x) for x in kv[j])
            out.append((self.arena[base + ko:base + ko + kl].tobytes(), self.arena[base + vo:base + vo + vl].tobytes()))
        return out
