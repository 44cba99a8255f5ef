/*
 * pegasus_b200.h — C ABI of the GPU-native (H100) LSM read/compaction engine for the Pegasus replica
 * server.  This is the drop-in boundary: everything a reference-side binding (the C++ class
 * that takes RocksDB's place behind `replication_app_base`, or a cgo/JNI stub) needs is declared
 * here with plain pointers and sizes.  No torch / CUDA / C++ types cross it, no exception does.
 *
 * Two layers, both exported by libpegasus_b200.so:
 *
 *   1. pgs_*       the device engine: partitions, HBM-resident sorted runs, compaction,
 *                  batched point lookup, range scan.   (what RocksDB's DB::* calls become)
 *   2. pgs_rrdb_*  the rrdb operator surface of one replica (`pegasus_server_impl`):
 *                  on_get / on_multi_get / on_batch_get / on_sortkey_count / on_ttl /
 *                  on_get_scanner / on_scan / on_clear_scanner / on_put ... with request and
 *                  response structs mirroring idl/rrdb.thrift.
 *
 * Citations are relative to the reference tree (apache/incubator-pegasus):
 *   plugin API ............ src/replica/replication_app_base.h:114-360
 *   read handlers ......... src/server/pegasus_read_service.h:52-85,
 *                           src/server/pegasus_server_impl.cpp:418-1549
 *   write handlers ........ src/server/pegasus_server_write.cpp:92-222,
 *                           src/server/rocksdb_wrapper.cpp:129-246
 *   compaction filter ..... src/server/key_ttl_compaction_filter.h:55-203
 *   manual compaction ..... src/server/pegasus_manual_compact_service.cpp:83-313,
 *                           src/server/pegasus_server_impl.cpp:3373-3456
 *   key / value schema .... src/base/pegasus_key_schema.h:41-183,
 *                           src/base/pegasus_value_schema.h:44-226
 *
 * Error convention (all `int32_t` returns and every `error` field): the integer values of
 * rocksdb::Status::Code, exactly as the reference puts them on the wire
 * (src/include/pegasus/error_def.h:57-69, PERR = -1000 - code).  CUDA faults map to
 * PGS_IO_ERROR, detected data damage to PGS_CORRUPTION.
 */
#ifndef PEGASUS_B200_H_
#define PEGASUS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PGS_API __attribute__((visibility("default")))

/* ---- status codes = rocksdb::Status::Code ------------------------------------------------ */
enum {
    PGS_OK = 0,
    PGS_NOT_FOUND = 1,
    PGS_CORRUPTION = 2,
    PGS_NOT_SUPPORTED = 3,
    PGS_INVALID_ARGUMENT = 4,
    PGS_IO_ERROR = 5,
    PGS_MERGE_IN_PROGRESS = 6,
    PGS_INCOMPLETE = 7,
    PGS_SHUTDOWN_IN_PROGRESS = 8,
    PGS_TIMED_OUT = 9,
    PGS_ABORTED = 10,
    PGS_BUSY = 11,
    PGS_EXPIRED = 12,
    PGS_TRY_AGAIN = 13
};

/* rrdb.thrift filter_type (idl/rrdb.thrift:27-33) */
enum { PGS_FT_NO_FILTER = 0, PGS_FT_MATCH_ANYWHERE = 1, PGS_FT_MATCH_PREFIX = 2, PGS_FT_MATCH_POSTFIX = 3 };

/* internal-key value types, as RocksDB's ValueType (dbformat.h, not in tree) */
enum { PGS_TYPE_DELETION = 0, PGS_TYPE_VALUE = 1 };

typedef struct pgs_engine pgs_engine;       /* one per GPU                                   */
typedef struct pgs_partition pgs_partition; /* one per replica (gpid) = one RocksDB instance */

typedef struct {
    const uint8_t *data;
    uint32_t len;
} pgs_blob;

/* ============================================================================================
 * 1. device engine
 * ========================================================================================== */

typedef struct {
    int32_t device;            /* CUDA ordinal; -1 = current                                  */
    uint32_t block_size;       /* target data block bytes; 0 -> 4096 (RocksDB default, never
                                  overridden by Pegasus: pegasus_server_impl_init.cpp:666-848) */
    uint32_t restart_interval; /* 0 -> 16 (pegasus_server_impl_init.cpp:716-718)              */
    uint32_t ctas_per_sm;      /* unused since round 2 (the walker sizes its own grid); kept for ABI stability              */
    uint32_t flags;            /* reserved and ignored; kept for ABI stability                                              */
} pgs_engine_config;

PGS_API int32_t pgs_engine_open(const pgs_engine_config *cfg, pgs_engine **out);
PGS_API void pgs_engine_close(pgs_engine *e);
/* the CUDA stream (cudaStream_t) every kernel of this engine is launched on; lets a harness
 * record events on it. */
PGS_API void *pgs_engine_stream(pgs_engine *e);
PGS_API int32_t pgs_engine_sync(pgs_engine *e);
/* number of kernels this engine has launched so far */
PGS_API uint64_t pgs_engine_launches(pgs_engine *e);
/* device time (CUDA events on the engine stream) of the kernels of the last pgs_get_batch /
 * pgs_range_scan(_many) call, without the host<->device copies around them */
PGS_API float pgs_engine_last_kernel_ms(pgs_engine *e);
/* data blocks fetched by the calling thread's last pgs_get_batch (one per run probed per key), and the run probes its
 * Bloom filters saved.  (These three getters are per calling thread: readers run concurrently.) */
PGS_API uint64_t pgs_engine_last_blocks_probed(pgs_engine *e);
PGS_API uint64_t pgs_engine_last_runs_skipped(pgs_engine *e);
/* thread-local description of the last failure on the calling thread */
PGS_API const char *pgs_last_error(void);

/* replaces rocksdb::DB::Open for one replica (pegasus_server_impl.cpp:1551-1860) */
PGS_API int32_t pgs_partition_create(pgs_engine *e, int32_t app_id, int32_t pidx,
                                     uint32_t data_version, pgs_partition **out);
PGS_API void pgs_partition_destroy(pgs_partition *p);

typedef struct {
    uint64_t run_id;
    int32_t level;
    uint32_t n_blocks;
    uint64_t n_records;
    uint64_t n_tombstones;
    uint64_t data_bytes;      /* encoded block bytes resident in HBM (incl. 16 B block padding) */
    uint64_t raw_key_bytes;   /* sum of user-key bytes  (SURVEY 8d: algorithmic bytes)          */
    uint64_t raw_value_bytes; /* sum of value bytes                                             */
    uint32_t max_ukey_len;
    uint32_t max_value_len;
    uint32_t max_block_size;
    uint32_t max_block_records;
    uint64_t smallest_seq;
    uint64_t largest_seq;
} pgs_run_info;

/* Install one sorted run (an SST's data blocks) in HBM.  `data` holds `n_blocks` RocksDB-format
 * data blocks (entries `varint shared, varint non_shared, varint value_len, key_delta, value`
 * over internal keys `user_key || fixed64_le(seq<<8|type)`, restart array, restart count; no
 * 5-byte trailer); block i occupies [blk_off[i], blk_off[i]+blk_size[i]) and every blk_off is a
 * multiple of 16.  The device builds its own index (last key, record count per block).
 * level 0: the run becomes the newest L0 run.  level>=1: newest run of that level.
 * Replaces flush / IngestExternalFile (rocksdb_wrapper.cpp:248-270). */
PGS_API int32_t pgs_run_upload(pgs_partition *p, int32_t level, const uint8_t *data,
                               uint64_t data_bytes, const uint64_t *blk_off,
                               const uint32_t *blk_size, uint32_t n_blocks, uint64_t *run_id_out);
/* Several runs in one call, in order (runs[0] is installed first).  The block bytes travel in 32 MB chunks; the device
 * index build of a chunk overlaps the copy of the next one, and the next run's bytes are on the link before the
 * current run's index is finished: with pinned host buffers the call takes the transfer time plus one short tail.
 * All or nothing: on an error no run of the call stays installed. */
typedef struct {
    const uint8_t *data;
    uint64_t data_bytes;
    const uint64_t *blk_off;
    const uint32_t *blk_size;
    uint32_t n_blocks;
    int32_t level;
} pgs_run_src;
PGS_API int32_t pgs_run_upload_many(pgs_partition *p, const pgs_run_src *runs, uint32_t n, uint64_t *run_ids_out);
/* Build one sorted run on the device from n flat records and install it, as the host builder plus pgs_run_upload would:
 * the blocks, their handles and the run's info are byte for byte those of pgs_run_builder_add_many + pgs_run_builder_finish
 * at the engine's block_size / restart_interval followed by pgs_run_upload (only the run id differs).  Records are in
 * internal-key order (user key ascending, then seq<<8|type strictly descending); record i's user key is
 * keys[key_off[i] .. key_off[i+1]), its value vals[val_off[i] .. val_off[i+1]).  Host arrays may be pageable or pinned.
 *   n == 0: PGS_OK, *run_id_out = 0, nothing resident.
 *   out of order (as pgs_run_builder_add returns), or offsets that are not ascending: PGS_INVALID_ARGUMENT.
 *   a user key over 4096 bytes, or a run past the index's 32-bit record / index-key offsets: PGS_NOT_SUPPORTED.
 * All or nothing: on an error the partition's run list is unchanged.
 * The whole input is resident on the device for the duration of the call, with about 4 * ceil(log2 n) + 25 bytes of
 * scratch per record besides. */
PGS_API int32_t pgs_run_build(pgs_partition *p, int32_t level, uint64_t n,
                              const uint8_t *keys, const uint64_t *key_off,
                              const uint8_t *vals, const uint64_t *val_off,
                              const uint64_t *seq, const uint8_t *type,
                              uint64_t *run_id_out);
/* pgs_run_build for n flat records in any order: they are sorted on the device into internal-key order (user keys bytewise as
 * unsigned bytes, a proper prefix first; equal user keys by seq<<8|type descending), then built as pgs_run_build builds.  The
 * installed run (blocks, handles, pgs_run_info) is byte for byte the one pgs_run_build makes from the same records stably sorted
 * into internal-key order; only the run id differs.  Shadowed versions are kept (compaction drops them).
 * Statuses, in this order of precedence:
 *   offsets (key_off / val_off) not ascending: PGS_INVALID_ARGUMENT;
 *   else a user key over 4096 bytes, or n > 0xFFFFFFF0: PGS_NOT_SUPPORTED;
 *   else two records with the same user key, seq and type (a duplicate internal key): PGS_INVALID_ARGUMENT;
 *   else pgs_run_build's statuses.
 *   n == 0: PGS_OK, *run_id_out = 0, nothing resident.
 * All or nothing: on an error the partition's run list is unchanged and every device buffer of the call is freed.
 * Device memory: while sorting, the input (key_off[n] + val_off[n] + 32 bytes, and 25 bytes per record), the sorted copy (the
 * same again) and the sort's scratch (60 bytes per record, plus about 1 KB per 4096 records); while building, the sorted copy,
 * pgs_run_build's scratch (about 4 * ceil(log2 n) + 25 bytes per record) and the run.  The input and the sort's scratch are
 * freed before the build's scratch is taken.
 * Rounds: one per 8 bytes of the longest prefix two user keys share, plus two; each round costs the records still tied. */
PGS_API int32_t pgs_run_build_unsorted(pgs_partition *p, int32_t level, uint64_t n,
                                       const uint8_t *keys, const uint64_t *key_off,
                                       const uint8_t *vals, const uint64_t *val_off,
                                       const uint64_t *seq, const uint8_t *type, uint64_t *run_id_out);
/* device times (ms) of the calling thread's last successful pgs_run_build or pgs_run_build_unsorted: [0] input copy, [1] block
 * plan (record, next-block, chain and scan passes), [2] block writing, [3] index and Bloom filter (the upload's two passes) */
PGS_API void pgs_run_build_last_ms(float *ms4);
/* device time (ms) of the sort and the gather of the sorted copy in the calling thread's last successful pgs_run_build_unsorted
 */
PGS_API float pgs_run_build_last_sort_ms(void);
PGS_API int32_t pgs_run_drop(pgs_partition *p, uint64_t run_id);
PGS_API int32_t pgs_run_info_get(pgs_partition *p, uint64_t run_id, pgs_run_info *out);
/* run ids in read order (newest first: L0 by recency, then L1, L2, ...) */
PGS_API int32_t pgs_run_list(pgs_partition *p, uint64_t *ids, uint32_t cap, uint32_t *n_out);
/* copy a run's raw blocks + handles back to the host (checkpoint / egress / tests) */
PGS_API int32_t pgs_run_download(pgs_partition *p, uint64_t run_id, uint8_t *data,
                                 uint64_t data_cap, uint64_t *blk_off, uint32_t *blk_size,
                                 uint32_t blk_cap);

/* ---- compaction ---------------------------------------------------------------------------
 * KeyWithTTLCompactionFilter snapshot (key_ttl_compaction_filter.h:140-157).  `ops` is the
 * binary form of the `user_specified_compaction` app-env produced by pgs_compaction_ops_parse.
 */
typedef struct {
    uint8_t enabled;       /* Factory::_enabled                                               */
    uint8_t validate_hash; /* replica.split.validate_partition_hash                            */
    uint8_t reserved[2];
    uint32_t data_version;
    uint32_t default_ttl;
    int32_t pidx;
    int32_t partition_version;
    const uint8_t *ops; /* may be NULL; a malformed table: pgs_compact returns PGS_INVALID_ARGUMENT */
    uint32_t ops_len;
} pgs_filter_params;

typedef struct {
    uint64_t new_run_id;
    uint64_t in_records, out_records;
    uint64_t in_bytes;  /* sum(user key + value) over input records  = "merged bytes"          */
    uint64_t out_bytes; /* sum(user key + value) over surviving records                        */
    uint64_t in_block_bytes, out_block_bytes;
    uint64_t dropped_shadowed;  /* older versions of a user key                                */
    uint64_t dropped_tombstone; /* deletions removed at the bottommost level                   */
    uint64_t dropped_expired;   /* Filter(): expire_ts <= now                                  */
    uint64_t dropped_user;      /* Filter(): user-specified delete op                          */
    uint64_t dropped_stale;     /* Filter(): stale split data                                  */
    uint64_t ttl_rewritten;     /* Filter(): value_changed                                     */
    uint32_t n_tiles;      /* segments of the merge                                               */
    uint32_t n_launches;
    float device_ms;       /* CUDA-event time of all compaction kernels                           */
    float merge_kernel_ms; /* k_walk + k_seg_scan + k_emit                                       */
    float walk_ms;         /* k_walk: the merge (decode, compare, filter, layout)                 */
    float emit_ms;         /* k_seg_scan + k_emit: block assembly and stores                      */
    uint32_t reserved;
} pgs_compact_result;

/* k-way merge of `k` runs of one partition into one new run at `out_level`, newest version of
 * each user key wins, tombstones dropped iff `bottommost` (-1 = derive from the partition: true
 * iff no older run stays outside the input set), Filter() fused.  `now` = epoch_now()
 * (pegasus_utils.h:39-41) passed explicitly.  Replaces DB::CompactRange
 * (pegasus_server_impl.cpp:3373-3394) and the background compaction job. */
PGS_API int32_t pgs_compact(pgs_partition *p, const uint64_t *run_ids, uint32_t k,
                            int32_t out_level, int32_t bottommost, const pgs_filter_params *fp,
                            uint32_t now, pgs_compact_result *out);

/* Same with flags.  KEEP_INPUTS leaves the input runs installed, DISCARD_OUTPUT does not install
 * the merged run (its buffers return to the pool): together they let a harness repeat one job. */
#define PGS_COMPACT_KEEP_INPUTS 1u
#define PGS_COMPACT_DISCARD_OUTPUT 2u
PGS_API int32_t pgs_compact_ex(pgs_partition *p, const uint64_t *run_ids, uint32_t k,
                               int32_t out_level, int32_t bottommost, const pgs_filter_params *fp,
                               uint32_t now, uint32_t flags, pgs_compact_result *out);

/* One compaction job of pgs_compact_many: the arguments pgs_compact_ex takes for one partition. */
typedef struct {
    pgs_partition *part;
    const uint64_t *run_ids;     /* the job's input runs, as pgs_compact takes them                 */
    uint32_t k;
    int32_t out_level;
    int32_t bottommost;          /* -1: derived per partition, as pgs_compact derives it            */
    const pgs_filter_params *fp; /* per job: pidx, partition_version, default_ttl, ops ... (may be NULL) */
} pgs_compact_job;
#define PGS_COMPACT_MANY_MAX_JOBS 4096u
/* Compactions of many partitions of one engine in one plan and one set of kernel launches on the engine stream.  Job i is by
 * definition pgs_compact_ex(jobs[i].part, jobs[i].run_ids, jobs[i].k, jobs[i].out_level, jobs[i].bottommost, jobs[i].fp, now,
 * flags, &out[i]): the same records, counters and run info, and the same reads afterwards.  Only the block layout may differ:
 * the segments are sized by the whole launch's weight and every segment starts a block, so block cuts (n_blocks, data_bytes,
 * max_block_size, max_block_records, out_block_bytes) can differ from a pgs_compact of the same job.
 *   launches: six, whatever n is (out[i].n_launches);
 *   out (n entries, may be NULL): out[i] = job i's own counters, run id and n_tiles (its segments); device_ms, merge_kernel_ms,
 *     walk_ms and emit_ms are the call's, repeated in every entry;
 *   installed runs: as pgs_compact, per job (inputs removed, the merged run installed only when non-empty); flags apply to
 *     every job.
 * Statuses, checked before anything is allocated or launched:
 *   jobs == NULL with n > 0, a job without a partition or run ids, k == 0, out_level < 0, a run given twice, the same partition
 *   in two jobs, partitions of different engines, a malformed ops table: PGS_INVALID_ARGUMENT;
 *   an unknown run: PGS_NOT_FOUND;
 *   n > PGS_COMPACT_MANY_MAX_JOBS, a job of more than 16 runs, a user key over 4096 bytes, or jobs whose joint geometry does not
 *   fit one launch (the widest user key of any job sizes the key rows of all of them): PGS_NOT_SUPPORTED -- split the call;
 *   n == 0: PGS_OK, nothing launched.
 * pgs_last_error() names the failing job.  All or nothing: on any error (a device allocation failure is PGS_IO_ERROR) no
 * partition's run list changes.
 * Device memory, all of it allocated before the first launch and held until the call returns: every job's merged run (about
 * its inputs' raw key and value bytes plus 23 bytes per record and 20 per block) and every job's scratch (about 16 +
 * (27 + the launch's widest user key, rounded up to 4) bytes per input record, plus the input blocks of two segments'
 * boundaries), a MergeParams (about 1.8 KB) per job. */
PGS_API int32_t pgs_compact_many(const pgs_compact_job *jobs, uint32_t n, uint32_t now, uint32_t flags,
                                 pgs_compact_result *out);

/* ---- partition split ------------------------------------------------------------------------
 * Splits partition `src` (index pidx of `src_count`) into its dst_count / src_count children on the
 * device.  Child i is partition pidx + i * src_count and receives, for every run of the parent, one
 * run at the same level holding the records with (pegasus_key_hash(key) % dst_count) / src_count == i
 * in the run's order: every version and tombstone with its trailer, values byte-identical, no filter.
 * Records with an empty user key (the empty write) are dropped and counted.  The reference's
 * local_partition_split (src/shell/commands/local_partition_split.cpp:238-283) routes records the
 * same way but refuses runs that hold deletions; here they are split.
 *   dst_count must be src_count * 2^n (n >= 1) and n_dst == dst_count / src_count; dst[i] may be
 *   NULL (child i is not built: the online split, where the parent itself keeps index 0).  Every
 *   other destination belongs to src's engine, has index pidx + i * src_count and no runs:
 *   PGS_INVALID_ARGUMENT otherwise, as for bad counts.  A destination may belong to another app
 *   (local_partition_split writes the children into a new table).  A destination with another
 *   data_version, or more than PGS_SPLIT_MAX_CHILDREN children: PGS_NOT_SUPPORTED.
 *   The parent is never modified.  The children's runs are installed only after every run of every
 *   child was built; on any error no child changes. */
#define PGS_SPLIT_MAX_CHILDREN 32
typedef struct {
    uint64_t records;     /* records of the child's runs                                          */
    uint64_t tombstones;
    uint64_t raw_bytes;   /* sum(user key + value)                                                */
    uint64_t block_bytes; /* encoded blocks                                                       */
    uint32_t runs;        /* runs installed                                                       */
    uint32_t reserved;
} pgs_split_child_result;
typedef struct {
    pgs_split_child_result child[PGS_SPLIT_MAX_CHILDREN];
    uint64_t in_records, in_bytes; /* over the parent's runs (in_bytes = sum(user key + value))  */
    uint64_t dropped_empty;        /* empty writes dropped                                         */
    float device_ms;               /* CUDA-event time from the first launch to the last           */
    float kernel_ms;               /* CUDA-event time of the split's kernels: the sum of the next three */
    float count_ms;                /* planner + counting walk                                      */
    float walk_ms;                 /* writing walk                                                 */
    float emit_ms;                 /* k_seg_scan + k_emit of every child                           */
    uint32_t n_launches;
} pgs_split_result;
PGS_API int32_t pgs_partition_split(pgs_partition *src, uint32_t src_count, uint32_t dst_count,
                                    pgs_partition *const *dst, uint32_t n_dst, pgs_split_result *out);

/* Parse the JSON of the `user_specified_compaction` env (compaction_operation.cpp:162-186) into
 * the binary ops table.  Invalid JSON / rules yield an empty table like the reference.  A pattern
 * longer than 65 535 bytes (it matches no key) is stored as the empty pattern; an op of more than
 * 65 535 rules: -PGS_INVALID_ARGUMENT.  Returns bytes written (<= cap) or a negative status. */
PGS_API int64_t pgs_compaction_ops_parse(const char *json, uint32_t json_len, uint32_t data_version,
                                         uint8_t *out, uint32_t cap, uint32_t *n_ops_out);

/* ---- batched point lookup: DB::Get / DB::MultiGet ------------------------------------------ */
typedef struct {
    int32_t status;     /* PGS_OK | PGS_NOT_FOUND                                             */
    uint32_t expire_ts; /* header field of the found record                                   */
    uint32_t value_off; /* user data (header stripped) inside the arena                       */
    uint32_t value_len;
    uint8_t expired;    /* found but hidden by TTL -> status is PGS_NOT_FOUND                 */
    uint8_t reserved[3];
} pgs_get_result;

/* keys: n raw Pegasus keys back to back, key i = keys[key_off[i] .. key_off[i+1]).
 * Values of found, unexpired records are written to `arena` (host memory).  A record whose
 * value does not fit gets PGS_INCOMPLETE and *arena_used is the total need.  value_off is 32-bit:
 * only the first 4 GiB - 1 bytes of the arena are used, whatever arena_cap says. */
PGS_API int32_t pgs_get_batch(pgs_partition *p, const uint8_t *keys, const uint32_t *key_off,
                              uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap,
                              pgs_get_result *results, uint64_t *arena_used);
/* The same for keys of several partitions of one engine in ONE launch (a batching front end's shape: concurrent handlers of
 * many replicas coalesced; SURVEY 8 f3): key i is looked up in parts[key_part[i]].  Results and arena as above. */
PGS_API int32_t pgs_get_batch_multi(pgs_partition *const *parts, uint32_t n_parts, const uint8_t *keys,
                                    const uint32_t *key_off, const uint32_t *key_part, uint32_t n, uint32_t now,
                                    uint8_t *arena, uint64_t arena_cap, pgs_get_result *results,
                                    uint64_t *arena_used);

/* ---- range scan: NewIterator + Seek + Next/Prev loop --------------------------------------- */
typedef struct {
    pgs_blob start, stop; /* raw keys                                                          */
    uint8_t start_inclusive, stop_inclusive;
    uint8_t reverse;
    uint8_t no_value;
    uint8_t key_mode;         /* 0: return the raw key (scan); 1: sort key only (multi_get)    */
    uint8_t return_expire_ts;
    uint8_t count_only;
    uint8_t validate_hash;    /* request flag && server flag, already combined                 */
    uint8_t prefix_same_as_start; /* ReadOptions of the data CF (pegasus_server_impl_init.cpp:835-840) */
    uint8_t skip_first_exclusive; /* unused: exclusiveness of `start` is start_inclusive        */
    uint8_t reserved[2];          /* reserved[0] = 1: `stop` is an iterate_upper_bound (sortkey_count) */
    int32_t hash_filter_type, sort_filter_type;
    pgs_blob hash_filter, sort_filter;
    uint32_t max_count;      /* loop guard `count < max_count`                                 */
    uint32_t max_iter_count; /* range_read_limiter max_count                                   */
    uint64_t max_iter_size;  /* range_read_limiter max_size, 0 = none                          */
    int32_t pidx, partition_version;
} pgs_scan_request;

typedef struct {
    uint32_t key_off, key_len;
    uint32_t value_off, value_len;
    uint32_t expire_ts;
} pgs_kv;

typedef struct {
    int32_t status;     /* iterator status: PGS_OK or an error                                 */
    uint32_t n_kvs;     /* records returned (= count unless count_only)                        */
    uint32_t count;     /* records in state kNormal                                            */
    uint32_t iter_count, expire_count, filter_count;
    uint64_t size;      /* sum(len(key)+len(value)) of returned records                        */
    uint8_t complete;   /* loop left through the stop key                                      */
    uint8_t iter_valid; /* iterator still valid when the loop ended                            */
    uint8_t reserved[2];
    uint32_t resume_len;/* raw key the iterator stands on (if iter_valid)                      */
    uint64_t arena_used;
} pgs_scan_result;

/* One scan; arena_cap is also its slice on the device, rounded up to 16 bytes.  pgs_kv's offsets are 32-bit, so a slice
 * holds at most 4 GiB - 16 bytes, whatever arena_cap says: an output that passes its slice or kv_cap records gets
 * PGS_ABORTED (retry with more room); an output that fits the slice but not arena_cap gets PGS_INCOMPLETE. */
PGS_API int32_t pgs_range_scan(pgs_partition *p, const pgs_scan_request *req, uint32_t now,
                               uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint32_t kv_cap,
                               uint8_t *resume_key, uint32_t resume_cap, pgs_scan_result *out);

/* Many independent scans in one launch (what a batching front-end in front of the SCAN / LOCAL_APP
 * thread pools submits).  Request i may use up to arena_stride bytes / kv_stride records on the
 * device; the outputs come back packed: request i's records are kvs[kv_base[i] .. kv_base[i+1]),
 * their offsets are relative to arena + arena_base[i] (arena_base / kv_base have n+1 entries),
 * its resume key (if iter_valid) is resume_keys + i*resume_stride.  For n > 1, arena_base[i+1] -
 * arena_base[i] is request i's arena_used rounded up to 16 (the padding bytes are unspecified);
 * for n == 1 it is arena_used.  kv_base is the exclusive prefix of n_kvs.  The device slice is
 * arena_stride rounded up to 16 and at most 4 GiB - 16 bytes (pgs_kv's offsets are 32-bit): an
 * output that passes it or kv_stride records gets PGS_ABORTED.  arena_cap must cover
 * arena_base[n] and kv_cap kv_base[n], or the call returns PGS_INCOMPLETE and leaves arena, kvs,
 * arena_base and kv_base unwritten. */
PGS_API int32_t pgs_range_scan_many(pgs_partition *p, const pgs_scan_request *reqs, uint32_t n,
                                    uint32_t now, uint64_t arena_stride, uint32_t kv_stride,
                                    uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs, uint64_t kv_cap,
                                    uint8_t *resume_keys, uint32_t resume_stride,
                                    pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base);
/* The same for FORWARD scans over several partitions of one engine in ONE launch (SURVEY 8 f3): request i merges the runs of
 * parts[req_part[i]] only.  A reverse request gets PGS_NOT_SUPPORTED (those go through pgs_range_scan_many).  Slices,
 * packing and statuses as for pgs_range_scan_many. */
PGS_API int32_t pgs_range_scan_many_multi(pgs_partition *const *parts, uint32_t n_parts, const pgs_scan_request *reqs,
                                          const uint32_t *req_part, uint32_t n, uint32_t now, uint64_t arena_stride,
                                          uint32_t kv_stride, uint8_t *arena, uint64_t arena_cap, pgs_kv *kvs,
                                          uint64_t kv_cap, uint8_t *resume_keys, uint32_t resume_stride,
                                          pgs_scan_result *results, uint64_t *arena_base, uint32_t *kv_base);

/* ============================================================================================
 * host-side helpers of the product (no device work)
 * ========================================================================================== */

/* pegasus_manual_compact_service.cpp:83-313, the rules only (no device work, no clock of its own): which manual-compaction
 * rule of the env map ("k\0v\0..." pairs as pgs_rrdb_start takes them) fires at now_ms, and with which CompactRange options.
 *   disabled .......... manual_compact.disabled == "true" (:122-145); nothing fires
 *   max_concurrent .... manual_compact.max_concurrent_running_count, INT_MAX when absent or unparsable (:147-166); <= 0: nothing fires
 *   once .............. manual_compact.once.trigger_time (unix seconds, buf2int64, > 0) newer than last_finish_ms / 1000 (:168-184)
 *   periodic .......... manual_compact.periodic.trigger_time = "H:M,H:M,...": some valid time of day t (today_midnight_s + seconds)
 *                       with last_finish_ms < t * 1000 < now_ms (:186-219); checked only when `once` did not fire
 *   options ........... <rule prefix>target_level: -1 or 1..num_levels, else -1; <rule prefix>bottommost_level_compaction:
 *                       "force" -> 1, anything else -> 0 (skip) (:231-272)
 * today_midnight_s: unix seconds of the local day's 00:00:00 (the reference asks localtime; pass -1 to derive it from now_ms). */
typedef struct {
    int32_t rule;                 /* 0 = none, 1 = once, 2 = periodic */
    int32_t disabled;
    int32_t max_concurrent_running_count;
    int32_t target_level;
    int32_t bottommost_force;
    int32_t reserved;
} pgs_manual_compact_decision;
PGS_API int32_t pgs_manual_compact_decide(const char *envs, uint32_t n_envs, uint64_t now_ms,
                                          uint64_t last_finish_ms, int64_t today_midnight_s,
                                          int32_t num_levels, pgs_manual_compact_decision *out);
/* parse_compression_types (pegasus_server_impl.cpp:3019-3060), the `rocksdb_compression_type` setting: "none|snappy|lz4|zstd"
 * compresses levels >= 2 with that type; "per_level:t0,t1,..." names every level, the last type repeats.  per_level[i] gets
 * RocksDB's CompressionType of level i (0 none, 1 snappy, 4 lz4, 7 zstd).  PGS_INVALID_ARGUMENT (and per_level untouched)
 * for anything else.  The SST writer of this library produces types 0 and 4. */
PGS_API int32_t pgs_parse_compression_types(const char *config, uint32_t num_levels, uint8_t *per_level);
/* check_manual_compact_state (:273-289): may a compaction be enqueued now?  1 = yes and *enqueue_ms becomes now_ms; 0 = one is
 * queued / running (*enqueue_ms != 0) or the last one finished less than min_interval_s ago (<= 0: no limit). */
PGS_API int32_t pgs_manual_compact_state_check(uint64_t now_ms, uint64_t last_finish_ms,
                                               int32_t min_interval_s, uint64_t *enqueue_ms);

/* pegasus_key_schema.h:41-98,150-165 */
PGS_API int32_t pgs_generate_key(const uint8_t *hk, uint32_t hk_len, const uint8_t *sk,
                                 uint32_t sk_len, uint8_t *out, uint32_t cap);
PGS_API int32_t pgs_generate_next_blob(const uint8_t *hk, uint32_t hk_len, const uint8_t *sk,
                                       uint32_t sk_len, int32_t with_sort_key, uint8_t *out,
                                       uint32_t cap);
PGS_API uint64_t pgs_key_hash(const uint8_t *raw_key, uint32_t len);
PGS_API uint64_t pgs_crc64(const uint8_t *data, uint64_t len, uint64_t init);

/* Sorted-run builder (the flush side: memtable -> data blocks).  Records must be added in
 * internal-key order (user key ascending, seq descending).  Produces exactly the layout
 * pgs_run_upload takes. */
typedef struct pgs_run_builder pgs_run_builder;
PGS_API pgs_run_builder *pgs_run_builder_new(uint32_t block_size, uint32_t restart_interval);
PGS_API int32_t pgs_run_builder_add(pgs_run_builder *b, const uint8_t *ukey, uint32_t ukey_len,
                                    uint64_t seq, uint8_t type, const uint8_t *value,
                                    uint32_t value_len);
/* bulk variant: n records, key i = keys[key_off[i]..key_off[i+1]), same for values */
PGS_API int32_t pgs_run_builder_add_many(pgs_run_builder *b, uint64_t n, const uint8_t *keys,
                                         const uint64_t *key_off, const uint8_t *vals,
                                         const uint64_t *val_off, const uint64_t *seq,
                                         const uint8_t *type);
PGS_API int32_t pgs_run_builder_finish(pgs_run_builder *b, const uint8_t **data,
                                       uint64_t *data_bytes, const uint64_t **blk_off,
                                       const uint32_t **blk_size, uint32_t *n_blocks);
PGS_API void pgs_run_builder_free(pgs_run_builder *b);

/* Decode raw blocks into flat records (egress / tests).  Two-call protocol: pass NULL outputs
 * to get the sizes. */
typedef struct {
    uint64_t n_records, key_bytes, value_bytes;
} pgs_decode_sizes;
PGS_API int32_t pgs_blocks_decode(const uint8_t *data, const uint64_t *blk_off,
                                  const uint32_t *blk_size, uint32_t n_blocks,
                                  pgs_decode_sizes *sizes, uint8_t *keys, uint64_t *key_off,
                                  uint8_t *vals, uint64_t *val_off, uint64_t *seq, uint8_t *type);

/* ============================================================================================
 * 2. rrdb operator surface of one replica  (pegasus_server_impl)
 * ========================================================================================== */

typedef struct pgs_server pgs_server;

typedef struct {
    /* [pegasus.server] knobs, defaults as pegasus_server_impl_init.cpp:456-511 */
    uint32_t rocksdb_max_iteration_count;          /* 0 -> 1000                               */
    uint32_t rocksdb_multi_get_max_iteration_count;/* 0 -> 3000                               */
    uint64_t rocksdb_multi_get_max_iteration_size; /* 0 -> 30 MB                              */
    uint32_t l0_compaction_trigger;                /* 0 -> 4                                  */
    uint64_t memtable_bytes;                       /* 0 -> 64 MB                              */
    uint8_t prefix_filter;                         /* rocksdb_filter_type == "prefix" (default 1) */
    uint8_t cluster_id;                            /* timetag cluster id, default 1           */
    uint8_t reserved[6];
    /* hot-key detection (hotkey_collector.cpp:38-75); pgs_rrdb_start rejects a bucket count that is not a prime >= 3 */
    uint32_t hotkey_buckets_num;                   /* 0 -> 37                                 */
    uint32_t hot_bucket_variance_threshold;        /* 0 -> 7                                  */
    uint32_t hot_key_variance_threshold;           /* 0 -> 5                                  */
    uint32_t max_seconds_to_detect_hotkey;         /* 0 -> 150                                */
} pgs_server_options;

/* replication_app_base::open/start: creates the partition on `e`, data version 1
 * (pegasus_server_impl_test.cpp:356-360). envs = "k1\0v1\0k2\0v2\0..." (n_envs pairs), the
 * app envs of replication_app_base.cpp:216-245. */
PGS_API int32_t pgs_rrdb_start(pgs_engine *e, int32_t app_id, int32_t pidx,
                               const pgs_server_options *opt, const char *envs, uint32_t n_envs,
                               pgs_server **out);
PGS_API void pgs_rrdb_stop(pgs_server *s);
PGS_API pgs_partition *pgs_rrdb_partition(pgs_server *s);
/* update_app_envs (pegasus_server_impl.cpp:2728-2741): default_ttl,
 * replica.split.validate_partition_hash, user_specified_compaction, manual_compact.* */
PGS_API int32_t pgs_rrdb_update_app_envs(pgs_server *s, const char *envs, uint32_t n_envs,
                                         uint32_t now);
PGS_API void pgs_rrdb_set_partition_version(pgs_server *s, int32_t partition_version);

/* responses own their bytes inside the server handle's response object */
typedef struct {
    int32_t error, app_id, partition_index;
    int32_t ttl_seconds;       /* on_ttl                                                      */
    int64_t count;             /* on_sortkey_count                                            */
    int64_t context_id;        /* scan                                                        */
    int32_t kv_count;          /* only_return_count (-1 = unset)                              */
    uint32_t n_kvs;
    const pgs_kv *kvs;         /* key/value offsets into arena                                */
    const uint32_t *hk_len;    /* batch_get: hash-key length of kvs[i].key (hk||sk)           */
    const uint8_t *arena;
    uint64_t arena_len;
    uint32_t iteration_count, expire_count, filter_count;
} pgs_response;

typedef struct pgs_response_buf pgs_response_buf; /* reusable response storage */
PGS_API pgs_response_buf *pgs_response_new(void);
PGS_API void pgs_response_free(pgs_response_buf *r);
PGS_API const pgs_response *pgs_response_view(pgs_response_buf *r);

typedef struct {
    pgs_blob hash_key;
    const pgs_blob *sort_keys;
    uint32_t n_sort_keys;
    int32_t max_kv_count, max_kv_size;
    uint8_t no_value, start_inclusive, stop_inclusive, reverse;
    pgs_blob start_sortkey, stop_sortkey;
    int32_t sort_key_filter_type;
    pgs_blob sort_key_filter_pattern;
} pgs_multi_get_request; /* idl/rrdb.thrift multi_get_request */

typedef struct {
    pgs_blob start_key, stop_key;
    uint8_t start_inclusive, stop_inclusive, no_value;
    uint8_t validate_partition_hash; /* default true when unset                               */
    uint8_t return_expire_ts, full_scan, only_return_count, reserved;
    int32_t batch_size;
    int32_t hash_key_filter_type;
    pgs_blob hash_key_filter_pattern;
    int32_t sort_key_filter_type;
    pgs_blob sort_key_filter_pattern;
} pgs_get_scanner_request; /* idl/rrdb.thrift get_scanner_request */

typedef struct {
    pgs_blob hash_key, sort_key;
} pgs_full_key;

/* read handlers (pegasus_read_service.h:52-68); `now` = epoch_now() made explicit */
PGS_API int32_t pgs_rrdb_get(pgs_server *s, pgs_blob raw_key, uint32_t now, pgs_response_buf *r);
PGS_API int32_t pgs_rrdb_ttl(pgs_server *s, pgs_blob raw_key, uint32_t now, pgs_response_buf *r);
PGS_API int32_t pgs_rrdb_multi_get(pgs_server *s, const pgs_multi_get_request *q, uint32_t now,
                                   pgs_response_buf *r);
PGS_API int32_t pgs_rrdb_batch_get(pgs_server *s, const pgs_full_key *keys, uint32_t n,
                                   uint32_t now, pgs_response_buf *r);
PGS_API int32_t pgs_rrdb_sortkey_count(pgs_server *s, pgs_blob hash_key, uint32_t now,
                                       pgs_response_buf *r);
PGS_API int32_t pgs_rrdb_get_scanner(pgs_server *s, const pgs_get_scanner_request *q,
                                     uint32_t now, pgs_response_buf *r);
PGS_API int32_t pgs_rrdb_scan(pgs_server *s, int64_t context_id, uint32_t now,
                              pgs_response_buf *r);
PGS_API void pgs_rrdb_clear_scanner(pgs_server *s, int64_t context_id);

/* many independent `get`s in one launch: what a batching front-end in front of the LOCAL_APP
 * thread pool would call. results[i].status / value in arena as pgs_get_batch. */
PGS_API int32_t pgs_rrdb_get_many(pgs_server *s, const uint8_t *keys, const uint32_t *key_off,
                                  uint32_t n, uint32_t now, uint8_t *arena, uint64_t arena_cap,
                                  pgs_get_result *results, uint64_t *arena_used);

/* write handlers -> memtable (pegasus_server_write.cpp:151-222, rocksdb_wrapper.cpp:129-219).
 * `decree` / `timestamp_us` are the mutation's; expire_ts_seconds as update_request.  Every write carries `now`
 * (epoch_now): a write that fills the memtable flushes it and may start the L0 compaction, whose filter needs the clock. */
PGS_API int32_t pgs_rrdb_put(pgs_server *s, pgs_blob raw_key, pgs_blob user_value,
                             uint32_t expire_ts_seconds, int64_t decree, uint64_t timestamp_us,
                             uint32_t now);
PGS_API int32_t pgs_rrdb_remove(pgs_server *s, pgs_blob raw_key, int64_t decree, uint32_t now);
/* on_batched_write_requests (src/server/pegasus_server_write.cpp:92-222): one decree's worth of batchable writes -- single puts
 * and removes -- applied as one batch by the replica's single writer.  count == 0 is RPC_REPLICATION_WRITE_EMPTY: an empty
 * record that only advances the decree.  The return value is the apply status the replication layer sees (kOk unless the
 * storage failed; an unknown operation is kInvalidArgument and nothing is applied); resp_errors[i] is what request i's client
 * sees.  The non-batchable writes (multi_put, multi_remove, incr, check_and_set, check_and_mutate) arrive alone in their
 * decree, as in the reference (`count == 1` is CHECKed there), through their own entry points: for pgs_rrdb_multi_put /
 * _multi_remove the return value is the *response* error (kInvalidArgument for an empty list, after the empty record was
 * written) and the apply status is kOk whenever the return is not a storage error (kIOError / kCorruption). */
typedef struct {
    uint32_t op; /* 0 = RPC_RRDB_RRDB_PUT, 1 = RPC_RRDB_RRDB_REMOVE */
    pgs_blob raw_key;
    pgs_blob value;              /* PUT: user data */
    uint32_t expire_ts_seconds;  /* PUT */
} pgs_write_request;
PGS_API int32_t pgs_rrdb_on_batched_writes(pgs_server *s, const pgs_write_request *reqs, uint32_t count, int64_t decree,
                                           uint64_t timestamp_us, uint32_t now, int32_t *resp_errors);
/* incr (pegasus_write_service_impl.h:264-342; RPC_RRDB_RRDB_INCR): read-before-write on the replica's single writer.  Absent,
 * expired or empty base = 0; a non-integer base or an int64 overflow is reported in *resp_error (kInvalidArgument, *new_value =
 * the old value on overflow) while the call still returns kOk and writes an empty record for the decree, as the reference
 * does.  expire_ts_seconds: 0 keeps the record's expiry, < 0 clears it, > 0 sets it. */
PGS_API int32_t pgs_rrdb_incr(pgs_server *s, pgs_blob raw_key, int64_t increment, int32_t expire_ts_seconds,
                              int64_t decree, uint64_t timestamp_us, uint32_t now, int32_t *resp_error,
                              int64_t *new_value);
/* check_and_set / check_and_mutate (pegasus_write_service_impl.h:436-530, 710-840; RPC_RRDB_RRDB_CHECK_AND_SET / _MUTATE): the
 * value of (hash_key, check_sort_key) is read, validate_check (:1144-1270) compares it with check_operand by check_type
 * (rrdb.thrift cas_check_type 0..17), and only if the check passes the writes are applied.  The call returns kOk whenever the
 * storage worked; res->error carries what the client sees: kOk, kTryAgain (check failed), kInvalidArgument (unsupported check
 * type / empty or bad mutate list / a value that is not an int64 for the integer compares).  A failed request still writes an
 * empty record so that the decree advances.  The checked value comes back in check_value_out (res->check_value_len = its full
 * length) when return_check_value is set. */
typedef struct {
    uint32_t operation; /* 0 = MO_PUT, 1 = MO_DELETE */
    pgs_blob sort_key;
    pgs_blob value;
    int32_t set_expire_ts_seconds;
} pgs_mutate;
typedef struct {
    pgs_blob hash_key, check_sort_key;
    int32_t check_type;
    pgs_blob check_operand;
    const pgs_mutate *mutate_list;
    uint32_t n_mutate;
    uint8_t return_check_value;
} pgs_check_and_mutate_request;
typedef struct {
    pgs_blob hash_key, check_sort_key;
    int32_t check_type;
    pgs_blob check_operand;
    uint8_t set_diff_sort_key; /* 0: the set goes to check_sort_key */
    pgs_blob set_sort_key, set_value;
    int32_t set_expire_ts_seconds;
    uint8_t return_check_value;
} pgs_check_and_set_request;
typedef struct {
    int32_t error;
    uint8_t check_value_returned, check_value_exist, reserved[2];
    uint32_t check_value_len;
} pgs_cas_result;
PGS_API int32_t pgs_rrdb_check_and_set(pgs_server *s, const pgs_check_and_set_request *req, int64_t decree,
                                       uint64_t timestamp_us, uint32_t now, pgs_cas_result *res,
                                       uint8_t *check_value_out, uint32_t check_value_cap);
PGS_API int32_t pgs_rrdb_check_and_mutate(pgs_server *s, const pgs_check_and_mutate_request *req, int64_t decree,
                                          uint64_t timestamp_us, uint32_t now, pgs_cas_result *res,
                                          uint8_t *check_value_out, uint32_t check_value_cap);
PGS_API int32_t pgs_rrdb_multi_put(pgs_server *s, pgs_blob hash_key, const pgs_blob *sort_keys,
                                   const pgs_blob *values, uint32_t n, uint32_t expire_ts_seconds,
                                   int64_t decree, uint64_t timestamp_us, uint32_t now);
PGS_API int32_t pgs_rrdb_multi_remove(pgs_server *s, pgs_blob hash_key, const pgs_blob *sort_keys,
                                      uint32_t n, int64_t decree, int64_t *count, uint32_t now);
/* flush_all_family_columns (pegasus_server_impl.cpp:3471): memtable -> L0 run in HBM, then the
 * L0 trigger check (L0 count >= trigger -> L0(+L1) -> L1 compaction with the filter at `now`).
 * `now` (epoch_now) also feeds the default-TTL substitution of puts (rocksdb_wrapper.cpp:280-288). */
PGS_API int32_t pgs_rrdb_flush(pgs_server *s, uint32_t now);
/* do_manual_compact (pegasus_server_impl.cpp:3373-3456): whole-CF CompactRange, bottommost
 * level forced. */
PGS_API int32_t pgs_rrdb_manual_compact(pgs_server *s, uint32_t now, pgs_compact_result *out);
/* pgs_rrdb_manual_compact of n replicas of one engine, the merges in one pgs_compact_many: every replica's memtable is
 * flushed, a stack deeper than 16 runs folded first, then its whole run list merged at the deepest level present (at least
 * 1), bottommost forced, and manual_compact_last_finish_ms set.  The replicas' writer locks are taken in address order and
 * held until the runs are installed.  out: n entries (may be NULL), replica i's result.  Replicas on different engines, or
 * one given twice: PGS_INVALID_ARGUMENT.  If the joint merge fails no replica's runs change; a memtable already flushed
 * stays flushed and a deep stack already folded stays folded, as with pgs_rrdb_manual_compact. */
PGS_API int32_t pgs_rrdb_manual_compact_many(pgs_server *const *servers, uint32_t n, uint32_t now,
                                             pgs_compact_result *out);
/* last_flushed_decree: the newest decree whose data lives in an HBM run (advanced by a memtable flush, like the decree the
 * reference persists in the SST meta CF); last_committed_decree: the newest decree applied to the memtable.  Nothing here is
 * durable across a process crash (no WAL / checkpoint yet: SURVEY 8 f4), so neither may drive replication-log GC. */
/* Partition split of a replica (the online split manager's copy_checkpoint_to_dir(flush = true) +
 * storage_apply_checkpoint, replica_split_manager.cpp:278, and local_partition_split): under the
 * parent's writer lock its memtable is flushed and its runs are snapshotted; the snapshot's
 * last_flushed_decree is the split's decree (*decree_out).  The parent then takes reads and writes
 * again while pgs_partition_split builds the children from the snapshot.  children[i] (n of them,
 * n == dst_count / src_count, NULL: not built) is a started, empty replica (no runs, empty memtable,
 * decree 0) of index parent.pidx + i * src_count on the parent's engine.  On success each child holds
 * its share of the snapshot, last_seq = the parent's (new writes win over copied versions),
 * committed and flushed decree = the split's decree, durable decree 0, and the parent's
 * manual_compact_last_finish_ms.  Errors as pgs_partition_split's; on an error no child changes. */
PGS_API int32_t pgs_rrdb_split(pgs_server *parent, uint32_t src_count, uint32_t dst_count,
                               pgs_server *const *children, uint32_t n, int64_t *decree_out);
PGS_API int64_t pgs_rrdb_last_flushed_decree(pgs_server *s);
PGS_API int64_t pgs_rrdb_last_committed_decree(pgs_server *s);
/* Checkpoints (first slice of SURVEY 8 f4; sync_checkpoint / storage_apply_checkpoint, pegasus_server_impl.cpp:1951-2336).
 * pgs_rrdb_sync_checkpoint flushes the memtable and writes every resident run as a BlockBasedTable file (section 8; LZ4 for
 * levels >= 2 like the reference's per-level compression) plus a MANIFEST (levels, file names, decree, sequence number,
 * data version) into `dir`/checkpoint.<last_flushed_decree>, the reference's directory naming; the decree becomes the
 * replica's last_durable_decree.  pgs_rrdb_apply_checkpoint replaces the replica's state (runs, memtable, scan contexts,
 * decrees) with that of a checkpoint directory: what learn / restore do.  Checkpoint files are plain SST images: a RocksDB
 * replica's uncompressed or LZ4 files of the same format version ingest the same way (pgs_sst_ingest). */
PGS_API int32_t pgs_rrdb_sync_checkpoint(pgs_server *s, const char *dir, uint32_t now, int64_t *decree_out);
PGS_API int64_t pgs_rrdb_last_durable_decree(pgs_server *s);
PGS_API int32_t pgs_rrdb_apply_checkpoint(pgs_server *s, const char *checkpoint_dir);
/* drops scan contexts older than 5 minutes (pegasus_server_impl.cpp:1377-1385 schedules the same expiry per context);
 * also runs implicitly on every scanner call. Returns the number of contexts dropped. */
PGS_API uint32_t pgs_rrdb_gc(pgs_server *s, uint32_t now);

/* on_detect_hotkey (pegasus_server_impl.cpp:3544-3566, hotkey_collector.cpp): the READ and WRITE hot-key collectors of the
 * replica.  START moves a STOPPED collector to COARSE_DETECTING; STOP clears it; QUERY returns the hot hash key once the
 * collector is FINISHED.  Returns a PGS_HOTKEY_ outcome; result_buf receives up to cap bytes of the hint, or of the hot hash
 * key of a successful QUERY, and *result_len its whole length.  Captures follow capacity_unit_calculator.cpp:158-403: reads
 * answered by the memtable and the handlers' own weights on the host, the misses of batched gets on the device
 * (k_hotkey_capture, next to k_get, only while the READ collector is active); scans capture nothing.  The collectors live on
 * the replica's partition, so pgs_get_batch / pgs_get_batch_multi / pgs_batcher_get on pgs_rrdb_partition(s) capture too. */
enum { PGS_HOTKEY_READ = 0, PGS_HOTKEY_WRITE = 1 };
enum { PGS_HOTKEY_START = 0, PGS_HOTKEY_STOP = 1, PGS_HOTKEY_QUERY = 2 };
enum { PGS_HOTKEY_OK = 0, PGS_HOTKEY_BUSY = 1, PGS_HOTKEY_INVALID_STATE = 2, PGS_HOTKEY_INVALID_PARAMETERS = 3 };
enum { PGS_HOTKEY_STOPPED = 0, PGS_HOTKEY_COARSE_DETECTING = 1, PGS_HOTKEY_FINE_DETECTING = 2, PGS_HOTKEY_FINISHED = 3 };
PGS_API int32_t pgs_rrdb_detect_hotkey(pgs_server *s, int32_t type, int32_t action, uint32_t now_s, char *result_buf,
                                       uint32_t cap, uint32_t *result_len);
/* one analysis step of both collectors at now_s (hotkey_collector::analyse_data); the library owns no threads, so the
 * binding calls it every hotkey_analyse_time_interval_s (10 s), like pgs_rrdb_gc.  Returns a status code. */
PGS_API int32_t pgs_rrdb_hotkey_analyse(pgs_server *s, uint32_t now_s);
/* a collector's PGS_HOTKEY_ state (-1: invalid type) */
PGS_API int32_t pgs_rrdb_hotkey_state(pgs_server *s, int32_t type);

/* ============================================================================================
 * 7. box-level placement: one engine per visible GPU
 * ==========================================================================================
 * A table is hash-partitioned and its replicas are independent (src/client/partition_resolver.cpp:48-51 picks
 * pidx = pegasus_key_hash(key) % partition_count; src/replica/replica_stub.h hosts one storage engine per gpid).
 * The router opens an engine on each of the first n_devices GPUs (0 = all visible) with the same configuration
 * (cfg->device is ignored) and pins replica (app_id, pidx) to GPU pidx % n.  No collective, no peer traffic. */
typedef struct pgs_router pgs_router;
PGS_API int32_t pgs_router_open(const pgs_engine_config *cfg, int32_t n_devices, pgs_router **out);
PGS_API void pgs_router_close(pgs_router *r); /* closes its engines: close their partitions / servers first */
PGS_API int32_t pgs_router_device_count(const pgs_router *r);
PGS_API int32_t pgs_router_device_for(const pgs_router *r, int32_t app_id, int32_t pidx); /* -1: no such */
PGS_API pgs_engine *pgs_router_engine_for(pgs_router *r, int32_t app_id, int32_t pidx);
/* pegasus_key_hash(hash_key, sort_key) % partition_count (src/base/pegasus_key_schema.h:150-165): the client-side half */
PGS_API uint32_t pgs_partition_index(const uint8_t *hash_key, uint32_t hash_key_len, const uint8_t *sort_key,
                                     uint32_t sort_key_len, uint32_t partition_count);

/* ============================================================================================
 * 8. BlockBasedTable images (SST egress + ingest), first slice
 * ==========================================================================================
 * format_version 2, no compression: data blocks with 5-byte trailers (type 0 + masked crc32c), legacy full Bloom
 * filter block (10 bits/key, whole user keys + HashkeyTransform prefixes), properties, metaindex, kBinarySearch index
 * with full internal keys, 53-byte footer.  What a replica writes for L0/L1 and what rocksdb_wrapper.cpp:248-270
 * (IngestExternalFile) reads.  Layout from RocksDB's public format description (SURVEY.md Appendix A): not yet
 * checked against a RocksDB build.  Compressed blocks / other format versions answer PGS_NOT_SUPPORTED.
 * The encode / decode pair works on host block runs (the layout of pgs_run_upload / pgs_run_download); export / ingest
 * wrap them around a resident run.  PGS_INCOMPLETE: the output did not fit, *out_size / *data_bytes / *n_blocks say
 * what is needed. */
PGS_API int32_t pgs_sst_encode(const uint8_t *data, const uint64_t *blk_off, const uint32_t *blk_size,
                               uint32_t n_blocks, uint8_t *out, uint64_t out_cap, uint64_t *out_size);
PGS_API int32_t pgs_sst_decode(const uint8_t *sst, uint64_t size, uint8_t *data, uint64_t data_cap,
                               uint64_t *blk_off, uint32_t *blk_size, uint32_t blk_cap, uint64_t *data_bytes,
                               uint32_t *n_blocks);
/* 1 / 0: the file's Bloom filter may contain / excludes `key` (a user key or a HashkeyTransform prefix); < 0: -status */
PGS_API int32_t pgs_sst_filter_may_match(const uint8_t *sst, uint64_t size, const uint8_t *key, uint32_t key_len);
PGS_API int32_t pgs_sst_export(pgs_partition *p, uint64_t run_id, uint8_t *out, uint64_t out_cap, uint64_t *out_size);
PGS_API int32_t pgs_sst_ingest(pgs_partition *p, int32_t level, const uint8_t *sst, uint64_t size, uint64_t *run_id_out);
/* compression: 0 = none, 4 = LZ4 (kLZ4Compression; what Pegasus configures for levels >= 2, pegasus_server_impl.cpp:3040-3056).
 * Data blocks are stored compressed when that saves 12.5 %; compress_format_version 2 (varint32 raw size | LZ4 block).
 * pgs_sst_decode / pgs_sst_ingest read either kind. */
PGS_API int32_t pgs_sst_encode_ex(const uint8_t *data, const uint64_t *blk_off, const uint32_t *blk_size,
                                  uint32_t n_blocks, uint32_t compression, uint8_t *out, uint64_t out_cap,
                                  uint64_t *out_size);
PGS_API int32_t pgs_sst_export_ex(pgs_partition *p, uint64_t run_id, uint32_t compression, uint8_t *out,
                                  uint64_t out_cap, uint64_t *out_size);
/* the raw LZ4 block codec used above (decompress: out_cap must be the exact raw size) */
PGS_API int32_t pgs_lz4_block(int32_t decompress, const uint8_t *in, uint64_t n, uint8_t *out, uint64_t out_cap,
                              uint64_t *out_size);
PGS_API uint32_t pgs_crc32c(const uint8_t *data, uint64_t len, uint32_t init);

/* ============================================================================================
 * 9. request-batching front end for point reads (SURVEY 8 f3), first slice
 * ========================================================================================== */
/* The read handlers of the reference run one blocking call per RPC on a thread pool (THREAD_POOL_LOCAL_APP,
 * src/server/config.ini:140-150; on_get pegasus_server_impl.cpp:418-494).  A batcher lets the calls of many threads over the
 * replicas `parts` (one engine) share launches: the first caller of a window waits up to max_wait_us for company (or until
 * max_batch requests are queued; 0 = 4096), then everything queued goes through ONE pgs_get_batch_multi launch; callers that
 * arrive meanwhile form the next window.  max_wait_us = 0: no waiting, a lone caller launches at once.
 * pgs_batcher_get blocks until the request's window is done: *result as pgs_get_batch fills it (status PGS_OK / PGS_NOT_FOUND
 * with `expired`, expire_ts, value_len); the value is copied to `value`; a value longer than value_cap gives status
 * PGS_INCOMPLETE with value_len = the need.  The return value is the launch's own status (PGS_OK unless the engine failed).
 * Close only when no call is in flight.  Answers come from the device only (the memtable-aware path is pgs_rrdb_get_many). */
typedef struct pgs_batcher pgs_batcher;
PGS_API int32_t pgs_batcher_open(pgs_partition *const *parts, uint32_t n_parts, uint32_t max_batch,
                                 uint32_t max_wait_us, pgs_batcher **out);
PGS_API void pgs_batcher_close(pgs_batcher *b);
PGS_API int32_t pgs_batcher_get(pgs_batcher *b, uint32_t part_slot, const uint8_t *key, uint32_t key_len,
                                uint32_t now, uint8_t *value, uint32_t value_cap, pgs_get_result *result);
/* requests served and launches made so far */
PGS_API void pgs_batcher_stats(pgs_batcher *b, uint64_t *requests, uint64_t *launches);

#ifdef __cplusplus
}
#endif
#endif /* PEGASUS_B200_H_ */
