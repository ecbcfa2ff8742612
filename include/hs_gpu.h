/*
 * hs_gpu.h -- C ABI of the H100-native covering-index engine (libhs_gpu.so).
 *
 * The reference (microsoft/hyperspace, Scala on the JVM) has no FFI boundary: its whole data path is three
 * Spark calls.  This header is the seam a maintainer binds with JNI / ctypes (see INTEGRATION.md); each entry
 * point names the reference interface whose body it replaces.  Paths below are relative to
 * src/main/scala/com/microsoft/hyperspace/ in the reference.
 *
 * Conventions: plain pointers and sizes only; strings are UTF-8, caller-owned, copied before return; every
 * function returns 0 on success or a negative HS_E* code and writes a message into (err, errlen) when non-NULL.
 * The library owns all device memory and every handle it returns until the matching *_free call.  There is no
 * CPU fallback: without a CUDA device hs_init fails with HS_ENODEVICE and nothing else can be called.
 * One hs_ctx drives one GPU: a main stream for the kernels plus one copy stream per direction for the staged / asynchronous
 * entry points; use one ctx per host thread / per rank.
 *
 * Environment switches (diagnostics and A/B measurements only; results are identical either way):
 *   HS_NO_CARRY=1      decode dictionary-encoded included columns to values instead of carrying 16-bit codes
 *                      (on several GPUs all ranks must agree)
 *   HS_LSD_SORT=1      sort the first key column with LSD passes over its high bytes + tie fix-up instead of the
 *                      shared-memory local sort (directly, or after one MSD pass)
 *   HS_NO_ZEROCOPY=1   decode aligned PLAIN pages into column arrays instead of reading them in place
 *   HS_IO_THREADS=n   host threads that read source files / write bucket files (default 16, at most half the cores)
 *   HS_TIMELINE=1      print the event timeline (H2D / build / D2H begin and end) of every staged or asynchronous call
 */
#ifndef HS_GPU_H
#define HS_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HS_ABI_VERSION 1

/* error codes */
#define HS_OK 0
#define HS_EINVAL (-1)       /* bad argument / unknown column / unsupported configuration */
#define HS_ENODEVICE (-2)    /* no CUDA device or CUDA runtime failure at init */
#define HS_ECUDA (-3)        /* CUDA error during execution */
#define HS_EFORMAT (-4)      /* malformed or unsupported Parquet input */
#define HS_EIO (-5)          /* file system error */
#define HS_EUNSUPPORTED (-6) /* valid input the GPU path does not handle yet (no CPU fallback exists) */
#define HS_ENOMEM (-7)
#define HS_ECOMM (-8)        /* NCCL / multi-GPU exchange failure */

/* physical column types (Parquet physical type x Spark SQL type actually supported on the GPU path) */
#define HS_TYPE_INT32 0  /* Spark int / date            */
#define HS_TYPE_INT64 1  /* Spark long / timestamp(us)  */
#define HS_TYPE_FLOAT 2
#define HS_TYPE_DOUBLE 3
#define HS_TYPE_BOOL 4   /* Spark boolean, one byte (0 / 1) per row: included columns of an index (written as PLAIN BOOLEAN
                            pages, bit-packed), projected columns of scans and joins; sources PLAIN or RLE.  Never an
                            indexed column (HS_EUNSUPPORTED before any source is decoded), a filter or a join key */
#define HS_TYPE_STRING 5 /* BYTE_ARRAY (Spark string / binary): indexed and included columns (one GPU), filter scan keys and
                            predicates, join keys (alone or with other key columns); compared in UTF8String byte order */
#define HS_TYPE_DECIMAL 6 /* hs_predicate literal only: a decimal, unscaled value in lo_i / hi_i, scale in `scale` */
#define HS_TYPE_DATE 7      /* hs_expr_node literal only: a date, days since the epoch in value_i */
#define HS_TYPE_TIMESTAMP 8 /* hs_expr_node literal only: a timestamp, microseconds since the epoch in value_i */

/* Spark timestamps and decimals.  Columns keep an int32 / int64 storage type; their Spark type comes from the Parquet
 * converted / logical type:
 *   TimestampType (INT96, INT64 TIMESTAMP_MICROS, INT64 TIMESTAMP_MILLIS): HS_TYPE_INT64, microseconds since the epoch
 *     (DateTimeUtils.fromJulianDay for INT96; millis x 1000); index files store INT64 TIMESTAMP_MICROS.  An INT96 value
 *     before 1900-01-01T00:00:00Z, millis whose micros overflow, and TIMESTAMP(NANOS) are HS_EUNSUPPORTED, as Spark 3.1
 *     refuses them.
 *   DecimalType(p, s), p <= 18 (INT32, INT64 or FIXED_LEN_BYTE_ARRAY): the unscaled value, HS_TYPE_INT32 for p <= 9 and
 *     HS_TYPE_INT64 above; index files store INT32 / INT64 DECIMAL(p, s).  Bucketed as Spark's Murmur3Hash does: hashLong
 *     of the unscaled value at every precision.  p > 18: HS_EUNSUPPORTED.
 * Result columns (hs_batch_column) come back as stored: int64 micros, int32 / int64 unscaled values; the caller knows the
 * schema. */

typedef struct hs_ctx hs_ctx;
typedef struct hs_index_result hs_index_result;
typedef struct hs_batch hs_batch;

/* ------------------------------------------------------------------------------------------------------------
 * Context
 * ---------------------------------------------------------------------------------------------------------- */

/* ABI version of the loaded library (== HS_ABI_VERSION it was built with). */
int hs_abi_version(void);
/* Static description: compile arch, CUDA version, build flags. */
const char* hs_build_info(void);

/* Create a context on CUDA device `device_id`.  `cuda_stream` may be NULL (the library creates its own
 * non-blocking stream) or a cudaStream_t owned by the caller (e.g. torch's current stream) on which every kernel
 * and copy of this ctx is then issued.  Replaces: the Spark executor pool a Hyperspace action runs on
 * (actions/Action.scala:84-105 runs op() on the driver thread; Spark schedules the tasks). */
int hs_init(int device_id, void* cuda_stream, hs_ctx** out, char* err, size_t errlen);
void hs_shutdown(hs_ctx* ctx);
/* Return cached device/pinned buffers to the driver. */
void hs_trim(hs_ctx* ctx);
/* Per-kernel timing: when enabled, the hot kernels are bracketed with CUDA events on the ctx stream; hs_profile_report
 * writes a JSON object {"kernel": {"launches": n, "ms": total}} covering the calls since the last report and resets
 * it.  Used by bench.py for the roofline of the dominant kernel.  k_range_bounds also reports "items": the (sorted file,
 * key range) work items it searched, one per window of the filter scans' key. */
void hs_profile_enable(hs_ctx* ctx, int on);
int hs_profile_report(hs_ctx* ctx, char* out_json, size_t outlen);
/* Page-locked host memory for file images handed to hs_create_index (a JNI direct ByteBuffer can wrap it); pageable
 * memory works too but copies at a fraction of the PCIe rate. */
void* hs_host_alloc(hs_ctx* ctx, size_t bytes);
void hs_host_free(hs_ctx* ctx, void* p);

/* Multi-GPU (one process per GPU).  Rank 0 calls hs_comm_unique_id and ships the 128 bytes to the other ranks
 * out of band; every rank then calls hs_comm_init.  Replaces: Spark's shuffle service behind
 * `indexData.repartition(numBuckets, indexedColumns)` (index/covering/CoveringIndex.scala:60). */
int hs_comm_unique_id(void* out_id128, char* err, size_t errlen);
int hs_comm_init(hs_ctx* ctx, int rank, int world_size, const void* id128, char* err, size_t errlen);

/* ------------------------------------------------------------------------------------------------------------
 * Write side: createIndex / refreshIndex(full|incremental) / optimizeIndex data path
 * ---------------------------------------------------------------------------------------------------------- */

typedef struct {
  const char* path;  /* read from the file system when data == NULL */
  const void* data;  /* whole Parquet file image; host memory, or device memory when on_device != 0
                        (device images must be 16-byte aligned) */
  uint64_t size;     /* image size in bytes (ignored when data == NULL) */
  int64_t file_id;   /* lineage id from FileIdTracker (index/IndexLogEntry.scala:627-703); -1 when lineage is off */
  int32_t on_device;
  int32_t reserved;
} hs_source_file;

#define HS_SAVE_OVERWRITE 0 /* create / refresh full / optimize  (covering/CoveringIndexTrait.scala:45-47) */
#define HS_SAVE_APPEND 1    /* incremental refresh into an existing version dir (CoveringIndexTrait.scala:87-93) */

#define HS_CODEC_UNCOMPRESSED 0
#define HS_CODEC_SNAPPY 1
#define HS_CODEC_GZIP 2 /* one gzip member per page */
#define HS_CODEC_LZ4 5  /* Hadoop's Lz4Codec framing, as Spark 2.4-3.1 write it */

#define HS_OUT_FILES 0  /* write <out_dir>/part-<bbbbb>-<uuid>_<bbbbb>.c000.parquet (the reference's effect) */
#define HS_OUT_HOST 1   /* keep the bucket file images in pinned host memory owned by the result handle */
#define HS_OUT_DEVICE 2 /* keep the bucket file images in device memory owned by the result handle */

typedef struct {
  const hs_source_file* files; /* this rank's share of the source files (all of them on one GPU) */
  int32_t n_files;
  const char* const* indexed_columns; /* resolved names, in IndexConfig order (CoveringIndex.scala:34) */
  int32_t n_indexed;
  const char* const* included_columns; /* CoveringIndex.scala:35 */
  int32_t n_included;
  int32_t num_buckets; /* spark.hyperspace.index.numBuckets, frozen in the log entry (CoveringIndex.scala:37) */
  int32_t save_mode;   /* HS_SAVE_* */
  int32_t output;      /* HS_OUT_* */
  int32_t lineage;     /* != 0: append `_data_file_id` (int64) from hs_source_file.file_id (CoveringIndex.scala:152-186) */
  const char* out_dir; /* ctx.indexDataPath = <index>/v__=<N> (actions/CreateActionBase.scala:32-37); HS_OUT_FILES only */
  const char* job_uuid; /* the <uuid> of the part file names; NULL -> generated */
  int64_t rows_per_page;      /* 0 -> 131072 */
  int64_t rows_per_row_group; /* 0 -> 4194304 */
  /* rows to drop: lineage ids whose rows must not reach the output (refreshIncremental's deleted files,
   * CoveringIndexTrait.scala:78-94).  Requires a `_data_file_id` column in the source files. */
  const int64_t* deleted_file_ids;
  int32_t n_deleted_file_ids;
  int32_t disable_dictionary; /* 0 (default): dictionary-encode columns whose distinct values fit a dictionary page, as
                                 parquet-mr does; != 0: PLAIN only */
  int32_t compression;        /* HS_CODEC_*: codec of the index pages, spark.sql.parquet.compression.codec.  HS_CODEC_SNAPPY is
                                 what Spark writes by default (files are then named ...c000.snappy.parquet,
                                 T/index/VacuumOutdatedActionTest.scala:67); GZIP and LZ4 files end in .c000.gz.parquet and
                                 .c000.lz4.parquet.  Other codecs are HS_EUNSUPPORTED. */
  int32_t reserved;
} hs_index_spec;

typedef struct {
  int64_t rows_in;       /* rows decoded on this rank */
  int64_t rows_out;      /* rows written by this rank (after the exchange) */
  int64_t bytes_in;      /* encoded source bytes consumed */
  int64_t bytes_out;     /* encoded index bytes produced */
  int64_t bytes_exchanged; /* bytes this rank sent through the all-to-all */
  int32_t files_out;
  int32_t gpu_launches;  /* kernels launched by this call */
  float ms_total;        /* CUDA-event time of the whole call on the ctx stream */
  float ms_h2d, ms_plan, ms_decode, ms_hash, ms_partition, ms_exchange, ms_sort, ms_gather, ms_encode, ms_d2h, ms_write;
} hs_stats;

/* Body of CoveringIndex.write(ctx, indexData, mode) (index/covering/CoveringIndex.scala:56-71): scan the source
 * Parquet, project indexed ++ included columns, bucket = pmod(murmur3(keys, 42), num_buckets), sort each bucket
 * ascending nulls-first on the indexed columns, and emit one Parquet file per non-empty bucket
 * (index/DataFrameWriterExtensions.scala:50-68).  All-or-nothing: on failure nothing is left in out_dir. */
int hs_create_index(hs_ctx* ctx, const hs_index_spec* spec, hs_index_result** out, hs_stats* stats, char* err,
                    size_t errlen);

/* ---- software pipelining across calls -------------------------------------------------------------------------------
 * One createIndex cannot overlap its own input and output copies: every index file depends on every source file (the hash
 * repartition), so the device->host drain of a call starts after its last source byte has arrived.  What CAN overlap are
 * the copies of NEIGHBOURING calls, in both directions at once (PCIe is full duplex) -- the overlap Spark gets from running
 * the scan tasks of one job beside the write tasks of another (index/DataFrameWriterExtensions.scala:76-80 hands the write
 * to Spark's task scheduler).  Three steps, each on its own CUDA stream of the ctx:
 *
 *   hs_stage_sources       host (or file system) Parquet images -> device, asynchronously on the H2D copy stream; footers
 *                          are parsed from host memory on the way.  The handle's descriptors (on_device = 1) are valid
 *                          inputs of hs_create_index[_async], hs_filter_scan and hs_bucket_join, which wait for the copy.
 *                          The caller's host images must stay valid until hs_staged_wait / hs_staged_free returns or a
 *                          call that consumed the descriptors has returned.
 *   hs_create_index_async  everything hs_create_index does up to the encoded index files in device memory (returns when
 *                          the kernels have run), then starts the device->host copy on the D2H copy stream.
 *   hs_pending_wait        waits for that copy (and writes the files for HS_OUT_FILES); yields the result + stats.
 *                          Consumes the handle, also on failure.
 *
 *   staged[i+1] = hs_stage_sources(...);  pending[i] = hs_create_index_async(staged[i]...);  hs_pending_wait(pending[i-1])
 *
 * keeps the H2D engine, the SMs and the D2H engine busy at the same time.  hs_create_index == async + wait. */
typedef struct hs_staged hs_staged;
typedef struct hs_pending hs_pending;
int hs_stage_sources(hs_ctx* ctx, const hs_source_file* files, int32_t n_files, hs_staged** out, char* err, size_t errlen);
int32_t hs_staged_num_files(const hs_staged* s);
int hs_staged_file(const hs_staged* s, int32_t i, hs_source_file* out); /* out->path points into the handle */
int hs_staged_wait(hs_staged* s, float* ms_copy); /* blocks until the copies have completed; ms_copy (optional): their
                                                      duration on the H2D stream */
void hs_staged_free(hs_staged* s); /* waits for the copies and for the ctx stream, then releases the device images */
int hs_create_index_async(hs_ctx* ctx, const hs_index_spec* spec, hs_pending** out, char* err, size_t errlen);
int hs_pending_wait(hs_pending* p, hs_index_result** out, hs_stats* stats, char* err, size_t errlen);
void hs_pending_cancel(hs_pending* p); /* waits for the copy and drops the result */

int32_t hs_result_num_files(const hs_index_result* r);
/* File i of the result: bucket id, file name (no directory), image pointer (host or device, NULL for
 * HS_OUT_FILES), image size, row count. */
int hs_result_file(const hs_index_result* r, int32_t i, int32_t* bucket, const char** name, const void** data,
                   uint64_t* size, int64_t* rows);
void hs_result_free(hs_index_result* r);

/* ------------------------------------------------------------------------------------------------------------
 * Read side: FilterIndexRule scan, JoinIndexRule bucket-aligned sort-merge join
 * ---------------------------------------------------------------------------------------------------------- */

typedef struct {
  const hs_source_file* files; /* index (or source) Parquet files */
  int32_t n_files;
  int32_t sorted_on_key;       /* != 0: every file is sorted ascending on key_column (index files) -> binary search;
                                  0: full predicate scan (appended source files under Hybrid Scan) */
  const char* key_column;      /* predicate column (first indexed column, covering/FilterIndexRule.scala:33-103) */
  const char* const* projected_columns;
  int32_t n_projected;
  int32_t has_lo, has_hi;      /* inclusive bounds lo <= key <= hi on an integer key.  A timestamp key compares them as
                                  micros since the epoch; a decimal key as integer VALUES, rescaled to its scale (lo = 10 on a
                                  decimal(9,2) key is 10.00, unscaled 1000), as Spark compares `price >= 10` */
  int64_t lo, hi;
  const int64_t* deleted_file_ids; /* Hybrid Scan: NOT (_data_file_id IN ids) (covering/CoveringIndexRuleUtils.scala:244-253) */
  int32_t n_deleted_file_ids;
  int32_t output;              /* HS_OUT_HOST (or 0): result columns in pinned host memory; HS_OUT_DEVICE: left in device
                                  memory for the next GPU operator (hs_batch_column then yields device pointers) */
  /* string / binary key column (HS_TYPE_STRING): the inclusive bounds as bytes, compared in UTF8String byte order (unsigned
   * bytes, the shorter value first on a common prefix); has_lo / has_hi say which are set, lo / hi are ignored.  Equality
   * -- the predicate of the reference's own filter-rule tests, `c3 == "facebook"` (T/index/E2EHyperspaceRulesTest.scala) --
   * is lo == hi. */
  const void* lo_bytes;
  const void* hi_bytes;
  uint32_t lo_len, hi_len;
} hs_scan_spec;

/* Executes the scan FilterIndexRule.applyIndex substitutes for the source scan
 * (index/covering/FilterIndexRule.scala:135-149; CoveringIndexRuleUtils.scala:98-130). */
int hs_filter_scan(hs_ctx* ctx, const hs_scan_spec* spec, hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* One comparison range on one column, a conjunct of a filter: lo <= column <= hi (strict where lo_strict / hi_strict say
 * so; has_lo / has_hi say which bounds exist, at least one must).  literal_type says which fields hold the bounds:
 * HS_TYPE_INT64 -> lo_i / hi_i, HS_TYPE_DOUBLE -> lo_f / hi_f, HS_TYPE_STRING -> lo_bytes / hi_bytes (lo_len / hi_len bytes,
 * at most 65535), HS_TYPE_DECIMAL -> lo_i / hi_i unscaled, with `scale`.
 * Timestamp columns take HS_TYPE_INT64 literals, microseconds since the epoch (a Spark timestamp literal's value).  Decimal
 * columns, and int32 / int64 columns against decimal literals, compare exactly, as Spark's decimal comparison does: an
 * HS_TYPE_INT64 literal is an integer value (`price > 10` is `price > 10.00` on a decimal(p,2)), and a literal with more
 * fractional digits than the column becomes the ceiling / floor bound with the right strictness.  Refused with
 * HS_EUNSUPPORTED, so that the caller keeps the conjunct in a Spark Filter (Spark compares them in double): HS_TYPE_DOUBLE
 * literals on decimal and timestamp columns, HS_TYPE_DECIMAL literals on float / double / timestamp / string columns.  The comparison is Spark 3.1's after its binary-comparison coercion: it happens in the wider of the
 * column's and the literal's types (int < long < float < double), so `int_col > 1.5` is `int_col >= 2`, a float column
 * against a double literal compares (double)f, and a float column against a long literal casts the literal to float;
 * NaN equals NaN and is greater than +inf, -0.0 equals 0.0 (SQLOrderingUtil.compareDoubles).  String columns take
 * HS_TYPE_STRING literals only, numeric columns numeric ones; boolean columns are not handled (HS_EUNSUPPORTED). */
typedef struct {
  const char* column;            /* any column of the files: int32 / int64 / float / double / string / timestamp / decimal */
  int32_t literal_type;          /* HS_TYPE_INT64, HS_TYPE_DOUBLE, HS_TYPE_STRING or HS_TYPE_DECIMAL */
  int32_t has_lo, has_hi;
  int32_t lo_strict, hi_strict;  /* 1: lo < x / x < hi; 0: inclusive */
  int32_t scale;                 /* HS_TYPE_DECIMAL: the literal's scale (0..38); ignored otherwise */
  int64_t lo_i, hi_i;
  double lo_f, hi_f;
  const void* lo_bytes;
  const void* hi_bytes;
  uint32_t lo_len, hi_len;
} hs_predicate;

/* The scan FilterIndexRule substitutes (FilterIndexRule.scala:58-101), with the conjunction of preds (at most 16) as the
 * filter: a row qualifies when every predicate holds, and a null never satisfies a bound.  spec gives files, sorted_on_key,
 * key_column (the column the files are sorted on; may be NULL when sorted_on_key is 0), projection, deleted_file_ids and
 * output; its own bounds (has_lo / has_hi) must be 0.  Sorted files are binary-searched on the predicates over key_column,
 * and the other predicates are evaluated over the rows inside those windows only.  Float and double keys are handled here
 * (hs_filter_scan, whose bounds are int64, refuses them). */
int hs_filter_scan_where(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds, hs_batch** out,
                         hs_stats* stats, char* err, size_t errlen);

/* A disjunction on one column -- Spark's In / InSet, and an Or whose branches all compare the same column: the row
 * qualifies when its value equals one of the n_values listed values or lies inside one of the n_ranges ranges.  Every `=`
 * and every range is evaluated as the hs_predicate of the same literal would be (the wider type decides, decimals compare
 * exactly, NaN equals NaN, -0.0 equals 0.0): this is Spark's In, which compares with the type's ordering (Spark 3.1's InSet,
 * used above 10 values, treats NaN and -0.0 differently in its interpreted and generated forms; this follows In).  A null
 * row never qualifies; a NULL inside the list never makes a row qualify, so the caller drops it.  n_values == 0 with no
 * ranges selects nothing.  The values are columnar, by literal_type: HS_TYPE_INT64 / HS_TYPE_DECIMAL (unscaled, with
 * `scale`) in values_i, HS_TYPE_DOUBLE in values_f, HS_TYPE_STRING as values_bytes[values_offsets[k] ..
 * values_offsets[k+1]) (n_values + 1 ascending offsets, each value at most 65535 bytes).  ranges[r].column is NULL or
 * `column`.  At most 2^24 values plus ranges per term (HS_EUNSUPPORTED above); string values on a numeric column, numeric
 * values on a string column, double values on decimal and timestamp columns: HS_EUNSUPPORTED.  A NULL array with a nonzero
 * count, or descending offsets: HS_EINVAL. */
typedef struct {
  const char* column;
  int32_t literal_type;        /* of the listed values: HS_TYPE_INT64 / HS_TYPE_DOUBLE / HS_TYPE_STRING / HS_TYPE_DECIMAL */
  int32_t scale;               /* HS_TYPE_DECIMAL */
  int64_t n_values;
  const int64_t* values_i;     /* INT64, DECIMAL (unscaled) */
  const double* values_f;      /* DOUBLE */
  const void* values_bytes;    /* STRING: value k = values_bytes[values_offsets[k] .. values_offsets[k+1]) */
  const uint64_t* values_offsets;
  const hs_predicate* ranges;  /* hs_predicate semantics; column NULL or == column */
  int32_t n_ranges;
  int32_t flags;               /* HS_TERM_* below; 0: the disjunction above, a null row never qualifying */
} hs_predicate_any;

/* hs_predicate_any.flags.  A term is true, false or unknown on each row, as in Spark's three-valued logic, and a row
 * qualifies only when every AND-ed term is true.  On a non-null row the term is true when the value lies in the term's set
 * (or matches its pattern) and false otherwise; on a null row it is unknown unless a NULL flag says otherwise.
 *   HS_TERM_NOT         Not(term): true <-> false, unknown stays (`c != 5`, `~c.isin(...)`, `NOT c LIKE '...'`).  The NULL
 *                       flags describe the term before NOT.
 *   HS_TERM_NULL_TRUE   a null row makes the term true: IsNull is NULL_TRUE with no values and no ranges, IsNotNull the same
 *                       with NOT.
 *   HS_TERM_NULL_FALSE  a null row makes the term false: EqualNullSafe(c, v) is the value v with NULL_FALSE, so that
 *                       NOT (c <=> v) keeps the null rows.
 *   HS_TERM_STARTS_WITH, HS_TERM_ENDS_WITH, HS_TERM_CONTAINS: StringStartsWith / StringEndsWith / StringContains, in bytes;
 *                       the empty pattern matches every non-null value.
 *   HS_TERM_LIKE        Like with the escape character '\': '%' matches any run of characters, '_' one UTF-8 character, and
 *                       the whole value must match.  A pattern ending in the escape character, or with the escape before
 *                       anything but '%', '_' and '\', is HS_EINVAL with Spark's message.  Values that are not valid UTF-8 are
 *                       not covered: Spark matches the decoded String.
 * A pattern term (one of the last four) has literal_type HS_TYPE_STRING, exactly one value -- the pattern, at most 65535
 * bytes -- and no ranges; on a non-string column it is HS_EUNSUPPORTED.  Both NULL flags, two pattern kinds, a malformed
 * pattern term or an unknown bit: HS_EINVAL. */
#define HS_TERM_NOT 1
#define HS_TERM_NULL_TRUE 2
#define HS_TERM_NULL_FALSE 4
#define HS_TERM_STARTS_WITH 8
#define HS_TERM_ENDS_WITH 16
#define HS_TERM_CONTAINS 32
#define HS_TERM_LIKE 64

/* hs_filter_scan_where with disjunction terms AND-ed to the predicates (n_preds + n_anys <= 16).  On sorted files a term on
 * key_column becomes many windows per file, one per disjoint range of its values; terms on other columns (and every term
 * on unsorted files) are evaluated per row.  file_buckets / num_buckets (optional: NULL / 0) give each file's bucket and
 * assert that the files are bucketed on key_column alone (Spark's bucket hash, as hs_create_index writes them): when the
 * key's windows are points only (listed values, ranges with lo == hi, equalities in preds) and the key is int32, int64,
 * string, timestamp or decimal, only the files of the points' buckets are opened, each point is searched only in the files
 * of its own bucket, and stats count only those files (a term on key_column that a null row makes true -- IS NULL,
 * NOT (k <=> v) -- turns this off: the null keys lie in their own bucket).  The rows are the same, in the same order (file,
 * then row), as without file_buckets.  Without terms and buckets this is hs_filter_scan_where. */
int hs_filter_scan_any(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds,
                       const hs_predicate_any* anys, int32_t n_anys, const int32_t* file_buckets, int32_t num_buckets,
                       hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* A comparison between two columns of the same row: `left OP right`, with NOT when flags has HS_TERM_NOT (`a != b` is NOT
 * of HS_CMP_EQ).  Spark 3.1 semantics:
 *   Nulls: a null on either side makes LT, LE, GT, GE and EQ unknown, so the row does not qualify, under NOT too.
 *          EQ_NULL_SAFE (`<=>`) is true on two nulls and false on one; NOT applies to that, so NOT (a <=> b) keeps the rows
 *          where exactly one side is null.
 *   Order: as the literal comparisons -- NaN equals NaN and is above +inf, -0.0 equals 0.0, strings in UTF8String byte
 *          order.
 *   Coercion (TypeCoercion and DecimalPrecision for BinaryComparison(attribute, attribute)), resolved once per call:
 *     the same type (int, long, float, double, string, binary, date, timestamp, decimal(p,s) of equal p and s): that type;
 *     int against long: long;
 *     int or long against float: float, the integer rounded to nearest (2^24 + 1 equals 16777216f);
 *     int, long or float against double: double;
 *     decimal against a decimal of another precision or scale, or against int / long (as decimal(10,0) / decimal(20,0)):
 *       exactly, the side of the smaller scale rescaled in 128 bits;
 *     decimal against float or double: double (the decimal rounded to nearest);
 *     date against timestamp: timestamp, the date's days times 86 400 000 000 micros (dates are UTC midnights, as the
 *       naive timestamp literals are UTC).
 *   Any other pair -- string against a number, date or timestamp; date or timestamp against a number; a boolean column --
 *   is HS_EUNSUPPORTED naming both columns and their Spark types.  A NULL name, an op outside HS_CMP_*, or a flag other
 *   than HS_TERM_NOT is HS_EINVAL; an unknown column fails as an unknown predicate column does.  Both names may be the
 *   same column. */
typedef struct {
  const char* left;
  const char* right;
  int32_t op;     /* HS_CMP_* */
  int32_t flags;  /* 0 or HS_TERM_NOT */
} hs_column_compare;

#define HS_CMP_LT 1
#define HS_CMP_LE 2
#define HS_CMP_GT 3
#define HS_CMP_GE 4
#define HS_CMP_EQ 5
#define HS_CMP_EQ_NULL_SAFE 6

/* hs_filter_scan_any with column comparisons AND-ed to the predicates and terms (n_preds + n_anys + n_cmps <= 16).  Both
 * columns of every comparison are decoded like other predicate columns (on sorted files, only inside the key's windows)
 * and the comparisons run per row.  A comparison makes no key window and prunes no bucket: when the key appears in the
 * filter only through comparisons, the scan of sorted files reads every row.  With n_cmps = 0 this is hs_filter_scan_any. */
int hs_filter_scan_cmp(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds,
                       const hs_predicate_any* anys, int32_t n_anys, const hs_column_compare* cmps, int32_t n_cmps,
                       const int32_t* file_buckets, int32_t num_buckets, hs_batch** out, hs_stats* stats, char* err,
                       size_t errlen);

typedef struct {
  const hs_source_file* left_files;  /* index files of the left side, any order; bucket id parsed from the name */
  int32_t n_left;
  const hs_source_file* right_files;
  int32_t n_right;
  const int32_t* left_buckets;       /* bucket id per left file  (BucketingUtils.getBucketId on the file name) */
  const int32_t* right_buckets;
  int32_t num_buckets;
  int32_t output;                    /* HS_OUT_HOST (or 0) / HS_OUT_DEVICE, as in hs_scan_spec */
  const char* left_key;              /* single join key on each side: int32 / int64 / string (timestamps and decimals too),
                                        the same Spark type on both */
  const char* right_key;
  const char* const* left_columns;   /* projected from the left side */
  int32_t n_left_columns;
  const char* const* right_columns;
  int32_t n_right_columns;
} hs_join_spec;

/* Inner equi-join bucket b of the left index with bucket b of the right index, no exchange -- what Spark plans
 * after JoinIndexRule.applyIndex (index/covering/JoinIndexRule.scala:653-687; T/index/E2EHyperspaceRulesTest.scala:487-512).
 * Buckets holding several files (after an incremental refresh) are merged first, as Spark's SortExec would. */
int hs_bucket_join(hs_ctx* ctx, const hs_join_spec* spec, hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* The same join on n_keys (1..8) AND-ed equalities left_keys[k] == right_keys[k], with a filter below each side -- the
 * joins JoinIndexRule rewrites (JoinIndexRule.scala:164-170 conditions, 569-616 column orders; T/index/covering/
 * JoinIndexRuleTest.scala:84-95 puts a Filter under both sides).  The keys come in the order of the indexes' indexed
 * columns: the left index's order, and the right columns they map to; both sides must have been bucketed and sorted on
 * the keys in that order.  Key columns are int32 / int64 / string (timestamps, decimals of precision <= 18), of the same
 * Spark type at each position -- a decimal's precision and scale included, and an int32 never pairs with a decimal(p <= 9)
 * although both are int32 here (float, double and
 * boolean keys: HS_EUNSUPPORTED; n_keys > 8: HS_EUNSUPPORTED; n_keys < 1: HS_EINVAL).  A row whose key has a null in any
 * column joins nothing, as in Spark's inner join.  left_preds / right_preds (at most 16 each) are conjunctions with the
 * semantics and refusals of hs_filter_scan_where; a row joins only when every predicate of its side holds.  Files,
 * buckets, projection and output come from spec, whose left_key / right_key must be NULL.  Output: the pairs in (bucket,
 * left sorted position, right sorted position) order, as hs_bucket_join.  With one key, no predicates and no nulls in the
 * keys this runs exactly what hs_bucket_join runs.  stats->ms_exchange (a one-GPU join exchanges nothing) reports the
 * side selection: the null and predicate masks and the compaction of both sides. */
int hs_bucket_join_where(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                         int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds, const hs_predicate* right_preds,
                         int32_t n_right_preds, hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* hs_bucket_join_where with hs_predicate_any terms AND-ed to each side's predicates (n_preds + n_anys <= 16 per side),
 * evaluated per row in the side selection.  No bucket pruning on join sides. */
int hs_bucket_join_any(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                       int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds, const hs_predicate_any* left_anys,
                       int32_t n_left_anys, const hs_predicate* right_preds, int32_t n_right_preds,
                       const hs_predicate_any* right_anys, int32_t n_right_anys, hs_batch** out, hs_stats* stats, char* err,
                       size_t errlen);

/* hs_bucket_join_any with hs_column_compare comparisons AND-ed to each side's filter (n_preds + n_anys + n_cmps <= 16 per
 * side); both columns of a comparison belong to that side.  They run per row in the side selection.  With no comparisons
 * this is hs_bucket_join_any. */
int hs_bucket_join_cmp(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                       int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds, const hs_predicate_any* left_anys,
                       int32_t n_left_anys, const hs_column_compare* left_cmps, int32_t n_left_cmps, const hs_predicate* right_preds,
                       int32_t n_right_preds, const hs_predicate_any* right_anys, int32_t n_right_anys,
                       const hs_column_compare* right_cmps, int32_t n_right_cmps, hs_batch** out, hs_stats* stats, char* err,
                       size_t errlen);

/* join_type of hs_bucket_join_exists: Spark 3.1's LeftSemi (EXISTS, IN-subquery) and LeftAnti (NOT EXISTS) */
#define HS_JOIN_LEFT_SEMI 1
#define HS_JOIN_LEFT_ANTI 2

/* The left semi or left anti join of hs_bucket_join_cmp's sides, bucket b of the left index with bucket b of the right
 * index and no exchange -- SortMergeJoinExec with joinType LeftSemi / LeftAnti, which JoinIndexRule rewrites as it does
 * an inner join (JoinIndexRule.scala:53-110 checks only for an equi-condition, a SortMergeJoin and linear children).
 * Keys, predicates, terms, comparisons, key types and their refusals (codes and messages) are hs_bucket_join_cmp's.
 * The output is left rows only, each at most once however many right rows it matches (duplicate left rows stay
 * duplicates), in (bucket, left sorted position) order:
 *   HS_JOIN_LEFT_SEMI  keeps a left row when some right row of its bucket has an equal key tuple; a left row with a null
 *                      in any key column is dropped.
 *   HS_JOIN_LEFT_ANTI  keeps a left row when no right row matches; a left row with a null in any key column matches
 *                      nothing and is KEPT.  This is not the null-aware anti join of NOT IN, which Spark 3.1 never plans
 *                      as a sort-merge join.
 * A right row with a null key, or that fails the right side's filter, matches nothing; a left row that fails the left
 * side's filter is never output.  A bucket whose right side is empty (or emptied by its filter) outputs none of its left
 * rows under semi and all of them under anti.  spec->n_right_columns must be 0 and spec->left_key / right_key NULL
 * (HS_EINVAL); the right side decodes only its key and filter columns.  A join_type other than HS_JOIN_* is HS_EINVAL.
 * stats->ms_sort reports the probe (k_join_exists and the compaction of the kept rows), stats->ms_exchange the side
 * selection, as for the inner join. */
int hs_bucket_join_exists(hs_ctx* ctx, const hs_join_spec* spec, int32_t join_type, const char* const* left_keys,
                          const char* const* right_keys, int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds,
                          const hs_predicate_any* left_anys, int32_t n_left_anys, const hs_column_compare* left_cmps,
                          int32_t n_left_cmps, const hs_predicate* right_preds, int32_t n_right_preds,
                          const hs_predicate_any* right_anys, int32_t n_right_anys, const hs_column_compare* right_cmps,
                          int32_t n_right_cmps, hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* join_type of hs_bucket_join_outer: Spark 3.1's LeftOuter, RightOuter and FullOuter */
#define HS_JOIN_LEFT_OUTER 3
#define HS_JOIN_RIGHT_OUTER 4
#define HS_JOIN_FULL_OUTER 5

/* The left, right or full outer join of hs_bucket_join_cmp's sides, bucket b of the left index with bucket b of the right
 * index and no exchange -- SortMergeJoinExec with joinType LeftOuter / RightOuter / FullOuter over Filter(left) and
 * Filter(right), which JoinIndexRule rewrites as it does an inner join (JoinIndexRule.scala:54 matches any join type).
 * Keys, predicates, terms, comparisons, key types and their refusals (codes and messages) are hs_bucket_join_cmp's.  Both
 * projections are allowed, and either may be empty; the batch holds the left columns, then the right ones.  A side whose
 * rows are output whether they match or not is preserved (the left side of LeftOuter, the right side of RightOuter, both
 * of FullOuter); the other side supplies nulls.
 *   A row that fails its side's filter is not output when its side is preserved, and matches nothing otherwise.  A row
 *   with a null in any key column matches nothing; on a preserved side it is output once, padded.
 *   HS_JOIN_LEFT_OUTER   every selected left row comes out once per matching right row, or once with every right column
 *                        null; order (bucket, left sorted position, right sorted position).
 *   HS_JOIN_RIGHT_OUTER  the mirror image, in (bucket, right sorted position, left sorted position) order; the columns are
 *                        still the left ones, then the right ones.
 *   HS_JOIN_FULL_OUTER   within each bucket, the bucket's HS_JOIN_LEFT_OUTER rows in the order above, then the bucket's
 *                        right rows that matched nothing, in right sorted position order, with every left column null.
 *                        Spark 3.1 gives a full outer join no output ordering; this order is the library's own.
 * Every column of a null-supplying side has a validity vector, even when no row was padded (both sides under FullOuter);
 * a padded value is 0, or a string of length 0.  More than 2^32 - 1 output rows is HS_EUNSUPPORTED, as for the inner
 * join.  A join_type other than the three above is HS_EINVAL.  stats->ms_sort reports the probe, the emit and the
 * placement of FullOuter's unmatched right rows, stats->ms_exchange the side selections, stats->rows_out the output rows. */
int hs_bucket_join_outer(hs_ctx* ctx, const hs_join_spec* spec, int32_t join_type, const char* const* left_keys,
                         const char* const* right_keys, int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds,
                         const hs_predicate_any* left_anys, int32_t n_left_anys, const hs_column_compare* left_cmps,
                         int32_t n_left_cmps, const hs_predicate* right_preds, int32_t n_right_preds,
                         const hs_predicate_any* right_anys, int32_t n_right_anys, const hs_column_compare* right_cmps,
                         int32_t n_right_cmps, hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* Arithmetic over the columns of a row, compared: `a + b < c`, `price * (1 - discount) > 100`, `k % 7 = 0`.  One side of
 * an hs_expr_compare is an array of hs_expr_node in postfix order (`a + b` is COLUMN a, COLUMN b, ADD); a side of one
 * COLUMN or LITERAL node is a bare column or literal.  Spark 3.1 semantics with spark.sql.ansi.enabled=false:
 *   Operands: int (byte and short count as int), long, float, double and decimal(p <= 18) columns, and literals.  An
 *     operation between two byte or short columns, and NEG of one, is HS_EUNSUPPORTED: Spark wraps it at 8 or 16 bits.  A
 *     HS_TYPE_INT32 literal is an int, HS_TYPE_INT64 a long, HS_TYPE_DOUBLE a double, and HS_TYPE_DECIMAL (unscaled
 *     value_i, `scale`) is decimal(max(digits, scale), scale).  String, binary, boolean, date and timestamp columns are
 *     HS_EUNSUPPORTED naming the column and its Spark type.
 *   Operand types (TypeCoercion.ImplicitTypeCasts, DecimalPrecision): int with long is long; int or long with float is
 *     float (the integer rounded to nearest); anything with double is double; decimal with int or long is decimal, an
 *     int column counting as decimal(10,0), a long column as decimal(20,0) and an integer literal as decimal(its digits,
 *     0); decimal with float or double is double.  DIV casts every operand to double (TypeCoercion.Division), so int / int
 *     is double.
 *   Nulls: a null operand makes the node null; so does a zero divisor of DIV and REM (0, 0.0 and -0.0 alike).
 *   Integers: ADD, SUB, MUL and NEG wrap in two's complement at the operand width (int arithmetic at 2^31); REM is Java's
 *     truncated remainder, the sign of the dividend, and MIN % -1 is 0.
 *   Float and double: every operation rounds to nearest on its own, never fused; REM is fmod.
 *   Decimals: exact.  ADD / SUB give scale max(s1,s2) and precision max(p1-s1, p2-s2) + scale + 1; MUL (p1+p2+1, s1+s2);
 *     REM (min(p1-s1, p2-s2) + max(s1,s2), max(s1,s2)).  A node whose result, or whose operands' wider type (max(p1-s1,
 *     p2-s2) + max(s1,s2)), would exceed 38 digits is HS_EUNSUPPORTED: Spark would bound or adjust it.  Decimal DIV is
 *     HS_EUNSUPPORTED, and so is a decimal of more than 18 digits that would have to become a double.
 *   The comparison: HS_CMP_* with HS_TERM_NOT, after hs_column_compare's coercion of the two sides' types (decimals up to
 *     38 digits compare exactly, the side of the smaller scale rescaled; a common decimal type above 38 digits is
 *     HS_EUNSUPPORTED).  NaN equals NaN and is above +inf; -0.0 equals 0.0.  A null side makes LT, LE, GT, GE and EQ
 *     unknown, under NOT too; EQ_NULL_SAFE is true on two null sides and false on one.
 *   Limits: at most 32 nodes per side (HS_EUNSUPPORTED) and a stack depth of 8 per side (HS_EUNSUPPORTED).  Stack underflow,
 *   values left over, an unknown kind, op or flag, a NULL column name, a HS_TYPE_INT32 literal outside int32 or a decimal
 *   scale outside 0..38 is HS_EINVAL. */
#define HS_EXPR_COLUMN 1
#define HS_EXPR_LITERAL 2
#define HS_EXPR_ADD 3
#define HS_EXPR_SUB 4
#define HS_EXPR_MUL 5
#define HS_EXPR_DIV 6
#define HS_EXPR_REM 7
#define HS_EXPR_NEG 8

/* Spark functions of columns inside an hs_expr_compare side: `year(d) = 1995`, `substring(s, 1, 2) = '13'`,
 * `datediff(a, b) > 30`, `abs(a - b) < 5`, `coalesce(x, 0) > 0.05`.  Each kind takes its arguments in postfix order below
 * it, like the arithmetic nodes; arithmetic, functions and comparisons nest freely within the limits above.  Spark 3.1
 * semantics with spark.sql.ansi.enabled=false:
 *   Literals besides the numeric ones: HS_TYPE_STRING (the bytes at `column`, value_i of them, at most 65535; a string),
 *     HS_TYPE_DATE (value_i days since the epoch, within int32) and HS_TYPE_TIMESTAMP (value_i microseconds since the epoch).
 *   YEAR QUARTER MONTH DAYOFMONTH DAYOFWEEK DAYOFYEAR WEEKOFYEAR (one date or timestamp) -> int.  Proleptic Gregorian, as
 *     LocalDate.ofEpochDay; DAYOFWEEK is 1 = Sunday .. 7 = Saturday; WEEKOFYEAR is the ISO-8601 week (weeks start on
 *     Monday, week 1 holds the year's first Thursday).  A timestamp is first cast to a date in UTC, the library's time
 *     zone (naive literals are UTC, hs_column_compare takes dates as UTC midnights): floorDiv(micros, 86 400 000 000).
 *   HOUR MINUTE SECOND (one timestamp) -> int: the UTC wall clock.  A date argument is HS_EUNSUPPORTED.
 *   DATE_ADD DATE_SUB (start: date or timestamp, then days) -> date: start +/- days in int arithmetic, wrapping at 2^31
 *     (Spark's DateAdd / DateSub).  days is an int literal or a byte, short or int column; a long, decimal or floating
 *     days is HS_EUNSUPPORTED (Spark would cast it).
 *   DATEDIFF (end, then start: each a date or timestamp) -> int: end - start in days, wrapping.
 *   LENGTH (string or binary) -> int: characters of a string, counted as UTF8String.numChars counts them (by the length
 *     each first byte announces), bytes of a binary.  Values that are not valid UTF-8 are not covered.
 *   SUBSTRING (string or binary, then pos, then len; pos and len HS_TYPE_INT32 literals, else HS_EINVAL) -> the argument's
 *     type: UTF8String.substringSQL / ByteArray.subStringSQL.  pos > 0 is 1-based, pos 0 is 1, a negative pos counts from
 *     the end; the end is start + len clamped to the int range, and start >= end gives the empty value.  The result
 *     refers to the argument's bytes: nothing is copied.
 *   ABS (a number) -> its type.  int and long wrap (abs(MIN) = MIN); float and double clear the sign (abs(-0.0) = 0.0,
 *     NaN stays NaN); decimals are exact.  A byte or short argument is HS_EUNSUPPORTED (Spark wraps at its width).
 *   COALESCE (value_i arguments, 2..8 and at most the values below it, else HS_EINVAL) -> findWiderCommonType of the
 *     arguments: the arithmetic's numeric widening (an integer literal counts as int or long here, decimal(10,0) or
 *     decimal(20,0) beside a decimal; a result above 38 digits is HS_EUNSUPPORTED), string with string, binary with
 *     binary, date with date, date with timestamp to timestamp.  The value is the first non-null argument; null only
 *     when every argument is.  Any other mix (a string with a number, for one) is HS_EUNSUPPORTED.  A date promoted to
 *     a timestamp is its UTC midnight in exact 128-bit micros, also for a date more than 106 751 991 days from the epoch
 *     (beyond the long micros range, where Spark's cast fails): the functions over it give that midnight's fields.
 *   Nulls: every function but COALESCE is null when any argument is null.
 *   The comparison, besides the numeric pairs above: string with string and binary with binary in UTF8String byte order;
 *     date with date in days; date or timestamp with timestamp in microseconds (a date is its UTC midnight), as
 *     hs_column_compare.  Any other pair with a string, binary, date or timestamp side is HS_EUNSUPPORTED, naming both
 *     sides' text and types -- except that a bare column of a type arithmetic refuses keeps the message "the column 'c'
 *     (type) cannot be used in arithmetic".  The argument of a function of the wrong type is HS_EUNSUPPORTED naming the
 *     function and the type. */
#define HS_EXPR_YEAR 9
#define HS_EXPR_QUARTER 10
#define HS_EXPR_MONTH 11
#define HS_EXPR_DAYOFMONTH 12
#define HS_EXPR_DAYOFWEEK 13
#define HS_EXPR_DAYOFYEAR 14
#define HS_EXPR_WEEKOFYEAR 15
#define HS_EXPR_HOUR 16
#define HS_EXPR_MINUTE 17
#define HS_EXPR_SECOND 18
#define HS_EXPR_DATE_ADD 19
#define HS_EXPR_DATE_SUB 20
#define HS_EXPR_DATEDIFF 21
#define HS_EXPR_LENGTH 22
#define HS_EXPR_SUBSTRING 23
#define HS_EXPR_ABS 24
#define HS_EXPR_COALESCE 25

typedef struct {
  int32_t kind;          /* HS_EXPR_* */
  const char* column;    /* HS_EXPR_COLUMN: the name; HS_TYPE_STRING literal: its bytes (value_i of them) */
  int32_t literal_type;  /* HS_EXPR_LITERAL: HS_TYPE_INT32 / INT64 / DOUBLE / DECIMAL / STRING / DATE / TIMESTAMP */
  int32_t scale;         /* HS_TYPE_DECIMAL literal */
  int64_t value_i;       /* INT32, INT64, DECIMAL (unscaled), DATE (days), TIMESTAMP (micros), STRING (length);
                            HS_EXPR_COALESCE: the argument count */
  double value_f;        /* DOUBLE */
} hs_expr_node;

typedef struct {
  const hs_expr_node* left;
  int32_t n_left;
  const hs_expr_node* right;
  int32_t n_right;
  int32_t op;     /* HS_CMP_* */
  int32_t flags;  /* 0 or HS_TERM_NOT */
} hs_expr_compare;

/* hs_filter_scan_cmp with expression comparisons AND-ed to the filter (n_preds + n_anys + n_cmps + n_exprs <= 16).  Their
 * columns are decoded like other predicate columns (on sorted files, only inside the key's windows) and they run per row.
 * An expression makes no key window and prunes no bucket.  With n_exprs = 0 this is hs_filter_scan_cmp. */
int hs_filter_scan_expr(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds,
                        const hs_predicate_any* anys, int32_t n_anys, const hs_column_compare* cmps, int32_t n_cmps,
                        const hs_expr_compare* exprs, int32_t n_exprs, const int32_t* file_buckets, int32_t num_buckets,
                        hs_batch** out, hs_stats* stats, char* err, size_t errlen);

/* join_type of hs_bucket_join_expr besides HS_JOIN_LEFT_SEMI .. HS_JOIN_FULL_OUTER: the inner join */
#define HS_JOIN_INNER 0

/* One bucket join of any type, with expression comparisons AND-ed to each side's filter (their columns belong to that
 * side; they run per row in the side selection).  join_type HS_JOIN_INNER is hs_bucket_join_cmp, HS_JOIN_LEFT_SEMI /
 * HS_JOIN_LEFT_ANTI hs_bucket_join_exists, HS_JOIN_*_OUTER hs_bucket_join_outer, with their rules and refusals; any other
 * join_type is HS_EINVAL.  With no expressions each is exactly that call. */
int hs_bucket_join_expr(hs_ctx* ctx, const hs_join_spec* spec, int32_t join_type, const char* const* left_keys,
                        const char* const* right_keys, int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds,
                        const hs_predicate_any* left_anys, int32_t n_left_anys, const hs_column_compare* left_cmps,
                        int32_t n_left_cmps, const hs_expr_compare* left_exprs, int32_t n_left_exprs,
                        const hs_predicate* right_preds, int32_t n_right_preds, const hs_predicate_any* right_anys,
                        int32_t n_right_anys, const hs_column_compare* right_cmps, int32_t n_right_cmps,
                        const hs_expr_compare* right_exprs, int32_t n_right_exprs, hs_batch** out, hs_stats* stats, char* err,
                        size_t errlen);

int64_t hs_batch_num_rows(const hs_batch* b);
int32_t hs_batch_on_device(const hs_batch* b); /* != 0: the column pointers are device pointers (output = HS_OUT_DEVICE) */
int32_t hs_batch_num_columns(const hs_batch* b);
/* Column i: name, HS_TYPE_*, pointer to num_rows values, pointer to one validity byte per row (NULL when the column
 * has no nulls; an outer join's null-supplying side always has one, see hs_bucket_join_outer); host pointers unless
 * hs_batch_on_device. */
int hs_batch_column(const hs_batch* b, int32_t i, const char** name, int32_t* type, const void** data,
                    const uint8_t** valid);
/* A HS_TYPE_STRING column: `data` of hs_batch_column points to the values' bytes back to back, and value r occupies
 * bytes [offsets[r], offsets[r + 1]) (num_rows + 1 offsets; a null has length 0).  HS_EINVAL for other columns. */
int hs_batch_string_offsets(const hs_batch* b, int32_t i, const uint64_t** offsets, uint64_t* total_bytes);
void hs_batch_free(hs_batch* b);

/* ------------------------------------------------------------------------------------------------------------
 * Verification of a written index (any size; bench.py checks the 1 B-row benchmark output with it on every run)
 * ---------------------------------------------------------------------------------------------------------- */

typedef struct {
  int64_t rows;               /* rows found in the files */
  int64_t bucket_mismatches;  /* rows whose pmod(murmur3(indexed columns, 42), num_buckets) != bucket id of their file */
  int64_t order_violations;   /* adjacent rows of one file whose indexed columns are not ascending, nulls first */
  uint64_t row_checksum;      /* sum over rows, mod 2^64, of a 64-bit mix of all the row's values (indexed ++ included order):
                                 independent of row order; changes when a value moves to another row */
  uint64_t column_checksum[16]; /* the same per column */
  int32_t n_columns;
  int32_t reserved;
} hs_verify_report;

/* The three properties the reference's write-path test pins (T/index/DataFrameWriterExtensionsTest.scala:93-158: bucket id
 * of every row == HashPartitioning's, every file sorted on the indexed columns, row multiset preserved), evaluated on the
 * GPU over whole index files.  buckets[i] is the bucket id of files[i] (BucketingUtils.getBucketId of its name). */
int hs_verify_index(hs_ctx* ctx, const hs_source_file* files, const int32_t* buckets, int32_t n_files,
                    const char* const* indexed_columns, int32_t n_indexed, const char* const* included_columns,
                    int32_t n_included, int32_t num_buckets, hs_verify_report* out, char* err, size_t errlen);
/* rows / row_checksum / column_checksum of rows [first_row, first_row + nrows) of the synthetic table T as generated
 * (never encoded): what hs_verify_index must report for an index built over those rows. */
int hs_synth_checksum(hs_ctx* ctx, int64_t first_row, int64_t nrows, int32_t ncols, hs_verify_report* out, char* err,
                      size_t errlen);

/* ------------------------------------------------------------------------------------------------------------
 * Kernel-level entry points (host arrays in, host arrays out).  They exist so the parity tests can pin each
 * kernel against the oracle in isolation; the JVM binding does not need them.
 * ---------------------------------------------------------------------------------------------------------- */

typedef struct {
  int32_t type;         /* HS_TYPE_* */
  int32_t reserved;     /* key columns: HS_KEY_DECIMAL or 0 */
  const void* data;     /* n values */
  const uint8_t* valid; /* one byte per row or NULL */
} hs_host_column;
/* hs_host_column.reserved of an int32 / int64 key column: its values are the unscaled values of a DecimalType(p <= 18),
 * bucketed as Spark does (hashLong of the unscaled value; for an int32 column that differs from an int's hash) */
#define HS_KEY_DECIMAL 1

/* K2: bucket id per row (int32) and the num_buckets-bin histogram (int64) of Spark's HashPartitioning. */
int hs_k_bucket_ids(hs_ctx* ctx, const hs_host_column* keys, int32_t nkeys, int64_t nrows, int32_t num_buckets,
                    int32_t* out_bucket, int64_t* out_hist, char* err, size_t errlen);
/* K3+K4: permutation ordering rows by (bucket, keys ascending nulls-first); bucket_offsets has num_buckets+1 entries. */
int hs_k_sort_perm(hs_ctx* ctx, const hs_host_column* keys, int32_t nkeys, int64_t nrows, int32_t num_buckets,
                   int64_t* out_perm, int64_t* out_bucket_offsets, char* err, size_t errlen);

/* K2+K3: the hash partition as createIndex runs it, alone.  Every row's bin is its bucket (HS_PART_LOCAL, what one GPU
 * does; HS_PART_PEER) or its owner bucket % world (HS_PART_OWNER, how several GPUs split their rows above 1024 buckets),
 * and the rows move stably into bin-major order:
 *   payload   npayload columns of 8-, 4- or 1-byte values (type gives the width; valid is not read -- validity travels as
 *             a 1-byte column) moved with the rows;
 *   codes     ncodes (0..4) uint16 columns moved as ONE 8-byte record per row, code j in bits [16 j, 16 j + 16) (the
 *             late-materialised dictionary columns of a build; up to 1024 bins only).
 * HS_PART_PEER: the runs leave as they do for the owners' memory on several GPUs, here to `world` buffers on this one:
 * bucket b's rows go to owner (b % world)'s buffer from row peer_base[b] on (num_buckets entries).  Owner o's buffer holds
 * owner_rows[o] rows and starts owner_shift[o] bytes (0 or 8; NULL: all 0) past a 16-byte boundary.  A peer layout
 * (peer_base) in another mode, or none in HS_PART_PEER, is refused with HS_EINVAL.
 * Every output buffer is filled with the byte `fill` on the device first and copied back whole, its 16 bytes of slack
 * included: out_payload[c] (nrows * width + 16 bytes) and out_records[0] (nrows * 8 + 16); with a peer layout
 * out_payload[c * world + o] (owner_shift[o] + owner_rows[o] * width + 16 bytes) and out_records[o] likewise.
 * out_offsets (optional, no peer layout): the nbins + 1 row offsets of the bins.  out_key_or_and (optional): the OR and
 * the AND of the sort encoding of the last key column over all rows, a null counted as 0 (they pick the sort's passes). */
#define HS_PART_LOCAL 0
#define HS_PART_OWNER 1
#define HS_PART_PEER 2
int hs_k_partition(hs_ctx* ctx, const hs_host_column* keys, int32_t nkeys, int64_t nrows, int32_t num_buckets,
                   const hs_host_column* payload, int32_t npayload, const uint16_t* const* codes, int32_t ncodes,
                   int32_t mode, int32_t world, const uint64_t* peer_base, const uint64_t* owner_rows,
                   const int32_t* owner_shift, int32_t fill, void* const* out_payload, void* const* out_records,
                   uint64_t* out_offsets, uint64_t* out_key_or_and, char* err, size_t errlen);

/* Synthetic table T of the benchmark (SURVEY.md section 8d): rows [first_row, first_row+nrows) of
 * (k:int64, v1:int64, v2:float64, v3:int32, v4:float32)[:ncols], generated and Parquet-encoded on the GPU into
 * n_files file images of row_groups_per_file row groups each (HS_OUT_HOST or HS_OUT_DEVICE).  dictionary != 0: low-cardinality
 * columns (v1, v3, v4) are PLAIN_DICTIONARY-encoded like a parquet-mr / pyarrow writer would; 0: PLAIN only. */
int hs_synth_table(hs_ctx* ctx, int64_t first_row, int64_t nrows, int32_t ncols, int32_t n_files,
                   int32_t row_groups_per_file, int32_t dictionary, int32_t output, hs_index_result** out, char* err,
                   size_t errlen);
/* the same with a page codec (HS_CODEC_*): the SNAPPY variant of T that SURVEY.md 8d asks for */
int hs_synth_table_ex(hs_ctx* ctx, int64_t first_row, int64_t nrows, int32_t ncols, int32_t n_files,
                      int32_t row_groups_per_file, int32_t dictionary, int32_t compression, int32_t output,
                      hs_index_result** out, char* err, size_t errlen);
/* Snappy-compresses n bytes of host memory on the GPU (the page compressor, fragment by fragment) into out (capacity cap);
 * kernel-level entry point for the parity tests: any Snappy decoder must give the input back. */
int hs_k_snappy_compress(hs_ctx* ctx, const void* in, uint64_t n, void* out, uint64_t cap, uint64_t* out_len, char* err,
                         size_t errlen);
/* The page decompressor on one raw Snappy stream of n bytes whose uncompressed length is out_len (Parquet's page header
 * carries it); *sequential = 1 when the stream's 64 KB blocks were not independent and one warp decoded it front to back.
 * HS_EFORMAT for a damaged stream.  Kernel-level entry point for the parity tests. */
int hs_k_snappy_decompress(hs_ctx* ctx, const void* in, uint64_t n, void* out, uint64_t out_len, int32_t* sequential, char* err,
                           size_t errlen);
/* The GZIP page decompressor (k_inflate) on one page body of n bytes -- one or more gzip members -- whose uncompressed
 * length is out_len.  HS_EFORMAT for a damaged stream; the message names the failed check.  Kernel-level entry point for
 * the parity tests. */
int hs_k_inflate(hs_ctx* ctx, const void* in, uint64_t n, void* out, uint64_t out_len, char* err, size_t errlen);
/* The LZ4 page decompressor (k_lz4) on one page body of n bytes whose uncompressed length is out_len: codec 7 (LZ4_RAW,
 * one block) or 5 (LZ4: Hadoop-framed blocks, or one raw block); any other codec is HS_EINVAL.  HS_EFORMAT for a damaged
 * body; the message names the failed check.  Kernel-level entry point for the parity tests. */
int hs_k_lz4(hs_ctx* ctx, int32_t codec, const void* in, uint64_t n, void* out, uint64_t out_len, char* err, size_t errlen);
/* The page decompressors over several blobs of one host buffer `in` (n_in bytes) in one launch, as the page reader makes
 * it.  Blob i is src_len[i] bytes at src_off[i] of `in`, decoded into dst_len[i] bytes at dst_off[i] of `out` (out_len
 * bytes); codec[i] is HS_CODEC_SNAPPY, HS_CODEC_GZIP, HS_CODEC_LZ4 or 7 (LZ4_RAW).  Its first prefix[i] bytes are stored
 * verbatim (a v2 page's level bytes); compressed[i] = 0 stores the blob whole.  Source and destination ranges must lie
 * in their buffers and destination ranges must not overlap (else HS_EINVAL).  The whole of `out` is first filled with the
 * byte `fill`, so bytes outside the destination ranges come back as `fill` unless a decoder strayed.  sequential
 * (optional, n_blobs entries): 1 where a snappy stream was decoded front to back by one lane.  HS_EFORMAT for a damaged
 * blob; the message names the codec and the failed check.  Kernel-level entry point for the decoder tests. */
int hs_k_decompress_blobs(hs_ctx* ctx, const void* in, uint64_t n_in, int32_t n_blobs, const uint64_t* src_off,
                          const uint32_t* src_len, const uint64_t* dst_off, const uint32_t* dst_len, const uint32_t* prefix,
                          const int32_t* compressed, const int32_t* codec, int32_t fill, void* out, uint64_t out_len,
                          int32_t* sequential, char* err, size_t errlen);
/* The page compressor of index builds on one page body of n bytes, through the same path as the encoder: codec HS_CODEC_GZIP
 * (one gzip member) or HS_CODEC_LZ4 (Hadoop-framed blocks, one per 64 KB); any other codec is HS_EINVAL.  *out_len is the
 * compressed size; HS_ENOMEM when it exceeds cap.  Kernel-level entry point for the parity tests. */
int hs_k_compress(hs_ctx* ctx, int32_t codec, const void* in, uint64_t n, void* out, uint64_t cap, uint64_t* out_len, char* err,
                  size_t errlen);

#ifdef __cplusplus
}
#endif
#endif /* HS_GPU_H */
