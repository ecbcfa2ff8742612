"""ctypes binding of libhs_gpu.so (the C ABI in include/hs_gpu.h).

This is the Python counterpart of the JNI stub shown in INTEGRATION.md.  There is no CPU fallback: if the shared
library is missing, or no CUDA device is visible, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import datetime
import decimal
import os
import weakref
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# HS_GPU_LIB: load another build of the same library (kernel A/B experiments); there is still no CPU fallback
LIB_PATH = os.environ.get("HS_GPU_LIB") or os.path.join(_HERE, "lib", "libhs_gpu.so")

HS_OK, HS_EINVAL, HS_ENODEVICE, HS_ECUDA, HS_EFORMAT, HS_EIO, HS_EUNSUPPORTED, HS_ENOMEM, HS_ECOMM = 0, -1, -2, -3, -4, -5, -6, -7, -8
HS_TYPE_INT32, HS_TYPE_INT64, HS_TYPE_FLOAT, HS_TYPE_DOUBLE, HS_TYPE_BOOL, HS_TYPE_STRING = range(6)
HS_TYPE_DECIMAL = 6  # predicate literals only: unscaled value in lo_i / hi_i, scale in `scale`
HS_SAVE_OVERWRITE, HS_SAVE_APPEND = 0, 1
HS_OUT_FILES, HS_OUT_HOST, HS_OUT_DEVICE = 0, 1, 2
# hs_predicate_any.flags
HS_TERM_NOT, HS_TERM_NULL_TRUE, HS_TERM_NULL_FALSE = 1, 2, 4
HS_TERM_STARTS_WITH, HS_TERM_ENDS_WITH, HS_TERM_CONTAINS, HS_TERM_LIKE = 8, 16, 32, 64
# hs_column_compare.op
HS_CMP_LT, HS_CMP_LE, HS_CMP_GT, HS_CMP_GE, HS_CMP_EQ, HS_CMP_EQ_NULL_SAFE = 1, 2, 3, 4, 5, 6
CMP_OPS = {"<": HS_CMP_LT, "<=": HS_CMP_LE, ">": HS_CMP_GT, ">=": HS_CMP_GE, "=": HS_CMP_EQ, "<=>": HS_CMP_EQ_NULL_SAFE}
HS_JOIN_LEFT_SEMI, HS_JOIN_LEFT_ANTI = 1, 2  # join_type of hs_bucket_join_exists
JOIN_TYPES = {"semi": HS_JOIN_LEFT_SEMI, "anti": HS_JOIN_LEFT_ANTI}
HS_JOIN_LEFT_OUTER, HS_JOIN_RIGHT_OUTER, HS_JOIN_FULL_OUTER = 3, 4, 5  # join_type of hs_bucket_join_outer
OUTER_JOIN_TYPES = {"left": HS_JOIN_LEFT_OUTER, "right": HS_JOIN_RIGHT_OUTER, "full": HS_JOIN_FULL_OUTER}
HS_JOIN_INNER = 0  # join_type of hs_bucket_join_expr, besides the five above
ALL_JOIN_TYPES = {"inner": HS_JOIN_INNER, **JOIN_TYPES, **OUTER_JOIN_TYPES}
# hs_expr_node.kind
HS_EXPR_COLUMN, HS_EXPR_LITERAL, HS_EXPR_ADD, HS_EXPR_SUB, HS_EXPR_MUL, HS_EXPR_DIV, HS_EXPR_REM, HS_EXPR_NEG = range(1, 9)
EXPR_OPS = {"+": HS_EXPR_ADD, "-": HS_EXPR_SUB, "*": HS_EXPR_MUL, "/": HS_EXPR_DIV, "%": HS_EXPR_REM, "neg": HS_EXPR_NEG}
# the function kinds, HS_EXPR_YEAR (9) .. HS_EXPR_COALESCE (25), by their Spark names
EXPR_FUNCS = {name: 9 + k for k, name in enumerate(
    ("year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute", "second", "date_add",
     "date_sub", "datediff", "length", "substring", "abs", "coalesce"))}
HS_EXPR_COALESCE = EXPR_FUNCS["coalesce"]
HS_TYPE_DATE, HS_TYPE_TIMESTAMP = 7, 8  # expression literals only
HS_CODEC_UNCOMPRESSED, HS_CODEC_SNAPPY, HS_CODEC_GZIP, HS_CODEC_LZ4 = 0, 1, 2, 5
HS_KEY_DECIMAL = 1  # hs_host_column.reserved of a decimal key column
PARTITION_MODES = {"local": 0, "owner": 1, "peer": 2}  # hs_k_partition's HS_PART_*

_NP_OF_TYPE = {HS_TYPE_INT32: np.int32, HS_TYPE_INT64: np.int64, HS_TYPE_FLOAT: np.float32, HS_TYPE_DOUBLE: np.float64,
               HS_TYPE_BOOL: np.uint8}
_TYPE_OF_NP = {np.dtype(np.int32): HS_TYPE_INT32, np.dtype(np.int64): HS_TYPE_INT64, np.dtype(np.float32): HS_TYPE_FLOAT,
               np.dtype(np.float64): HS_TYPE_DOUBLE, np.dtype(np.bool_): HS_TYPE_BOOL, np.dtype(np.uint8): HS_TYPE_BOOL}


class HyperspaceGpuError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libhs_gpu error {code}: {message}")
        self.code = code
        self.message = message


class SourceFile(C.Structure):
    _fields_ = [("path", C.c_char_p), ("data", C.c_void_p), ("size", C.c_uint64), ("file_id", C.c_int64),
                ("on_device", C.c_int32), ("reserved", C.c_int32)]


class IndexSpec(C.Structure):
    _fields_ = [("files", C.POINTER(SourceFile)), ("n_files", C.c_int32),
                ("indexed_columns", C.POINTER(C.c_char_p)), ("n_indexed", C.c_int32),
                ("included_columns", C.POINTER(C.c_char_p)), ("n_included", C.c_int32),
                ("num_buckets", C.c_int32), ("save_mode", C.c_int32), ("output", C.c_int32), ("lineage", C.c_int32),
                ("out_dir", C.c_char_p), ("job_uuid", C.c_char_p),
                ("rows_per_page", C.c_int64), ("rows_per_row_group", C.c_int64),
                ("deleted_file_ids", C.POINTER(C.c_int64)), ("n_deleted_file_ids", C.c_int32), ("disable_dictionary", C.c_int32),
                ("compression", C.c_int32), ("reserved", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("rows_in", C.c_int64), ("rows_out", C.c_int64), ("bytes_in", C.c_int64), ("bytes_out", C.c_int64),
                ("bytes_exchanged", C.c_int64), ("files_out", C.c_int32), ("gpu_launches", C.c_int32),
                ("ms_total", C.c_float), ("ms_h2d", C.c_float), ("ms_plan", C.c_float), ("ms_decode", C.c_float),
                ("ms_hash", C.c_float), ("ms_partition", C.c_float), ("ms_exchange", C.c_float), ("ms_sort", C.c_float),
                ("ms_gather", C.c_float), ("ms_encode", C.c_float), ("ms_d2h", C.c_float), ("ms_write", C.c_float)]

    def as_dict(self) -> Dict[str, float]:
        return {n: getattr(self, n) for n, _ in self._fields_}


class ScanSpec(C.Structure):
    _fields_ = [("files", C.POINTER(SourceFile)), ("n_files", C.c_int32), ("sorted_on_key", C.c_int32),
                ("key_column", C.c_char_p), ("projected_columns", C.POINTER(C.c_char_p)), ("n_projected", C.c_int32),
                ("has_lo", C.c_int32), ("has_hi", C.c_int32), ("lo", C.c_int64), ("hi", C.c_int64),
                ("deleted_file_ids", C.POINTER(C.c_int64)), ("n_deleted_file_ids", C.c_int32), ("output", C.c_int32),
                ("lo_bytes", C.c_char_p), ("hi_bytes", C.c_char_p), ("lo_len", C.c_uint32), ("hi_len", C.c_uint32)]


class PredicateSpec(C.Structure):
    _fields_ = [("column", C.c_char_p), ("literal_type", C.c_int32), ("has_lo", C.c_int32), ("has_hi", C.c_int32),
                ("lo_strict", C.c_int32), ("hi_strict", C.c_int32), ("scale", C.c_int32),
                ("lo_i", C.c_int64), ("hi_i", C.c_int64), ("lo_f", C.c_double), ("hi_f", C.c_double),
                ("lo_bytes", C.c_char_p), ("hi_bytes", C.c_char_p), ("lo_len", C.c_uint32), ("hi_len", C.c_uint32)]


class PredicateAnySpec(C.Structure):
    _fields_ = [("column", C.c_char_p), ("literal_type", C.c_int32), ("scale", C.c_int32), ("n_values", C.c_int64),
                ("values_i", C.c_void_p), ("values_f", C.c_void_p), ("values_bytes", C.c_void_p), ("values_offsets", C.c_void_p),
                ("ranges", C.POINTER(PredicateSpec)), ("n_ranges", C.c_int32), ("flags", C.c_int32)]


class ColumnCompareSpec(C.Structure):
    _fields_ = [("left", C.c_char_p), ("right", C.c_char_p), ("op", C.c_int32), ("flags", C.c_int32)]


class ExprNodeSpec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_char_p), ("literal_type", C.c_int32), ("scale", C.c_int32),
                ("value_i", C.c_int64), ("value_f", C.c_double)]


class ExprCompareSpec(C.Structure):
    _fields_ = [("left", C.POINTER(ExprNodeSpec)), ("n_left", C.c_int32), ("right", C.POINTER(ExprNodeSpec)),
                ("n_right", C.c_int32), ("op", C.c_int32), ("flags", C.c_int32)]


class JoinSpec(C.Structure):
    _fields_ = [("left_files", C.POINTER(SourceFile)), ("n_left", C.c_int32),
                ("right_files", C.POINTER(SourceFile)), ("n_right", C.c_int32),
                ("left_buckets", C.POINTER(C.c_int32)), ("right_buckets", C.POINTER(C.c_int32)),
                ("num_buckets", C.c_int32), ("output", C.c_int32),
                ("left_key", C.c_char_p), ("right_key", C.c_char_p),
                ("left_columns", C.POINTER(C.c_char_p)), ("n_left_columns", C.c_int32),
                ("right_columns", C.POINTER(C.c_char_p)), ("n_right_columns", C.c_int32)]


class VerifyReport(C.Structure):
    _fields_ = [("rows", C.c_int64), ("bucket_mismatches", C.c_int64), ("order_violations", C.c_int64),
                ("row_checksum", C.c_uint64), ("column_checksum", C.c_uint64 * 16), ("n_columns", C.c_int32),
                ("reserved", C.c_int32)]

    def as_dict(self) -> Dict[str, object]:
        return {"rows": self.rows, "bucket_mismatches": self.bucket_mismatches, "order_violations": self.order_violations,
                "row_checksum": int(self.row_checksum),
                "column_checksum": [int(self.column_checksum[i]) for i in range(self.n_columns)]}


class HostColumn(C.Structure):
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("data", C.c_void_p), ("valid", C.c_void_p)]


# every symbol include/hs_gpu.h declares; tests/test_abi.py checks the library exports all of them
EXPORTED_SYMBOLS = [
    "hs_abi_version", "hs_build_info", "hs_init", "hs_shutdown", "hs_trim", "hs_host_alloc", "hs_host_free", "hs_profile_enable", "hs_profile_report",
    "hs_comm_unique_id", "hs_comm_init", "hs_create_index", "hs_result_num_files", "hs_result_file", "hs_result_free",
    "hs_filter_scan", "hs_bucket_join", "hs_batch_num_rows", "hs_batch_on_device", "hs_batch_num_columns", "hs_batch_column", "hs_batch_free",
    "hs_k_bucket_ids", "hs_k_sort_perm", "hs_synth_table",
    "hs_stage_sources", "hs_staged_num_files", "hs_staged_file", "hs_staged_wait", "hs_staged_free",
    "hs_create_index_async", "hs_pending_wait", "hs_pending_cancel", "hs_verify_index", "hs_synth_checksum",
    "hs_synth_table_ex", "hs_k_snappy_compress", "hs_k_snappy_decompress", "hs_batch_string_offsets", "hs_filter_scan_where",
    "hs_bucket_join_where", "hs_k_inflate", "hs_filter_scan_any", "hs_bucket_join_any", "hs_k_lz4", "hs_k_compress",
    "hs_filter_scan_cmp", "hs_bucket_join_cmp", "hs_bucket_join_exists", "hs_bucket_join_outer", "hs_filter_scan_expr",
    "hs_bucket_join_expr", "hs_k_partition", "hs_k_decompress_blobs",
]

_lib: Optional[C.CDLL] = None


def load_library() -> C.CDLL:
    """Loads libhs_gpu.so; raises if it has not been built (``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise HyperspaceGpuError(HS_ENODEVICE, f"{LIB_PATH} is missing: build it with __graft_entry__.build(); "
                                               "there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    err = (C.c_char_p, C.c_size_t)
    L.hs_abi_version.restype = C.c_int
    L.hs_build_info.restype = C.c_char_p
    L.hs_init.restype = C.c_int
    L.hs_init.argtypes = [C.c_int, C.c_void_p, C.POINTER(C.c_void_p), *err]
    L.hs_shutdown.restype = None
    L.hs_shutdown.argtypes = [C.c_void_p]
    L.hs_trim.restype = None
    L.hs_trim.argtypes = [C.c_void_p]
    L.hs_host_alloc.restype = C.c_void_p
    L.hs_host_alloc.argtypes = [C.c_void_p, C.c_size_t]
    L.hs_host_free.restype = None
    L.hs_host_free.argtypes = [C.c_void_p, C.c_void_p]
    L.hs_profile_enable.restype = None
    L.hs_profile_enable.argtypes = [C.c_void_p, C.c_int]
    L.hs_profile_report.restype = C.c_int
    L.hs_profile_report.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.hs_comm_unique_id.restype = C.c_int
    L.hs_comm_unique_id.argtypes = [C.c_void_p, *err]
    L.hs_comm_init.restype = C.c_int
    L.hs_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, *err]
    L.hs_create_index.restype = C.c_int
    L.hs_create_index.argtypes = [C.c_void_p, C.POINTER(IndexSpec), C.POINTER(C.c_void_p), C.POINTER(Stats), *err]
    L.hs_result_num_files.restype = C.c_int32
    L.hs_result_num_files.argtypes = [C.c_void_p]
    L.hs_result_file.restype = C.c_int
    L.hs_result_file.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_char_p), C.POINTER(C.c_void_p),
                                 C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]
    L.hs_result_free.restype = None
    L.hs_result_free.argtypes = [C.c_void_p]
    # the read-side calls, from the parameter groups of include/hs_gpu.h: scan head, join head, one side's filter
    # (predicates, terms, comparisons, expression comparisons: a call takes the first one, two, three or all four), the
    # files' buckets, outputs
    scan = [C.c_void_p, C.POINTER(ScanSpec)]
    join = [C.c_void_p, C.POINTER(JoinSpec), C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_int32]
    side_x = [C.POINTER(PredicateSpec), C.c_int32, C.POINTER(PredicateAnySpec), C.c_int32, C.POINTER(ColumnCompareSpec), C.c_int32,
              C.POINTER(ExprCompareSpec), C.c_int32]
    side = side_x[:6]
    buckets = [C.c_void_p, C.c_int32]
    out = [C.POINTER(C.c_void_p), C.POINTER(Stats), *err]
    for name, args in (("hs_filter_scan", [*scan, *out]),
                       ("hs_filter_scan_where", [*scan, *side[:2], *out]),
                       ("hs_filter_scan_any", [*scan, *side[:4], *buckets, *out]),
                       ("hs_filter_scan_cmp", [*scan, *side, *buckets, *out]),
                       ("hs_bucket_join", [*join[:2], *out]),
                       ("hs_bucket_join_where", [*join, *side[:2], *side[:2], *out]),
                       ("hs_bucket_join_any", [*join, *side[:4], *side[:4], *out]),
                       ("hs_bucket_join_cmp", [*join, *side, *side, *out]),
                       ("hs_bucket_join_exists", [*join[:2], C.c_int32, *join[2:], *side, *side, *out]),
                       ("hs_bucket_join_outer", [*join[:2], C.c_int32, *join[2:], *side, *side, *out]),
                       ("hs_filter_scan_expr", [*scan, *side_x, *buckets, *out]),
                       ("hs_bucket_join_expr", [*join[:2], C.c_int32, *join[2:], *side_x, *side_x, *out])):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = args
    L.hs_batch_num_rows.restype = C.c_int64
    L.hs_batch_num_rows.argtypes = [C.c_void_p]
    L.hs_batch_on_device.restype = C.c_int32
    L.hs_batch_on_device.argtypes = [C.c_void_p]
    L.hs_batch_num_columns.restype = C.c_int32
    L.hs_batch_num_columns.argtypes = [C.c_void_p]
    L.hs_batch_column.restype = C.c_int
    L.hs_batch_column.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.POINTER(C.c_void_p),
                                  C.POINTER(C.c_void_p)]
    L.hs_batch_free.restype = None
    L.hs_batch_free.argtypes = [C.c_void_p]
    L.hs_k_bucket_ids.restype = C.c_int
    L.hs_k_bucket_ids.argtypes = [C.c_void_p, C.POINTER(HostColumn), C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, *err]
    L.hs_k_sort_perm.restype = C.c_int
    L.hs_k_sort_perm.argtypes = [C.c_void_p, C.POINTER(HostColumn), C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, *err]
    L.hs_k_partition.restype = C.c_int
    L.hs_k_partition.argtypes = [C.c_void_p, C.POINTER(HostColumn), C.c_int32, C.c_int64, C.c_int32, C.POINTER(HostColumn), C.c_int32,
                                 C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, *err]
    L.hs_synth_table.restype = C.c_int
    L.hs_synth_table.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.POINTER(C.c_void_p), *err]
    L.hs_stage_sources.restype = C.c_int
    L.hs_stage_sources.argtypes = [C.c_void_p, C.POINTER(SourceFile), C.c_int32, C.POINTER(C.c_void_p), *err]
    L.hs_staged_num_files.restype = C.c_int32
    L.hs_staged_num_files.argtypes = [C.c_void_p]
    L.hs_staged_file.restype = C.c_int
    L.hs_staged_file.argtypes = [C.c_void_p, C.c_int32, C.POINTER(SourceFile)]
    L.hs_staged_wait.restype = C.c_int
    L.hs_staged_wait.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.hs_staged_free.restype = None
    L.hs_staged_free.argtypes = [C.c_void_p]
    L.hs_create_index_async.restype = C.c_int
    L.hs_create_index_async.argtypes = [C.c_void_p, C.POINTER(IndexSpec), C.POINTER(C.c_void_p), *err]
    L.hs_pending_wait.restype = C.c_int
    L.hs_pending_wait.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(Stats), *err]
    L.hs_pending_cancel.restype = None
    L.hs_pending_cancel.argtypes = [C.c_void_p]
    L.hs_verify_index.restype = C.c_int
    L.hs_verify_index.argtypes = [C.c_void_p, C.POINTER(SourceFile), C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_char_p), C.c_int32,
                                  C.POINTER(C.c_char_p), C.c_int32, C.c_int32, C.POINTER(VerifyReport), *err]
    L.hs_synth_checksum.restype = C.c_int
    L.hs_synth_checksum.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(VerifyReport), *err]
    L.hs_synth_table_ex.restype = C.c_int
    L.hs_synth_table_ex.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.POINTER(C.c_void_p), *err]
    L.hs_k_snappy_compress.restype = C.c_int
    L.hs_k_snappy_compress.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), *err]
    L.hs_batch_string_offsets.restype = C.c_int
    L.hs_batch_string_offsets.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    L.hs_k_snappy_decompress.restype = C.c_int
    L.hs_k_snappy_decompress.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_int32), *err]
    L.hs_k_inflate.restype = C.c_int
    L.hs_k_inflate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, *err]
    L.hs_k_lz4.restype = C.c_int
    L.hs_k_lz4.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, *err]
    L.hs_k_decompress_blobs.restype = C.c_int
    L.hs_k_decompress_blobs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_int32), *err]
    L.hs_k_compress.restype = C.c_int
    L.hs_k_compress.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), *err]
    if L.hs_abi_version() != 1:
        raise HyperspaceGpuError(HS_EINVAL, f"ABI version mismatch: library {L.hs_abi_version()}, binding 1")
    _lib = L
    return L


def _check(rc: int, err) -> None:
    if rc != HS_OK:
        raise HyperspaceGpuError(rc, err.value.decode("utf-8", "replace"))


def _cstr_array(names: Sequence[str]):
    arr = (C.c_char_p * max(1, len(names)))()
    for i, n in enumerate(names):
        arr[i] = n.encode()
    return arr


@dataclass
class FileImage:
    """One Parquet file handed to the engine: a path, or an in-memory image (host bytes / numpy uint8 / device pointer)."""
    path: Optional[str] = None
    data: Optional[object] = None   # bytes, numpy uint8 array, or int (raw pointer)
    size: int = 0
    file_id: int = -1
    on_device: bool = False


_EPOCH = datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc)


def timestamp_micros(v: datetime.datetime) -> int:
    """A Spark timestamp literal's value: microseconds since the epoch (a naive datetime is UTC)."""
    if v.tzinfo is None:
        v = v.replace(tzinfo=datetime.timezone.utc)
    return (v - _EPOCH) // datetime.timedelta(microseconds=1)


def decimal_unscaled(v: decimal.Decimal) -> Tuple[int, int]:
    """(unscaled value, scale) of a finite decimal literal; the unscaled value must fit in 64 bits."""
    if not v.is_finite():
        raise ValueError(f"decimal literal {v} is not finite")
    sign, digits, exp = v.as_tuple()
    unscaled = int("".join(map(str, digits)) or "0") * (-1 if sign else 1)
    if exp > 0:
        unscaled, exp = unscaled * 10 ** exp, 0
    if not -2**63 <= unscaled < 2**63:
        raise ValueError(f"decimal literal {v} has more than 18 significant digits")
    return unscaled, -exp


def _literal_type(lo, hi) -> int:
    """HS_TYPE_* of a predicate's literals: str / bytes -> string, int / datetime -> long (it must fit in 64 bits; a datetime
    is a timestamp's micros), float -> double, decimal.Decimal -> decimal (an int beside a Decimal is a decimal of scale 0)."""
    kinds = set()
    for v in (lo, hi):
        if v is None:
            continue
        if isinstance(v, (bool, np.bool_)):
            raise ValueError("a boolean literal cannot bound a range")
        if isinstance(v, datetime.datetime):
            kinds.add(HS_TYPE_INT64)
        elif isinstance(v, decimal.Decimal):
            decimal_unscaled(v)
            kinds.add(HS_TYPE_DECIMAL)
        elif isinstance(v, (str, bytes, bytearray)):
            kinds.add(HS_TYPE_STRING)
        elif isinstance(v, (int, np.integer)):
            if not -2**63 <= int(v) < 2**63:
                raise ValueError(f"integer literal {v} does not fit in a long")
            kinds.add(HS_TYPE_INT64)
        elif isinstance(v, (float, np.floating)):
            kinds.add(HS_TYPE_DOUBLE)
        else:
            raise ValueError(f"unsupported literal {v!r}")
    if not kinds:
        raise ValueError("a predicate needs a lower or an upper bound")
    if HS_TYPE_STRING in kinds and len(kinds) > 1:
        raise ValueError("a predicate cannot mix string and numeric bounds")
    if HS_TYPE_DOUBLE in kinds:
        return HS_TYPE_DOUBLE
    return HS_TYPE_DECIMAL if HS_TYPE_DECIMAL in kinds else kinds.pop()


def _predicate_array(predicates: Sequence[tuple]):
    """``(column, lo, lo_strict, hi, hi_strict)`` tuples -> (hs_predicate array, count).  A range whose two bounds are
    literals of different numeric types (int and float, decimal and float, int and decimal), or decimals of different
    scales, becomes two comparisons, each in its own type."""
    split = []
    for column, lo, lo_strict, hi, hi_strict in predicates:
        kinds = {_literal_type(lo, None), _literal_type(None, hi)} if lo is not None and hi is not None else set()
        mixed = len(kinds) == 2 and HS_TYPE_STRING not in kinds
        if kinds == {HS_TYPE_DECIMAL}:
            mixed = decimal_unscaled(lo)[1] != decimal_unscaled(hi)[1]
        if mixed:
            split += [(column, lo, lo_strict, None, False), (column, None, False, hi, hi_strict)]
        else:
            split.append((column, lo, lo_strict, hi, hi_strict))
    preds = (PredicateSpec * max(1, len(split)))()
    for p, (column, lo, lo_strict, hi, hi_strict) in zip(preds, split):
        p.column = column.encode()
        p.literal_type = _literal_type(lo, hi)
        p.has_lo, p.has_hi = int(lo is not None), int(hi is not None)
        p.lo_strict, p.hi_strict = int(bool(lo_strict)), int(bool(hi_strict))
        for side, v in (("lo", lo), ("hi", hi)):
            if v is None:
                continue
            if p.literal_type == HS_TYPE_STRING:
                b = v.encode("utf-8") if isinstance(v, str) else bytes(v)
                setattr(p, side + "_bytes", b)
                setattr(p, side + "_len", len(b))
            elif p.literal_type == HS_TYPE_INT64:
                setattr(p, side + "_i", timestamp_micros(v) if isinstance(v, datetime.datetime) else int(v))
            elif p.literal_type == HS_TYPE_DECIMAL:  # one scale per predicate: bounds of two scales were split above
                unscaled, p.scale = decimal_unscaled(decimal.Decimal(v))
                setattr(p, side + "_i", unscaled)
            else:
                setattr(p, side + "_f", float(v))
    return preds, len(split)


def any_values(values) -> Tuple[int, int, object]:
    """The listed values of an IN term as (HS_TYPE_* literal type, decimal scale, values): an int64 or float64 numpy array,
    or a list of bytes for strings.  None is dropped.  Spark casts the list to its widest type: a float among numbers
    makes every value a double; a Decimal among ints makes every value a decimal, all brought to the largest scale
    exactly; datetimes are timestamps' micros (longs).  Numpy int / float arrays pass without a Python object per value.
    Raises ValueError for strings mixed with numbers and for booleans or other values."""
    if isinstance(values, np.ndarray) and values.dtype.kind in "iu":
        return HS_TYPE_INT64, 0, np.ascontiguousarray(values, dtype=np.int64)
    if isinstance(values, np.ndarray) and values.dtype.kind == "f":
        return HS_TYPE_DOUBLE, 0, np.ascontiguousarray(values, dtype=np.float64)
    if isinstance(values, np.ndarray) and values.dtype.kind == "b":
        raise ValueError("a boolean list cannot be compared")
    vals = [v for v in (values.tolist() if isinstance(values, np.ndarray) else values) if v is not None]
    kinds = set()
    for v in vals:
        if isinstance(v, (bool, np.bool_)):
            raise ValueError("a boolean literal cannot be listed in IN")
        if isinstance(v, (str, bytes, bytearray, np.str_, np.bytes_)):
            kinds.add("s")
        elif isinstance(v, (float, np.floating)):
            kinds.add("f")
        elif isinstance(v, decimal.Decimal):
            kinds.add("d")
        elif isinstance(v, (int, np.integer, datetime.datetime)):
            kinds.add("i")
        else:
            raise ValueError(f"unsupported literal {v!r} in IN")
    if "s" in kinds and len(kinds) > 1:
        raise ValueError("an IN list cannot mix string and numeric values")
    if "s" in kinds:
        return HS_TYPE_STRING, 0, [v.encode("utf-8") if isinstance(v, str) else bytes(v) for v in vals]
    ints = [timestamp_micros(v) if isinstance(v, datetime.datetime) else v for v in vals]
    if "f" in kinds:
        return HS_TYPE_DOUBLE, 0, np.array([float(v) for v in ints], dtype=np.float64)
    if "d" in kinds:
        scale = max(decimal_unscaled(v)[1] for v in ints if isinstance(v, decimal.Decimal))
        out = []
        for v in ints:
            unscaled, sc = decimal_unscaled(v) if isinstance(v, decimal.Decimal) else (int(v), 0)
            unscaled *= 10 ** (scale - sc)
            if not -2**63 <= unscaled < 2**63:
                raise ValueError(f"decimal literal {v} has more than 18 significant digits at scale {scale}")
            out.append(unscaled)
        return HS_TYPE_DECIMAL, scale, np.array(out, dtype=np.int64)
    for v in ints:
        if not -2**63 <= int(v) < 2**63:
            raise ValueError(f"integer literal {v} does not fit in a long")
    return HS_TYPE_INT64, 0, np.array([int(v) for v in ints], dtype=np.int64)


def _one_literal_type(lo, hi):
    """The bounds of one range of a disjunction as literals of one type: decimals (and an int beside a decimal) at the
    larger of their scales, exactly; other mixes are left for _predicate_array to refuse."""
    if lo is None or hi is None or not ({type(lo), type(hi)} & {decimal.Decimal}):
        return lo, hi
    if any(isinstance(v, (float, np.floating)) for v in (lo, hi)):
        return lo, hi
    lo, hi = decimal.Decimal(lo), decimal.Decimal(hi)
    scale = max(decimal_unscaled(lo)[1], decimal_unscaled(hi)[1])
    q = decimal.Decimal(1).scaleb(-scale)
    return lo.quantize(q), hi.quantize(q)


def _any_array(terms: Sequence[tuple]):
    """``(column, values, ranges)`` or ``(column, values, ranges, flags)`` terms -> (hs_predicate_any array, count, buffers
    to keep alive).  values go through any_values; ranges are ``(lo, lo_strict, hi, hi_strict)`` tuples with
    _predicate_array's literal typing; flags are HS_TERM_* (a pattern term lists its pattern as its one value)."""
    keep = []
    arr = (PredicateAnySpec * max(1, len(terms)))()
    for a, (column, values, ranges, *flags) in zip(arr, terms):
        a.column = column.encode()
        a.flags = flags[0] if flags else 0
        lt, scale, vals = any_values(values)
        a.literal_type, a.scale, a.n_values = lt, scale, len(vals)
        if lt == HS_TYPE_STRING:
            offs = np.zeros(len(vals) + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(v) for v in vals], dtype=np.uint64) if vals else []
            blob = np.frombuffer(b"".join(vals) or b"\0", dtype=np.uint8)
            keep += [offs, blob]
            a.values_bytes, a.values_offsets = blob.ctypes.data, offs.ctypes.data
        else:
            keep.append(vals)
            if lt == HS_TYPE_DOUBLE:
                a.values_f = vals.ctypes.data
            else:
                a.values_i = vals.ctypes.data
        ranges = [(lo, ls, hi, hs) for (lo, hi), (_, ls, _, hs) in ((_one_literal_type(r[0], r[2]), r) for r in ranges)]
        rp, nr = _predicate_array([(column, lo, ls, hi, hs) for lo, ls, hi, hs in ranges])
        if nr != len(ranges):
            raise ValueError("a range of an OR must have bounds of one literal type")
        keep.append(rp)
        a.ranges, a.n_ranges = rp, nr
    return arr, len(terms), keep


def _cmp_array(compares: Sequence[tuple]):
    """``(left, op, right)`` or ``(left, op, right, flags)`` comparisons -> (hs_column_compare array, count, names to keep
    alive).  op is one of CMP_OPS's keys ("<", "<=", ">", ">=", "=", "<=>") or an HS_CMP_* code; flags is 0 or HS_TERM_NOT."""
    keep = []
    arr = (ColumnCompareSpec * max(1, len(compares)))()
    for c, (left, op, right, *flags) in zip(arr, compares):
        names = [n.encode() if n is not None else None for n in (left, right)]
        keep += names
        c.left, c.right = names
        c.op = CMP_OPS[op] if isinstance(op, str) else op
        c.flags = flags[0] if flags else 0
    return arr, len(compares), keep


def expr_literal(v) -> Tuple[int, int, int, float]:
    """A Python literal of an expression as (literal_type, scale, value_i, value_f), as py4j hands it to Spark: an int that
    fits in 32 bits is an int, a larger one a long; a float is a double; a Decimal is a decimal of its own scale (its
    unscaled value must fit in 64 bits).  bool and anything else raise ValueError."""
    if isinstance(v, (bool, np.bool_)):
        raise ValueError(f"a boolean literal ({v!r}) cannot be used in arithmetic")
    if isinstance(v, (int, np.integer)):
        v = int(v)
        if not -2**63 <= v < 2**63:
            raise ValueError(f"the integer literal {v} does not fit in a long")
        return (HS_TYPE_INT32 if -2**31 <= v < 2**31 else HS_TYPE_INT64), 0, v, 0.0
    if isinstance(v, (float, np.floating)):
        return HS_TYPE_DOUBLE, 0, 0, float(v)
    if isinstance(v, decimal.Decimal):
        if not v.is_finite():
            raise ValueError(f"the decimal literal {v} is not finite")
        sign, digits, exp = v.as_tuple()
        scale = max(0, -exp)
        unscaled = int(v.scaleb(scale))
        if not -2**63 <= unscaled < 2**63:
            raise ValueError(f"the decimal literal {v} has more than 18 digits")
        return HS_TYPE_DECIMAL, scale, unscaled, 0.0
    raise ValueError(f"the literal {v!r} cannot be used in arithmetic")


def _expr_nodes(nodes: Sequence[tuple]):
    """One side of an expression comparison, postfix: ``("column", name)``, ``("literal", value)`` (typed by expr_literal;
    str and bytes are HS_TYPE_STRING literals, datetime.date HS_TYPE_DATE days and datetime.datetime HS_TYPE_TIMESTAMP
    micros), an operator ``(op,)`` with op one of EXPR_OPS's keys ("+", "-", "*", "/", "%", "neg") or EXPR_FUNCS's
    ("year" .. "abs"), ``("coalesce", n)``, or an HS_EXPR_* code; a raw ``(kind, column, literal_type, scale, value_i,
    value_f)`` tuple passes as it is.  Returns (array, count, keep)."""
    keep = []
    arr = (ExprNodeSpec * max(1, len(nodes)))()
    for x, node in zip(arr, nodes):
        tag = node[0]
        if tag == "column":
            name = node[1].encode() if node[1] is not None else None
            keep.append(name)
            x.kind, x.column = HS_EXPR_COLUMN, name
        elif tag == "literal" and isinstance(node[1], (str, bytes)):
            b = node[1].encode("utf-8") if isinstance(node[1], str) else bytes(node[1])
            buf = C.create_string_buffer(b, max(1, len(b)))
            keep.append(buf)
            x.kind, x.literal_type, x.value_i = HS_EXPR_LITERAL, HS_TYPE_STRING, len(b)
            x.column = C.addressof(buf)
        elif tag == "literal" and isinstance(node[1], datetime.datetime):
            x.kind, x.literal_type, x.value_i = HS_EXPR_LITERAL, HS_TYPE_TIMESTAMP, timestamp_micros(node[1])
        elif tag == "literal" and isinstance(node[1], datetime.date):
            x.kind, x.literal_type, x.value_i = HS_EXPR_LITERAL, HS_TYPE_DATE, (node[1] - datetime.date(1970, 1, 1)).days
        elif tag == "literal":
            x.kind = HS_EXPR_LITERAL
            x.literal_type, x.scale, x.value_i, x.value_f = expr_literal(node[1])
        elif tag == "coalesce":
            x.kind, x.value_i = HS_EXPR_COALESCE, node[1]
        elif tag in EXPR_FUNCS:
            x.kind = EXPR_FUNCS[tag]
        elif len(node) == 6:
            name = node[1].encode() if node[1] is not None else None
            keep.append(name)
            x.kind, x.column, x.literal_type, x.scale, x.value_i, x.value_f = node[0], name, *node[2:]
        else:
            x.kind = EXPR_OPS[tag] if isinstance(tag, str) else tag
    return arr, len(nodes), keep


def _expr_array(exprs: Sequence[tuple]):
    """``(left nodes, op, right nodes)`` or ``(left nodes, op, right nodes, flags)`` expression comparisons -> (hs_expr_compare
    array, count, buffers to keep alive).  Nodes are _expr_nodes'; op and flags are _cmp_array's."""
    keep = []
    arr = (ExprCompareSpec * max(1, len(exprs)))()
    for e, (left, op, right, *flags) in zip(arr, exprs):
        la, nl, k1 = _expr_nodes(left)
        ra, nr, k2 = _expr_nodes(right)
        keep += [la, ra, k1, k2]
        e.left, e.n_left, e.right, e.n_right = la, nl, ra, nr
        e.op = CMP_OPS[op] if isinstance(op, str) else op
        e.flags = flags[0] if flags else 0
    return arr, len(exprs), keep


def _filter_args(*parts, first=0):
    """One side's filter as the arguments of its parameter group: ``parts`` are its predicates (see _predicate_array),
    then, for the calls that take them, its terms (_any_array), its comparisons (_cmp_array) and its expression
    comparisons (_expr_array); each becomes an array and its count.  first=1: parts start at the terms.  Returns
    (arguments, buffers to keep alive)."""
    args, keep = [], []
    for build, part in zip((_predicate_array, _any_array, _cmp_array, _expr_array)[first:], parts):
        arr, n, *k = build(part)
        args += [arr, n]
        keep += k
    return args, keep


def _source_array(files: Sequence[FileImage]):
    keep = []
    arr = (SourceFile * max(1, len(files)))()
    for i, f in enumerate(files):
        arr[i].path = f.path.encode() if f.path else None
        arr[i].file_id = f.file_id
        arr[i].on_device = 1 if f.on_device else 0
        if f.data is None:
            arr[i].data = None
            arr[i].size = 0
        elif isinstance(f.data, int):
            arr[i].data = f.data
            arr[i].size = f.size
        elif isinstance(f.data, np.ndarray):
            a = np.ascontiguousarray(f.data).view(np.uint8)
            keep.append(a)
            arr[i].data = a.ctypes.data
            arr[i].size = a.nbytes
        else:
            b = bytes(f.data)
            buf = C.create_string_buffer(b, len(b))
            keep.append(buf)
            arr[i].data = C.addressof(buf)
            arr[i].size = len(b)
    return arr, keep


@dataclass
class ResultFile:
    bucket: int
    name: str
    ptr: Optional[int]
    size: int
    rows: int


class IndexResult:
    """Owns an hs_index_result handle."""

    def __init__(self, ctx: "Context", handle: int, output: int):
        self._ctx, self._h, self.output = ctx, handle, output
        ctx._results.add(self)  # a result must not outlive its context: Context.close() frees the stragglers
        L = load_library()
        self.files: List[ResultFile] = []
        for i in range(L.hs_result_num_files(handle)):
            b, nm, p, sz, rows = C.c_int32(), C.c_char_p(), C.c_void_p(), C.c_uint64(), C.c_int64()
            L.hs_result_file(handle, i, C.byref(b), C.byref(nm), C.byref(p), C.byref(sz), C.byref(rows))
            self.files.append(ResultFile(b.value, nm.value.decode(), p.value, sz.value, rows.value))

    def host_bytes(self, i: int) -> bytes:
        assert self.output == HS_OUT_HOST
        f = self.files[i]
        return C.string_at(f.ptr, f.size)

    def host_view(self, i: int) -> np.ndarray:
        assert self.output == HS_OUT_HOST
        f = self.files[i]
        return np.ctypeslib.as_array((C.c_uint8 * f.size).from_address(f.ptr))

    def as_sources(self) -> List[FileImage]:
        """The result's in-memory images as engine inputs (host or device)."""
        return [FileImage(path=f.name, data=f.ptr, size=f.size, on_device=self.output == HS_OUT_DEVICE) for f in self.files]

    def free(self) -> None:
        if self._h:
            load_library().hs_result_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Staged:
    """Source file images on their way to device memory (hs_stage_sources); ``as_sources()`` feeds create_index[_async]."""

    def __init__(self, ctx: "Context", handle: int, keep):
        self._ctx, self._h, self._keep = ctx, handle, keep
        ctx._results.add(self)
        L = load_library()
        self.files: List[FileImage] = []
        for i in range(L.hs_staged_num_files(handle)):
            sf = SourceFile()
            L.hs_staged_file(handle, i, C.byref(sf))
            self.files.append(FileImage(path=sf.path.decode() if sf.path else None, data=sf.data, size=sf.size,
                                        file_id=sf.file_id, on_device=True))

    def as_sources(self) -> List[FileImage]:
        return list(self.files)

    def wait(self) -> float:
        """Blocks until the copies have completed; returns their duration on the H2D stream in ms."""
        ms = C.c_float(0)
        if self._h and load_library().hs_staged_wait(self._h, C.byref(ms)) != HS_OK:
            raise HyperspaceGpuError(HS_ECUDA, "hs_staged_wait failed")
        return float(ms.value)

    def free(self) -> None:
        if self._h:
            load_library().hs_staged_free(self._h)
            self._h = None
            self._keep = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Pending:
    """A createIndex whose index files are draining to the host (hs_create_index_async); ``wait()`` yields the result."""

    def __init__(self, ctx: "Context", handle: int, output: int, keep):
        self._ctx, self._h, self.output, self._keep = ctx, handle, output, keep
        ctx._results.add(self)

    def wait(self) -> Tuple[IndexResult, Dict[str, float]]:
        assert self._h, "already waited for"
        res, st = C.c_void_p(), Stats()
        err = C.create_string_buffer(1024)
        h, self._h = self._h, None
        _check(load_library().hs_pending_wait(h, C.byref(res), C.byref(st), err, len(err)), err)
        self._keep = None
        return IndexResult(self._ctx, res.value, self.output), st.as_dict()

    def free(self) -> None:
        if self._h:
            load_library().hs_pending_cancel(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Batch:
    """An hs_batch: result columns in pinned host memory, exposed as zero-copy numpy views.  The views are valid until
    ``free()`` (or garbage collection of the Batch); copy them if they must outlive it."""

    def __init__(self, handle: int, ctx: "Context" = None):
        L = load_library()
        self._h = handle
        if ctx is not None:
            ctx._results.add(self)
        self.num_rows = L.hs_batch_num_rows(handle)
        self.on_device = bool(L.hs_batch_on_device(handle))
        self.columns: List[Tuple[str, np.ndarray, Optional[np.ndarray]]] = []
        self.device_columns: List[Tuple[str, int, int]] = []  # (name, HS_TYPE_*, device pointer) when on_device
        n = self.num_rows
        for i in range(L.hs_batch_num_columns(handle)):
            nm, ty, d, v = C.c_char_p(), C.c_int32(), C.c_void_p(), C.c_void_p()
            L.hs_batch_column(handle, i, C.byref(nm), C.byref(ty), C.byref(d), C.byref(v))
            if self.on_device:
                self.device_columns.append((nm.value.decode(), ty.value, d.value))
                continue
            if ty.value == HS_TYPE_STRING:  # bytes back to back + num_rows + 1 offsets -> an object array of bytes
                off_p, total = C.c_void_p(), C.c_uint64()
                L.hs_batch_string_offsets(handle, i, C.byref(off_p), C.byref(total))
                offs = np.ctypeslib.as_array((C.c_uint64 * (n + 1)).from_address(off_p.value)) if n else np.zeros(1, np.uint64)
                blob = C.string_at(d.value, total.value) if total.value else b""
                data = np.empty(n, dtype=object)
                o = offs.tolist()
                for r in range(n):
                    data[r] = blob[o[r]:o[r + 1]]
                valid = None
                if v.value:
                    valid = np.ctypeslib.as_array((C.c_uint8 * n).from_address(v.value)).copy() if n else np.empty(0, np.uint8)
                self.columns.append((nm.value.decode(), data, valid))
                continue
            dt = np.dtype(_NP_OF_TYPE[ty.value])
            if n:
                data = np.ctypeslib.as_array((C.c_uint8 * (n * dt.itemsize)).from_address(d.value)).view(dt)
            else:
                data = np.empty(0, dt)
            valid = None
            if v.value:
                valid = np.ctypeslib.as_array((C.c_uint8 * n).from_address(v.value)) if n else np.empty(0, np.uint8)
            self.columns.append((nm.value.decode(), data, valid))

    def column(self, name: str) -> np.ndarray:
        for n, d, _ in self.columns:
            if n == name:
                return d
        raise KeyError(name)

    def free(self) -> None:
        if self._h:
            self.columns = []
            load_library().hs_batch_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """One GPU, one stream (hs_ctx)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        L = load_library()
        h = C.c_void_p()
        err = C.create_string_buffer(1024)
        _check(L.hs_init(device, stream, C.byref(h), err, len(err)), err)
        self._h = h.value
        self.device = device
        self.rank, self.world = 0, 1
        self._results = weakref.WeakSet()

    def close(self) -> None:
        if self._h:
            for r in list(self._results):
                r.free()
            load_library().hs_shutdown(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def trim(self) -> None:
        load_library().hs_trim(self._h)

    def profile_enable(self, on: bool = True) -> None:
        load_library().hs_profile_enable(self._h, 1 if on else 0)

    def profile_report(self) -> Dict[str, Dict[str, float]]:
        import json

        buf = C.create_string_buffer(1 << 16)
        rc = load_library().hs_profile_report(self._h, buf, len(buf))
        if rc != HS_OK:
            raise HyperspaceGpuError(rc, "hs_profile_report failed")
        return json.loads(buf.value.decode())

    def host_alloc(self, nbytes: int) -> np.ndarray:
        """Pinned host buffer (owned by the context's pool) as a numpy uint8 view."""
        p = load_library().hs_host_alloc(self._h, nbytes)
        if not p:
            raise HyperspaceGpuError(HS_ENOMEM, f"cannot pin {nbytes} bytes")
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))

    def host_free(self, arr: np.ndarray) -> None:
        load_library().hs_host_free(self._h, arr.ctypes.data)

    # ---- multi-GPU --------------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_comm_unique_id(buf, err, len(err)), err)
        return buf.raw

    def comm_init(self, rank: int, world: int, unique_id: bytes) -> None:
        err = C.create_string_buffer(1024)
        idbuf = C.create_string_buffer(unique_id, 128)
        _check(load_library().hs_comm_init(self._h, rank, world, idbuf, err, len(err)), err)
        self.rank, self.world = rank, world

    # ---- write side ----------------------------------------------------------------------------------
    def stage_sources(self, files: Sequence[FileImage]) -> Staged:
        """Starts copying host / file-system Parquet images to the device on the ctx's H2D copy stream."""
        src, keep = _source_array(files)
        h = C.c_void_p()
        err = C.create_string_buffer(1024)
        _check(load_library().hs_stage_sources(self._h, src, len(files), C.byref(h), err, len(err)), err)
        return Staged(self, h.value, (src, keep, list(files)))

    def create_index_async(self, files: Sequence[FileImage], indexed: Sequence[str], included: Sequence[str], num_buckets: int,
                           **kw) -> Pending:
        """create_index up to the encoded files in device memory; the device->host copy continues on the D2H copy stream."""
        spec, keep = self._index_spec(files, indexed, included, num_buckets, **kw)
        h = C.c_void_p()
        err = C.create_string_buffer(1024)
        _check(load_library().hs_create_index_async(self._h, C.byref(spec), C.byref(h), err, len(err)), err)
        return Pending(self, h.value, spec.output, keep)

    def verify_index(self, files: Sequence[FileImage], buckets: Sequence[int], indexed: Sequence[str], included: Sequence[str],
                     num_buckets: int) -> Dict[str, object]:
        src, keep = _source_array(files)
        ic, nc = _cstr_array(indexed), _cstr_array(included)
        bk = (C.c_int32 * max(1, len(buckets)))(*buckets)
        rep = VerifyReport()
        err = C.create_string_buffer(1024)
        _check(load_library().hs_verify_index(self._h, src, bk, len(files), ic, len(indexed), nc, len(included), num_buckets,
                                              C.byref(rep), err, len(err)), err)
        return rep.as_dict()

    def synth_checksum(self, first_row: int, nrows: int, ncols: int = 5) -> Dict[str, object]:
        rep = VerifyReport()
        err = C.create_string_buffer(1024)
        _check(load_library().hs_synth_checksum(self._h, first_row, nrows, ncols, C.byref(rep), err, len(err)), err)
        return rep.as_dict()

    def _index_spec(self, files, indexed, included, num_buckets, out_dir=None, output=HS_OUT_FILES, job_uuid=None,
                    save_mode=HS_SAVE_OVERWRITE, lineage=False, deleted_file_ids=(), rows_per_page=0, rows_per_row_group=0,
                    dictionary=True, compression=HS_CODEC_UNCOMPRESSED):
        src, keep = _source_array(files)
        ic, nc = _cstr_array(indexed), _cstr_array(included)
        spec = IndexSpec()
        spec.files, spec.n_files = src, len(files)
        spec.indexed_columns, spec.n_indexed = ic, len(indexed)
        spec.included_columns, spec.n_included = nc, len(included)
        spec.num_buckets, spec.save_mode, spec.output, spec.lineage = num_buckets, save_mode, output, 1 if lineage else 0
        spec.out_dir = out_dir.encode() if out_dir else None
        spec.job_uuid = job_uuid.encode() if job_uuid else None
        spec.rows_per_page, spec.rows_per_row_group = rows_per_page, rows_per_row_group
        dl = (C.c_int64 * max(1, len(deleted_file_ids)))(*deleted_file_ids)
        spec.deleted_file_ids, spec.n_deleted_file_ids = dl, len(deleted_file_ids)
        spec.disable_dictionary = 0 if dictionary else 1
        spec.compression = compression
        return spec, (src, keep, ic, nc, dl)

    def create_index(self, files: Sequence[FileImage], indexed: Sequence[str], included: Sequence[str], num_buckets: int,
                     **kw) -> Tuple[IndexResult, Dict[str, float]]:
        """hs_create_index.  Keywords: out_dir, output (HS_OUT_*), job_uuid, save_mode, lineage, deleted_file_ids,
        rows_per_page, rows_per_row_group, dictionary, compression (HS_CODEC_*)."""
        spec, keep = self._index_spec(files, indexed, included, num_buckets, **kw)
        res, st = C.c_void_p(), Stats()
        err = C.create_string_buffer(1024)
        _check(load_library().hs_create_index(self._h, C.byref(spec), C.byref(res), C.byref(st), err, len(err)), err)
        return IndexResult(self, res.value, spec.output), st.as_dict()

    def synth_table(self, first_row: int, nrows: int, ncols: int = 5, n_files: int = 1, row_groups_per_file: int = 1,
                    output: int = HS_OUT_HOST, dictionary: bool = True, compression: int = HS_CODEC_UNCOMPRESSED) -> IndexResult:
        L = load_library()
        res = C.c_void_p()
        err = C.create_string_buffer(1024)
        _check(L.hs_synth_table_ex(self._h, first_row, nrows, ncols, n_files, row_groups_per_file, 1 if dictionary else 0,
                                   compression, output, C.byref(res), err, len(err)), err)
        return IndexResult(self, res.value, output)

    def k_snappy_compress(self, data: bytes) -> bytes:
        """The GPU page compressor on a host buffer (parity tests: any Snappy decoder must give `data` back)."""
        cap = 64 + len(data) + len(data) // 5
        out = C.create_string_buffer(cap)
        n = C.c_uint64(0)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_snappy_compress(self._h, data, len(data), out, cap, C.byref(n), err, len(err)), err)
        return out.raw[:n.value]

    def k_snappy_decompress(self, stream: bytes, uncompressed_len: int) -> Tuple[bytes, bool]:
        """The GPU page decompressor on one raw Snappy stream; returns (bytes, decoded front-to-back by one warp?)."""
        out = C.create_string_buffer(max(1, uncompressed_len))
        seq = C.c_int32(0)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_snappy_decompress(self._h, stream, len(stream), out, uncompressed_len, C.byref(seq), err,
                                                     len(err)), err)
        return out.raw[:uncompressed_len], bool(seq.value)

    def k_inflate(self, stream: bytes, uncompressed_len: int) -> bytes:
        """The GZIP page decompressor on one page body (one or more gzip members) of `uncompressed_len` bytes."""
        out = C.create_string_buffer(max(1, uncompressed_len))
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_inflate(self._h, stream, len(stream), out, uncompressed_len, err, len(err)), err)
        return out.raw[:uncompressed_len]

    def k_lz4(self, stream: bytes, uncompressed_len: int, codec: int = 7) -> bytes:
        """The LZ4 page decompressor on one page body of `uncompressed_len` bytes: codec 7 (LZ4_RAW, one block) or 5 (LZ4:
        Hadoop-framed blocks, or one raw block)."""
        out = C.create_string_buffer(max(1, uncompressed_len))
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_lz4(self._h, codec, stream, len(stream), out, uncompressed_len, err, len(err)), err)
        return out.raw[:uncompressed_len]

    def k_decompress_blobs(self, data: bytes, blobs, out_len: int, fill: int = 0) -> Tuple[bytes, List[bool]]:
        """The page decompressors over several blobs of `data` in one launch.  blobs: (src_off, src_len, dst_off, dst_len,
        prefix, compressed, codec) per blob.  Returns the whole output buffer of out_len bytes, pre-filled with `fill`, and
        per blob whether a snappy stream was decoded front to back by one lane."""
        cols = list(zip(*blobs)) if blobs else [()] * 7
        arrs = [np.ascontiguousarray(c, dtype=t) for c, t in zip(cols, (np.uint64, np.uint32, np.uint64, np.uint32, np.uint32,
                                                                          np.int32, np.int32))]
        out = C.create_string_buffer(max(1, out_len))
        seq = (C.c_int32 * max(1, len(blobs)))()
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_decompress_blobs(self._h, data, len(data), len(blobs), *(a.ctypes.data for a in arrs), fill,
                                                    out, out_len, seq, err, len(err)), err)
        return out.raw[:out_len], [bool(seq[i]) for i in range(len(blobs))]

    def k_compress(self, data: bytes, codec: int) -> bytes:
        """The index page compressor on one page body: HS_CODEC_GZIP (one gzip member) or HS_CODEC_LZ4 (Hadoop-framed
        blocks, one group per 64 KB)."""
        cap = 64 + len(data) + len(data) // 64 + 64 * (len(data) // 65536 + 1)
        out = C.create_string_buffer(cap)
        n = C.c_uint64(0)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_compress(self._h, codec, data, len(data), out, cap, C.byref(n), err, len(err)), err)
        return out.raw[:n.value]

    # ---- read side ----------------------------------------------------------------------------------
    def _read(self, fn, *args) -> Tuple[Batch, Dict[str, float]]:
        """Calls the read-side entry point fn with the context, args and the outputs: (result batch, stats)."""
        res, st = C.c_void_p(), Stats()
        err = C.create_string_buffer(1024)
        _check(fn(self._h, *args, C.byref(res), C.byref(st), err, len(err)), err)
        return Batch(res.value, self), st.as_dict()

    def filter_scan(self, files: Sequence[FileImage], key: str, projected: Sequence[str], lo=None, hi=None, sorted_on_key: bool = True, deleted_file_ids: Sequence[int] = (),
                    output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        spec, keep = self._scan_spec(files, key, projected, sorted_on_key, deleted_file_ids, output)
        spec.has_lo, spec.has_hi = int(lo is not None), int(hi is not None)
        if isinstance(lo, (str, bytes)) or isinstance(hi, (str, bytes)):  # string / binary key: bounds as bytes
            lob = (lo.encode() if isinstance(lo, str) else lo) if lo is not None else b""
            hib = (hi.encode() if isinstance(hi, str) else hi) if hi is not None else b""
            spec.lo_bytes, spec.lo_len, spec.hi_bytes, spec.hi_len = lob, len(lob), hib, len(hib)
            spec.lo, spec.hi = 0, 0
        else:
            spec.lo, spec.hi = lo or 0, hi or 0
        return self._read(load_library().hs_filter_scan, C.byref(spec))

    @staticmethod
    def _scan_spec(files, key, projected, sorted_on_key, deleted_file_ids, output):
        """The hs_scan_spec of the filter scans, and the arrays it points into."""
        src, src_keep = _source_array(files)
        pc = _cstr_array(projected)
        dl = (C.c_int64 * max(1, len(deleted_file_ids)))(*deleted_file_ids)
        spec = ScanSpec()
        spec.files, spec.n_files, spec.sorted_on_key = src, len(files), 1 if sorted_on_key else 0
        spec.key_column = key.encode() if key else None
        spec.projected_columns, spec.n_projected = pc, len(projected)
        spec.deleted_file_ids, spec.n_deleted_file_ids = dl, len(deleted_file_ids)
        spec.output = output
        return spec, (src, src_keep, pc, dl)

    def _filter_scan(self, fn, files, key, projected, parts, sorted_on_key, deleted_file_ids, output, buckets=None):
        """Runs the filter scan fn on the scan's spec and one filter (_filter_args' parts), then, for the calls that take
        them, buckets: (file_buckets or None, num_buckets)."""
        spec, keep = self._scan_spec(files, key, projected, sorted_on_key, deleted_file_ids, output)
        args, keep_filter = _filter_args(*parts)
        if buckets is not None:
            fb = None if buckets[0] is None else np.ascontiguousarray(buckets[0], dtype=np.int32)
            args += [None, 0] if fb is None else [fb.ctypes.data, buckets[1]]
        return self._read(fn, C.byref(spec), *args)

    def filter_scan_where(self, files: Sequence[FileImage], key: Optional[str], projected: Sequence[str], predicates: Sequence[tuple],
                          sorted_on_key: bool = True, deleted_file_ids: Sequence[int] = (), output: int = HS_OUT_HOST
                          ) -> Tuple[Batch, Dict[str, float]]:
        """hs_filter_scan_where: rows where every predicate holds.  A predicate is ``(column, lo, lo_strict, hi, hi_strict)``
        with None for a missing bound; the literal type follows the Python value (int -> long, float -> double, str / bytes
        -> string) and the engine applies Spark's comparison coercion."""
        return self._filter_scan(load_library().hs_filter_scan_where, files, key, projected, (predicates,), sorted_on_key,
                                 deleted_file_ids, output)

    def filter_scan_any(self, files: Sequence[FileImage], key: Optional[str], projected: Sequence[str], predicates: Sequence[tuple],
                        terms: Sequence[tuple], sorted_on_key: bool = True, deleted_file_ids: Sequence[int] = (),
                        file_buckets: Optional[Sequence[int]] = None, num_buckets: int = 0, output: int = HS_OUT_HOST
                        ) -> Tuple[Batch, Dict[str, float]]:
        """hs_filter_scan_any: filter_scan_where's predicates AND-ed with disjunction terms ``(column, values, ranges)``:
        the row's value equals one of `values` (see any_values) or lies in one of `ranges` (``(lo, lo_strict, hi,
        hi_strict)``).  A fourth element gives the term's HS_TERM_* flags: NOT, a null outcome, or a string pattern.  file_buckets / num_buckets: the bucket of every file of an index bucketed on `key` alone, for
        skipping the files a point lookup cannot hit."""
        return self._filter_scan(load_library().hs_filter_scan_any, files, key, projected, (predicates, terms), sorted_on_key,
                                 deleted_file_ids, output, (file_buckets, num_buckets))

    def filter_scan_cmp(self, files: Sequence[FileImage], key: Optional[str], projected: Sequence[str], predicates: Sequence[tuple],
                        terms: Sequence[tuple], compares: Sequence[tuple], sorted_on_key: bool = True,
                        deleted_file_ids: Sequence[int] = (), file_buckets: Optional[Sequence[int]] = None, num_buckets: int = 0,
                        output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_filter_scan_cmp: filter_scan_any with comparisons between two columns of the row AND-ed to the predicates and
        terms, each ``(left, op, right)`` with op one of "<", "<=", ">", ">=", "=", "<=>" and an optional fourth element,
        HS_TERM_NOT.  The engine applies Spark's coercion of the two columns' types."""
        return self._filter_scan(load_library().hs_filter_scan_cmp, files, key, projected, (predicates, terms, compares),
                                 sorted_on_key, deleted_file_ids, output, (file_buckets, num_buckets))

    def filter_scan_expr(self, files: Sequence[FileImage], key: Optional[str], projected: Sequence[str], predicates: Sequence[tuple],
                         terms: Sequence[tuple], compares: Sequence[tuple], exprs: Sequence[tuple], sorted_on_key: bool = True,
                         deleted_file_ids: Sequence[int] = (), file_buckets: Optional[Sequence[int]] = None, num_buckets: int = 0,
                         output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_filter_scan_expr: filter_scan_cmp with expression comparisons AND-ed to the filter, each ``(left nodes, op,
        right nodes)`` with an optional fourth element, HS_TERM_NOT.  Nodes are postfix: ``("column", name)``,
        ``("literal", value)`` and operators ``("+",)``, ``("-",)``, ``("*",)``, ``("/",)``, ``("%",)``, ``("neg",)``.
        The engine types them as Spark 3.1 does."""
        return self._filter_scan(load_library().hs_filter_scan_expr, files, key, projected, (predicates, terms, compares, exprs),
                                 sorted_on_key, deleted_file_ids, output, (file_buckets, num_buckets))

    def _join_spec(self, left, left_buckets, right, right_buckets, num_buckets, left_key, right_key, left_columns, right_columns,
                   output):
        ls, k1 = _source_array(left)
        rs, k2 = _source_array(right)
        lc, rc = _cstr_array(left_columns), _cstr_array(right_columns)
        lb = (C.c_int32 * max(1, len(left_buckets)))(*left_buckets)
        rb = (C.c_int32 * max(1, len(right_buckets)))(*right_buckets)
        spec = JoinSpec()
        spec.left_files, spec.n_left, spec.right_files, spec.n_right = ls, len(left), rs, len(right)
        spec.left_buckets, spec.right_buckets, spec.num_buckets = lb, rb, num_buckets
        spec.left_key = left_key.encode() if left_key is not None else None
        spec.right_key = right_key.encode() if right_key is not None else None
        spec.left_columns, spec.n_left_columns = lc, len(left_columns)
        spec.right_columns, spec.n_right_columns = rc, len(right_columns)
        spec.output = output
        return spec, (ls, k1, rs, k2, lc, rc, lb, rb)

    def bucket_join(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                    right_buckets: Sequence[int], num_buckets: int, left_key: str, right_key: str,
                    left_columns: Sequence[str], right_columns: Sequence[str], output: int = HS_OUT_HOST
                    ) -> Tuple[Batch, Dict[str, float]]:
        spec, keep = self._join_spec(left, left_buckets, right, right_buckets, num_buckets, left_key, right_key, left_columns,
                                     right_columns, output)
        return self._read(load_library().hs_bucket_join, C.byref(spec))

    def _join_where_args(self, left, left_buckets, right, right_buckets, num_buckets, left_keys, right_keys, left_columns,
                         right_columns, left_predicates, right_predicates, output):
        """What every multi-key join passes alike: the spec (and the arrays it points into), the key name arrays, and each
        side's predicate array with its count."""
        if len(left_keys) != len(right_keys):
            raise ValueError("left_keys and right_keys must pair up")
        spec, keep = self._join_spec(left, left_buckets, right, right_buckets, num_buckets, None, None, left_columns,
                                     right_columns, output)
        return (spec, keep, _cstr_array(left_keys), _cstr_array(right_keys), _predicate_array(left_predicates),
                _predicate_array(right_predicates))

    def _bucket_join(self, fn, join_type, left, left_buckets, right, right_buckets, num_buckets, left_keys, right_keys,
                     left_columns, right_columns, left_parts, right_parts, output):
        """Runs the multi-key join fn on its join head (after the spec, join_type when it is not None) and the two sides'
        filters (_filter_args' parts)."""
        spec, keep, lk, rk, lp, rp = self._join_where_args(left, left_buckets, right, right_buckets, num_buckets, left_keys,
                                                           right_keys, left_columns, right_columns, left_parts[0],
                                                           right_parts[0], output)
        largs, k1 = _filter_args(*left_parts[1:], first=1)
        rargs, k2 = _filter_args(*right_parts[1:], first=1)
        head = [C.byref(spec)] + ([] if join_type is None else [join_type])
        return self._read(fn, *head, lk, rk, len(left_keys), *lp, *largs, *rp, *rargs)

    def bucket_join_where(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                          right_buckets: Sequence[int], num_buckets: int, left_keys: Sequence[str], right_keys: Sequence[str],
                          left_columns: Sequence[str], right_columns: Sequence[str], left_predicates: Sequence[tuple] = (),
                          right_predicates: Sequence[tuple] = (), output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_bucket_join_where: inner join on left_keys[k] == right_keys[k] for every k (in the order of the indexes' indexed
        columns), keeping on each side only the rows where every predicate of that side holds.  Predicates are
        filter_scan_where's ``(column, lo, lo_strict, hi, hi_strict)`` tuples.  Rows with a null key join nothing.  The
        side selection's time is in ``ms_exchange``."""
        return self._bucket_join(load_library().hs_bucket_join_where, None, left, left_buckets, right, right_buckets, num_buckets,
                                 left_keys, right_keys, left_columns, right_columns, (left_predicates,), (right_predicates,),
                                 output)

    def bucket_join_any(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                        right_buckets: Sequence[int], num_buckets: int, left_keys: Sequence[str], right_keys: Sequence[str],
                        left_columns: Sequence[str], right_columns: Sequence[str], left_predicates: Sequence[tuple] = (),
                        right_predicates: Sequence[tuple] = (), left_terms: Sequence[tuple] = (), right_terms: Sequence[tuple] = (),
                        output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_bucket_join_any: bucket_join_where with filter_scan_any's disjunction terms on either side."""
        return self._bucket_join(load_library().hs_bucket_join_any, None, left, left_buckets, right, right_buckets, num_buckets,
                                 left_keys, right_keys, left_columns, right_columns, (left_predicates, left_terms),
                                 (right_predicates, right_terms), output)

    def bucket_join_cmp(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                        right_buckets: Sequence[int], num_buckets: int, left_keys: Sequence[str], right_keys: Sequence[str],
                        left_columns: Sequence[str], right_columns: Sequence[str], left_predicates: Sequence[tuple] = (),
                        right_predicates: Sequence[tuple] = (), left_terms: Sequence[tuple] = (), right_terms: Sequence[tuple] = (),
                        left_compares: Sequence[tuple] = (), right_compares: Sequence[tuple] = (),
                        output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_bucket_join_cmp: bucket_join_any with filter_scan_cmp's comparisons on either side."""
        return self._bucket_join(load_library().hs_bucket_join_cmp, None, left, left_buckets, right, right_buckets, num_buckets,
                                 left_keys, right_keys, left_columns, right_columns, (left_predicates, left_terms, left_compares),
                                 (right_predicates, right_terms, right_compares), output)

    def bucket_join_exists(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                           right_buckets: Sequence[int], num_buckets: int, left_keys: Sequence[str], right_keys: Sequence[str],
                           left_columns: Sequence[str], join_type="semi", left_predicates: Sequence[tuple] = (),
                           right_predicates: Sequence[tuple] = (), left_terms: Sequence[tuple] = (), right_terms: Sequence[tuple] = (),
                           left_compares: Sequence[tuple] = (), right_compares: Sequence[tuple] = (),
                           output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_bucket_join_exists: the left semi (``join_type="semi"``) or left anti (``"anti"``) join of bucket_join_cmp's
        sides.  The batch holds left_columns only, each kept left row once, in (bucket, left sorted position) order.  Semi
        drops left rows with a null key; anti keeps them.  join_type may also be an HS_JOIN_* code (others are refused
        by the library)."""
        if isinstance(join_type, str) and join_type not in JOIN_TYPES:
            raise ValueError(f"join_type must be one of {sorted(JOIN_TYPES)} or an HS_JOIN_* code, not {join_type!r}")
        jt = JOIN_TYPES[join_type] if isinstance(join_type, str) else join_type
        return self._bucket_join(load_library().hs_bucket_join_exists, jt, left, left_buckets, right, right_buckets, num_buckets,
                                 left_keys, right_keys, left_columns, [], (left_predicates, left_terms, left_compares),
                                 (right_predicates, right_terms, right_compares), output)

    def bucket_join_outer(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                          right_buckets: Sequence[int], num_buckets: int, left_keys: Sequence[str], right_keys: Sequence[str],
                          left_columns: Sequence[str], right_columns: Sequence[str], join_type="left",
                          left_predicates: Sequence[tuple] = (), right_predicates: Sequence[tuple] = (),
                          left_terms: Sequence[tuple] = (), right_terms: Sequence[tuple] = (), left_compares: Sequence[tuple] = (),
                          right_compares: Sequence[tuple] = (), output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_bucket_join_outer: the left (``join_type="left"``), right (``"right"``) or full (``"full"``) outer join of
        bucket_join_cmp's sides.  The batch holds left_columns, then right_columns; a row padded on one side has that
        side's columns null (their validity is 0), and every column of a side that may be padded has a validity array.
        join_type may also be an HS_JOIN_* code (others are refused by the library)."""
        if isinstance(join_type, str) and join_type not in OUTER_JOIN_TYPES:
            raise ValueError(f"join_type must be one of {sorted(OUTER_JOIN_TYPES)} or an HS_JOIN_* code, not {join_type!r}")
        jt = OUTER_JOIN_TYPES[join_type] if isinstance(join_type, str) else join_type
        return self._bucket_join(load_library().hs_bucket_join_outer, jt, left, left_buckets, right, right_buckets, num_buckets,
                                 left_keys, right_keys, left_columns, right_columns, (left_predicates, left_terms, left_compares),
                                 (right_predicates, right_terms, right_compares), output)

    def bucket_join_expr(self, left: Sequence[FileImage], left_buckets: Sequence[int], right: Sequence[FileImage],
                         right_buckets: Sequence[int], num_buckets: int, left_keys: Sequence[str], right_keys: Sequence[str],
                         left_columns: Sequence[str], right_columns: Sequence[str], join_type="inner",
                         left_predicates: Sequence[tuple] = (), right_predicates: Sequence[tuple] = (),
                         left_terms: Sequence[tuple] = (), right_terms: Sequence[tuple] = (), left_compares: Sequence[tuple] = (),
                         right_compares: Sequence[tuple] = (), left_exprs: Sequence[tuple] = (), right_exprs: Sequence[tuple] = (),
                         output: int = HS_OUT_HOST) -> Tuple[Batch, Dict[str, float]]:
        """hs_bucket_join_expr: the join of any type -- ``join_type`` "inner" (bucket_join_cmp), "semi" / "anti"
        (bucket_join_exists: right_columns must be empty) or "left" / "right" / "full" (bucket_join_outer) -- with
        filter_scan_expr's expression comparisons on either side.  join_type may also be an HS_JOIN_* code (others are
        refused by the library)."""
        if isinstance(join_type, str) and join_type not in ALL_JOIN_TYPES:
            raise ValueError(f"join_type must be one of {sorted(ALL_JOIN_TYPES)} or an HS_JOIN_* code, not {join_type!r}")
        jt = ALL_JOIN_TYPES[join_type] if isinstance(join_type, str) else join_type
        return self._bucket_join(load_library().hs_bucket_join_expr, jt, left, left_buckets, right, right_buckets, num_buckets,
                                 left_keys, right_keys, left_columns, right_columns,
                                 (left_predicates, left_terms, left_compares, left_exprs),
                                 (right_predicates, right_terms, right_compares, right_exprs), output)

    # ---- kernel-level entry points ----------------------------------------------------------------------------------
    @staticmethod
    def _host_columns(cols: Sequence[np.ndarray], valids, decimal=None):
        keep = []
        arr = (HostColumn * max(1, len(cols)))()
        for i, c in enumerate(cols):
            c = np.ascontiguousarray(c)
            keep.append(c)
            arr[i].type = _TYPE_OF_NP[c.dtype]
            arr[i].reserved = HS_KEY_DECIMAL if decimal is not None and decimal[i] else 0
            arr[i].data = c.ctypes.data
            v = None if valids is None else valids[i]
            if v is not None:
                v = np.ascontiguousarray(v.astype(np.uint8))
                keep.append(v)
                arr[i].valid = v.ctypes.data
            else:
                arr[i].valid = None
        return arr, keep

    def k_bucket_ids(self, keys: Sequence[np.ndarray], num_buckets: int, valids=None) -> Tuple[np.ndarray, np.ndarray]:
        n = len(keys[0])
        arr, keep = self._host_columns(keys, valids)
        out = np.empty(n, dtype=np.int32)
        hist = np.zeros(num_buckets, dtype=np.int64)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_bucket_ids(self._h, arr, len(keys), n, num_buckets, out.ctypes.data, hist.ctypes.data,
                                              err, len(err)), err)
        return out, hist

    def k_sort_perm(self, keys: Sequence[np.ndarray], num_buckets: int, valids=None) -> Tuple[np.ndarray, np.ndarray]:
        n = len(keys[0])
        arr, keep = self._host_columns(keys, valids)
        perm = np.empty(n, dtype=np.int64)
        offs = np.empty(num_buckets + 1, dtype=np.int64)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_sort_perm(self._h, arr, len(keys), n, num_buckets, perm.ctypes.data, offs.ctypes.data,
                                             err, len(err)), err)
        return perm, offs

    def k_partition(self, keys: Sequence[np.ndarray], num_buckets: int, valids=None, decimal=None,
                    payload: Sequence[np.ndarray] = (), codes: Sequence[np.ndarray] = (), mode="local", world: int = 1,
                    peer_base=None, owner_rows=None, owner_shift=None, fill: int = 0xA5) -> Dict[str, object]:
        """hs_k_partition: the hash partition alone.  decimal[i]: key i holds a decimal's unscaled values.  payload: columns
        of 8, 4 or 1 byte values; codes: 0..4 uint16 columns.  mode "local", "owner" or "peer" (or an HS_PART_* code); a
        peer layout is peer_base (num_buckets rows) with owner_rows (world buffer sizes, rows) and owner_shift (bytes).
        Returns the output buffers as bytes, slack included: "payload" (per column: one uint8 array, or with a peer layout
        one per owner), "records" (likewise, None without codes), "offsets" (the bins' nbins + 1 offsets, None with a peer
        layout) and "key_or_and"."""
        n = len(keys[0])
        karr, keep = self._host_columns(keys, valids, decimal)
        parr, pkeep = self._host_columns(payload, None)
        code_cols = [np.ascontiguousarray(c, dtype=np.uint16) for c in codes]
        code_ptrs = (C.c_void_p * max(1, len(code_cols)))(*[c.ctypes.data for c in code_cols])
        owners = world if peer_base is not None else 1
        rows = [int(r) for r in owner_rows] if peer_base is not None else [n]
        shift = [int(s) for s in owner_shift] if owner_shift is not None and peer_base is not None else [0] * owners
        base = np.ascontiguousarray(peer_base, dtype=np.uint64) if peer_base is not None else None
        rows_arr = np.ascontiguousarray(rows, dtype=np.uint64)
        shift_arr = np.ascontiguousarray(shift, dtype=np.int32)

        def buffers(width):
            return [np.empty(shift[o] + rows[o] * width + 16, dtype=np.uint8) for o in range(owners)]
        outs = [buffers(np.ascontiguousarray(p).dtype.itemsize) for p in payload]
        recs = buffers(8) if code_cols else []
        out_ptrs = (C.c_void_p * max(1, len(outs) * owners))(*[b.ctypes.data for col in outs for b in col])
        rec_ptrs = (C.c_void_p * max(1, owners))(*[b.ctypes.data for b in recs])
        nbins = world if mode in ("owner", PARTITION_MODES["owner"]) else num_buckets
        offs = np.zeros(nbins + 1, dtype=np.uint64)
        or_and = np.zeros(2, dtype=np.uint64)
        err = C.create_string_buffer(1024)
        _check(load_library().hs_k_partition(
            self._h, karr, len(keys), n, num_buckets, parr, len(payload), code_ptrs if code_cols else None, len(code_cols),
            PARTITION_MODES.get(mode, mode), world, None if base is None else base.ctypes.data,
            rows_arr.ctypes.data if base is not None else None, shift_arr.ctypes.data if base is not None else None, fill,
            out_ptrs, rec_ptrs if code_cols else None, offs.ctypes.data, or_and.ctypes.data, err, len(err)), err)
        single = base is None
        return {"payload": [col[0] if single else col for col in outs],
                "records": (recs[0] if single else recs) if code_cols else None,
                "offsets": offs if single else None, "key_or_and": (int(or_and[0]), int(or_and[1]))}
