"""ctypes binding of libcitus_gpu.so (include/citus_gpu.h).

This module is plumbing for tests and bench.py: the product is the C-ABI library.  It
fails loudly when the library is missing or cannot be loaded -- there is no CPU fallback
on this path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcitus_gpu.so")

CG_OK, CG_EINVAL, CG_ECUDA, CG_ENOMEM, CG_ECORRUPT, CG_ETABLEFULL, CG_EUNSUPPORTED, CG_ERETRY_UNPACKED, CG_ECOMM = range(9)
CG_COMM_ID_BYTES = 128
CG_COMM_SUM, CG_COMM_MIN, CG_COMM_MAX = 0, 1, 2
CG_TYPE_INT, CG_TYPE_FLOAT = 0, 1
CG_OP = {"<": 0, "<=": 1, "=": 2, ">=": 3, ">": 4, "<>": 5, "in": 6, "not in": 7, "is null": 8, "is not null": 9,
         "col <": 16, "col <=": 17, "col =": 18, "col >=": 19, "col >": 20, "col <>": 21}
CG_AGG_COUNT_STAR, CG_AGG_COUNT, CG_AGG_SUM, CG_AGG_MIN, CG_AGG_MAX = range(5)
CG_AGG_BIT_AND, CG_AGG_BIT_OR, CG_AGG_BOOL_AND, CG_AGG_BOOL_OR = range(5, 9)
CG_AGG_VARIANCE = 9
CG_VAR_POP, CG_VAR_SAMP, CG_STDDEV_POP, CG_STDDEV_SAMP = range(4)
CG_WORD_ADD, CG_WORD_MIN, CG_WORD_MAX, CG_WORD_FADD, CG_WORD_FMIN, CG_WORD_FMAX = range(6)
CG_WORD_AND, CG_WORD_OR = 6, 7
CG_GEN_UNIFORM, CG_GEN_SEQUENCE = 0, 1
CG_MAX_QUALS, CG_MAX_AGGS, CG_MAX_GROUP_COLS = 8, 8, 4
CG_MAX_QEXPR, CG_QX_AND, CG_QX_OR = 16, -1, -2
CG_MAX_FILTER_QUALS = 8
CG_MAX_WORDS = 32
CG_MAX_IN_LISTS, CG_MAX_IN_VALUES, CG_IN_REFUTE_MAX = 8, 1024, 100
CG_MAX_CASE_ARMS = 16
CG_CASE_NULL, CG_CASE_CONST, CG_CASE_PRODUCT = 0, 1, 2
CG_PSTATE_PACKED_DIRTY, CG_PSTATE_WIDE_DIRTY, CG_PSTATE_READ_PACKED_DIRECT, CG_PSTATE_TABLE_INITIALISED = 1, 2, 4, 8


class CgSkipNode(C.Structure):
    _fields_ = [
        ("has_minmax", C.c_int32), ("compression_type", C.c_int32),
        ("min_value", C.c_int64), ("max_value", C.c_int64),
        ("row_count", C.c_uint64), ("value_offset", C.c_uint64), ("value_length", C.c_uint64),
        ("exists_offset", C.c_uint64), ("exists_length", C.c_uint64),
        ("decompressed_size", C.c_uint64), ("compression_level", C.c_int32), ("reserved", C.c_int32),
    ]


class CgStripe(C.Structure):
    _fields_ = [
        ("id", C.c_uint64), ("file_offset", C.c_uint64), ("data_length", C.c_uint64),
        ("row_count", C.c_uint64), ("first_row_number", C.c_uint64),
        ("column_count", C.c_uint32), ("chunk_row_count", C.c_uint32),
        ("chunk_count", C.c_uint32), ("skipnode_base", C.c_uint32),
    ]


class CgColumnDesc(C.Structure):
    _fields_ = [("attlen", C.c_int32), ("type_class", C.c_int32)]


class CgRelation(C.Structure):
    _fields_ = [
        ("pages", C.c_void_p), ("nblocks", C.c_uint64),
        ("stripes", C.POINTER(CgStripe)), ("nstripes", C.c_int32),
        ("nodes", C.POINTER(CgSkipNode)), ("nnodes", C.c_int32),
        ("columns", C.POINTER(CgColumnDesc)), ("natts", C.c_int32),
    ]


class CgQual(C.Structure):
    _fields_ = [("column", C.c_int32), ("op", C.c_int32), ("konst", C.c_int64)]


class CgInList(C.Structure):
    _fields_ = [("first", C.c_int32), ("nvalues", C.c_int32), ("nnulls", C.c_int32), ("reserved", C.c_int32)]


class CgAggSpec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("nfactors", C.c_int32), ("column", C.c_int32 * 3),
                ("is_float", C.c_int32), ("a", C.c_int64 * 3), ("b", C.c_int64 * 3),
                ("term_abs_bound", C.c_int64)]


class CgCaseArm(C.Structure):
    _fields_ = [("nwhen", C.c_int32), ("when", C.c_int8 * CG_MAX_QEXPR), ("form", C.c_int32), ("nfactors", C.c_int32),
                ("column", C.c_int32 * 3), ("a", C.c_int64 * 3), ("b", C.c_int64 * 3)]


class CgScanDesc(C.Structure):
    _fields_ = [("nquals", C.c_int32), ("quals", CgQual * CG_MAX_QUALS),
                ("enable_qual_pushdown", C.c_int32), ("ngroup_cols", C.c_int32),
                ("group_cols", C.c_int32 * CG_MAX_GROUP_COLS), ("naggs", C.c_int32),
                ("aggs", CgAggSpec * CG_MAX_AGGS), ("expected_groups", C.c_int64),
                ("nqual_expr", C.c_int32), ("qual_expr", C.c_int8 * CG_MAX_QEXPR), ("reserved", C.c_int32),
                ("nfilter_quals", C.c_int32), ("filter_quals", CgQual * CG_MAX_FILTER_QUALS),
                ("nfilter_expr", C.c_int32 * CG_MAX_AGGS), ("filter_expr", (C.c_int8 * CG_MAX_QEXPR) * CG_MAX_AGGS),
                ("narg_expr", C.c_int32 * CG_MAX_AGGS), ("arg_expr", (C.c_int8 * CG_MAX_QEXPR) * CG_MAX_AGGS),
                ("composite_key", C.c_int32), ("key_col_min", C.c_int64 * CG_MAX_GROUP_COLS),
                ("key_col_max", C.c_int64 * CG_MAX_GROUP_COLS),
                ("nin_lists", C.c_int32), ("in_lists", CgInList * CG_MAX_IN_LISTS),
                ("nin_values", C.c_int32), ("in_values", C.c_int64 * CG_MAX_IN_VALUES),
                ("case_first", C.c_int32 * CG_MAX_AGGS), ("case_narms", C.c_int32 * CG_MAX_AGGS), ("ncase_arms", C.c_int32),
                ("reserved2", C.c_int32), ("case_arms", CgCaseArm * CG_MAX_CASE_ARMS)]


class CgScanStats(C.Structure):
    _fields_ = [("rows_scanned", C.c_int64), ("rows_removed_by_filter", C.c_int64),
                ("chunk_groups_filtered", C.c_int64), ("rows_passed", C.c_int64),
                ("chunk_groups_scanned", C.c_int64), ("bytes_scanned", C.c_int64),
                ("kernel_ms", C.c_double), ("h2d_bytes", C.c_int64)]


class CgJoinSide(C.Structure):
    _fields_ = [("d_cols", C.POINTER(C.c_void_p)), ("d_nulls", C.POINTER(C.c_void_p)), ("ncols", C.c_int32),
                ("key", C.c_int32), ("nrows", C.c_int64)]


class CgGenColumn(C.Structure):
    _fields_ = [("attlen", C.c_int32), ("kind", C.c_int32), ("lo", C.c_int64), ("hi", C.c_int64),
                ("null_ppm", C.c_uint32), ("reserved", C.c_uint32)]


# every symbol include/citus_gpu.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("cg_last_error", C.c_char_p, []),
    ("cg_init", C.c_int, [C.c_int]),
    ("cg_device_count", C.c_int, [C.POINTER(C.c_int)]),
    ("cg_synchronize", C.c_int, []),
    ("cg_shutdown", None, []),
    ("cg_set_stream", C.c_int, [C.c_void_p]),
    ("cg_kernel_launches", C.c_uint64, []),
    ("cg_partition_copy_bytes", C.c_int, [_P, C.c_int64, C.c_int32, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    ("cg_partition_copy_serialize", C.c_int, [_P, C.c_int64, C.c_int32, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, _P]),
    ("cg_join_count_sum", C.c_int, [_P, _P, _P, C.c_int64, _P, _P, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                   C.POINTER(C.c_uint64)]),
    ("cg_partial_dense_words_enqueue", C.c_int, [_P, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    ("cg_partial_check", C.c_int, [_P]),
    ("cg_partial_packed_state", C.c_int, [_P, _P, C.c_uint64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                          C.POINTER(C.c_uint64)]),
    ("cg_gen_set_compression", C.c_int, [C.c_int32]),
    ("cg_jit_launches", C.c_uint64, []),
    ("cg_jit_compiles", C.c_uint64, []),
    ("cg_jit_compile_check", C.c_int, [C.POINTER(CgScanDesc), C.POINTER(CgColumnDesc), C.c_int32, C.c_int64, C.c_int64, C.c_int64,
                                      C.POINTER(C.c_int32), C.c_char_p, C.c_size_t]),
    ("cg_jit_compile_check_nullable", C.c_int, [C.POINTER(CgScanDesc), C.POINTER(CgColumnDesc), C.c_int32, C.c_int64, C.c_int64,
                                               C.c_int64, C.c_uint32, C.POINTER(C.c_int32), C.c_char_p, C.c_size_t]),
    ("cg_set_option", C.c_int, [C.c_char_p, C.c_int64]),
    ("cg_numa_bind", C.c_int, [C.POINTER(C.c_int32)]),
    ("cg_numa_unbind", C.c_int, []),
    ("cg_profile_begin", C.c_int, []),
    ("cg_profile_collect", C.c_int, [C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    ("cg_shard_stage", C.c_int, [C.POINTER(CgRelation), _P, C.c_int32, C.POINTER(_P)]),
    ("cg_shard_free", None, [_P]),
    ("cg_shard_device_bytes", C.c_uint64, [_P]),
    ("cg_shard_rows", C.c_uint64, [_P]),
    ("cg_shard_narrow_bytes", C.c_uint64, [_P]),
    ("cg_shard_narrow_column", C.c_int32, [_P, C.c_int32]),
    ("cg_shard_narrow_image", C.c_int, [_P, C.c_int64, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_uint32), _P, C.c_uint64,
                                        C.POINTER(C.c_uint64)]),
    ("cg_narrow_plan", C.c_int, [C.c_int64, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_uint64)]),
    ("cg_partial_create", C.c_int, [C.POINTER(CgScanDesc), C.POINTER(CgColumnDesc), C.c_int32, C.c_int64,
                                    C.c_int64, C.c_int64, C.POINTER(_P)]),
    ("cg_partial_free", None, [_P]),
    ("cg_partial_reset", C.c_int, [_P]),
    ("cg_partial_set_packing", C.c_int, [_P, C.c_int32]),
    ("cg_scan_shard", C.c_int, [_P, C.POINTER(CgScanDesc), _P, C.POINTER(CgScanStats)]),
    ("cg_scan_shard_rows", C.c_int, [_P, C.POINTER(CgScanDesc), _P, C.c_int32, C.c_int64, _P, _P, C.POINTER(C.c_int64),
                                     C.POINTER(CgScanStats)]),
    ("cg_relation_register", C.c_int, [C.POINTER(CgRelation)]),
    ("cg_relation_unregister", C.c_int, [C.POINTER(CgRelation)]),
    ("cg_scan_relation", C.c_int, [C.POINTER(CgRelation), C.POINTER(CgScanDesc), _P, C.POINTER(CgScanStats)]),
    ("cg_partial_ngroups", C.c_int, [_P, C.POINTER(C.c_int64)]),
    ("cg_partial_fetch", C.c_int, [_P, C.c_int64, _P, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_int64)]),
    ("cg_partial_fetch_ex", C.c_int, [_P, C.c_int64, _P, _P, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_int64)]),
    ("cg_partial_layout", C.c_int, [_P, C.POINTER(C.c_int32), _P, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    ("cg_partial_export_device", C.c_int, [_P, C.c_int64, _P, _P, _P, C.POINTER(C.c_int64)]),
    ("cg_partial_merge_rows", C.c_int, [_P, _P, _P, _P, C.c_int64]),
    ("cg_partial_dense_words", C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    ("cg_partition_index", C.c_int, [_P, _P, C.c_int64, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P]),
    ("cg_partition_scatter", C.c_int, [_P, C.c_int64, C.c_int32, _P, C.c_int32, _P, _P]),
    ("cg_partition_scatter_ordered", C.c_int, [_P, C.c_int64, C.c_int32, _P, _P, C.c_int32, _P, _P]),
    ("cg_relation_bounds", C.c_int, [C.POINTER(CgRelation), C.POINTER(CgScanDesc), C.POINTER(C.c_int64),
                                     C.POINTER(C.c_int64), _P, C.POINTER(C.c_int64)]),
    ("cg_relation_key_bounds", C.c_int, [C.POINTER(CgRelation), C.POINTER(CgScanDesc), _P, _P]),
    ("cg_group_key_decode", C.c_int, [C.POINTER(CgScanDesc), C.c_int64, _P, _P, _P]),
    ("cg_group_key_encode", C.c_int, [C.POINTER(CgScanDesc), C.c_int64, _P, _P, _P]),
    ("cg_selected_chunk_mask", C.c_int, [C.POINTER(CgRelation), C.c_int32, C.POINTER(CgScanDesc), _P,
                                         C.POINTER(C.c_int64)]),
    ("cg_numeric_out", C.c_int, [C.c_int64, C.c_uint64, C.c_int32, C.c_char_p, C.c_size_t]),
    ("cg_numeric_div_out", C.c_int, [C.c_int64, C.c_uint64, C.c_int32, C.c_int64, C.c_char_p, C.c_size_t]),
    ("cg_numeric_var_out", C.c_int, [C.c_int32, C.c_int64, C.c_int64, C.c_uint64, _P, C.c_int32, C.c_char_p, C.c_size_t,
                                     C.POINTER(C.c_int32)]),
    ("cg_gen_relation", C.c_int, [C.POINTER(CgGenColumn), C.c_int32, C.c_uint64, C.c_uint64, C.c_uint64,
                                  C.c_uint64, C.c_uint32, C.c_int32, C.POINTER(_P)]),
    ("cg_write_relation", C.c_int, [C.POINTER(CgColumnDesc), C.c_int32, _P, _P, C.c_uint64, C.c_uint64,
                                    C.c_uint32, C.POINTER(_P)]),
    ("cg_gen_relation_view", C.c_int, [_P, C.POINTER(CgRelation)]),
    ("cg_gen_relation_free", None, [_P]),
    ("cg_join_rows", C.c_int, [_P, _P, _P, C.c_int64, _P, _P, _P, C.c_int64, C.c_int64, _P, _P, _P, C.POINTER(C.c_int64)]),
    ("cg_join_aggregate", C.c_int, [C.POINTER(CgJoinSide), C.POINTER(CgJoinSide), C.POINTER(CgColumnDesc), C.POINTER(CgScanDesc), _P,
                                    C.POINTER(CgScanStats)]),
    ("cg_partial_merge_values", C.c_int, [_P, C.c_int64, _P, _P, _P, _P, _P, _P, _P]),
    ("cg_agg_column", C.c_int, [C.c_int32, C.c_int32, _P, _P, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                               C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("cg_comm_unique_id", C.c_int, [_P]),
    ("cg_comm_init", C.c_int, [_P, C.c_int32, C.c_int32]),
    ("cg_comm_rank", C.c_int, [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("cg_comm_destroy", C.c_int, []),
    ("cg_comm_barrier", C.c_int, []),
    ("cg_comm_peer_window", C.c_int, []),
    ("cg_comm_allreduce_i64", C.c_int, [_P, C.c_int32, C.c_int32]),
    ("cg_comm_combine", C.c_int, [_P, C.c_int32, C.c_int32]),
    ("cg_comm_repartition_exchange", C.c_int, [C.c_int32, _P, _P, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _P, _P,
                                              C.POINTER(C.c_int64)]),
    ("cg_comm_exchange_wait", C.c_int, [C.c_int32]),
    ("cg_comm_exchange_result", C.c_int, [C.c_int32, _P, C.POINTER(C.c_int64), _P, C.POINTER(C.c_int32), C.POINTER(C.c_uint64),
                                         C.POINTER(C.c_double)]),
    ("cg_comm_exchange_plan", C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.POINTER(C.c_int32)]),
    ("cg_comm_peer_plan", C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P]),
]

_lib = None


class CitusGpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[{code}] {msg}")
        self.code = code


def lib():
    """Loads libcitus_gpu.so; raises if it is missing (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -m citus_b200.build` (nvcc, sm_90a)")
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise CitusGpuError(rc, lib().cg_last_error().decode())
