"""ctypes binding of libpinot_b200.so (include/pinot_b200.h + include/pinot_b200_host.h).

There is NO fallback: if the shared library is missing or no CUDA device is present, importing / initialising fails
loudly.  The library is built in-tree by ``python -m pinot_b200.build`` (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpinot_b200.so")

PB200_OK = 0
E_INVALID, E_UNSUPPORTED, E_CUDA, E_NOMEM, E_LIMIT = -1, -2, -3, -4, -5

INT, LONG, FLOAT, DOUBLE, STRING = 0, 1, 2, 3, 4
FWD_DICT_FIXEDBIT, FWD_DICT_SORTED, FWD_RAW_FIXEDBYTE = 0, 1, 2
AGG_CODES = {"COUNT": 0, "SUM": 1, "MIN": 2, "MAX": 3, "AVG": 4, "DISTINCTCOUNT": 5, "PERCENTILE": 6,
             "VARPOP": 7, "VARSAMP": 8, "STDDEVPOP": 9, "STDDEVSAMP": 10, "FIRSTWITHTIME": 11, "LASTWITHTIME": 12,
             "DISTINCTSUM": 13, "DISTINCTAVG": 14, "DISTINCTCOUNTHLL": 15}
FILTER_CODES = {"AND": 0, "OR": 1, "NOT": 2, "EQ": 3, "NEQ": 4, "IN": 5, "NOT_IN": 6, "RANGE": 7, "REGEXP_LIKE": 8}
REGIMES = {0: "NONE", 1: "ARRAY", 2: "INT_MAP", 3: "LONG_MAP", 4: "ARRAY_MAP"}
OPERATOR_KINDS = {0: "AGGREGATION", 1: "GROUP_BY", 2: "NON_SCAN_AGGREGATION", 3: "EMPTY", 4: "STAR_TREE"}


class Pb200Error(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"pb200 error {code}: {message}")
        self.code = code


class UnsupportedQueryError(Pb200Error):
    """PB200_E_UNSUPPORTED / PB200_E_LIMIT: the caller must run the reference's own operator for this query."""


class ColDesc(C.Structure):
    _fields_ = [("fwd_kind", C.c_int32), ("stored_type", C.c_int32), ("bits_per_value", C.c_int32),
                ("cardinality", C.c_int32), ("flags", C.c_int32), ("reserved", C.c_int32), ("fwd", C.c_void_p),
                ("fwd_bytes", C.c_uint64), ("dict", C.c_void_p), ("dict_bytes", C.c_uint64), ("inv", C.c_void_p),
                ("inv_bytes", C.c_uint64)]


class FilterNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("column", C.c_int32), ("num_children", C.c_int32), ("lo", C.c_int32),
                ("hi", C.c_int32), ("num_ids", C.c_int32), ("ids", C.POINTER(C.c_int32)), ("raw_lo", C.c_double),
                ("raw_hi", C.c_double), ("raw_flags", C.c_int32), ("reserved", C.c_int32)]


class Agg(C.Structure):
    _fields_ = [("function", C.c_int32), ("column", C.c_int32)]


class Query(C.Structure):
    _fields_ = [("num_filter_nodes", C.c_int32), ("num_group_by", C.c_int32), ("num_aggs", C.c_int32),
                ("num_groups_limit", C.c_int32), ("max_initial_result_holder_capacity", C.c_int32),
                ("flags", C.c_int32), ("filter", C.POINTER(FilterNode)), ("group_by_columns", C.POINTER(C.c_int32)),
                ("aggs", C.POINTER(Agg)), ("reduce_world", C.c_int32), ("reserved", C.c_int32),
                ("merged_docs_bound", C.c_int64)]


class ResultMeta(C.Structure):
    _fields_ = [("num_groups", C.c_int32), ("num_group_by", C.c_int32), ("num_aggs", C.c_int32),
                ("regime", C.c_int32), ("groups_limit_reached", C.c_int32), ("reserved", C.c_int32),
                ("num_docs_scanned", C.c_int64), ("num_entries_scanned_in_filter", C.c_int64),
                ("num_entries_scanned_post_filter", C.c_int64), ("num_total_docs", C.c_int64),
                ("device_ms", C.c_double)]


class SynthCol(C.Structure):
    _fields_ = [("cardinality", C.c_int32), ("value_base", C.c_int32), ("value_step", C.c_int32),
                ("with_inverted", C.c_int32), ("seed", C.c_uint64)]


class HColumn(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data_type", C.c_int32), ("has_dictionary", C.c_int32),
                ("bits_per_value", C.c_int32), ("cardinality", C.c_int32), ("is_sorted", C.c_int32),
                ("dict_entry_bytes", C.c_int32), ("fwd", C.c_void_p), ("fwd_bytes", C.c_uint64), ("dict", C.c_void_p),
                ("dict_bytes", C.c_uint64), ("inv", C.c_void_p), ("inv_bytes", C.c_uint64)]


class DomainCol(C.Structure):
    _fields_ = [("column", C.c_int32), ("stored_type", C.c_int32), ("num_parts", C.c_int32), ("reserved", C.c_int32),
                ("parts", C.POINTER(C.c_void_p)), ("cardinalities", C.POINTER(C.c_int32)),
                ("entry_bytes", C.POINTER(C.c_int32))]


class HLiteral(C.Structure):
    _fields_ = [("i", C.c_int64), ("d", C.c_double), ("s", C.c_char_p)]


class HFilterNode(C.Structure):
    _fields_ = [("type", C.c_int32), ("column", C.c_char_p), ("num_children", C.c_int32),
                ("lower_inclusive", C.c_int32), ("upper_inclusive", C.c_int32), ("lower_unbounded", C.c_int32),
                ("upper_unbounded", C.c_int32), ("num_values", C.c_int32), ("values_offset", C.c_int32)]


class HAgg(C.Structure):
    _fields_ = [("function", C.c_int32), ("column", C.c_char_p)]


class AggArg(C.Structure):  # pb200_agg_arg
    _fields_ = [("p", C.c_double), ("time_column", C.c_int32), ("value_type", C.c_int32)]


class HAggArg(C.Structure):  # pb200h_agg_arg
    _fields_ = [("p", C.c_double), ("time_column", C.c_char_p), ("value_type", C.c_int32)]


class HQuery(C.Structure):
    _fields_ = [("num_filter_nodes", C.c_int32), ("filter", C.POINTER(HFilterNode)), ("literals", C.POINTER(HLiteral)),
                ("num_group_by", C.c_int32), ("group_by", C.POINTER(C.c_char_p)), ("num_aggs", C.c_int32),
                ("aggs", C.POINTER(HAgg)), ("num_groups_limit", C.c_int32),
                ("max_initial_result_holder_capacity", C.c_int32), ("merge_segments", C.c_int32),
                ("skip_star_tree", C.c_int32), ("reduce_world", C.c_int32), ("no_count_carrier", C.c_int32),
                ("merged_docs_bound", C.c_int64), ("agg_filter_nodes", C.POINTER(HFilterNode)),
                ("agg_filter_start", C.POINTER(C.c_int32)), ("agg_filter_count", C.POINTER(C.c_int32))]


MAX_ORDER_BY = 8
ORDER_AGG, ORDER_GROUP_BY, ORDER_POST = 0, 1, 2


class OrderItem(C.Structure):
    _fields_ = [("kind", C.c_int32), ("index", C.c_int32), ("descending", C.c_int32)]


class OrderBy(C.Structure):
    _fields_ = [("num_items", C.c_int32), ("trim_size", C.c_int32), ("items", OrderItem * MAX_ORDER_BY)]


MAX_HAVING_NODES = 32
HAVING_CODES = {"AND": 0, "OR": 1, "NOT": 2, "RANGE": 3, "EQ": 4, "NEQ": 5}
HAVING_LO_UNBOUNDED, HAVING_HI_UNBOUNDED, HAVING_LO_EXCLUSIVE, HAVING_HI_EXCLUSIVE = 1, 2, 4, 8


class HavingNode(C.Structure):
    _fields_ = [("op", C.c_int32), ("num_children", C.c_int32), ("agg", C.c_int32), ("flags", C.c_int32),
                ("lo", C.c_double), ("hi", C.c_double)]


class Having(C.Structure):
    _fields_ = [("num_nodes", C.c_int32), ("reserved", C.c_int32), ("nodes", HavingNode * MAX_HAVING_NODES)]


MAX_POST_NODES = 16
POST_CODES = {"AGG": 0, "LIT": 1, "ADD": 2, "SUB": 3, "MUL": 4, "DIV": 5, "NEG": 6}   # PB200_POST_*


class PostNode(C.Structure):  # pb200_post_node
    _fields_ = [("op", C.c_int32), ("agg", C.c_int32), ("value", C.c_double)]


class PostProgram(C.Structure):  # pb200_post_program
    _fields_ = [("num_nodes", C.c_int32), ("reserved", C.c_int32), ("nodes", PostNode * MAX_POST_NODES)]


class PostAggs(C.Structure):  # pb200_post_aggs
    _fields_ = [("num_programs", C.c_int32), ("reserved", C.c_int32), ("programs", PostProgram * MAX_ORDER_BY)]


class SelectOrder(C.Structure):
    _fields_ = [("column", C.c_int32), ("descending", C.c_int32)]


class Selection(C.Structure):
    _fields_ = [("num_columns", C.c_int32), ("columns", C.POINTER(C.c_int32)), ("num_order_items", C.c_int32),
                ("order", SelectOrder * MAX_ORDER_BY), ("limit", C.c_int64)]


class HSelectOrder(C.Structure):
    _fields_ = [("column", C.c_char_p), ("descending", C.c_int32)]


class HSelection(C.Structure):
    _fields_ = [("num_columns", C.c_int32), ("columns", C.POINTER(C.c_char_p)), ("num_order_items", C.c_int32),
                ("order", HSelectOrder * MAX_ORDER_BY), ("limit", C.c_int64)]


MAX_SELECT_LIMIT = 1_000_000


class TransformOp(C.Structure):
    _fields_ = [("op", C.c_int32), ("reserved", C.c_int32), ("i", C.c_int64), ("d", C.c_double)]


class ExprProgram(C.Structure):  # pb200_expr_program
    _fields_ = [("num_ops", C.c_int32), ("reserved", C.c_int32), ("ops", C.POINTER(TransformOp))]


EXPR_OPS = {"EQ": 0, "NEQ": 1, "IN": 2, "NOT_IN": 3, "RANGE": 4}   # PB200_EXPR_*
T_COND, T_AND, T_OR, T_NOT, T_CASE = 27, 28, 29, 30, 31               # PB200_T_* of CASE WHEN programs
COND_RANGE, COND_BITSET = 0, 1                                         # PB200_COND_*
MAX_EXPR_CONDS = 32


class ExprCond(C.Structure):  # pb200_expr_cond
    _fields_ = [("column", C.c_int32), ("kind", C.c_int32), ("args", C.POINTER(C.c_int64))]


class ExprConds(C.Structure):  # pb200_expr_conds
    _fields_ = [("num_conds", C.c_int32), ("reserved", C.c_int32), ("conds", C.POINTER(ExprCond)), ("num_words", C.c_int64),
                ("words", C.POINTER(C.c_uint32))]


class ExprPredicate(C.Structure):  # pb200_expr_predicate
    _fields_ = [("program", ExprProgram), ("op", C.c_int32), ("flags", C.c_int32), ("lo", C.c_double), ("hi", C.c_double),
                ("num_values", C.c_int32), ("reserved", C.c_int32), ("values", C.POINTER(C.c_double))]


class HStarMetric(C.Structure):
    _fields_ = [("function", C.c_int32), ("reserved", C.c_int32), ("column", C.c_char_p), ("fwd", C.c_void_p),
                ("fwd_bytes", C.c_uint64)]


class HStarTreeConfig(C.Structure):
    _fields_ = [("num_dimensions", C.c_int32), ("dimensions", C.POINTER(C.c_char_p)), ("num_skip_star", C.c_int32),
                ("skip_star", C.POINTER(C.c_char_p)), ("num_pairs", C.c_int32), ("pairs", C.POINTER(HAgg)),
                ("max_leaf_records", C.c_int32)]


class HStarTreeBuildInfo(C.Structure):
    _fields_ = [("num_star_docs", C.c_int64), ("num_base_docs", C.c_int64), ("num_nodes", C.c_int32),
                ("reserved", C.c_int32), ("phase_ms", C.c_double * 4)]


STAR_BUILD_PHASES = ("base", "construct", "aggregate", "encode")


# every symbol include/pinot_b200.h and include/pinot_b200_host.h declare (checked by tests/test_abi.py)
EXPORTED_SYMBOLS = [
    "pb200_init", "pb200_shutdown", "pb200_last_error", "pb200_abi_version", "pb200_device_info", "pb200_tuning_set",
    "pb200_segment_register", "pb200_segment_release", "pb200_segment_device_bytes", "pb200_execute", "pb200_execute_ordered",
    "pb200_result_meta_get", "pb200_result_group_keys", "pb200_result_agg", "pb200_result_agg_dict_ids",
    "pb200_result_distinct", "pb200_result_fetch", "pb200_result_free", "pb200_result_device_buffers", "pb200_result_finalize",
    "pb200_synth_segment", "pb200_segment_read_index", "pb200_segment_column_info",
    "pb200h_segment_create", "pb200h_segment_adopt", "pb200h_segment_load_dir", "pb200h_segment_destroy",
    "pb200h_segment_device", "pb200h_segment_num_docs", "pb200h_segment_num_columns", "pb200h_segment_column_index",
    "pb200h_segment_column_name", "pb200h_segment_column_info", "pb200h_dictionary_get", "pb200h_execute", "pb200h_execute_ordered",
    "pb200h_explain", "pb200h_startree_attach", "pb200h_domain_build", "pb200h_segment_bind_domain",
    "pb200h_result_to_datatable", "pb200h_cache_create", "pb200h_cache_acquire", "pb200h_cache_release", "pb200h_cache_evict",
    "pb200h_cache_stats", "pb200h_cache_destroy",
    "pb200_domain_create", "pb200_domain_from_segments", "pb200_domain_column_info", "pb200_domain_dictionary",
    "pb200_domain_release", "pb200_segment_bind_domain", "pb200_segment_local_ids",
    "pb200_last_phases", "pb200_result_columns", "pb200_doc_mask_upload", "pb200_doc_mask_free", "pb200_roaring_validate", "pb200_comm_unique_id", "pb200_comm_init", "pb200_comm_shutdown", "pb200_result_combine",
    "pb200_execute_selection", "pb200_result_selection", "pb200h_execute_selection",
    "pb200_execute_distinct", "pb200h_execute_distinct",
    "pb200_execute_args", "pb200h_execute_args", "pb200_result_histogram", "pb200_result_moments",
    "pb200_segment_derive_column", "pb200h_segment_derive",
    "pb200h_startree_build", "pb200h_startree_get",
    "pb200_execute_having", "pb200h_execute_having", "pb200_execute_agg_args", "pb200h_execute_agg_args",
    "pb200_match_pattern", "pb200_result_exact_sum", "pb200_execute_exprs", "pb200_expr_doc_masks",
    "pb200_execute_post", "pb200h_execute_post", "pb200_execute_exprs_cond",
]

_LIB = None


def load() -> C.CDLL:
    """Loads the shared library (no compute).  Raises if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -m pinot_b200.build` (there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    L.pb200_last_error.restype = C.c_char_p
    L.pb200_init.argtypes = [i32, C.POINTER(vp)]
    L.pb200_shutdown.argtypes = [vp]
    L.pb200_device_info.argtypes = [vp, C.POINTER(i64)]
    L.pb200_tuning_set.argtypes = [vp, C.c_char_p, i64]
    L.pb200_segment_register.argtypes = [vp, C.c_char_p, i32, i32, C.POINTER(ColDesc), C.POINTER(vp)]
    L.pb200_segment_release.argtypes = [vp, vp]
    L.pb200_segment_device_bytes.restype = i64
    L.pb200_segment_device_bytes.argtypes = [vp]
    L.pb200_execute.argtypes = [vp, C.POINTER(Query), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_ordered.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_args.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(C.c_double), C.POINTER(vp), i32,
                                     C.POINTER(vp)]
    L.pb200_execute_having.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(C.c_double), C.POINTER(Having),
                                       C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_agg_args.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(AggArg), C.POINTER(Having),
                                         C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_exprs.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(AggArg), C.POINTER(Having),
                                      C.POINTER(ExprProgram), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_exprs_cond.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(AggArg), C.POINTER(Having),
                                           C.POINTER(ExprProgram), C.POINTER(ExprConds), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_post.argtypes = [vp, C.POINTER(Query), C.POINTER(OrderBy), C.POINTER(AggArg), C.POINTER(Having),
                                     C.POINTER(PostAggs), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_expr_doc_masks.argtypes = [vp, i32, C.POINTER(ExprPredicate), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_result_histogram.restype = i64
    L.pb200_result_histogram.argtypes = [vp, i32, i32, vp, vp, i64]
    L.pb200_result_moments.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    L.pb200_result_meta_get.argtypes = [vp, C.POINTER(ResultMeta)]
    L.pb200_result_group_keys.argtypes = [vp, vp]
    L.pb200_result_agg.argtypes = [vp, i32, vp, vp]
    L.pb200_result_agg_dict_ids.argtypes = [vp, i32, vp]
    L.pb200_result_exact_sum.argtypes = [vp, i32, C.POINTER(i64)]
    L.pb200_result_distinct.restype = i64
    L.pb200_result_distinct.argtypes = [vp, i32, i32, vp, i64]
    L.pb200_result_fetch.argtypes = [vp, vp, vp, vp, vp]
    L.pb200_result_free.argtypes = [vp]
    L.pb200_result_device_buffers.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(i64)]
    L.pb200_result_finalize.argtypes = [vp, vp]
    L.pb200_synth_segment.argtypes = [vp, C.c_char_p, i32, i32, C.POINTER(SynthCol), C.POINTER(vp)]
    L.pb200_segment_read_index.restype = i64
    L.pb200_segment_read_index.argtypes = [vp, vp, i32, i32, vp, C.c_uint64]
    L.pb200_segment_column_info.argtypes = [vp, i32, C.POINTER(i64)]
    L.pb200h_segment_create.argtypes = [vp, C.c_char_p, i32, i32, C.POINTER(HColumn), C.POINTER(vp)]
    L.pb200h_segment_adopt.argtypes = [vp, vp, i32, i32, C.POINTER(C.c_char_p), C.POINTER(vp)]
    L.pb200h_segment_load_dir.argtypes = [vp, C.c_char_p, C.POINTER(vp)]
    L.pb200h_segment_destroy.argtypes = [vp]
    L.pb200h_segment_device.restype = vp
    L.pb200h_segment_device.argtypes = [vp]
    L.pb200h_segment_num_docs.argtypes = [vp]
    L.pb200h_segment_num_columns.argtypes = [vp]
    L.pb200h_segment_column_index.argtypes = [vp, C.c_char_p]
    L.pb200h_segment_column_name.restype = C.c_char_p
    L.pb200h_segment_column_name.argtypes = [vp, i32]
    L.pb200h_segment_column_info.argtypes = [vp, i32, C.POINTER(i32)]
    L.pb200h_dictionary_get.argtypes = [vp, i32, i32, C.POINTER(C.c_double), C.POINTER(i64), C.c_char_p, i32]
    L.pb200h_execute.argtypes = [vp, C.POINTER(HQuery), C.POINTER(vp), i32, C.POINTER(vp), C.POINTER(i32)]
    L.pb200h_execute_ordered.argtypes = [vp, C.POINTER(HQuery), C.POINTER(OrderBy), C.POINTER(vp), i32, C.POINTER(vp),
                                         C.POINTER(i32)]
    L.pb200h_execute_args.argtypes = [vp, C.POINTER(HQuery), C.POINTER(OrderBy), C.POINTER(C.c_double), C.POINTER(vp), i32,
                                      C.POINTER(vp), C.POINTER(i32)]
    L.pb200h_execute_having.argtypes = [vp, C.POINTER(HQuery), C.POINTER(OrderBy), C.POINTER(C.c_double), C.POINTER(Having),
                                        C.POINTER(vp), i32, C.POINTER(vp), C.POINTER(i32)]
    L.pb200h_execute_agg_args.argtypes = [vp, C.POINTER(HQuery), C.POINTER(OrderBy), C.POINTER(HAggArg), C.POINTER(Having),
                                          C.POINTER(vp), i32, C.POINTER(vp), C.POINTER(i32)]
    L.pb200h_execute_post.argtypes = [vp, C.POINTER(HQuery), C.POINTER(OrderBy), C.POINTER(HAggArg), C.POINTER(Having),
                                      C.POINTER(PostAggs), C.POINTER(vp), i32, C.POINTER(vp), C.POINTER(i32)]
    L.pb200h_explain.argtypes = [vp, C.POINTER(HQuery), vp, C.c_char_p, i32]
    L.pb200h_startree_attach.argtypes = [vp, vp, vp, C.c_uint64, i32, i32, C.POINTER(C.c_char_p), C.POINTER(vp),
                                         C.POINTER(C.c_uint64), i32, C.POINTER(HStarMetric)]
    L.pb200_execute_selection.argtypes = [vp, C.POINTER(Query), C.POINTER(Selection), C.POINTER(vp), i32, i32, C.POINTER(vp)]
    L.pb200_result_selection.argtypes = [vp, C.POINTER(i64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.pb200h_execute_selection.argtypes = [vp, C.POINTER(HQuery), C.POINTER(HSelection), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_execute_distinct.argtypes = [vp, C.POINTER(Query), C.POINTER(Selection), C.POINTER(vp), i32, i32, C.POINTER(vp)]
    L.pb200h_execute_distinct.argtypes = [vp, C.POINTER(HQuery), C.POINTER(HSelection), C.POINTER(vp), i32, C.POINTER(vp)]
    L.pb200_result_columns.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.pb200_roaring_validate.argtypes = [vp, C.c_uint64, C.c_int64]
    L.pb200_doc_mask_upload.argtypes = [vp, i32, vp, C.c_int64, C.POINTER(vp)]
    L.pb200_doc_mask_free.argtypes = [vp, vp]
    L.pb200_match_pattern.argtypes = [vp, C.c_char_p, i32, C.POINTER(vp), C.POINTER(i32), C.POINTER(vp)]
    L.pb200_last_phases.argtypes = [C.POINTER(C.c_double)]
    L.pb200_comm_unique_id.argtypes = [vp]
    L.pb200_comm_init.argtypes = [vp, vp, i32, i32]
    L.pb200_comm_shutdown.argtypes = [vp]
    L.pb200_result_combine.argtypes = [vp, vp, i32, C.POINTER(i32)]
    L.pb200h_cache_create.argtypes = [vp, i64, C.POINTER(vp)]
    L.pb200h_cache_acquire.argtypes = [vp, C.c_char_p, C.c_uint64, C.c_char_p, i64, C.POINTER(vp)]
    L.pb200h_cache_release.argtypes = [vp, vp]
    L.pb200h_cache_evict.argtypes = [vp, C.c_char_p, C.c_uint64]
    L.pb200h_cache_stats.argtypes = [vp, C.POINTER(i64)]
    L.pb200h_cache_destroy.argtypes = [vp]
    L.pb200h_result_to_datatable.restype = i64
    L.pb200h_result_to_datatable.argtypes = [C.POINTER(HQuery), vp, vp, vp, C.c_uint64]
    L.pb200h_domain_build.argtypes = [vp, C.POINTER(vp), i32, i32, C.POINTER(C.c_char_p), C.POINTER(vp)]
    L.pb200h_segment_bind_domain.argtypes = [vp, vp, vp]
    L.pb200_domain_create.argtypes = [vp, i32, C.POINTER(DomainCol), C.POINTER(vp)]
    L.pb200_domain_from_segments.argtypes = [vp, C.POINTER(vp), i32, i32, C.POINTER(i32), C.POINTER(vp)]
    L.pb200_domain_column_info.argtypes = [vp, i32, C.POINTER(i64)]
    L.pb200_domain_dictionary.restype = i64
    L.pb200_domain_dictionary.argtypes = [vp, i32, vp, C.c_uint64]
    L.pb200_domain_release.argtypes = [vp, vp]
    L.pb200_segment_bind_domain.argtypes = [vp, vp, vp]
    L.pb200_segment_local_ids.restype = i64
    L.pb200_segment_local_ids.argtypes = [vp, i32, vp, i64]
    L.pb200_segment_derive_column.argtypes = [vp, vp, i32, i32, C.POINTER(TransformOp), C.POINTER(i32)]
    L.pb200h_segment_derive.argtypes = [vp, vp, C.c_char_p, C.POINTER(i32)]
    L.pb200h_startree_build.argtypes = [vp, vp, C.POINTER(HStarTreeConfig), C.POINTER(HStarTreeBuildInfo)]
    L.pb200h_startree_get.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(C.c_uint64), C.POINTER(vp)]
    _LIB = L
    return L


def check(rc: int):
    if rc == PB200_OK:
        return
    msg = load().pb200_last_error().decode("utf-8", "replace")
    if rc in (E_UNSUPPORTED, E_LIMIT):
        raise UnsupportedQueryError(rc, msg)
    raise Pb200Error(rc, msg)
