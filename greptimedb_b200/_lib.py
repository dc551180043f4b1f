"""ctypes binding of libb200promql.so (the C ABI declared in include/b200promql.h).

There is no CPU fallback: if the shared library is missing this module raises, and if no CUDA
device is present `Context()` raises with the library's own error message.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2P_LIB_PATH") or os.path.join(_HERE, "libb200promql.so")  # override: tuning experiments only

# every symbol include/b200promql.h declares (tests/test_abi.py checks the .so exports them all)
EXPORTED_SYMBOLS = [
    "b2p_create", "b2p_destroy", "b2p_last_error", "b2p_version", "b2p_set_stream", "b2p_use_own_stream", "b2p_sync", "b2p_num_steps",
    "b2p_last_slow_series", "b2p_last_h2d_bytes", "b2p_last_warp_tier_series", "b2p_last_kernel_ms", "b2p_launch_count",
    "b2p_series_offsets_dev", "b2p_range_eval_dev", "b2p_range_udf_dev", "b2p_instant_select_dev",
    "b2p_group_aggregate_dev", "b2p_range_group_sum_dev", "b2p_group_finalize_dev", "b2p_histogram_quantile_dev",
    "b2p_group_index_create_dev", "b2p_group_index_destroy", "b2p_group_aggregate_indexed_dev",
    "b2p_range_group_sum_indexed_dev", "b2p_range_group_sum_fused", "b2p_group_aggregate_partial_dev",
    "b2p_comm_unique_id", "b2p_comm_init", "b2p_comm_destroy", "b2p_allreduce_partials_dev",
    "b2p_range_group_sum_allreduce_dev", "b2p_allreduce_columns_dev", "b2p_histogram_fold_dev", "b2p_range_histogram_fold",
    "b2p_column_reduce_dev", "b2p_host_scan_series", "b2p_range_eval", "b2p_range_udf", "b2p_instant_select", "b2p_group_aggregate",
    "b2p_histogram_quantile", "b2p_synth_fill_dev",
    "b2p_binary_op_dev", "b2p_scalar_op_dev", "b2p_count_valid_words_dev", "b2p_binary_op", "b2p_scalar_op",
    "b2p_plan_range_create", "b2p_plan_set_instant", "b2p_plan_set_histogram_quantile", "b2p_plan_push_batch", "b2p_plan_execute", "b2p_plan_num_series", "b2p_plan_destroy",
    "b2p_plan_last_error", "b2p_plan_set_scalar_op", "b2p_plan_binary_create",
    "b2p_setop_dev", "b2p_setop", "b2p_plan_setop_create",
    "b2p_instant_fn_dev", "b2p_instant_fn", "b2p_scalar_calculate_dev", "b2p_scalar_calculate",
    "b2p_plan_set_function", "b2p_plan_scalar_create",
    "b2p_topk_dev", "b2p_topk", "b2p_plan_topk_create",
    "b2p_group_quantile_dev", "b2p_group_quantile", "b2p_plan_aggregate_create",
    "b2p_count_values_dev", "b2p_count_values", "b2p_plan_count_values_create",
    "b2p_subquery_dev", "b2p_subquery", "b2p_plan_subquery_create",
    "b2p_histogram_fold", "b2p_plan_histogram_quantile_create",
    "b2p_sort_cells_dev", "b2p_sort_cells", "b2p_plan_sort_create",
    "b2p_absent_dev", "b2p_absent", "b2p_plan_absent_create",
    "b2p_range_eval_fields_dev", "b2p_instant_select_fields_dev", "b2p_range_eval_fields", "b2p_instant_select_fields",
    "b2p_plan_range_create_fields", "b2p_sort_cells_fields_dev", "b2p_sort_cells_fields",
    "b2p_instant_select_fields_i64_dev", "b2p_instant_select_fields_i64", "b2p_group_aggregate_i64_dev",
    "b2p_group_aggregate_i64", "b2p_topk_i64_dev", "b2p_topk_i64", "b2p_count_values_i64_dev", "b2p_count_values_i64",
    "b2p_sort_cells_i64_dev", "b2p_sort_cells_i64", "b2p_i64_to_f64_dev", "b2p_i64_to_f64",
    "b2p_step_fn_dev", "b2p_step_fn", "b2p_instant_timestamp_dev", "b2p_instant_timestamp",
    "b2p_plan_empty_metric_create", "b2p_plan_set_timestamp",
    "b2p_plan_label_replace_create", "b2p_plan_label_join_create", "b2p_label_regex_check", "b2p_label_regex_replace",
    "b2p_plan_set_label_columns",
    "b2p_topk_allgather_dev", "b2p_last_exchange_bytes", "b2p_topk_shard_plan", "b2p_topk_shard_candidates_dev",
    "b2p_topk_shard_merge_dev", "b2p_topk_shard_mark_dev",
    "b2p_quantile_allreduce_dev", "b2p_quantile_shard_plan", "b2p_quantile_shard_pass_dev",
    "b2p_quantile_shard_advance_dev",
    "b2p_count_values_shard_heights_dev", "b2p_count_values_allgather_dev", "b2p_count_values_allgather_i64_dev",
    "b2p_count_values_shard_plan", "b2p_count_values_shard_pack_dev", "b2p_count_values_shard_pack_i64_dev",
    "b2p_count_values_shard_merge_dev", "b2p_count_values_shard_merge_i64_dev",
    "b2p_sort_shard_counts_dev", "b2p_sort_cells_allgather_dev", "b2p_sort_cells_allgather_fields_dev",
    "b2p_sort_cells_allgather_i64_dev", "b2p_sort_shard_pack_dev", "b2p_sort_shard_pack_i64_dev",
    "b2p_sort_shard_merge_dev", "b2p_sort_shard_merge_i64_dev",
]


class RangeParams(C.Structure):
    """struct b2p_range_params"""
    _fields_ = [("fn_id", C.c_int32), ("filter_nan", C.c_int32), ("start", C.c_int64), ("end", C.c_int64),
                ("interval", C.c_int64), ("range", C.c_int64), ("offset", C.c_int64),
                ("param0", C.c_double), ("param1", C.c_double)]


class B200LibraryMissing(ImportError):
    pass


_lib = None


def load() -> C.CDLL:
    """Load libb200promql.so; fail loudly when it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200LibraryMissing(
            f"{LIB_PATH} is missing — build it with greptimedb_b200/csrc/build.sh "
            "(or __graft_entry__.build()).  There is no CPU fallback for the GPU path.")
    L = C.CDLL(LIB_PATH)
    vp, i64, u64, u32, i32, dbl = C.c_void_p, C.c_int64, C.c_uint64, C.c_uint32, C.c_int32, C.c_double
    P = C.POINTER(RangeParams)
    sig = {
        "b2p_create": (vp, [C.c_int]),
        "b2p_destroy": (None, [vp]),
        "b2p_last_error": (C.c_char_p, []),
        "b2p_version": (C.c_char_p, []),
        "b2p_set_stream": (C.c_int, [vp, vp]),
        "b2p_use_own_stream": (C.c_int, [vp]),
        "b2p_sync": (C.c_int, [vp]),
        "b2p_num_steps": (i64, [i64, i64, i64]),
        "b2p_last_slow_series": (i64, [vp]),
        "b2p_last_h2d_bytes": (i64, [vp]),
        "b2p_last_warp_tier_series": (i64, [vp]),
        "b2p_last_kernel_ms": (dbl, [vp, C.c_int]),
        "b2p_launch_count": (i64, [vp]),
        "b2p_series_offsets_dev": (C.c_int, [vp, vp, u64, u32, vp]),
        "b2p_range_eval_dev": (C.c_int, [vp, P, vp, vp, vp, u64, u32, vp, vp]),
        "b2p_range_udf_dev": (C.c_int, [vp, i32, vp, vp, u64, vp, vp, u64, i64, dbl, dbl, vp, vp]),
        "b2p_instant_select_dev": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, u64, u32, vp, vp]),
        "b2p_group_aggregate_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_range_group_sum_dev": (C.c_int, [vp, P, vp, vp, vp, u64, u32, vp, u32, vp, vp]),
        "b2p_group_finalize_dev": (C.c_int, [vp, i32, vp, vp, u64]),
        "b2p_group_index_create_dev": (C.c_int, [vp, vp, u32, u32, C.POINTER(vp)]),
        "b2p_group_index_destroy": (None, [vp, vp]),
        "b2p_group_aggregate_indexed_dev": (C.c_int, [vp, i32, vp, vp, vp, u64, vp, vp]),
        "b2p_range_group_sum_indexed_dev": (C.c_int, [vp, P, vp, vp, vp, u64, u32, vp, u32, u32, vp, vp]),
        "b2p_range_group_sum_fused": (C.c_int, [vp, P, vp]),
        "b2p_group_aggregate_partial_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, u32, u64, vp, vp, vp]),
        "b2p_comm_unique_id": (C.c_int, [vp, C.c_size_t]),
        "b2p_comm_init": (C.c_int, [vp, vp, C.c_size_t, C.c_int, C.c_int]),
        "b2p_comm_destroy": (C.c_int, [vp]),
        "b2p_allreduce_partials_dev": (C.c_int, [vp, i32, vp, vp, vp, u64]),
        "b2p_range_group_sum_allreduce_dev": (C.c_int, [vp, P, vp, vp, vp, u64, u32, vp, i32, vp, vp]),
        "b2p_allreduce_columns_dev": (C.c_int, [vp, vp, vp, u32]),
        "b2p_histogram_fold_dev": (C.c_int, [vp, dbl, vp, vp, vp, u32, vp, vp, u64, vp, vp]),
        "b2p_range_histogram_fold": (C.c_int, [vp, P, vp, vp, vp, vp, u64, u32, dbl, vp, vp, vp, u32, vp, vp]),
        "b2p_histogram_quantile_dev": (C.c_int, [vp, dbl, vp, u32, vp, vp, u32, u64, vp, vp]),
        "b2p_column_reduce_dev": (C.c_int, [vp, vp, u32, u64, vp, vp]),
        "b2p_host_scan_series": (C.c_int, [vp, vp, vp, u64, u32, u32, vp, vp, vp, vp]),
        "b2p_range_eval": (C.c_int, [vp, P, vp, vp, vp, vp, u64, u32, vp, vp, vp]),
        "b2p_range_udf": (C.c_int, [vp, i32, vp, vp, u64, vp, vp, u64, i64, dbl, dbl, vp, vp]),
        "b2p_instant_select": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, vp, u64, u32, vp, vp]),
        "b2p_group_aggregate": (C.c_int, [vp, i32, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_histogram_quantile": (C.c_int, [vp, dbl, vp, u32, vp, vp, u32, u64, vp, vp]),
        "b2p_synth_fill_dev": (C.c_int, [vp, u64, u64, u32, i64, i64, u32, i32, u64, vp, vp, vp]),
        "b2p_binary_op_dev": (C.c_int, [vp, i32, i32, vp, vp, vp, u32, vp, vp, vp, u32, u64, u64, vp, vp]),
        "b2p_scalar_op_dev": (C.c_int, [vp, i32, i32, i32, dbl, vp, vp, u64, u64, vp, vp]),
        "b2p_count_valid_words_dev": (C.c_int, [vp, vp, u64, u64, vp]),
        "b2p_binary_op": (C.c_int, [vp, i32, i32, vp, vp, vp, u32, vp, vp, vp, u32, u64, u64, vp, vp]),
        "b2p_scalar_op": (C.c_int, [vp, i32, i32, i32, dbl, vp, vp, u64, u64, vp, vp]),
        "b2p_plan_range_create": (vp, [vp, C.c_char_p, P, C.c_char_p, C.c_char_p, C.POINTER(C.c_char_p), i32, C.c_char_p,
                                       C.POINTER(C.c_char_p), i32]),
        "b2p_plan_set_instant": (C.c_int, [vp, i64]),
        "b2p_plan_set_histogram_quantile": (C.c_int, [vp, C.c_char_p, dbl]),
        "b2p_plan_set_label_columns": (C.c_int, [vp, C.POINTER(C.c_char_p), i32]),
        "b2p_plan_push_batch": (C.c_int, [vp, vp, vp]),
        "b2p_plan_execute": (C.c_int, [vp, vp, vp]),
        "b2p_plan_num_series": (i64, [vp]),
        "b2p_plan_destroy": (None, [vp]),
        "b2p_plan_last_error": (C.c_char_p, []),
        "b2p_plan_set_scalar_op": (C.c_int, [vp, i32, dbl, i32, i32]),
        "b2p_plan_binary_create": (vp, [vp, i32, i32, vp, vp, C.c_char_p, C.POINTER(C.c_char_p), i32, C.c_char_p]),
        "b2p_setop_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_setop": (C.c_int, [vp, i32, vp, vp, vp, u32, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_plan_setop_create": (vp, [vp, i32, vp, vp, C.c_char_p, C.POINTER(C.c_char_p), i32]),
        "b2p_instant_fn_dev": (C.c_int, [vp, i32, dbl, dbl, vp, vp, u64, u64, vp, vp]),
        "b2p_instant_fn": (C.c_int, [vp, i32, dbl, dbl, vp, vp, u64, u64, vp, vp]),
        "b2p_scalar_calculate_dev": (C.c_int, [vp, vp, vp, vp, u32, u64, vp, vp]),
        "b2p_scalar_calculate": (C.c_int, [vp, vp, vp, vp, u32, u64, vp, vp]),
        "b2p_topk_dev": (C.c_int, [vp, i32, dbl, vp, vp, vp, vp, u64, vp]),
        "b2p_topk": (C.c_int, [vp, i32, dbl, vp, vp, vp, u32, u32, vp, u64, vp]),
        "b2p_plan_topk_create": (vp, [vp, i32, dbl, vp, C.c_char_p, C.POINTER(C.c_char_p), i32]),
        "b2p_group_quantile_dev": (C.c_int, [vp, dbl, vp, vp, vp, u64, vp, vp]),
        "b2p_group_quantile": (C.c_int, [vp, dbl, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_plan_aggregate_create": (vp, [vp, C.c_char_p, dbl, vp, C.c_char_p, C.POINTER(C.c_char_p), i32]),
        "b2p_count_values_dev": (C.c_int, [vp, vp, vp, vp, u64, vp, vp]),
        "b2p_count_values": (C.c_int, [vp, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_plan_count_values_create": (vp, [vp, C.c_char_p, vp, C.c_char_p, C.POINTER(C.c_char_p), i32]),
        "b2p_subquery_dev": (C.c_int, [vp, P, i64, i64, vp, vp, u32, u64, vp, vp]),
        "b2p_subquery": (C.c_int, [vp, P, i64, i64, vp, vp, u32, u64, vp, vp]),
        "b2p_plan_subquery_create": (vp, [vp, C.c_char_p, P, vp]),
        "b2p_histogram_fold": (C.c_int, [vp, dbl, vp, vp, vp, u32, vp, vp, u32, u64, vp, vp]),
        "b2p_plan_histogram_quantile_create": (vp, [vp, C.c_char_p, dbl, vp]),
        "b2p_sort_cells_dev": (C.c_int, [vp, i32, vp, vp, u32, u64, vp, vp]),
        "b2p_sort_cells": (C.c_int, [vp, i32, vp, vp, u32, u64, vp, vp]),
        "b2p_plan_sort_create": (vp, [vp, C.c_char_p, vp, C.POINTER(C.c_char_p), i32]),
        "b2p_absent_dev": (C.c_int, [vp, vp, u32, u64, vp, vp]),
        "b2p_absent": (C.c_int, [vp, vp, u32, u64, vp, vp]),
        "b2p_plan_absent_create": (vp, [vp, i64, i64, i64, C.c_char_p, C.c_char_p, C.POINTER(C.c_char_p),
                                        C.POINTER(C.c_char_p), i32, vp]),
        "b2p_range_eval_fields_dev": (C.c_int, [vp, P, vp, vp, vp, i32, vp, u64, u32, vp, vp]),
        "b2p_instant_select_fields_dev": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, i32, vp, u64, u32, vp, vp]),
        "b2p_range_eval_fields": (C.c_int, [vp, P, vp, vp, vp, i32, vp, vp, u64, u32, vp, vp]),
        "b2p_instant_select_fields": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, i32, vp, vp, u64, u32, vp, vp]),
        "b2p_plan_range_create_fields": (vp, [vp, C.c_char_p, P, C.c_char_p, C.POINTER(C.c_char_p), i32,
                                              C.POINTER(C.c_char_p), i32, C.c_char_p, C.POINTER(C.c_char_p), i32]),
        "b2p_sort_cells_fields_dev": (C.c_int, [vp, i32, vp, i32, vp, u32, u64, vp, vp]),
        "b2p_sort_cells_fields": (C.c_int, [vp, i32, vp, i32, vp, u32, u64, vp, vp]),
        "b2p_instant_select_fields_i64_dev": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, i32, vp, u64, u32, vp, vp]),
        "b2p_instant_select_fields_i64": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, i32, vp, vp, u64, u32, vp, vp]),
        "b2p_group_aggregate_i64_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_group_aggregate_i64": (C.c_int, [vp, i32, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_topk_i64_dev": (C.c_int, [vp, i32, dbl, vp, vp, vp, vp, u64, vp]),
        "b2p_topk_i64": (C.c_int, [vp, i32, dbl, vp, vp, vp, u32, u32, vp, u64, vp]),
        "b2p_count_values_i64_dev": (C.c_int, [vp, vp, vp, vp, u64, vp, vp]),
        "b2p_count_values_i64": (C.c_int, [vp, vp, vp, vp, u32, u32, u64, vp, vp]),
        "b2p_sort_cells_i64_dev": (C.c_int, [vp, i32, vp, vp, u32, u64, vp, vp]),
        "b2p_sort_cells_i64": (C.c_int, [vp, i32, vp, vp, u32, u64, vp, vp]),
        "b2p_i64_to_f64_dev": (C.c_int, [vp, vp, u64, vp]),
        "b2p_i64_to_f64": (C.c_int, [vp, vp, u64, vp]),
        "b2p_plan_set_function": (C.c_int, [vp, C.c_char_p, C.POINTER(dbl), i32]),
        "b2p_plan_scalar_create": (vp, [vp, vp]),
        "b2p_step_fn_dev": (C.c_int, [vp, i32, vp, vp, u64, u64, vp]),
        "b2p_step_fn": (C.c_int, [vp, i32, vp, vp, u64, u64, vp]),
        "b2p_instant_timestamp_dev": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, u64, u32, vp, vp]),
        "b2p_instant_timestamp": (C.c_int, [vp, i64, i64, i64, i64, i64, vp, vp, vp, u64, u32, vp, vp]),
        "b2p_plan_empty_metric_create": (vp, [vp, i64, i64, i64, C.c_char_p, C.c_char_p, i32, dbl]),
        "b2p_plan_set_timestamp": (C.c_int, [vp, i64]),
        "b2p_plan_label_replace_create": (vp, [vp, vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p]),
        "b2p_plan_label_join_create": (vp, [vp, vp, C.c_char_p, C.c_char_p, C.POINTER(C.c_char_p), i32]),
        "b2p_label_regex_check": (C.c_int, [C.c_char_p]),
        "b2p_label_regex_replace": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, u64, C.POINTER(u64)]),
        "b2p_topk_allgather_dev": (C.c_int, [vp, i32, dbl, vp, vp, vp, vp, u64, vp]),
        "b2p_last_exchange_bytes": (i64, [vp]),
        "b2p_topk_shard_plan": (C.c_int, [vp, dbl, vp, u32, u64, i32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32),
                                          C.POINTER(u64), C.POINTER(u64)]),
        "b2p_topk_shard_candidates_dev": (C.c_int, [vp, i32, dbl, vp, vp, vp, vp, u64, vp, i32, u32, u32, vp, vp]),
        "b2p_topk_shard_merge_dev": (C.c_int, [vp, dbl, vp, u32, u64, i32, u32, u32, vp, vp]),
        "b2p_topk_shard_mark_dev": (C.c_int, [vp, i32, dbl, vp, vp, vp, vp, u64, vp, i32, u32, vp, vp]),
        "b2p_quantile_allreduce_dev": (C.c_int, [vp, dbl, vp, vp, vp, u64, vp, vp]),
        "b2p_quantile_shard_plan": (C.c_int, [vp, u32, u64, C.POINTER(u32), C.POINTER(u64), C.POINTER(u64)]),
        "b2p_quantile_shard_pass_dev": (C.c_int, [vp, dbl, vp, vp, vp, u64, u32, u32, vp]),
        "b2p_quantile_shard_advance_dev": (C.c_int, [vp, dbl, u32, u64, u32, u32, vp, u32, vp, vp, C.POINTER(u64)]),
        "b2p_count_values_shard_heights_dev": (C.c_int, [vp, vp, vp, u64, vp]),
        "b2p_count_values_allgather_dev": (C.c_int, [vp, vp, vp, vp, u64, vp, vp, vp]),
        "b2p_count_values_allgather_i64_dev": (C.c_int, [vp, vp, vp, vp, u64, vp, vp, vp]),
        "b2p_count_values_shard_plan": (C.c_int, [vp, vp, i32, u32, u64, C.POINTER(u32), C.POINTER(u64)]),
        "b2p_count_values_shard_pack_dev": (C.c_int, [vp, vp, vp, vp, u64, vp, i32, i32, u32, vp]),
        "b2p_count_values_shard_pack_i64_dev": (C.c_int, [vp, vp, vp, vp, u64, vp, i32, i32, u32, vp]),
        "b2p_count_values_shard_merge_dev": (C.c_int, [vp, vp, i32, u32, u64, u32, vp, vp, vp]),
        "b2p_count_values_shard_merge_i64_dev": (C.c_int, [vp, vp, i32, u32, u64, u32, vp, vp, vp]),
        "b2p_sort_shard_counts_dev": (C.c_int, [vp, vp, u32, u64, vp]),
        "b2p_sort_cells_allgather_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, u64, vp, vp, vp]),
        "b2p_sort_cells_allgather_fields_dev": (C.c_int, [vp, i32, vp, i32, vp, vp, u32, u64, vp, vp, vp]),
        "b2p_sort_cells_allgather_i64_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, u64, vp, vp, vp]),
        "b2p_sort_shard_pack_dev": (C.c_int, [vp, i32, vp, i32, vp, vp, u32, u64, u64, vp]),
        "b2p_sort_shard_pack_i64_dev": (C.c_int, [vp, i32, vp, vp, vp, u32, u64, u64, vp]),
        "b2p_sort_shard_merge_dev": (C.c_int, [vp, i32, i32, vp, i32, vp, vp, vp]),
        "b2p_sort_shard_merge_i64_dev": (C.c_int, [vp, i32, vp, i32, vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        f = getattr(L, name)  # AttributeError here means the .so does not match the header
        f.restype = res
        f.argtypes = args
    _lib = L
    return L
