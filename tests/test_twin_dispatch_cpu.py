"""The Python side of the C ABI's twin entry points, checked without a GPU: _lib.SIGNATURES declares every twin with
its base's arguments (plus the scale before the stream for a _scaled twin), and _lib.call reaches the twin the
arguments ask for, with the scale just before the stream."""
import ctypes as C

import pytest
import torch

from monolith_b200 import _lib

# SIGNATURES as written out symbol by symbol before the twins were declared per family:
# name -> (restype name, [argtype names])
SNAPSHOT = {
    "mono_last_error": ("c_char_p", []),
    "mono_abi_version": ("c_int", []),
    "mono_kernel_launch_count": ("c_long", []),
    "mono_xstep_window_bytes": ("c_long", ["c_int", "c_long", "c_int"]),
    "mono_xstep_create": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "LP_c_void_p"]),
    "mono_xstep_destroy": ("c_int", ["c_void_p"]),
    "mono_xstep_prepare": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_void_p"]),
    "mono_xstep_forward": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_void_p", "c_long", "c_int", "c_void_p",
        "c_long", "c_int", "c_void_p"]),
    "mono_xstep_backward": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_void_p", "c_int", "c_void_p",
        "c_long", "c_void_p"]),
    "mono_bench_tower_scratch_floats": ("c_long", []),
    "mono_bench_tower_grad": ("c_int", ["c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p", "c_void_p",
        "c_void_p", "c_void_p", "c_long", "c_void_p"]),
    "mono_set_option": ("c_int", ["c_char_p", "c_long"]),
    "mono_get_option": ("c_long", ["c_char_p"]),
    "mono_mtable_create": ("c_int", ["LP_TableCfg", "c_int", "c_int", "LP_c_void_p"]),
    "mono_mtable_destroy": ("c_int", ["c_void_p"]),
    "mono_mtable_num_tables": ("c_int", ["c_void_p"]),
    "mono_mtable_table_index": ("c_int", ["c_void_p", "c_char_p"]),
    "mono_mtable_table_name": ("c_char_p", ["c_void_p", "c_int"]),
    "mono_mtable_dim": ("c_int", ["c_void_p", "c_int"]),
    "mono_mtable_slice_size": ("c_int", ["c_void_p", "c_int"]),
    "mono_mtable_state_floats": ("c_int", ["c_void_p", "c_int"]),
    "mono_mtable_size": ("c_int", ["c_void_p", "c_int", "LP_c_long", "c_void_p"]),
    "mono_mtable_max_update_ts": ("c_long", ["c_void_p", "c_int"]),
    "mono_mtable_counters": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_int", "c_void_p"]),
    "mono_mtable_lookup": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_mtable_fused_offsets": ("c_int", ["c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_mtable_fused_lookup": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_int", "c_long", "c_void_p",
        "c_void_p"]),
    "mono_mtable_set_hash_filter": ("c_int", ["c_void_p", "c_int", "c_long", "c_uint", "c_void_p", "c_void_p", "c_int",
        "c_void_p"]),
    "mono_mtable_hash_filter_cells": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p"]),
    "mono_mtable_contains": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_mtable_lookup_pool": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_void_p", "c_long", "c_int", "c_void_p",
        "c_long", "c_int", "c_void_p"]),
    "mono_mtable_pool_backward": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p", "c_long", "c_int",
        "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_long", "c_void_p"]),
    "mono_mtable_lookup_pool_parts": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p"]),
    "mono_mtable_pool_backward_parts": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long", "c_long",
        "c_void_p"]),
    "mono_mtable_lookup_pool_parts_bf16": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p"]),
    "mono_mtable_pool_backward_parts_bf16": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long",
        "c_long", "c_void_p"]),
    "mono_mtable_optimize": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_long", "c_long",
        "c_uint", "c_void_p"]),
    "mono_mtable_fused_optimize": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p",
        "c_void_p", "c_long", "c_long", "c_int", "c_uint", "c_void_p"]),
    "mono_mtable_assign": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_long", "c_uint", "c_void_p"]),
    "mono_mtable_assign_add": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_long", "c_uint",
        "c_void_p"]),
    "mono_mtable_reinitialize": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p", "c_long",
        "c_void_p"]),
    "mono_mtable_evict": ("c_int", ["c_void_p", "c_int", "c_long", "c_void_p"]),
    "mono_mtable_lookup_entry": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_mtable_export": ("c_int", ["c_void_p", "c_int", "LP_c_long", "c_long", "c_void_p", "c_void_p", "LP_c_long",
        "c_void_p"]),
    "mono_mtable_restore_rows": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_reorder_by_indices": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_int", "c_void_p", "c_int",
        "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_dedup": ("c_int", ["c_int", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p", "c_void_p",
        "c_void_p"]),
    "mono_sharding_sparse_fids": ("c_int", ["c_int", "c_void_p", "c_void_p", "LP_ShardingFeature", "c_int", "c_int",
        "c_int", "c_int", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p",
        "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_unique_key_with_value_and_offset": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p",
        "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_ragged_split_by_indices": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_long", "c_void_p", "c_int", "c_int",
        "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_fill_with_offset_map": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p", "c_long",
        "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_fill_with_offset_map_grad": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p",
        "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_mtable_lookup_f16": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_sharding_sparse_fids_v5": ("c_int", ["c_int", "c_void_p", "c_void_p", "LP_ShardingFeature", "c_int", "c_int",
        "c_int", "c_int", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p",
        "c_void_p", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_normalize_merged_split": ("c_int", ["c_int", "c_void_p", "c_long", "c_void_p", "c_long", "c_void_p",
        "c_void_p", "c_void_p"]),
    "mono_round_to_f16": ("c_int", ["c_int", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_embedding_to_layout_f16in": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p"]),
    "mono_embedding_to_layout_f16in_bf16": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p"]),
    "mono_fill_with_offset_map_f16": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p",
        "c_long", "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_fill_with_offset_map_grad_f16": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p",
        "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_grouping_create": ("c_int", ["c_int", "LP_c_void_p"]),
    "mono_grouping_destroy": ("c_int", ["c_void_p"]),
    "mono_grouping_build": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_int", "c_void_p", "c_void_p",
        "c_void_p", "LP_c_long", "c_void_p"]),
    "mono_grouping_reduce": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_int",
        "c_void_p", "c_void_p"]),
    "mono_peer_create": ("c_int", ["c_int", "c_int", "c_int", "c_long", "LP_c_void_p"]),
    "mono_peer_destroy": ("c_int", ["c_void_p"]),
    "mono_peer_detach": ("c_int", ["c_void_p"]),
    "mono_peer_handle": ("c_int", ["c_void_p", "c_void_p"]),
    "mono_peer_attach": ("c_int", ["c_void_p", "c_void_p", "c_int"]),
    "mono_peer_local": ("c_int", ["c_void_p", "LP_c_void_p"]),
    "mono_peer_barrier": ("c_int", ["c_void_p", "c_void_p"]),
    "mono_peer_put": ("c_int", ["c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_peer_get": ("c_int", ["c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_mtable_lookup_push": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_void_p", "c_void_p", "c_long", "c_void_p",
        "c_void_p"]),
    "mono_grouping_reduce_push": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_int",
        "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_gather_pool": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_void_p", "c_long", "c_int", "c_int", "c_void_p",
        "c_long", "c_int", "c_void_p"]),
    "mono_gather_pool_grad": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_void_p", "c_long",
        "c_int", "c_int", "c_void_p", "c_void_p"]),
    "mono_scatter_grad_rows": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_void_p",
        "c_long", "c_int", "c_int", "c_void_p", "c_long", "c_void_p"]),
    "mono_embedding_to_layout": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long", "c_void_p",
        "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p"]),
    "mono_embedding_to_layout_grad": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p"]),
    "mono_gather_pool_bf16": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_void_p", "c_long", "c_int", "c_int",
        "c_void_p", "c_long", "c_int", "c_void_p"]),
    "mono_gather_pool_grad_bf16": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_void_p", "c_long",
        "c_int", "c_int", "c_void_p", "c_void_p"]),
    "mono_scatter_grad_rows_bf16": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_void_p",
        "c_long", "c_int", "c_int", "c_void_p", "c_long", "c_void_p"]),
    "mono_embedding_to_layout_bf16": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p"]),
    "mono_embedding_to_layout_grad_bf16": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p"]),
    "mono_reduce_and_split": ("c_int", ["c_int", "LP_ReduceFeature", "c_int", "c_void_p", "c_void_p"]),
    "mono_reduce_and_split_grad": ("c_int", ["c_int", "LP_ReduceFeature", "c_int", "c_void_p", "c_void_p"]),
    "mono_reduce_and_split_bf16": ("c_int", ["c_int", "LP_ReduceFeature", "c_int", "c_void_p", "c_void_p"]),
    "mono_reduce_and_split_grad_bf16": ("c_int", ["c_int", "LP_ReduceFeature", "c_int", "c_void_p", "c_void_p"]),
    "mono_mtable_note_update_ts": ("c_int", ["c_void_p", "c_int", "c_long"]),
    "mono_global_norm": ("c_int", ["c_int", "LP_NormTensor", "c_int", "c_float", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_mtable_pool_backward_parts_scaled": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long",
        "c_long", "c_void_p", "c_void_p"]),
    "mono_mtable_pool_backward_parts_bf16_scaled": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long",
        "c_long", "c_void_p", "c_void_p"]),
    "mono_embedding_to_layout_grad_scaled": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p",
        "c_void_p"]),
    "mono_embedding_to_layout_grad_bf16_scaled": ("c_int", ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p",
        "c_long", "c_void_p", "c_int", "c_void_p", "c_int", "c_int", "LP_SliceTask", "c_int", "c_void_p", "c_void_p",
        "c_void_p"]),
    "mono_gather_pool_grad_scaled": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_void_p", "c_long",
        "c_int", "c_int", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_gather_pool_grad_bf16_scaled": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_void_p",
        "c_long", "c_int", "c_int", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_scatter_grad_rows_scaled": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_long", "c_int", "c_int", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_scatter_grad_rows_bf16_scaled": ("c_int", ["c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_long", "c_int", "c_int", "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_mtable_pool_backward_scaled": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_long", "c_void_p", "c_long",
        "c_int", "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_long", "c_void_p", "c_void_p"]),
    "mono_reduce_and_split_grad_scaled": ("c_int", ["c_int", "LP_ReduceFeature", "c_int", "c_void_p", "c_void_p",
        "c_void_p"]),
    "mono_reduce_and_split_grad_bf16_scaled": ("c_int", ["c_int", "LP_ReduceFeature", "c_int", "c_void_p", "c_void_p",
        "c_void_p"]),
    "mono_grouping_reduce_scaled": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_void_p", "c_long", "c_int",
        "c_void_p", "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_push_scaled": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_void_p", "c_long",
        "c_int", "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_xstep_backward_scaled": ("c_int", ["c_void_p", "c_void_p", "c_long", "c_int", "c_void_p", "c_int", "c_void_p",
        "c_long", "c_void_p", "c_void_p"]),
    "mono_xstep_forward_parts": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p"]),
    "mono_xstep_forward_parts_bf16": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p"]),
    "mono_xstep_backward_parts": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long", "c_void_p"]),
    "mono_xstep_backward_parts_bf16": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long",
        "c_void_p"]),
    "mono_xstep_backward_parts_scaled": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_void_p"]),
    "mono_xstep_backward_parts_bf16_scaled": ("c_int", ["c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_long",
        "c_void_p", "c_void_p"]),
    "mono_grouping_build_parts": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_int", "c_void_p",
        "c_void_p", "c_void_p", "LP_c_long", "c_void_p"]),
    "mono_gather_pool_parts": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p"]),
    "mono_gather_pool_parts_bf16": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p"]),
    "mono_grouping_reduce_parts": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_parts_bf16": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p",
        "c_void_p"]),
    "mono_grouping_reduce_parts_scaled": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p",
        "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_parts_bf16_scaled": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p",
        "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_push_parts": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p",
        "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_push_parts_bf16": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p",
        "c_void_p", "c_long", "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_push_parts_scaled": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int", "c_void_p",
        "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_grouping_reduce_push_parts_bf16_scaled": ("c_int", ["c_void_p", "c_void_p", "LP_PoolPartC", "c_int",
        "c_void_p", "c_void_p", "c_long", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_ckpt_last_error": ("c_char_p", []),
    "mono_ckpt_writer_open": ("c_int", ["c_char_p", "c_char_p", "c_int", "LP_c_void_p"]),
    "mono_ckpt_writer_begin_table": ("c_int", ["c_void_p", "c_char_p", "LP_SegmentCfg", "c_int"]),
    "mono_ckpt_writer_add": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_long", "c_long", "c_void_p",
        "LP_c_long"]),
    "mono_ckpt_writer_end_table": ("c_int", ["c_void_p"]),
    "mono_ckpt_writer_close": ("c_int", ["c_void_p", "c_int"]),
    "mono_ckpt_reader_open": ("c_int", ["c_char_p", "c_char_p", "c_int", "LP_c_void_p"]),
    "mono_ckpt_reader_next_table": ("c_int", ["c_void_p", "c_char_p", "c_int", "LP_c_long", "LP_c_int"]),
    "mono_ckpt_reader_read": ("c_int", ["c_void_p", "LP_SegmentCfg", "c_int", "c_void_p", "c_void_p", "c_long",
        "LP_c_long"]),
    "mono_ckpt_reader_close": ("c_int", ["c_void_p"]),
    "mono_ckpt_encode_entry": ("c_long", ["LP_SegmentCfg", "c_int", "c_long", "c_void_p", "c_void_p", "c_long"]),
    "mono_ckpt_decode_entry": ("c_int", ["LP_SegmentCfg", "c_int", "c_void_p", "c_long", "LP_c_long", "c_void_p"]),
    "mono_ckpt_crc32c": ("c_uint", ["c_void_p", "c_long"]),
    "mono_ckpt_masked_crc32c": ("c_uint", ["c_void_p", "c_long"]),
    "mono_ckpt_snappy_compress": ("c_long", ["c_void_p", "c_long", "c_void_p", "c_long"]),
    "mono_ckpt_snappy_uncompress": ("c_long", ["c_void_p", "c_long", "c_void_p", "c_long"]),
    "mono_mtable_lookup_host": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p"]),
    "mono_mtable_lookup_pool_host": ("c_int", ["c_void_p", "c_int", "c_void_p", "c_void_p", "c_long", "c_long", "c_int",
        "c_void_p"]),
    "mono_mtable_optimize_host": ("c_int", ["c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_void_p", "c_long",
        "c_long", "c_uint"]),

}
SUFFIXES = ("_bf16_scaled", "_scaled", "_bf16")


def _names(sig):
  return {k: (r.__name__, [a.__name__ for a in args]) for k, (r, args) in sig.items()}


def test_signatures_are_the_snapshot():
  assert _names(_lib.SIGNATURES) == SNAPSHOT


def _twins():
  """(twin, base, bf16, scaled) of every twin in the snapshot."""
  out = []
  for name in SNAPSHOT:
    for sfx in SUFFIXES:
      if name.endswith(sfx):
        out.append((name, name[:-len(sfx)], "_bf16" in sfx, sfx.endswith("_scaled")))
        break
  return out


def test_twin_families():
  twins = _twins()
  assert len(twins) == 35
  for name, base, bf16, scaled in twins:
    assert base in SNAPSHOT, name
    res, args = SNAPSHOT[name]
    b_res, b_args = SNAPSHOT[base]
    assert res == b_res and args == (b_args[:-1] + ["c_void_p"] + b_args[-1:] if scaled else b_args), name
  for f16, f32 in (("mono_embedding_to_layout_f16in", "mono_embedding_to_layout"),
                   ("mono_fill_with_offset_map_f16", "mono_fill_with_offset_map"),
                   ("mono_fill_with_offset_map_grad_f16", "mono_fill_with_offset_map_grad"),
                   ("mono_mtable_lookup_f16", "mono_mtable_lookup")):
    assert SNAPSHOT[f16] == SNAPSHOT[f32], f16


class _Recorder:
  """Stands in for the loaded library: every symbol records its name and arguments and returns `status`."""

  def __init__(self, status=0):
    self.calls, self.status = [], status

  def mono_last_error(self):
    return b"bad argument"

  def __getattr__(self, name):
    def fn(*args):
      self.calls.append((name, args))
      return self.status
    return fn


@pytest.fixture
def rec(monkeypatch):
  r = _Recorder()
  monkeypatch.setattr(_lib, "load", lambda: r)
  return r


def test_call_reaches_every_twin(rec):
  scale, stream = C.c_void_p(0x5CA1E), C.c_void_p(0x57AE)
  bases = {base for _, base, _, _ in _twins()}
  for name, base, bf16, scaled in _twins():
    rec.calls.clear()
    _lib.call(base, 1, "two", 3.0, bf16=bf16, scale=scale if scaled else None, stream=stream)
    assert rec.calls == [(name, (1, "two", 3.0) + ((scale,) if scaled else ()) + (stream,))], name
  for base in bases:   # no twin asked for: the base itself, never its _scaled twin with a NULL scale
    rec.calls.clear()
    _lib.call(base, 7, stream=stream)
    assert rec.calls == [(base, (7, stream))], base


@pytest.mark.parametrize("base, kw", [("mono_gather_pool", dict(scale=C.c_void_p(1))),
                                      ("mono_mtable_pool_backward", dict(bf16=True)),
                                      ("mono_xstep_forward", dict(bf16=True)),
                                      ("mono_dedup", dict(bf16=True, scale=C.c_void_p(1))),
                                      ("mono_no_such_call", {})])
def test_call_refuses_undeclared_twins(rec, base, kw):
  with pytest.raises(KeyError):
    _lib.call(base, 1, stream=None, **kw)
  assert rec.calls == []


def test_call_checks_the_status(monkeypatch):
  monkeypatch.setattr(_lib, "load", lambda: _Recorder(status=-1))
  with pytest.raises(_lib.MonoError, match="InvalidArgument: bad argument"):
    _lib.call("mono_gather_pool", 1, stream=None)
  with pytest.raises(ValueError, match="^bad argument$"):
    _lib.call("mono_fill_with_offset_map", 1, stream=None, value_error=True)


def test_row_offsets():
  ro, n = _lib.row_offsets(torch.tensor([0, 2, 2, 5], dtype=torch.int64), 99)
  assert ro.dtype == torch.int32 and ro.is_contiguous() and ro.tolist() == [0, 2, 2, 5] and n == 3
  assert _lib.row_offsets(None, 99) == (None, 99)
  assert _lib.PART_POOLINGS == {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN, "firstn": _lib.POOL_FIRSTN}
  assert _lib.POOLINGS == {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}
