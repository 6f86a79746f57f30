"""ctypes binding of libmono_emb.so (the C ABI in include/mono_emb.h).

This is the same kind of stub a reference maintainer would write to call the engine from
monolith/native_training (see INTEGRATION.md): plain pointers and sizes, no torch types.  The helpers at the
end turn torch tensors and streams into those pointers and choose a call's _bf16 or _scaled twin.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmono_emb.so")


class SegmentCfg(C.Structure):  # mono_segment_cfg
  _fields_ = [("dim", C.c_int32), ("init_type", C.c_int32), ("init_a", C.c_float),
              ("init_b", C.c_float), ("opt_type", C.c_int32), ("opt_p", C.c_float * 6)]


class TableCfg(C.Structure):  # mono_table_cfg
  _fields_ = [("name", C.c_char_p), ("n_segments", C.c_int32),
              ("segments", C.POINTER(SegmentCfg)), ("initial_capacity", C.c_uint64),
              ("default_expire_days", C.c_uint32), ("n_slot_expire", C.c_int32),
              ("slot_ids", C.POINTER(C.c_uint32)), ("slot_expire_days", C.POINTER(C.c_uint32)),
              ("init_seed", C.c_uint64)]


class SliceTask(C.Structure):  # mono_slice_task
  _fields_ = [("nfl_idx", C.c_int32), ("slice_start", C.c_int32), ("dim", C.c_int32),
              ("pooling", C.c_int32), ("max_seq_len", C.c_int32), ("out_tensor", C.c_int32),
              ("out_row_stride", C.c_int32), ("out_col", C.c_int32), ("accumulate", C.c_int32)]


class PoolPartC(C.Structure):  # mono_pool_part
  _fields_ = [("table", C.c_int32), ("fids_dev", C.c_void_p), ("n_fids", C.c_int64),
              ("row_offsets_dev", C.c_void_p), ("n_rows", C.c_int64), ("pooling", C.c_int32),
              ("rows_dev", C.c_void_p), ("stride", C.c_int64), ("col", C.c_int32), ("max_seq_len", C.c_int32)]


class ShardingFeature(C.Structure):  # mono_sharding_feature
  _fields_ = [("n_fids", C.c_int64), ("n_rows", C.c_int64), ("table", C.c_int32), ("dims_sum", C.c_int32),
              ("shared", C.c_int32)]


class ReduceSlice(C.Structure):  # mono_reduce_slice
  _fields_ = [("dim", C.c_int32), ("out_dev", C.c_void_p), ("stride", C.c_int64)]


class ReduceFeature(C.Structure):  # mono_reduce_feature
  _fields_ = [("splits_dev", C.c_void_p), ("batch_size", C.c_int64), ("rows_dev", C.c_void_p), ("n_rows", C.c_int64),
              ("row_stride", C.c_int64), ("dim", C.c_int32), ("pooling", C.c_int32),
              ("slices", C.POINTER(ReduceSlice)), ("n_slices", C.c_int32)]


class NormTensor(C.Structure):  # mono_norm_tensor
  _fields_ = [("data_dev", C.c_void_p), ("n", C.c_int64), ("dtype", C.c_int32)]


MAX_POOL_PARTS = 1024  # MONO_MAX_POOL_PARTS
MAX_NORM_TENSORS = 4096  # MONO_MAX_NORM_TENSORS
DTYPE_F32, DTYPE_BF16 = 0, 1
OPT_SGD, OPT_ADAGRAD, OPT_FTRL, OPT_ADAM = 0, 1, 2, 3
OPT_MOMENTUM, OPT_RMSPROP, OPT_RMSPROPV2, OPT_ADADELTA, OPT_AMSGRAD = 4, 5, 6, 7, 8
OPT_MOVING_AVERAGE, OPT_GROUP_ADAGRAD = 9, 10
INIT_ZEROS, INIT_ONES, INIT_CONSTANT, INIT_UNIFORM = 0, 1, 2, 3
POOL_SUM, POOL_MEAN, POOL_FIRSTN = 0, 1, 2
FLAG_IDS_UNIQUE, FLAG_DEDUP_SUM = 1, 2

_p = C.c_void_p
_i32, _i64, _u32 = C.c_int32, C.c_int64, C.c_uint32

_BF16, _SCALED, _ALL = ("_bf16",), ("_scaled",), ("_bf16", "_scaled", "_bf16_scaled")


def _twins(base, restype, argtypes, twins):
  """`base` and its twins: a "_bf16" twin takes the base's arguments, a "_scaled" one adds the device pointer of the
  gradient scale just before the stream."""
  return {base + t: (restype, argtypes[:-1] + [_p] + argtypes[-1:] if t.endswith("_scaled") else argtypes)
          for t in ("",) + twins}


_LOOKUP = [_p, _p, _p, _p, _p]
_FILL = [_i32, _p, _p, _i32, _p, _p, _i64, _p, _p, _i64, _p, _p, _p]
_FILL_GRAD = [_i32, _p, _p, _i32, _p, _p, _p, _p, _i64, _p, _p, _p]
_LAYOUT = [_i32, _p, _p, _i32, _p, _i64, _p, _i32, _p, _i32, _i32, C.POINTER(SliceTask), _i32, _p, _p]

# name -> (restype, argtypes); every symbol include/mono_emb.h declares
SIGNATURES = {
    "mono_last_error": (C.c_char_p, []),
    "mono_abi_version": (_i32, []),
    "mono_kernel_launch_count": (_i64, []),
    "mono_xstep_window_bytes": (_i64, [_i32, _i64, _i32]),
    "mono_xstep_create": (C.c_int, [_p, _i32, _p, _i64, C.POINTER(_p)]),
    "mono_xstep_destroy": (C.c_int, [_p]),
    "mono_xstep_prepare": (C.c_int, [_p, _p, _i64, _p]),
    "mono_xstep_forward": (C.c_int, [_p, _p, _i64, _p, _i64, _i32, _p, _i64, _i32, _p]),
    **_twins("mono_xstep_backward", C.c_int, [_p, _p, _i64, _i32, _p, _i32, _p, _i64, _p], _SCALED),
    "mono_bench_tower_scratch_floats": (_i64, []),
    "mono_bench_tower_grad": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _p, _i64, _p]),
    "mono_set_option": (C.c_int, [C.c_char_p, _i64]),
    "mono_get_option": (_i64, [C.c_char_p]),
    "mono_mtable_create": (C.c_int, [C.POINTER(TableCfg), _i32, _i32, C.POINTER(_p)]),
    "mono_mtable_destroy": (C.c_int, [_p]),
    "mono_mtable_num_tables": (_i32, [_p]),
    "mono_mtable_table_index": (_i32, [_p, C.c_char_p]),
    "mono_mtable_table_name": (C.c_char_p, [_p, _i32]),
    "mono_mtable_dim": (_i32, [_p, _i32]),
    "mono_mtable_slice_size": (_i32, [_p, _i32]),
    "mono_mtable_state_floats": (_i32, [_p, _i32]),
    "mono_mtable_size": (C.c_int, [_p, _i32, C.POINTER(_i64), _p]),
    "mono_mtable_max_update_ts": (_i64, [_p, _i32]),
    "mono_mtable_counters": (C.c_int, [_p, _i32, _p, _i32, _p]),
    "mono_mtable_lookup": (C.c_int, _LOOKUP),
    "mono_mtable_fused_offsets": (C.c_int, [_p, _p, _i32, _p, _p, _p]),
    "mono_mtable_fused_lookup": (C.c_int, [_p, _p, _p, _i32, _i64, _p, _p]),
    "mono_mtable_set_hash_filter": (C.c_int, [_p, _i32, _i64, _u32, _p, _p, _i32, _p]),
    "mono_mtable_hash_filter_cells": (C.c_int, [_p, _i32, _p, _i64, _p]),
    "mono_mtable_contains": (C.c_int, [_p, _i32, _p, _i64, _p, _p]),
    "mono_mtable_lookup_pool": (C.c_int, [_p, _i32, _p, _p, _i64, _i32, _p, _i64, _i32, _p]),
    **_twins("mono_mtable_pool_backward", C.c_int,
             [_p, _i32, _p, _i64, _p, _i64, _i32, _p, _i64, _i32, _p, _i64, _i64, _p], _SCALED),
    **_twins("mono_mtable_lookup_pool_parts", C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p], _BF16),
    **_twins("mono_mtable_pool_backward_parts", C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p, _i64, _i64, _p], _ALL),
    "mono_mtable_optimize": (C.c_int, [_p, _p, _p, _p, _p, _i64, _i64, _u32, _p]),
    "mono_mtable_fused_optimize": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i32, _u32, _p]),
    "mono_mtable_assign": (C.c_int, [_p, _p, _p, _p, _i64, _u32, _p]),
    "mono_mtable_assign_add": (C.c_int, [_p, _p, _p, _p, _i64, _u32, _p]),
    "mono_mtable_reinitialize": (C.c_int, [_p, _i32, _p, _i64, _p, _i64, _p]),
    "mono_mtable_evict": (C.c_int, [_p, _i32, _i64, _p]),
    "mono_mtable_lookup_entry": (C.c_int, [_p, _i32, _p, _i64, _p, _p]),
    "mono_mtable_export": (C.c_int, [_p, _i32, C.POINTER(_i64), _i64, _p, _p, C.POINTER(_i64), _p]),
    "mono_mtable_restore_rows": (C.c_int, [_p, _i32, _p, _i64, _p, _p]),
    "mono_reorder_by_indices": (C.c_int, [_i32, _p, _p, _i32, _i32, _p, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "mono_dedup": (C.c_int, [_i32, _p, _i64, _p, _p, _p, _p, _p]),
    "mono_sharding_sparse_fids": (C.c_int, [_i32, _p, _p, C.POINTER(ShardingFeature), _i32, _i32, _i32, _i32, _p, _p,
                                            _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "mono_unique_key_with_value_and_offset": (C.c_int, [_i32, _p, _p, _i32, _p, _p, _p, _p, _p, _p, _p, _p]),
    "mono_ragged_split_by_indices": (C.c_int, [_i32, _p, _p, _i64, _p, _i32, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "mono_fill_with_offset_map": (C.c_int, _FILL),
    "mono_fill_with_offset_map_grad": (C.c_int, _FILL_GRAD),
    "mono_mtable_lookup_f16": (C.c_int, _LOOKUP),
    "mono_sharding_sparse_fids_v5": (C.c_int, [_i32, _p, _p, C.POINTER(ShardingFeature), _i32, _i32, _i32, _i32, _p,
                                               _p, _p, _p, _p, _p, _p, _p, _p, _p, _i32, _p, _p, _p, _p]),
    "mono_normalize_merged_split": (C.c_int, [_i32, _p, _i64, _p, _i64, _p, _p, _p]),
    "mono_round_to_f16": (C.c_int, [_i32, _p, _i64, _p, _p]),
    **_twins("mono_embedding_to_layout_f16in", C.c_int, _LAYOUT, _BF16),
    "mono_fill_with_offset_map_f16": (C.c_int, _FILL),
    "mono_fill_with_offset_map_grad_f16": (C.c_int, _FILL_GRAD),
    "mono_grouping_create": (C.c_int, [_i32, C.POINTER(_p)]),
    "mono_grouping_destroy": (C.c_int, [_p]),
    "mono_grouping_build": (C.c_int, [_p, _p, _i64, _i32, _i32, _p, _p, _p, C.POINTER(_i64), _p]),
    **_twins("mono_grouping_reduce", C.c_int, [_p, _p, _i64, _i32, _p, _i64, _i32, _p, _p], _SCALED),
    "mono_peer_create": (C.c_int, [_i32, _i32, _i32, _i64, C.POINTER(_p)]),
    "mono_peer_destroy": (C.c_int, [_p]),
    "mono_peer_detach": (C.c_int, [_p]),
    "mono_peer_handle": (C.c_int, [_p, _p]),
    "mono_peer_attach": (C.c_int, [_p, _p, _i32]),
    "mono_peer_local": (C.c_int, [_p, C.POINTER(_p)]),
    "mono_peer_barrier": (C.c_int, [_p, _p]),
    "mono_peer_put": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "mono_peer_get": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p]),
    "mono_mtable_lookup_push": (C.c_int, [_p, _i32, _p, _p, _p, _i64, _p, _p]),
    **_twins("mono_grouping_reduce_push", C.c_int, [_p, _p, _i64, _i32, _p, _i64, _i32, _p, _p, _i64, _p, _p],
             _SCALED),
    **_twins("mono_gather_pool", C.c_int, [_i32, _p, _p, _p, _i64, _i32, _i32, _p, _i64, _i32, _p], _BF16),
    **_twins("mono_gather_pool_grad", C.c_int, [_i32, _p, _i64, _i32, _p, _p, _i64, _i32, _i32, _p, _p], _ALL),
    **_twins("mono_scatter_grad_rows", C.c_int, [_i32, _p, _i64, _i32, _p, _i64, _p, _i64, _i32, _i32, _p, _i64, _p],
             _ALL),
    **_twins("mono_embedding_to_layout", C.c_int, _LAYOUT, _BF16),
    **_twins("mono_embedding_to_layout_grad", C.c_int, _LAYOUT, _ALL),
    **_twins("mono_reduce_and_split", C.c_int, [_i32, C.POINTER(ReduceFeature), _i32, _p, _p], _BF16),
    **_twins("mono_reduce_and_split_grad", C.c_int, [_i32, C.POINTER(ReduceFeature), _i32, _p, _p], _ALL),
    "mono_mtable_note_update_ts": (C.c_int, [_p, _i32, _i64]),
    "mono_global_norm": (C.c_int, [_i32, C.POINTER(NormTensor), _i32, C.c_float, _p, _p, _p]),
    **_twins("mono_xstep_forward_parts", C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p], _BF16),
    **_twins("mono_xstep_backward_parts", C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p, _i64, _p], _ALL),
    "mono_grouping_build_parts": (C.c_int, [_p, _p, C.POINTER(PoolPartC), _i32, _i32, _p, _p, _p, C.POINTER(_i64),
                                            _p]),
    **_twins("mono_gather_pool_parts", C.c_int, [_p, _p, _p, C.POINTER(PoolPartC), _i32, _p], _BF16),
    **_twins("mono_grouping_reduce_parts", C.c_int, [_p, _p, C.POINTER(PoolPartC), _i32, _p, _p], _ALL),
    **_twins("mono_grouping_reduce_push_parts", C.c_int, [_p, _p, C.POINTER(PoolPartC), _i32, _p, _p, _i64, _p, _p],
             _ALL),
    "mono_ckpt_last_error": (C.c_char_p, []),
    "mono_ckpt_writer_open": (C.c_int, [C.c_char_p, C.c_char_p, _i32, C.POINTER(_p)]),
    "mono_ckpt_writer_begin_table": (C.c_int, [_p, C.c_char_p, C.POINTER(SegmentCfg), _i32]),
    "mono_ckpt_writer_add": (C.c_int, [_p, _p, _p, _i64, _i64, _p, C.POINTER(_i64)]),
    "mono_ckpt_writer_end_table": (C.c_int, [_p]),
    "mono_ckpt_writer_close": (C.c_int, [_p, _i32]),
    "mono_ckpt_reader_open": (C.c_int, [C.c_char_p, C.c_char_p, _i32, C.POINTER(_p)]),
    "mono_ckpt_reader_next_table": (C.c_int, [_p, C.c_char_p, _i32, C.POINTER(_i64), C.POINTER(_i32)]),
    "mono_ckpt_reader_read": (C.c_int, [_p, C.POINTER(SegmentCfg), _i32, _p, _p, _i64, C.POINTER(_i64)]),
    "mono_ckpt_reader_close": (C.c_int, [_p]),
    "mono_ckpt_encode_entry": (_i64, [C.POINTER(SegmentCfg), _i32, _i64, _p, _p, _i64]),
    "mono_ckpt_decode_entry": (C.c_int, [C.POINTER(SegmentCfg), _i32, _p, _i64, C.POINTER(_i64), _p]),
    "mono_ckpt_crc32c": (C.c_uint32, [_p, _i64]),
    "mono_ckpt_masked_crc32c": (C.c_uint32, [_p, _i64]),
    "mono_ckpt_snappy_compress": (_i64, [_p, _i64, _p, _i64]),
    "mono_ckpt_snappy_uncompress": (_i64, [_p, _i64, _p, _i64]),
    "mono_mtable_lookup_host": (C.c_int, [_p, _p, _p, _p]),
    "mono_mtable_lookup_pool_host": (C.c_int, [_p, _i32, _p, _p, _i64, _i64, _i32, _p]),
    "mono_mtable_optimize_host": (C.c_int, [_p, _p, _p, _p, _p, _i64, _i64, _u32]),
}

_lib = None


class MonoError(RuntimeError):
  pass


def load():
  """Loads the CUDA library; raises loudly if it has not been built (no fallback)."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(monolith_b200 has no CPU fallback)")
  lib = C.CDLL(LIB_PATH)
  for name, (res, args) in SIGNATURES.items():
    fn = getattr(lib, name)
    fn.restype = res
    fn.argtypes = args
  _lib = lib
  return lib


def check(status, value_error: bool = False):
  """Raises MonoError for a failed call's status; with value_error, an invalid argument (-1) raises ValueError with
  the engine's message alone."""
  if status != 0:
    msg = load().mono_last_error()
    msg = msg.decode() if msg else ''
    if status == -1 and value_error:
      raise ValueError(msg)
    kinds = {-1: "InvalidArgument", -2: "ResourceExhausted", -3: "CudaError", -4: "Internal"}
    raise MonoError(f"{kinds.get(status, status)}: {msg}")


def call(base: str, *args, bf16: bool = False, scale=None, stream, value_error: bool = False):
  """Calls `base`, or its twin: `base`_bf16 for bf16=True, `base`[_bf16]_scaled for a scale pointer, which goes just
  before the stream.  The symbol is looked up on the loaded library at every call; a twin SIGNATURES does not
  declare raises KeyError.  The status goes to check()."""
  name = base + ("_bf16" if bf16 else "") + ("" if scale is None else "_scaled")
  if name not in SIGNATURES:
    raise KeyError(f"{name} is not a C entry point")
  check(getattr(load(), name)(*args, *(() if scale is None else (scale,)), stream), value_error)


def ptr(t):
  """A tensor's device pointer (None for None)."""
  return None if t is None else C.c_void_p(t.data_ptr())


def stream(device):
  """The current CUDA stream of `device`."""
  return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


# pooling name -> mono pooling code: the calls that pool one flat feature take SUM and MEAN, PoolPart FIRSTN too
POOLINGS = {"sum": POOL_SUM, "mean": POOL_MEAN}
PART_POOLINGS = dict(POOLINGS, firstn=POOL_FIRSTN)


def row_offsets(offsets, n_rows: int, device=None):
  """-> (offsets as contiguous int32 on `device` (None: where they are), their row count), or (None, n_rows) without
  offsets (one FID per row)."""
  if offsets is None:
    return None, n_rows
  offsets = offsets.to(device=device, dtype=torch.int32).contiguous()
  return offsets, offsets.numel() - 1
