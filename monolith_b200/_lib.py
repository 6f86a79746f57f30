"""ctypes binding of libmono_emb.so (the C ABI in include/mono_emb.h).

This is the same kind of stub a reference maintainer would write to call the engine from
monolith/native_training (see INTEGRATION.md): plain pointers and sizes, no torch types.
"""
import ctypes as C
import os

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


MAX_POOL_PARTS = 1024  # MONO_MAX_POOL_PARTS
OPT_SGD, OPT_ADAGRAD, OPT_FTRL, OPT_ADAM = 0, 1, 2, 3
OPT_MOMENTUM, OPT_RMSPROP, OPT_RMSPROPV2, OPT_ADADELTA, OPT_AMSGRAD = 4, 5, 6, 7, 8
OPT_MOVING_AVERAGE, OPT_GROUP_ADAGRAD = 9, 10
INIT_ZEROS, INIT_ONES, INIT_CONSTANT, INIT_UNIFORM = 0, 1, 2, 3
POOL_SUM, POOL_MEAN, POOL_FIRSTN = 0, 1, 2
FLAG_IDS_UNIQUE, FLAG_DEDUP_SUM = 1, 2

_p = C.c_void_p
_i32, _i64, _u32 = C.c_int32, C.c_int64, C.c_uint32

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
    "mono_xstep_backward": (C.c_int, [_p, _p, _i64, _i32, _p, _i32, _p, _i64, _p]),
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
    "mono_mtable_lookup": (C.c_int, [_p, _p, _p, _p, _p]),
    "mono_mtable_fused_offsets": (C.c_int, [_p, _p, _i32, _p, _p, _p]),
    "mono_mtable_fused_lookup": (C.c_int, [_p, _p, _p, _i32, _i64, _p, _p]),
    "mono_mtable_set_hash_filter": (C.c_int, [_p, _i32, _i64, _u32, _p, _p, _i32, _p]),
    "mono_mtable_contains": (C.c_int, [_p, _i32, _p, _i64, _p, _p]),
    "mono_mtable_lookup_pool": (C.c_int, [_p, _i32, _p, _p, _i64, _i32, _p, _i64, _i32, _p]),
    "mono_mtable_pool_backward": (C.c_int, [_p, _i32, _p, _i64, _p, _i64, _i32, _p, _i64, _i32, _p, _i64, _i64, _p]),
    "mono_mtable_lookup_pool_parts": (C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p]),
    "mono_mtable_pool_backward_parts": (C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p, _i64, _i64, _p]),
    "mono_mtable_lookup_pool_parts_bf16": (C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p]),
    "mono_mtable_pool_backward_parts_bf16": (C.c_int, [_p, C.POINTER(PoolPartC), _i32, _p, _i64, _i64, _p]),
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
    "mono_grouping_create": (C.c_int, [_i32, C.POINTER(_p)]),
    "mono_grouping_destroy": (C.c_int, [_p]),
    "mono_grouping_build": (C.c_int, [_p, _p, _i64, _i32, _i32, _p, _p, _p, C.POINTER(_i64), _p]),
    "mono_grouping_reduce": (C.c_int, [_p, _p, _i64, _i32, _p, _i64, _i32, _p, _p]),
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
    "mono_grouping_reduce_push": (C.c_int, [_p, _p, _i64, _i32, _p, _i64, _i32, _p, _p, _i64, _p, _p]),
    "mono_gather_pool": (C.c_int, [_i32, _p, _p, _p, _i64, _i32, _i32, _p, _i64, _i32, _p]),
    "mono_gather_pool_grad": (C.c_int, [_i32, _p, _i64, _i32, _p, _p, _i64, _i32, _i32, _p, _p]),
    "mono_scatter_grad_rows": (C.c_int, [_i32, _p, _i64, _i32, _p, _i64, _p, _i64, _i32, _i32, _p, _i64, _p]),
    "mono_embedding_to_layout": (C.c_int, [_i32, _p, _p, _i32, _p, _i64, _p, _i32, _p, _i32, _i32,
                                           C.POINTER(SliceTask), _i32, _p, _p]),
    "mono_embedding_to_layout_grad": (C.c_int, [_i32, _p, _p, _i32, _p, _i64, _p, _i32, _p, _i32, _i32,
                                                C.POINTER(SliceTask), _i32, _p, _p]),
    "mono_gather_pool_bf16": (C.c_int, [_i32, _p, _p, _p, _i64, _i32, _i32, _p, _i64, _i32, _p]),
    "mono_gather_pool_grad_bf16": (C.c_int, [_i32, _p, _i64, _i32, _p, _p, _i64, _i32, _i32, _p, _p]),
    "mono_scatter_grad_rows_bf16": (C.c_int, [_i32, _p, _i64, _i32, _p, _i64, _p, _i64, _i32, _i32, _p, _i64, _p]),
    "mono_embedding_to_layout_bf16": (C.c_int, [_i32, _p, _p, _i32, _p, _i64, _p, _i32, _p, _i32, _i32,
                                                C.POINTER(SliceTask), _i32, _p, _p]),
    "mono_embedding_to_layout_grad_bf16": (C.c_int, [_i32, _p, _p, _i32, _p, _i64, _p, _i32, _p, _i32, _i32,
                                                     C.POINTER(SliceTask), _i32, _p, _p]),
    "mono_mtable_note_update_ts": (C.c_int, [_p, _i32, _i64]),
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


def check(status):
  if status != 0:
    msg = load().mono_last_error()
    kinds = {-1: "InvalidArgument", -2: "ResourceExhausted", -3: "CudaError", -4: "Internal"}
    raise MonoError(f"{kinds.get(status, status)}: {msg.decode() if msg else ''}")
