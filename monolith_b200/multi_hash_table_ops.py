"""MultiHashTable — host-side mirror of monolith/native_training/multi_hash_table_ops.py.

Same method names, argument meaning and tensor layouts as the reference class
(ref: multi_hash_table_ops.py:186-548): tables are ordered by sorted name (:72,83); ids of all tables
travel as one ragged tensor (values + row_splits, :113-136,528-548) and values as one flat float
tensor.  Instead of TF ops over a CPU cuckoo map, every method calls the sm_90a kernels through
the C ABI (include/mono_emb.h).  Tensors are torch CUDA tensors on the table's device (int64 ids,
float32 values); the mutating methods return `self` where the reference returns a copied wrapper
around the same resource handle (:419-423).
"""
import ctypes as C
import dataclasses
import time
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .entry import HashTableConfigInstance, to_c_table_cfgs


def _ptr(t: Optional[torch.Tensor]):
  return None if t is None else C.c_void_p(t.data_ptr())


def _stream(device) -> C.c_void_p:
  return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ids(t, device) -> torch.Tensor:
  t = torch.as_tensor(t, dtype=torch.int64, device=device) if not isinstance(t, torch.Tensor) else t
  if t.dtype != torch.int64 or t.device != device:
    t = t.to(device=device, dtype=torch.int64)
  return t.reshape(-1).contiguous()


def _f32(t, device) -> torch.Tensor:
  t = torch.as_tensor(t, dtype=torch.float32, device=device) if not isinstance(t, torch.Tensor) else t
  if t.dtype != torch.float32 or t.device != device:
    t = t.to(device=device, dtype=torch.float32)
  return t.contiguous()


@dataclasses.dataclass
class PoolPart:
  """One feature's slice of a step for lookup_pool_parts / pool_backward_parts: the FIDs of table `slot`, pooled by
  `pooling` ("sum", "mean" or "firstn") into rows (row_offsets: CSR [n_rows + 1] int32, None = one FID per row), and
  the output or gradient rows `rows` ([n_rows, >= col + dim] float32 or bfloat16, the table's dim values start at
  column `col`).  bfloat16 rows go to the engine's bf16 calls: the tables and all arithmetic stay float32, outputs are
  rounded once to bfloat16 (nearest even) and gradients are widened exactly to float32.

  "firstn" is a sequence feature (the reference's FirstN combiner): row r holds max_seq_len positions of dim floats
  from column `col` on ([n_rows, >= col + max_seq_len * dim]; a [B, L, dim] tensor viewed as [B, L * dim] with
  col 0), position j being the row of the row's j-th FID, zeros past the row's FIDs; FIDs past max_seq_len are not
  looked up, and on the backward get a zero gradient.  max_seq_len is set for "firstn" only."""
  slot: str
  fids: torch.Tensor
  row_offsets: Optional[torch.Tensor] = None
  pooling: str = "sum"
  rows: Optional[torch.Tensor] = None
  col: int = 0
  max_seq_len: int = 0

  def __post_init__(self):
    if self.pooling not in ("sum", "mean", "firstn"):
      raise ValueError(f"PoolPart.pooling must be 'sum', 'mean' or 'firstn', not {self.pooling!r}")
    if not isinstance(self.max_seq_len, int) or isinstance(self.max_seq_len, bool):
      raise ValueError("PoolPart.max_seq_len must be an int")
    if self.pooling == "firstn" and self.max_seq_len < 1:
      raise ValueError("PoolPart.max_seq_len must be >= 1 for 'firstn'")
    if self.pooling != "firstn" and self.max_seq_len != 0:
      raise ValueError("PoolPart.max_seq_len is set for 'firstn' only")
    if not isinstance(self.col, int) or self.col < 0:
      raise ValueError("PoolPart.col must be a non-negative int")
    if self.rows is not None and (not isinstance(self.rows, torch.Tensor) or self.rows.dim() != 2):
      raise ValueError("PoolPart.rows must be a 2-D tensor")


class MultiHashTable:
  """Maps int64 FIDs to float32 embeddings, K named tables behind one handle."""
  NAME_PREFIX = "MonolithMultiHashTable"

  def __init__(self, configs: Dict[str, HashTableConfigInstance], device=None, name_suffix: str = ""):
    self._lib = _lib.load()
    if not torch.cuda.is_available():
      raise RuntimeError("monolith_b200 needs a CUDA device (there is no CPU fallback)")
    self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if self._device.index is None:
      self._device = torch.device("cuda", torch.cuda.current_device())
    self._table_names: Tuple[str, ...] = tuple(sorted(configs.keys()))
    self._configs = {k: configs[k] for k in self._table_names}
    self._dims = tuple(self._configs[k].table_config.dim_size for k in self._table_names)
    self._shared_name = "_".join([MultiHashTable.NAME_PREFIX, name_suffix])
    arr, keep = to_c_table_cfgs(self._configs)
    h = C.c_void_p()
    _lib.check(self._lib.mono_mtable_create(arr, len(self._table_names), self._device.index, C.byref(h)))
    self._h = h
    del keep
    for k, name in enumerate(self._table_names):  # the library sorts by name too
      assert self._lib.mono_mtable_table_name(self._h, k).decode() == name
      assert self._lib.mono_mtable_dim(self._h, k) == self._dims[k]
    self._slices = tuple(self._lib.mono_mtable_slice_size(self._h, k) for k in range(len(self._dims)))

  @classmethod
  def from_configs(cls, configs: Dict[str, HashTableConfigInstance], *args, **kwargs) -> "MultiHashTable":
    """ref: multi_hash_table_ops.py:270-283."""
    return cls(configs, *args, **kwargs)

  def close(self):
    if getattr(self, "_h", None):
      self._lib.mono_mtable_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass

  # ---- properties -------------------------------------------------------------------------
  @property
  def table_names(self):
    return self._table_names

  @property
  def shared_name(self):
    return self._shared_name

  @property
  def device(self):
    return self._device

  @property
  def handle(self):
    return self._h

  def get_table_dim_sizes(self):
    """ref: multi_hash_table_ops.py:485-486."""
    return self._dims

  def learning_rates(self) -> List[float]:
    """ref: self._learning_rate = stack(learning_rate_list) (:202), one per segment, table order."""
    out = []
    for name in self._table_names:
      out += self._configs[name].call_learning_rate_fns()
    return out

  def size(self, name: Optional[str] = None):
    """Live keys (ref: EmbeddingHashTableInterface::Size).  Synchronises."""
    names = [name] if name else self._table_names
    res = {}
    for n in names:
      v = C.c_int64()
      _lib.check(self._lib.mono_mtable_size(self._h, self._table_names.index(n), C.byref(v),
                                            _stream(self._device)))
      res[n] = v.value
    return res[name] if name else res

  # ---- ragged packing (ref: get_ragged_id / get_flat_value / get_embeddings :528-548) -------
  def get_ragged_id(self, slot_to_id: Dict[str, torch.Tensor]) -> Tuple[torch.Tensor, List[int]]:
    parts, splits = [], [0]
    for name in self._table_names:
      t = _ids(slot_to_id[name], self._device) if name in slot_to_id else None
      n = 0 if t is None else t.numel()
      if n:
        parts.append(t)
      splits.append(splits[-1] + n)
    for k in slot_to_id:
      if k not in self._table_names:
        raise KeyError(f"unknown table {k}")
    values = torch.cat(parts) if parts else torch.empty(0, dtype=torch.int64, device=self._device)
    return values, splits

  def get_flat_value(self, slot_to_value: Dict[str, torch.Tensor]) -> torch.Tensor:
    parts = [
        _f32(slot_to_value[name], self._device).reshape(-1) for name in self._table_names if name in slot_to_value
    ]
    return torch.cat(parts) if parts else torch.empty(0, dtype=torch.float32, device=self._device)

  def get_embeddings(self, splits: Sequence[int], flat: torch.Tensor) -> Dict[str, torch.Tensor]:
    d, off = {}, 0
    for k, name in enumerate(self._table_names):
      n = splits[k + 1] - splits[k]
      d[name] = flat[off:off + n * self._dims[k]].view(n, self._dims[k])
      off += n * self._dims[k]
    return d

  def _split_arr(self, splits: Sequence[int]):
    if len(splits) != len(self._table_names) + 1:
      raise ValueError(f"id_split must have {len(self._table_names) + 1} entries")
    return (C.c_int64 * len(splits))(*[int(s) for s in splits])

  # ---- BaseMultiTypeHashTable API (ref: multi_type_hash_table.py:38-96) -----------------------
  def lookup(self, slot_to_id: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """ref: multi_hash_table_ops.py:382-390.  Miss -> zeros; never inserts."""
    values, splits = self.get_ragged_id(slot_to_id)
    flat = self.raw_lookup(values, splits)
    emb = self.get_embeddings(splits, flat)
    return {k: v for k, v in emb.items() if k in slot_to_id}

  def assign(self, slot_to_id_and_value: Dict[str, Tuple[torch.Tensor, torch.Tensor]], req_time: int = 0,
             ids_unique: bool = False):
    """ref: multi_hash_table_ops.py:349-357."""
    values, splits = self.get_ragged_id({k: v[0] for k, v in slot_to_id_and_value.items()})
    flat = self.get_flat_value({k: v[1] for k, v in slot_to_id_and_value.items()})
    return self.raw_assign(values, splits, flat, req_time, ids_unique)

  def assign_add(self, slot_to_id_and_value: Dict[str, Tuple[torch.Tensor, torch.Tensor]], req_time: int = 0,
                 ids_unique: bool = False):
    """ref: multi_hash_table_ops.py:359-374 (per-id serial semantics for duplicate ids)."""
    values, splits = self.get_ragged_id({k: v[0] for k, v in slot_to_id_and_value.items()})
    flat = self.get_flat_value({k: v[1] for k, v in slot_to_id_and_value.items()})
    self._check_values(values, splits, flat)
    _lib.check(self._lib.mono_mtable_assign_add(self._h, _ptr(values), self._split_arr(splits), _ptr(flat),
                                                int(req_time), _lib.FLAG_IDS_UNIQUE if ids_unique else 0,
                                                _stream(self._device)))
    return self

  def reinitialize(self, slot: str, ids: torch.Tensor):
    """ref: multi_hash_table_ops.py:376-380; status -1 unknown table, 0 inserted, 1 re-initialised."""
    ids = _ids(ids, self._device)
    status = torch.empty(ids.numel(), dtype=torch.int32, device=self._device)
    k = self._table_names.index(slot) if slot in self._table_names else -1
    _lib.check(self._lib.mono_mtable_reinitialize(self._h, k, _ptr(ids), ids.numel(), _ptr(status),
                                                  int(time.time()), _stream(self._device)))
    return self, status

  def apply_gradients(self, slot_to_id_and_grad: Dict[str, Tuple[torch.Tensor, torch.Tensor]],
                      global_step: int = 0, req_time: int = 0, enable_dedup: bool = False,
                      ids_unique: bool = False):
    """ref: multi_hash_table_ops.py:398-407 -> MonolithMultiHashTableOptimize."""
    values, splits = self.get_ragged_id({k: v[0] for k, v in slot_to_id_and_grad.items()})
    flat = self.get_flat_value({k: v[1] for k, v in slot_to_id_and_grad.items()})
    return self.raw_apply_gradients(values, splits, flat, global_step, req_time, enable_dedup, ids_unique)

  def as_op(self, *args, **kwargs):
    return self

  # ---- RawMultiTypeHashTable API (ref: multi_hash_table_ops.py:492-526) ------------------------
  def raw_lookup(self, ids: torch.Tensor, id_split: Sequence[int]) -> torch.Tensor:
    ids = _ids(ids, self._device)
    total = sum((id_split[k + 1] - id_split[k]) * self._dims[k] for k in range(len(self._dims)))
    out = torch.empty(total, dtype=torch.float32, device=self._device)
    if id_split[-1] != ids.numel():
      raise ValueError("id_split does not cover ids")
    _lib.check(self._lib.mono_mtable_lookup(self._h, _ptr(ids), self._split_arr(id_split), _ptr(out),
                                            _stream(self._device)))
    return out

  def _check_values(self, ids, id_split, flat):
    if id_split[-1] != ids.numel():
      raise ValueError("id_split does not cover ids")
    need = sum((id_split[k + 1] - id_split[k]) * self._dims[k] for k in range(len(self._dims)))
    if flat.numel() < need:  # ref: LengthTooShort, multi_hash_table_update_op.cc:41-45
      raise ValueError(f"The length of tensor `value` is too short. Currently value {flat.numel()}")

  def raw_apply_gradients(self, ids: torch.Tensor, id_split: Sequence[int], flat_grad: torch.Tensor,
                          global_step: int = 0, req_time: int = 0, enable_dedup: bool = False,
                          ids_unique: bool = False):
    ids, flat_grad = _ids(ids, self._device), _f32(flat_grad, self._device).reshape(-1)
    self._check_values(ids, id_split, flat_grad)
    lr = self.learning_rates()
    lr_arr = (C.c_float * len(lr))(*lr)
    flags = (_lib.FLAG_IDS_UNIQUE if ids_unique else 0) | (_lib.FLAG_DEDUP_SUM if enable_dedup else 0)
    _lib.check(self._lib.mono_mtable_optimize(self._h, _ptr(ids), self._split_arr(id_split), _ptr(flat_grad),
                                              lr_arr, int(req_time), int(global_step), flags,
                                              _stream(self._device)))
    return self

  def raw_assign(self, ids: torch.Tensor, id_split: Sequence[int], flat_value: torch.Tensor, req_time: int = 0,
                 ids_unique: bool = False):
    ids, flat_value = _ids(ids, self._device), _f32(flat_value, self._device).reshape(-1)
    self._check_values(ids, id_split, flat_value)
    _lib.check(self._lib.mono_mtable_assign(self._h, _ptr(ids), self._split_arr(id_split), _ptr(flat_value),
                                            int(req_time), _lib.FLAG_IDS_UNIQUE if ids_unique else 0,
                                            _stream(self._device)))
    return self

  # ---- fused ops for sync training (ref: multi_hash_table_ops.py:438-483) ----------------------
  def fused_offsets(self, fused_slot_size: Sequence[int], num_of_shards: int):
    K = len(self._dims)
    if len(fused_slot_size) != num_of_shards * K:
      raise ValueError("fused_slot_size must have num_of_shards * num_tables entries")
    ss = (C.c_int32 * len(fused_slot_size))(*[int(x) for x in fused_slot_size])
    emb_splits = (C.c_int32 * num_of_shards)()
    id_off = (C.c_int32 * (num_of_shards * K + 1))()
    emb_off = (C.c_int32 * (num_of_shards * K + 1))()
    _lib.check(self._lib.mono_mtable_fused_offsets(self._h, ss, num_of_shards, emb_splits, id_off, emb_off))
    return ss, list(emb_splits), list(id_off), list(emb_off)

  def fused_lookup(self, ids: torch.Tensor, fused_slot_size: Sequence[int], num_of_shards: int, req_time: int = 0,
                   out: Optional[torch.Tensor] = None):
    """ref: multi_hash_table_ops.py:442-454 -> MonolithMultiHashTableFusedLookup.
    Returns (embeddings, embedding_splits, id_offsets, embedding_offsets, indices)."""
    ids = _ids(ids, self._device)
    ss, emb_splits, id_off, emb_off = self.fused_offsets(fused_slot_size, num_of_shards)
    if id_off[-1] != ids.numel():
      raise ValueError("fused_slot_size does not cover ids")
    if out is None:
      out = torch.empty(emb_off[-1], dtype=torch.float32, device=self._device)
    elif out.numel() < emb_off[-1] or out.dtype != torch.float32 or not out.is_contiguous():
      raise ValueError("fused_lookup: out must be a contiguous float32 buffer of at least emb_offsets[-1] floats")
    _lib.check(self._lib.mono_mtable_fused_lookup(self._h, _ptr(ids), ss, num_of_shards, int(req_time), _ptr(out),
                                                  _stream(self._device)))
    return out, emb_splits, id_off, emb_off, ids

  def fused_apply_gradient(self, ids: torch.Tensor, indices: torch.Tensor, fused_slot_size: Sequence[int],
                           id_grads: torch.Tensor, id_offsets: Sequence[int], grad_offsets: Sequence[int],
                           global_step: int, req_time: int, num_of_shards: int,
                           enable_grad_accumulation: bool = False, ids_unique: bool = True):
    """ref: multi_hash_table_ops.py:458-483 -> MonolithMultiHashTableFusedOptimize.
    ids_unique: ids are unique inside each (shard, table) segment (what fused_reorder_by_indices
    produces); the same FID may still appear once per shard and is then applied in shard order."""
    ids, id_grads = _ids(ids, self._device), _f32(id_grads, self._device).reshape(-1)
    ss = (C.c_int32 * len(fused_slot_size))(*[int(x) for x in fused_slot_size])
    io = (C.c_int32 * len(id_offsets))(*[int(x) for x in id_offsets])
    go = (C.c_int32 * len(grad_offsets))(*[int(x) for x in grad_offsets])
    lr = self.learning_rates()
    lr_arr = (C.c_float * len(lr))(*lr)
    flags = (_lib.FLAG_IDS_UNIQUE if (ids_unique and not enable_grad_accumulation) else 0) | \
            (_lib.FLAG_DEDUP_SUM if enable_grad_accumulation else 0)
    _lib.check(self._lib.mono_mtable_fused_optimize(self._h, _ptr(ids), ss, _ptr(id_grads), io, go, lr_arr,
                                                    int(req_time), int(global_step), num_of_shards, flags,
                                                    _stream(self._device)))
    return self

  # ---- engine extensions -------------------------------------------------------------------
  def lookup_push(self, slot: str, ids: torch.Tensor, counts: Sequence[int], window, region_off: int,
                  dst_row_off: Sequence[int]):
    """Owner-side lookup fused with the row exchange: ids = counts[0] ids of rank 0, counts[1] of rank 1, ...;
    rank r's rows are stored into r's peer window at region_off + dst_row_off[r] rows (mono_mtable_lookup_push)."""
    k = self._table_names.index(slot)
    n = window.world
    _lib.check(self._lib.mono_mtable_lookup_push(
        self._h, k, _ptr(ids), (C.c_int64 * n)(*[int(x) for x in counts]), window._h, int(region_off),
        (C.c_int64 * n)(*[int(x) for x in dst_row_off]), _stream(self._device)))

  def lookup_pool(self, slot: str, fids: torch.Tensor, row_offsets: Optional[torch.Tensor] = None,
                  pooling: str = "sum", out: Optional[torch.Tensor] = None, out_col: int = 0) -> torch.Tensor:
    """Fused probe + gather + SUM/MEAN pool (one kernel): the hot forward.  Equivalent to
    lookup() followed by embedding_combiners.ReduceSum/ReduceMean (ref: embedding_combiners.py:41-70)."""
    k = self._table_names.index(slot)
    fids = _ids(fids, self._device)
    if row_offsets is not None:
      row_offsets = row_offsets.to(device=self._device, dtype=torch.int32).contiguous()
      n_rows = row_offsets.numel() - 1
    else:
      n_rows = fids.numel()
    if out is None:
      out = torch.empty(n_rows, self._dims[k], dtype=torch.float32, device=self._device)
    stride = out.stride(0) if out.dim() == 2 else self._dims[k]
    pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
    _lib.check(self._lib.mono_mtable_lookup_pool(self._h, k, _ptr(fids), _ptr(row_offsets), n_rows, pool,
                                                 _ptr(out), stride, out_col, _stream(self._device)))
    return out

  def pool_backward(self, slot: str, fids: torch.Tensor, pooled_grad: torch.Tensor,
                    row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum", req_time: int = 0,
                    global_step: int = 0, grad_col: int = 0):
    """Fused backward of lookup_pool: scatters the pooled-row gradients to the unique FIDs, applies one
    sparse optimizer step per FID and bumps the expiry timestamp (upsert), deterministically and without
    a per-unique gradient buffer.  Equivalent to fused_embedding_to_layout_grad / ScatterGrad followed by
    apply_gradients on the deduplicated ids (ref: distributed_ps.py:1321-1332,1390-1395)."""
    k = self._table_names.index(slot)
    fids = _ids(fids, self._device)
    pooled_grad = _f32(pooled_grad, self._device)
    if row_offsets is not None:
      row_offsets = row_offsets.to(device=self._device, dtype=torch.int32).contiguous()
      n_rows = row_offsets.numel() - 1
    else:
      n_rows = fids.numel()
    stride = pooled_grad.stride(0) if pooled_grad.dim() == 2 else self._dims[k]
    lr = self._configs[slot].call_learning_rate_fns()
    lr_arr = (C.c_float * len(lr))(*lr)
    pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
    _lib.check(self._lib.mono_mtable_pool_backward(self._h, k, _ptr(fids), fids.numel(), _ptr(row_offsets), n_rows,
                                                   pool, _ptr(pooled_grad), stride, grad_col, lr_arr, int(req_time),
                                                   int(global_step), _stream(self._device)))
    return self

  @staticmethod
  def _parts_dtype(parts: Sequence[PoolPart], dtype=None):
    """The row dtype of a parts call: `dtype` if given, else the one dtype of the rows passed in, else float32."""
    if dtype is None:
      given = {p.rows.dtype for p in parts if p.rows is not None}
      if len(given) > 1:
        raise ValueError(f"part rows mix dtypes {sorted(str(d) for d in given)}")
      dtype = given.pop() if given else torch.float32
    if dtype not in (torch.float32, torch.bfloat16):
      raise ValueError(f"part rows must be float32 or bfloat16, not {dtype}")
    return dtype

  def _parts_arr(self, parts: Sequence[PoolPart], forward: bool, dtype=None):
    """-> (mono_pool_part array, tensors that must stay alive over the call, the parts' row tensors); rows of the
    call's dtype (_parts_dtype)."""
    if len(parts) > _lib.MAX_POOL_PARTS:
      raise ValueError(f"at most {_lib.MAX_POOL_PARTS} parts per call")
    dtype = self._parts_dtype(parts, dtype)
    arr = (_lib.PoolPartC * max(len(parts), 1))()
    keep, outs = [], []
    for i, p in enumerate(parts):
      if p.slot not in self._table_names:
        raise KeyError(f"unknown table {p.slot}")
      k = self._table_names.index(p.slot)
      fids = _ids(p.fids, self._device)
      ro = None
      if p.row_offsets is not None:
        ro = p.row_offsets.to(device=self._device, dtype=torch.int32).contiguous()
        n_rows = ro.numel() - 1
      else:
        n_rows = fids.numel()
      width = self._dims[k] * (p.max_seq_len if p.pooling == "firstn" else 1)
      rows = p.rows
      if rows is None:
        if not forward:
          raise ValueError("pool_backward_parts: every part needs its gradient rows")
        rows = torch.empty(n_rows, width, dtype=dtype, device=self._device)
      if rows.dtype != dtype:
        raise ValueError(f"part rows are {rows.dtype}, the call's rows are {dtype}")
      if rows.device != self._device or rows.stride(1) != 1:
        raise ValueError("part rows must be on the table's device with unit column stride")
      if rows.shape[0] < n_rows or rows.shape[1] < p.col + width:
        raise ValueError("part rows are smaller than [n_rows, col + dim] ([n_rows, col + max_seq_len * dim] for "
                         "'firstn')")
      keep += [fids, ro]
      outs.append(rows)
      arr[i] = _lib.PoolPartC(k, fids.data_ptr(), fids.numel(), None if ro is None else ro.data_ptr(), n_rows,
                              {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN, "firstn": _lib.POOL_FIRSTN}[p.pooling],
                              rows.data_ptr(), rows.stride(0), p.col, p.max_seq_len)
    return arr, keep, outs

  def lookup_pool_parts(self, parts: Sequence[PoolPart], dtype: Optional[torch.dtype] = None) -> List[torch.Tensor]:
    """lookup_pool over many features and tables in one call (mono_mtable_lookup_pool_parts): every part's rows
    are bit-identical to lookup_pool on that part alone; parts served by the same kernel share one launch.  A
    "firstn" part writes its [n_rows, max_seq_len, dim] positions (see PoolPart).  A part without `rows` gets a new
    [n_rows, dim] tensor ([n_rows, max_seq_len * dim] for "firstn": .view(n_rows, max_seq_len, dim) gives the
    sequence); returns each part's rows, in part order.

    The call's row dtype is `dtype` if given, else that of the rows passed in (all alike), else float32.  With
    torch.bfloat16 (mono_mtable_lookup_pool_parts_bf16) every row is the float32 result rounded once to bfloat16."""
    dtype = self._parts_dtype(parts, dtype)
    arr, keep, outs = self._parts_arr(parts, forward=True, dtype=dtype)
    fn = (self._lib.mono_mtable_lookup_pool_parts_bf16 if dtype == torch.bfloat16 else
          self._lib.mono_mtable_lookup_pool_parts)
    _lib.check(fn(self._h, arr, len(parts), _stream(self._device)))
    del keep
    return outs

  def pool_backward_parts(self, parts: Sequence[PoolPart], req_time: int = 0, global_step: int = 0):
    """pool_backward over many features and tables in one call (mono_mtable_pool_backward_parts): the parts
    of one table are ONE batch in part order, so a FID that several features share gets one optimizer step
    with the sum of all its terms; the claim, sort and run list run once for the whole call.  A "firstn" part's
    occurrence j of row r takes position j of the row's gradient, or zeros for j >= max_seq_len: the FID is still
    inserted, bumped and stepped (with a zero gradient) as the reference's ScatterGrad leaves it.

    Every part's rows share one dtype, float32 or bfloat16; bfloat16 gradients (mono_mtable_pool_backward_parts_bf16)
    give exactly the bits of this call on the rows widened to float32."""
    dtype = self._parts_dtype(parts)
    arr, keep, _ = self._parts_arr(parts, forward=False, dtype=dtype)
    lr = self.learning_rates()
    lr_arr = (C.c_float * max(len(lr), 1))(*lr)
    fn = (self._lib.mono_mtable_pool_backward_parts_bf16 if dtype == torch.bfloat16 else
          self._lib.mono_mtable_pool_backward_parts)
    _lib.check(fn(self._h, arr, len(parts), lr_arr, int(req_time), int(global_step), _stream(self._device)))
    del keep
    return self

  def set_hash_filter(self, slot: str, capacity: int, default_threshold: int, slot_thresholds: Optional[Dict[int, int]] = None):
    """Attach a counting admission filter to table `slot` (ref: hash_filter_ops.create_hash_filters; thresholds:
    HashTableConfigInstance slot_occurrence_threshold / SlotOccurrenceThresholdConfig): a FID absent from the table is
    inserted only once it has been seen `threshold` times before (0 = never filter)."""
    k = self._table_names.index(slot)
    st = slot_thresholds or {}
    ks = (C.c_uint32 * max(len(st), 1))(*[int(x) for x in st.keys()])
    vs = (C.c_uint32 * max(len(st), 1))(*[int(x) for x in st.values()])
    _lib.check(self._lib.mono_mtable_set_hash_filter(self._h, k, int(capacity), int(default_threshold), ks, vs, len(st),
                                                     _stream(self._device)))
    return self

  def contains(self, slot: str, ids: torch.Tensor) -> torch.Tensor:
    ids = _ids(ids, self._device)
    out = torch.empty(ids.numel(), dtype=torch.uint8, device=self._device)
    _lib.check(self._lib.mono_mtable_contains(self._h, self._table_names.index(slot), _ptr(ids), ids.numel(),
                                              _ptr(out), _stream(self._device)))
    return out.bool()

  def evict(self, slot: str, max_update_time: int):
    """ref: CuckooEmbeddingHashTable::Evict; the reference runs it from a background thread."""
    _lib.check(self._lib.mono_mtable_evict(self._h, self._table_names.index(slot), int(max_update_time),
                                           _stream(self._device)))
    return self

  def lookup_entry(self, slot: str, ids: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Full rows: emb, optimizer state, found flag and last_update_ts (ref: LookupEntry/EntryDump)."""
    k = self._table_names.index(slot)
    ids = _ids(ids, self._device)
    D, S = self._dims[k], self._lib.mono_mtable_state_floats(self._h, k)
    raw = torch.empty(ids.numel(), D + S + 2, dtype=torch.float32, device=self._device)
    _lib.check(self._lib.mono_mtable_lookup_entry(self._h, k, _ptr(ids), ids.numel(), _ptr(raw),
                                                  _stream(self._device)))
    meta = raw[:, D + S:].contiguous().view(torch.int32)
    return {"num": raw[:, :D], "opt": raw[:, D:D + S], "found": meta[:, 0].bool(),
            "last_update_ts_sec": meta[:, 1].to(torch.int64) & 0xFFFFFFFF, "raw": raw}

  def export(self, slot: str, chunk: int = 1 << 20):
    """Yields (ids, raw_rows) chunks of every live row (checkpoint writer side)."""
    k = self._table_names.index(slot)
    D, S = self._dims[k], self._lib.mono_mtable_state_floats(self._h, k)
    cursor, n = C.c_int64(0), C.c_int64(0)
    while cursor.value >= 0:
      ids = torch.empty(chunk, dtype=torch.int64, device=self._device)
      rows = torch.empty(chunk, D + S + 2, dtype=torch.float32, device=self._device)
      _lib.check(self._lib.mono_mtable_export(self._h, k, C.byref(cursor), chunk, _ptr(ids), _ptr(rows),
                                              C.byref(n), _stream(self._device)))
      if n.value:
        yield ids[:n.value], rows[:n.value]

  # ---- checkpoints in the reference's on-disk format (checkpoint.py, csrc/ckpt.cu) -------------
  @property
  def configs(self):
    return self._configs

  def entry_width(self, slot: str) -> int:
    """floats per exported row: dim + optimizer state + found + last_update_ts."""
    k = self._table_names.index(slot)
    return self._dims[k] + self._lib.mono_mtable_state_floats(self._h, k) + 2

  def max_update_ts(self, slot: str) -> int:
    """ref: EmbeddingHashTableTfBridge::max_update_ts_sec."""
    return int(self._lib.mono_mtable_max_update_ts(self._h, self._table_names.index(slot)))

  def note_update_ts(self, slot: str, ts: int):
    _lib.check(self._lib.mono_mtable_note_update_ts(self._h, self._table_names.index(slot), int(ts)))
    return self

  def save(self, basename: str, nshards: int = -1) -> "MultiHashTable":
    """ref: multi_hash_table_ops.py:409-415 -> MonolithMultiHashTableSave: `<basename>-%05d-of-%05d` (Snappy
    TFRecords of EntryDump) + `<basename>.meta-%05d-of-%05d`; expired entries are not written."""
    from . import checkpoint
    checkpoint.save(self, basename, nshards)
    return self

  def restore(self, basename: str) -> "MultiHashTable":
    """ref: multi_hash_table_ops.py:417-420 -> MonolithMultiHashTableRestore."""
    from . import checkpoint
    checkpoint.restore(self, basename)
    return self

  def restore_rows(self, slot: str, ids: torch.Tensor, raw_rows: torch.Tensor):
    k = self._table_names.index(slot)
    ids, raw_rows = _ids(ids, self._device), _f32(raw_rows, self._device)
    _lib.check(self._lib.mono_mtable_restore_rows(self._h, k, _ptr(ids), ids.numel(), _ptr(raw_rows),
                                                  _stream(self._device)))
    return self
