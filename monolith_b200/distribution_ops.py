"""Dedup / shard / pooling ops around the table — mirror of the hot-path subset of
monolith/native_training/distribution_ops.py (ref: fused_reorder_by_indices :218-258,
fused_gather_embeddings_by_input :816-889, fused_embedding_to_layout :528-700).
All tensors are torch CUDA tensors; the work is done by the kernels in csrc/{dedup,layout}.cu.
"""
import ctypes as C
import dataclasses
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib


def _ptr(t):
  return None if t is None else C.c_void_p(t.data_ptr())


def _stream(device):
  return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


_TOWER_DTYPES = (torch.float32, torch.bfloat16)


def _tower_dtype(dtype, what):
  """The dtype of the tensors a tower reads or writes: float32, or bfloat16 (the *_bf16 kernels)."""
  if dtype not in _TOWER_DTYPES:
    raise ValueError(f"{what} must be torch.float32 or torch.bfloat16, not {dtype}")
  return dtype


def fused_reorder_by_indices(inputs: Sequence[torch.Tensor], num_of_shards: int, dim_sizes: Sequence[int],
                             rank0_empty_shard: Optional[bool] = None):
  """ref: distribution_ops.py:218-258 / FusedReorderByIndices (runtime/ops/fused_reorder_by_indices.cc).

  Returns (output, shard_sizes, sharded_slot_sizes, emb_offset_sz, fused_embedding_offsets); the two
  size vectors come back as Python lists (they size the all-to-all), the rest stay on the device.
  """
  lib = _lib.load()
  if rank0_empty_shard is None:  # ref: distribution_ops.py:253-256
    rank0_empty_shard = os.environ.get('MONOLITH_SYNC_EMPTY_RANK0_PS_SHARD', '1') == '1' and num_of_shards > 4
  if len(inputs) != len(dim_sizes):
    raise ValueError("inputs and dim_sizes must have the same length")
  device = inputs[0].device
  ids = torch.cat([t.reshape(-1).to(torch.int64) for t in inputs]) if inputs else torch.empty(0, dtype=torch.int64)
  K = len(inputs)
  splits = [0]
  for t in inputs:
    splits.append(splits[-1] + t.numel())
  M = splits[-1]
  out = torch.empty(max(M, 1), dtype=torch.int64, device=device)
  offs = torch.empty(max(M, 1), dtype=torch.int32, device=device)
  c_split = (C.c_int64 * (K + 1))(*splits)
  c_dims = (C.c_int32 * K)(*[int(d) for d in dim_sizes])
  shard_sizes = (C.c_int32 * num_of_shards)()
  slot_sizes = (C.c_int32 * (num_of_shards * K))()
  n_unique = C.c_int64(0)
  _lib.check(lib.mono_reorder_by_indices(device.index, _ptr(ids), c_split, K, num_of_shards, c_dims,
                                         1 if rank0_empty_shard else 0, _ptr(out), None, _ptr(offs), shard_sizes,
                                         slot_sizes, C.byref(n_unique), _stream(device)))
  emb_offset_sz = [t.numel() for t in inputs]
  return out[:n_unique.value], list(shard_sizes), list(slot_sizes), emb_offset_sz, offs[:M]


def unique_with_inverse(ids: torch.Tensor, sync: bool = True):
  """First-occurrence dedup of one id list (tf.unique order).  Returns (unique, inverse[, n_unique])."""
  lib = _lib.load()
  ids = ids.reshape(-1).to(torch.int64).contiguous()
  n = ids.numel()
  uniq = torch.empty(max(n, 1), dtype=torch.int64, device=ids.device)
  inv = torch.empty(max(n, 1), dtype=torch.int32, device=ids.device)
  n_dev = torch.zeros(1, dtype=torch.int32, device=ids.device)
  n_host = C.c_int64(0)
  _lib.check(lib.mono_dedup(ids.device.index, _ptr(ids), n, _ptr(uniq), _ptr(inv), _ptr(n_dev),
                            C.byref(n_host) if sync else None, _stream(ids.device)))
  if sync:
    return uniq[:n_host.value], inv[:n]
  return uniq, inv[:n], n_dev


def sharding_sparse_fids(features: Dict[str, Tuple[torch.Tensor, torch.Tensor]], feature_table: Dict[str, str],
                         feature_dims_sum: Dict[str, int], num_of_shards: int, shared_features: Sequence[str] = (),
                         reorder_fn=None):
  """Outputs of the reference's ShardingSparseFids (version 3+, unique = true) from per-feature FID lists —
  ref: ShardingSparseFidsOp::FillFidList / CreateOffsetTensor, NT/data/kernels/parse_sparse_feature.cc:187-330;
  Python model: NT/data/parse_sparse_feature_test.py:87-240 (SURVEY §8 row a2).

  features[name] = (fids int64[n], row_splits int64[rows + 1]) — CSR over the samples of the batch (a shared
  feature has ONE row).  Returns a dict:
    fid_list       list of K*N int64 tensors, index = table_index * N + shard (tables in sorted-name order): the
                   (table, shard) list is the concatenation, over the table's features in sorted-name order, of
                   each feature's distinct FIDs of that shard in first-occurrence order
    fid_offset     int64[M] holding the reference's uint64: (table_index * N + shard) << 32 | float offset of the
                   FID's row inside that (table, shard) list, rows of feature f being dims_sum[f] floats wide
    feature_offset int32[#(feature, row) + 1]; nfl_offset int32[#features + 1] holding the reference's uint32 bits
                   (bit 31 = shared, so a shared feature's entry is negative), features in sorted-name order — all
                   three are what fused_embedding_to_layout[_grad] takes as they are
  The dedup / shard / offset work is ONE FusedReorderByIndices launch over the features as lists (per-list
  dims = dims_sum, shard-major / list-minor output, bit-exact kernel); the rest is index arithmetic on device.
  (The reference dedups per (feature, shard); FIDs carry their slot, so features never share a FID.)"""
  N = int(num_of_shards)
  if reorder_fn is None:
    reorder_fn = lambda lists, n, dims: fused_reorder_by_indices(lists, n, dims, rank0_empty_shard=False)
  names = sorted(features)
  tables = sorted({feature_table[n] for n in names})
  t_idx = {t: i for i, t in enumerate(tables)}
  order = sorted(names, key=lambda n: (t_idx[feature_table[n]], n))      # table-major, feature-minor
  F, K = len(order), len(tables)
  lists = [features[n][0].reshape(-1).to(torch.int64) for n in order]
  dims = [int(feature_dims_sum[n]) for n in order]
  device = lists[0].device if lists else torch.device("cpu")
  out, _, slot_sizes, _, offs = reorder_fn(lists, N, dims)
  slot = torch.as_tensor([int(x) for x in slot_sizes], dtype=torch.int64).reshape(N, F)
  width = slot * torch.as_tensor(dims, dtype=torch.int64).reshape(1, F)
  flat_id = torch.cumsum(slot.reshape(-1), 0) - slot.reshape(-1)           # exclusive, shard-major / list-minor
  flat_emb = torch.cumsum(width.reshape(-1), 0) - width.reshape(-1)
  id_base, emb_base = flat_id.reshape(N, F), flat_emb.reshape(N, F)
  first = {}                                                               # first / last list index of every table
  for j, n in enumerate(order):
    k = t_idx[feature_table[n]]
    first.setdefault(k, [j, j])[1] = j
  fid_list = []
  for k in range(K):
    j0, j1 = first[k]
    for n in range(N):
      b = int(id_base[n, j0])
      e = int(id_base[n, j1] + slot[n, j1])
      fid_list.append(out[b:e])
  # fid_offset blocks, computed in list order, emitted in sorted-feature-name order
  occ_start = [0]
  for l in lists:
    occ_start.append(occ_start[-1] + l.numel())
  wrap = (1 << 64) % N
  blocks = {}
  for j, n in enumerate(order):
    v = lists[j]
    k = t_idx[feature_table[n]]
    shard = torch.remainder(torch.remainder(v, N) + wrap * (v < 0).to(torch.int64), N)   # (uint64)fid % N
    base = emb_base[:, first[k][0]].to(device)
    local = offs[occ_start[j]:occ_start[j + 1]].to(torch.int64) - base[shard]
    blocks[n] = ((k * N + shard) << 32) | local
  feature_offset, nfl_offset, pieces, total = [], [], [], 0
  shared = set(shared_features)
  for n in names:
    nfl_offset.append(len(feature_offset) | ((1 << 31) if n in shared else 0))
    rs = [int(x) for x in features[n][1].reshape(-1).tolist()]
    feature_offset.extend(total + r for r in rs[:-1])
    total += rs[-1]
    pieces.append(blocks[n])
  feature_offset.append(total)
  nfl_offset.append(len(feature_offset))
  fid_offset = torch.cat(pieces) if pieces else torch.empty(0, dtype=torch.int64, device=device)
  return {"fid_list": fid_list, "fid_offset": fid_offset,
          "feature_offset": torch.as_tensor(feature_offset, dtype=torch.int32, device=device),
          "nfl_offset": torch.as_tensor([v - (1 << 32) if v >> 31 else v for v in nfl_offset], dtype=torch.int32,
                                        device=device),
          "table_names": tables, "feature_names": names}


def gather_pool(fused_embeddings: torch.Tensor, fused_embedding_offsets: torch.Tensor, dim: int,
                row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
                out: Optional[torch.Tensor] = None, out_col: int = 0, dtype: torch.dtype = torch.float32) -> torch.Tensor:
  """out[r] = pool_{m in row r} fused_embeddings[offsets[m]:offsets[m]+dim]
  (ref: FusedGatherKernel, runtime/ops/map_id_to_embedding.cu.cc:30-74, + per-row pool).
  The pooled rows are float32 or bfloat16: out's dtype when out is given, else `dtype`.  bfloat16 rows are the
  float32 results rounded once to nearest even; the fused buffer stays float32."""
  dtype = _tower_dtype(out.dtype if out is not None else dtype, "gather_pool's output")
  lib = _lib.load()
  dev = fused_embeddings.device
  offs = fused_embedding_offsets.to(torch.int32).contiguous()
  n_rows = offs.numel() if row_offsets is None else row_offsets.numel() - 1
  if row_offsets is not None:
    row_offsets = row_offsets.to(torch.int32).contiguous()
  if out is None:
    out = torch.empty(n_rows, dim, dtype=dtype, device=dev)
  pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
  fn = lib.mono_gather_pool_bf16 if dtype == torch.bfloat16 else lib.mono_gather_pool
  _lib.check(fn(dev.index, _ptr(fused_embeddings), _ptr(offs), _ptr(row_offsets), n_rows, dim,
                                  pool, _ptr(out), out.stride(0), out_col, _stream(dev)))
  return out


def gather_pool_grad(pooled_grad: torch.Tensor, fused_embedding_offsets: torch.Tensor, dim: int, total_floats: int,
                     row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum", grad_col: int = 0):
  """Backward of gather_pool: scatter-add pooled grads to the fused row buffer
  (ref: FusedGatherGradKernel, map_id_to_embedding.cu.cc:75-118).  pooled_grad is float32 or bfloat16 (widened
  exactly); the returned buffer is float32."""
  bf16 = _tower_dtype(pooled_grad.dtype, "pooled_grad") == torch.bfloat16
  lib = _lib.load()
  dev = pooled_grad.device
  offs = fused_embedding_offsets.to(torch.int32).contiguous()
  n_rows = offs.numel() if row_offsets is None else row_offsets.numel() - 1
  if row_offsets is not None:
    row_offsets = row_offsets.to(torch.int32).contiguous()
  grad = torch.zeros(total_floats, dtype=torch.float32, device=dev)
  pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
  fn = lib.mono_gather_pool_grad_bf16 if bf16 else lib.mono_gather_pool_grad
  _lib.check(fn(dev.index, _ptr(pooled_grad), pooled_grad.stride(0), grad_col, _ptr(offs), _ptr(row_offsets), n_rows,
                dim, pool, _ptr(grad), _stream(dev)))
  return grad


def scatter_grad_rows(pooled_grad: torch.Tensor, fused_embedding_offsets: torch.Tensor, dim: int,
                      grad_fused: torch.Tensor, row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
                      grad_col: int = 0):
  """Deterministic (sort-based, atomics-free) scatter of pooled-row grads into the fused row buffer
  `grad_fused` (written in place; rows nobody refers to are left as they are).  pooled_grad is float32 or
  bfloat16 (widened exactly); grad_fused must be float32."""
  bf16 = _tower_dtype(pooled_grad.dtype, "pooled_grad") == torch.bfloat16
  if grad_fused.dtype != torch.float32:
    raise ValueError(f"grad_fused must be torch.float32, not {grad_fused.dtype}")
  lib = _lib.load()
  dev = pooled_grad.device
  offs = fused_embedding_offsets.to(torch.int32).contiguous()
  n_rows = offs.numel() if row_offsets is None else row_offsets.numel() - 1
  if row_offsets is not None:
    row_offsets = row_offsets.to(torch.int32).contiguous()
  pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
  fn = lib.mono_scatter_grad_rows_bf16 if bf16 else lib.mono_scatter_grad_rows
  _lib.check(fn(dev.index, _ptr(pooled_grad), pooled_grad.stride(0), grad_col, _ptr(offs), offs.numel(),
                _ptr(row_offsets), n_rows, dim, pool, _ptr(grad_fused), grad_fused.numel(), _stream(dev)))
  return grad_fused


class Grouping:
  """One grouping of a batch's FID occurrences, shared by the sharded forward and backward
  (mono_grouping_*).  build(): dedup + bucket by owner = fid mod num_shards; reduce(): deterministic
  per-FID sum of pooled-row gradients in the bucketed order."""

  def __init__(self, device):
    self._lib = _lib.load()
    self.device = torch.device(device)
    h = C.c_void_p()
    _lib.check(self._lib.mono_grouping_create(self.device.index, C.byref(h)))
    self._h = h
    self.dim = 0

  def __del__(self):
    try:
      if self._h:
        self._lib.mono_grouping_destroy(self._h)
        self._h = None
    except Exception:
      pass

  def build(self, fids: torch.Tensor, num_shards: int, dim: int):
    """Returns (unique fids shard-major, occurrence row offsets int32[M], shard_sizes list)."""
    fids = fids.reshape(-1).contiguous()
    M = fids.numel()
    uniq = torch.empty(max(M, 1), dtype=torch.int64, device=self.device)
    offs = torch.empty(max(M, 1), dtype=torch.int32, device=self.device)
    counts = (C.c_int32 * num_shards)()
    n_u = C.c_int64(0)
    _lib.check(self._lib.mono_grouping_build(self._h, _ptr(fids), M, num_shards, dim, _ptr(uniq), _ptr(offs), counts,
                                             C.byref(n_u), _stream(self.device)))
    self.dim = dim
    self._keep = fids  # the grouping refers to positions of this tensor until the next build
    return uniq[:n_u.value], offs[:M], list(counts)

  def reduce(self, pooled_grad: torch.Tensor, out_rows: torch.Tensor, row_offsets: Optional[torch.Tensor] = None,
             pooling: str = "sum", grad_col: int = 0):
    n_rows = self._keep.numel() if row_offsets is None else row_offsets.numel() - 1
    if row_offsets is not None:
      row_offsets = row_offsets.to(torch.int32).contiguous()
    pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
    _lib.check(self._lib.mono_grouping_reduce(self._h, _ptr(pooled_grad), pooled_grad.stride(0), grad_col,
                                              _ptr(row_offsets), n_rows, pool, _ptr(out_rows), _stream(self.device)))
    return out_rows

  def reduce_push(self, pooled_grad: torch.Tensor, shard_sizes: Sequence[int], window: "PeerWindow", region_off: int,
                  dst_row_off: Sequence[int], row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
                  grad_col: int = 0):
    """reduce() whose output rows are stored into the owners' windows (fused gradient exchange)."""
    n_rows = self._keep.numel() if row_offsets is None else row_offsets.numel() - 1
    if row_offsets is not None:
      row_offsets = row_offsets.to(torch.int32).contiguous()
    pool = {"sum": _lib.POOL_SUM, "mean": _lib.POOL_MEAN}[pooling]
    n = window.world
    _lib.check(self._lib.mono_grouping_reduce_push(
        self._h, _ptr(pooled_grad), pooled_grad.stride(0), grad_col, _ptr(row_offsets), n_rows, pool,
        (C.c_int64 * n)(*[int(x) for x in shard_sizes]), window._h, int(region_off),
        (C.c_int64 * n)(*[int(x) for x in dst_row_off]), _stream(self.device)))


class _RawCuda:
  """__cuda_array_interface__ carrier for a raw device pointer (torch.as_tensor makes a view of it)."""

  def __init__(self, ptr: int, nbytes: int, owner):
    self.owner = owner
    self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class PeerWindow:
  """One rank's NVLink window (mono_peer_*): device memory mapped into every peer process of the node.
  Construction is collective over `group` (the 64-byte IPC handles are all-gathered)."""

  def __init__(self, device, world: int, rank: int, nbytes: int, group=None):
    import torch.distributed as dist
    self._lib = _lib.load()
    self.device = torch.device(device)
    self.world, self.rank, self.nbytes = world, rank, int(nbytes)
    h = C.c_void_p()
    _lib.check(self._lib.mono_peer_create(self.device.index, world, rank, self.nbytes, C.byref(h)))
    self._h = h
    if world > 1:
      buf = (C.c_uint8 * 64)()
      _lib.check(self._lib.mono_peer_handle(self._h, buf))
      mine = torch.tensor(list(buf), dtype=torch.uint8, device=self.device)
      allh = torch.empty(64 * world, dtype=torch.uint8, device=self.device)
      dist.all_gather_into_tensor(allh, mine, group=group)
      raw = bytes(allh.cpu().tolist())
      _lib.check(self._lib.mono_peer_attach(self._h, raw, world))
      dist.barrier(group=group)   # every rank has mapped every window before anyone stores
    p = C.c_void_p()
    _lib.check(self._lib.mono_peer_local(self._h, C.byref(p)))
    self._local = torch.as_tensor(_RawCuda(p.value, self.nbytes, self), device=self.device)

  def close(self, group=None):
    """Collective teardown: unmap the peers, rank barrier, free."""
    if getattr(self, "_h", None):
      import torch.distributed as dist
      self._local = None
      _lib.check(self._lib.mono_peer_detach(self._h))
      if self.world > 1:
        dist.barrier(group=group)
      self._lib.mono_peer_destroy(self._h)
      self._h = None

  def view(self, offset: int, count: int, dtype: torch.dtype) -> torch.Tensor:
    """`count` items of `dtype` of THIS rank's window starting at byte `offset`."""
    nb = count * torch.empty(0, dtype=dtype).element_size()
    return self._local[offset:offset + nb].view(dtype)

  def barrier(self):
    _lib.check(self._lib.mono_peer_barrier(self._h, _stream(self.device)))

  def put(self, region_off: int, dst_off: Sequence[int], src: torch.Tensor, src_off: Sequence[int],
          nbytes: Sequence[int]):
    """nbytes[r] bytes of src (+ src_off[r]) -> rank r's window at region_off + dst_off[r]."""
    n = self.world
    arr = lambda xs: (C.c_int64 * n)(*[int(x) for x in xs])
    _lib.check(self._lib.mono_peer_put(self._h, int(region_off), arr(dst_off), _ptr(src), arr(src_off), arr(nbytes),
                                       _stream(self.device)))


  def get(self, region_off: int, src_off: Sequence[int], dst: torch.Tensor, dst_off: Sequence[int],
          nbytes: Sequence[int]):
    """nbytes[r] bytes of rank r's window at region_off + src_off[r] -> dst (+ dst_off[r], bytes)."""
    n = self.world
    arr = lambda xs: (C.c_int64 * n)(*[int(x) for x in xs])
    _lib.check(self._lib.mono_peer_get(self._h, int(region_off), arr(src_off), _ptr(dst), arr(dst_off), arr(nbytes),
                                       _stream(self.device)))


# ---- generic fused layout op ------------------------------------------------------------------
@dataclasses.dataclass
class SliceTask:
  """One (layout, slice_config) pair of the reference's FeatureConfigs, flattened
  (ref: idl/matrix/proto/example.proto:177-220; runtime/ops/fused_embedding_to_layout.cc:229-286)."""
  nfl_idx: int
  slice_start: int
  dim: int
  pooling: int  # _lib.POOL_*
  max_seq_len: int
  out_tensor: int
  out_row_stride: int
  out_col: int
  accumulate: int


def _tasks_arr(tasks: Sequence[SliceTask]):
  arr = (_lib.SliceTask * len(tasks))()
  for i, t in enumerate(tasks):
    for f, _ in _lib.SliceTask._fields_:
      setattr(arr[i], f, int(getattr(t, f)))
  return arr


def _ptr_table(tensors: Sequence[torch.Tensor], device):
  return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device=device)


def _check_layout_inputs(fid_offset, feature_offset, nfl_offset, rows, rows_name, rows_dtype=torch.float32):
  """-> the device of the index tensors.  The C ABI reads fid_offset as uint64, feature_offset as int32 and
  nfl_offset as uint32 words: a tensor of another dtype would be silently reinterpreted, so it is refused."""
  want = (("fid_offset", fid_offset, torch.int64), ("feature_offset", feature_offset, torch.int32),
          ("nfl_offset", nfl_offset, torch.int32))
  for name, t, dt in want:
    if not isinstance(t, torch.Tensor) or t.dtype != dt:
      raise ValueError(f"{name} must be a {dt} tensor, not {getattr(t, 'dtype', type(t).__name__)}")
  dev = fid_offset.device
  for name, t, _ in want:
    if t.device.type != "cuda" or t.device != dev:
      raise ValueError(f"{name} must be a CUDA tensor on {dev if dev.type == 'cuda' else 'a CUDA device'}, "
                       f"not on {t.device}")
    if not t.is_contiguous():
      raise ValueError(f"{name} must be contiguous")
  for t in rows:
    if t.dtype != rows_dtype or t.device != dev:
      raise ValueError(f"{rows_name} must be {rows_dtype} tensors on {dev}, not {t.dtype} on {t.device}")
  return dev


def fused_embedding_to_layout(embeddings_list: Sequence[torch.Tensor], emb_strides: Sequence[int],
                              fid_offset: torch.Tensor, feature_offset: torch.Tensor, nfl_offset: torch.Tensor,
                              batch_size: int, tasks: Sequence[SliceTask], out_shapes: Sequence[Sequence[int]],
                              dtype: torch.dtype = torch.float32):
  """ref: distribution_ops.fused_embedding_to_layout (versions 3/4/5) -> MonolithEmbeddingToLayoutV*.
  fid_offset: uint64 viewed as int64 tensor; nfl_offset: uint32 viewed as int32 tensor (sharding_sparse_fids'
  outputs as they are).  Raises ValueError for any other dtype, a non-CUDA or non-contiguous index tensor, or
  embeddings that are not float32 on the same device.  dtype: of the outputs, float32 or bfloat16 (the float32
  results rounded once to nearest even; the tasks' strides and columns then count bfloat16 elements)."""
  bf16 = _tower_dtype(dtype, "dtype") == torch.bfloat16
  dev = _check_layout_inputs(fid_offset, feature_offset, nfl_offset, embeddings_list, "embeddings_list")
  lib = _lib.load()
  outs = [torch.zeros(*s, dtype=dtype, device=dev) for s in out_shapes]
  embs = [e.contiguous() for e in embeddings_list]
  ep, op = _ptr_table(embs, dev), _ptr_table(outs, dev)
  st = torch.tensor(list(emb_strides), dtype=torch.int32, device=dev)
  fn = lib.mono_embedding_to_layout_bf16 if bf16 else lib.mono_embedding_to_layout
  _lib.check(fn(dev.index, _ptr(ep), _ptr(st), len(embs), _ptr(fid_offset), fid_offset.numel(), _ptr(feature_offset),
                feature_offset.numel(), _ptr(nfl_offset), nfl_offset.numel(), batch_size, _tasks_arr(tasks), len(tasks),
                _ptr(op), _stream(dev)))
  return outs


def fused_embedding_to_layout_grad(emb_sizes: Sequence[int], emb_strides: Sequence[int], fid_offset: torch.Tensor,
                                   feature_offset: torch.Tensor, nfl_offset: torch.Tensor, batch_size: int,
                                   tasks: Sequence[SliceTask], out_grads: Sequence[torch.Tensor]):
  """ref: MonolithEmbeddingToLayoutGradV* (fused_embedding_to_layout.cc:697-948).  The index tensors as in
  fused_embedding_to_layout; out_grads all float32 or all bfloat16 (widened exactly) on their device.  The
  returned embedding gradients are float32."""
  dtype = _tower_dtype(out_grads[0].dtype if len(out_grads) else torch.float32, "out_grads")
  if any(g.dtype != dtype for g in out_grads):
    raise ValueError(f"out_grads must be all torch.float32 or all torch.bfloat16, not {[g.dtype for g in out_grads]}")
  dev = _check_layout_inputs(fid_offset, feature_offset, nfl_offset, out_grads, "out_grads", dtype)
  lib = _lib.load()
  grads = [torch.zeros(n, dtype=torch.float32, device=dev) for n in emb_sizes]
  og = [g.contiguous() for g in out_grads]
  gp, op = _ptr_table(grads, dev), _ptr_table(og, dev)
  st = torch.tensor(list(emb_strides), dtype=torch.int32, device=dev)
  fn = lib.mono_embedding_to_layout_grad_bf16 if dtype == torch.bfloat16 else lib.mono_embedding_to_layout_grad
  _lib.check(fn(dev.index, _ptr(gp), _ptr(st), len(grads), _ptr(fid_offset), fid_offset.numel(), _ptr(feature_offset),
                feature_offset.numel(), _ptr(nfl_offset), nfl_offset.numel(), batch_size, _tasks_arr(tasks), len(tasks),
                _ptr(op), _stream(dev)))
  return grads
