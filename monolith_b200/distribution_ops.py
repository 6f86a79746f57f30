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
from ._lib import ptr, stream
from .clip_ops import scale_ptr


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
  _lib.check(lib.mono_reorder_by_indices(device.index, ptr(ids), c_split, K, num_of_shards, c_dims,
                                         1 if rank0_empty_shard else 0, ptr(out), None, ptr(offs), shard_sizes,
                                         slot_sizes, C.byref(n_unique), stream(device)))
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
  _lib.check(lib.mono_dedup(ids.device.index, ptr(ids), n, ptr(uniq), ptr(inv), ptr(n_dev),
                            C.byref(n_host) if sync else None, stream(ids.device)))
  if sync:
    return uniq[:n_host.value], inv[:n]
  return uniq, inv[:n], n_dev


def sharding_sparse_fids(features: Dict[str, Tuple[torch.Tensor, torch.Tensor]], feature_table: Dict[str, str],
                         feature_dims_sum: Dict[str, int], num_of_shards: int, shared_features: Sequence[str] = (),
                         reorder_fn=None, *, unique: bool = True, sync: bool = True, version: int = 4,
                         batch_size: Optional[int] = None):
  """Outputs of the reference's ShardingSparseFids (versions 3 and 4) from per-feature FID lists —
  ref: ShardingSparseFidsOp::FillFidList / CreateOffsetTensor, NT/data/kernels/parse_sparse_feature.cc:187-330,
  version 4: parse_sparse_feature.h:714-920; Python model: NT/data/parse_sparse_feature_test.py:87-301 (SURVEY §8
  row a2).

  features[name] = (fids int64[n], row_splits int64[rows + 1]) — CSR over the samples of the batch (a shared
  feature has ONE row).  Returns a dict:
    fid_list       list of K*N int64 tensors, index = table_index * N + shard (tables in sorted-name order): the
                   (table, shard) list is the concatenation, over the table's features in sorted-name order, of
                   each feature's FIDs of that shard: its distinct FIDs in first-occurrence order (unique=True) or
                   every occurrence in input order (unique=False).  None with sync=False (its sizes are on the device)
    fid_offset     int64[M] holding the reference's uint64: (table_index * N + shard) << 32 | float offset of the
                   FID's row inside that (table, shard) list, rows of feature f being dims_sum[f] floats wide
    feature_offset int32[#(feature, row) + 1]; nfl_offset int32[#features + 1] holding the reference's uint32 bits
                   (bit 31 = shared, so a shared feature's entry is negative), features in sorted-name order — all
                   three are what fused_embedding_to_layout[_grad] takes as they are
  and, for CUDA inputs without reorder_fn (one mono_sharding_sparse_fids call, all outputs made on the device):
    fid_list_row_splits        K*N int64 tensors [0, c1, c1 + c2, ...], FID counts of the (table, shard) list's features
    fid_list_fused             the version-4 fid_list: the lists shard-major, table-minor, in one int64 tensor; with
                               sync=False its first sum(fid_list_shard_row_length) of M entries
    fid_list_table_row_length  int32[N*K], list (shard n, table k) at n * K + k
    fid_list_shard_row_length  int32[N]
    fid_list_emb_row_length    int32[N*K], floats of each list
  sync=True reads the N*K list lengths back to slice fid_list (one synchronisation); sync=False makes no host round
  trip.  reorder_fn (the CPU twin: lists, N, dims -> fused_reorder_by_indices' outputs) keeps the version-3
  unique outputs only and the adapter's own index arithmetic.
  version=5 (the reference's default without GPU embeddings, parse_sparse_feature.cc:287-404; CUDA inputs, one
  mono_sharding_sparse_fids_v5 call) adds, all int32 on the device and written there:
    fid_list_row_splits_size   K*N one-element tensors: the table's feature count + 1
    nfl_size, feature_size, fid_size, batch_size   one-element tensors: F + 1, #(feature, row) + 1, M, batch size
    emb_size                   int32[K*N], table-major (index table_index * N + shard): floats of each list
  batch_size defaults to the row count the non-shared features share (ValueError if they differ, or if every
  feature is shared).
  (The reference dedups per (feature, shard); FIDs carry their slot, so features never share a FID.)"""
  N = int(num_of_shards)
  names = sorted(features)
  if version not in (3, 4, 5):
    raise ValueError(f"version must be 3, 4 or 5, not {version!r}")
  if reorder_fn is None and names and features[names[0]][0].is_cuda:
    v5 = None
    if version == 5:
      v5 = _v5_batch_size(features, names, set(shared_features), batch_size)
    return _sharding_sparse_fids_device(features, feature_table, feature_dims_sum, N, shared_features, unique, sync,
                                        v5)
  if version == 5:
    raise ValueError("version=5 needs CUDA inputs and no reorder_fn")
  if not unique or not sync:
    raise ValueError("unique=False and sync=False need CUDA inputs and no reorder_fn")
  if reorder_fn is None:
    reorder_fn = lambda lists, n, dims: fused_reorder_by_indices(lists, n, dims, rank0_empty_shard=False)
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


def _v5_batch_size(features, names, shared, batch_size):
  if batch_size is not None:
    if int(batch_size) < 0:
      raise ValueError("batch_size must not be negative")
    return int(batch_size)
  rows = {features[n][1].numel() - 1 for n in names if n not in shared}
  if len(rows) != 1:
    raise ValueError("batch_size is needed: the non-shared features do not give one row count "
                     f"({sorted(rows) if rows else 'every feature is shared'})")
  return rows.pop()


def _sharding_sparse_fids_device(features, feature_table, feature_dims_sum, N, shared_features, unique, sync,
                                 v5_batch_size=None):
  lib = _lib.load()
  names = sorted(features)
  tables = sorted({feature_table[n] for n in names})
  t_idx = {t: i for i, t in enumerate(tables)}
  F, K = len(names), len(tables)
  device = features[names[0]][0].device
  fids = [features[n][0].reshape(-1).to(torch.int64) for n in names]
  splits = [features[n][1].reshape(-1).to(device=device, dtype=torch.int64) for n in names]
  shared = set(shared_features)
  recs = (_lib.ShardingFeature * F)()
  for i, n in enumerate(names):
    recs[i].n_fids, recs[i].n_rows = fids[i].numel(), splits[i].numel() - 1
    recs[i].table, recs[i].dims_sum, recs[i].shared = t_idx[feature_table[n]], int(feature_dims_sum[n]), n in shared
  M, R = sum(t.numel() for t in fids), sum(t.numel() - 1 for t in splits)
  fids, splits = torch.cat(fids), torch.cat(splits)
  i32 = dict(dtype=torch.int32, device=device)
  fused = torch.empty(max(M, 1), dtype=torch.int64, device=device)
  fid_offset = torch.empty(max(M, 1), dtype=torch.int64, device=device)
  feature_offset, nfl_offset = torch.empty(R + 1, **i32), torch.empty(F + 1, **i32)
  row_splits = torch.empty(N * (F + K), dtype=torch.int64, device=device)
  table_len, shard_len, emb_len = torch.empty(N * K, **i32), torch.empty(N, **i32), torch.empty(N * K, **i32)
  host_len = (C.c_int32 * (N * K))() if sync else None
  args = (device.index, ptr(fids), ptr(splits), recs, F, K, N, 1 if unique else 0, ptr(fused), ptr(fid_offset),
          ptr(feature_offset), ptr(nfl_offset), ptr(row_splits), ptr(table_len), ptr(shard_len), ptr(emb_len),
          None, host_len)
  if v5_batch_size is None:
    _lib.check(lib.mono_sharding_sparse_fids(*args, stream(device)))
  else:
    rs_size, emb_size, sizes = torch.empty(K * N, **i32), torch.empty(K * N, **i32), torch.empty(4, **i32)
    _lib.check(lib.mono_sharding_sparse_fids_v5(*args, v5_batch_size, ptr(rs_size), ptr(emb_size), ptr(sizes),
                                                stream(device)))
  # lists of table k: features first[k] .. first[k + 1] - 1 in table-major order; row splits block of (n, k) at
  # n * (F + K) + first[k] + k
  per_table = [sum(1 for n in names if t_idx[feature_table[n]] == k) for k in range(K)]
  first = [0]
  for c in per_table:
    first.append(first[-1] + c)
  rs_list = [row_splits[n * (F + K) + first[k] + k:n * (F + K) + first[k + 1] + k + 1] for k in range(K)
             for n in range(N)]
  fid_list = None
  if sync:
    lens = list(host_len)
    starts = [0]
    for x in lens:
      starts.append(starts[-1] + x)
    fid_list = [fused[starts[n * K + k]:starts[n * K + k + 1]] for k in range(K) for n in range(N)]
    fused = fused[:starts[-1]]
  else:
    fused = fused[:M]
  out = {"fid_list": fid_list, "fid_offset": fid_offset[:M], "feature_offset": feature_offset, "nfl_offset": nfl_offset,
         "table_names": tables, "feature_names": names, "fid_list_row_splits": rs_list, "fid_list_fused": fused,
         "fid_list_table_row_length": table_len, "fid_list_shard_row_length": shard_len,
         "fid_list_emb_row_length": emb_len}
  if v5_batch_size is not None:
    out.update({"fid_list_row_splits_size": [rs_size[i:i + 1] for i in range(K * N)], "nfl_size": sizes[0:1],
                "feature_size": sizes[1:2], "fid_size": sizes[2:3], "batch_size": sizes[3:4], "emb_size": emb_size})
  return out


def normalize_merged_split(row_split: torch.Tensor, row_split_size: torch.Tensor, *, sync: bool = True) -> torch.Tensor:
  """ref: distribution_ops.normalize_merged_split / MonolithNormalizeMergedSplit (RT/ops/normalize_merged_split_op.cc
  :33-90): row_split (int64, CUDA) holds len(row_split_size) row splits end to end, split i being row_split_size[i]
  entries that start at 0; the result (int64[len(row_split) + 1 - len(row_split_size)]) joins them, every later
  split's entries after its first shifted by the sum of the last entries of the splits before it.  E.g. [0, 2, 5, 5,
  9, 0, 0, 3, 4] with sizes [5, 4] gives [0, 2, 5, 5, 9, 9, 12, 13].  One device kernel (mono_normalize_merged_split).
  sync=True checks on the device that every size is >= 1 and that they add up to len(row_split), and raises
  ValueError otherwise (one synchronisation); sync=False makes no host round trip."""
  lib = _lib.load()
  dev = row_split.device
  rs = row_split.reshape(-1).to(torch.int64).contiguous()
  sz = row_split_size.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
  n, m = rs.numel(), sz.numel()
  if m > n or (m == 0 and n > 0):
    raise ValueError(f"normalize_merged_split: {m} merged splits for {n} entries")
  out = torch.empty(n + 1 - m if m else 0, dtype=torch.int64, device=dev)
  bad = torch.zeros(1, dtype=torch.int32, device=dev)
  _lib.check(lib.mono_normalize_merged_split(dev.index, ptr(rs), n, ptr(sz), m, ptr(out), ptr(bad), stream(dev)))
  if sync and int(bad.item()):
    raise ValueError("normalize_merged_split: every row_split_size must be >= 1 and they must add up to row_split's "
                     "length")
  return out


def round_to_f16(x: torch.Tensor) -> torch.Tensor:
  """x (float32, CUDA) rounded once to fp16, nearest even, by one kernel (mono_round_to_f16)."""
  if x.dtype != torch.float32 or x.device.type != "cuda":
    raise ValueError(f"round_to_f16 takes a CUDA float32 tensor, not {x.dtype} on {x.device}")
  x = x.contiguous()
  out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
  _lib.check(_lib.load().mono_round_to_f16(x.device.index, ptr(x), x.numel(), ptr(out), stream(x.device)))
  return out


def gather_pool(fused_embeddings: torch.Tensor, fused_embedding_offsets: torch.Tensor, dim: int,
                row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
                out: Optional[torch.Tensor] = None, out_col: int = 0, dtype: torch.dtype = torch.float32) -> torch.Tensor:
  """out[r] = pool_{m in row r} fused_embeddings[offsets[m]:offsets[m]+dim]
  (ref: FusedGatherKernel, runtime/ops/map_id_to_embedding.cu.cc:30-74, + per-row pool).
  The pooled rows are float32 or bfloat16: out's dtype when out is given, else `dtype`.  bfloat16 rows are the
  float32 results rounded once to nearest even; the fused buffer stays float32."""
  dtype = _tower_dtype(out.dtype if out is not None else dtype, "gather_pool's output")
  dev = fused_embeddings.device
  offs = fused_embedding_offsets.to(torch.int32).contiguous()
  row_offsets, n_rows = _lib.row_offsets(row_offsets, offs.numel())
  if out is None:
    out = torch.empty(n_rows, dim, dtype=dtype, device=dev)
  _lib.call("mono_gather_pool", dev.index, ptr(fused_embeddings), ptr(offs), ptr(row_offsets), n_rows, dim,
            _lib.POOLINGS[pooling], ptr(out), out.stride(0), out_col, bf16=dtype == torch.bfloat16, stream=stream(dev))
  return out


def gather_pool_grad(pooled_grad: torch.Tensor, fused_embedding_offsets: torch.Tensor, dim: int, total_floats: int,
                     row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum", grad_col: int = 0,
                     scale: Optional[torch.Tensor] = None):
  """Backward of gather_pool: scatter-add pooled grads to the fused row buffer
  (ref: FusedGatherGradKernel, map_id_to_embedding.cu.cc:75-118).  pooled_grad is float32 or bfloat16 (widened
  exactly); the returned buffer is float32.  scale: a one-element float32 tensor on pooled_grad's device (the
  reference kernel's `input * scale`): each gradient element is multiplied by it in float32 before the MEAN
  division (mono_gather_pool_grad[_bf16]_scaled)."""
  _tower_dtype(pooled_grad.dtype, "pooled_grad")
  scale_ptr(scale, pooled_grad.device, "scale")
  grad = torch.zeros(total_floats, dtype=torch.float32, device=pooled_grad.device)
  _gather_pool_grad_into(grad, pooled_grad, fused_embedding_offsets, dim, row_offsets, pooling, grad_col, scale)
  return grad


def _gather_pool_grad_into(grad, pooled_grad, fused_embedding_offsets, dim, row_offsets, pooling, grad_col, scale):
  """gather_pool_grad's launch: scatter-adds into the float32 buffer `grad`; scale is checked by the caller."""
  dev = pooled_grad.device
  offs = fused_embedding_offsets.to(torch.int32).contiguous()
  row_offsets, n_rows = _lib.row_offsets(row_offsets, offs.numel())
  _lib.call("mono_gather_pool_grad", dev.index, ptr(pooled_grad), pooled_grad.stride(0), grad_col, ptr(offs),
            ptr(row_offsets), n_rows, dim, _lib.POOLINGS[pooling], ptr(grad), bf16=pooled_grad.dtype == torch.bfloat16,
            scale=ptr(scale), stream=stream(dev))


def scatter_grad_rows(pooled_grad: torch.Tensor, fused_embedding_offsets: torch.Tensor, dim: int,
                      grad_fused: torch.Tensor, row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
                      grad_col: int = 0, scale: Optional[torch.Tensor] = None):
  """Deterministic (sort-based, atomics-free) scatter of pooled-row grads into the fused row buffer
  `grad_fused` (written in place; rows nobody refers to are left as they are).  pooled_grad is float32 or
  bfloat16 (widened exactly); grad_fused must be float32.  scale: as gather_pool_grad's; the result is bit for bit
  this call on pooled_grad multiplied by it in float32 (mono_scatter_grad_rows[_bf16]_scaled)."""
  bf16 = _tower_dtype(pooled_grad.dtype, "pooled_grad") == torch.bfloat16
  if grad_fused.dtype != torch.float32:
    raise ValueError(f"grad_fused must be torch.float32, not {grad_fused.dtype}")
  dev = pooled_grad.device
  sp = scale_ptr(scale, dev, "scale")
  offs = fused_embedding_offsets.to(torch.int32).contiguous()
  row_offsets, n_rows = _lib.row_offsets(row_offsets, offs.numel())
  _lib.call("mono_scatter_grad_rows", dev.index, ptr(pooled_grad), pooled_grad.stride(0), grad_col, ptr(offs),
            offs.numel(), ptr(row_offsets), n_rows, dim, _lib.POOLINGS[pooling], ptr(grad_fused), grad_fused.numel(),
            bf16=bf16, scale=sp, stream=stream(dev))
  return grad_fused


# ---- ReduceSum / ReduceMean / FusedReduceSumAndSplit / FusedReduceAndSplitGPU ------------------------------------
# ref: distribution_ops.py:689-884 and RT/ops/reduce_op.{cc,cu.cc}.  Every function below is one call of
# mono_reduce_and_split[_grad][_bf16]: see include/mono_emb.h for the arithmetic.

def _poolings(pooling, n):
  ps = [pooling] * n if isinstance(pooling, str) else list(pooling)
  if len(ps) != n or any(p not in _lib.POOLINGS for p in ps):
    raise ValueError(f"pooling must be 'sum', 'mean' or one of them per feature, not {pooling!r}")
  return ps


def _rows2d(t, what):
  if t.dim() != 2 or t.dtype != torch.float32 or (t.size(0) > 1 and t.stride(1) != 1):
    raise ValueError(f"{what} must be a 2-D float32 tensor with unit column stride")
  return t


def _reduce_split_call(backward, splits, rows, slices, poolings, bad_splits, scale=None):
  """splits[f]: int32 [B + 1]; rows[f]: [n_f, D_f] float32 (read forward, written backward); slices[f]: the 2-D
  tensors of feature f's slices (written forward, read backward), all float32 or all bfloat16.  scale (backward
  only): the clip_ops.scale_ptr of the gradient scale, or None for the unscaled call."""
  F = len(splits)
  flat = [t for s in slices for t in s]
  dtype = _tower_dtype(flat[0].dtype if flat else torch.float32, "the slice tensors")
  if any(t.dtype != dtype or t.dim() != 2 or (t.size(0) > 1 and t.stride(1) != 1) for t in flat):
    raise ValueError("the slice tensors must be 2-D with unit column stride and all float32 or all bfloat16")
  dev = splits[0].device if F else torch.device("cuda", torch.cuda.current_device())
  keep = []
  recs = (_lib.ReduceFeature * max(F, 1))()
  for f in range(F):
    sl = (_lib.ReduceSlice * max(len(slices[f]), 1))()
    for j, t in enumerate(slices[f]):
      sl[j].dim, sl[j].out_dev, sl[j].stride = t.size(1), t.data_ptr(), t.stride(0)
    keep.append(sl)
    r = rows[f]
    recs[f].splits_dev, recs[f].batch_size = splits[f].data_ptr(), splits[f].numel() - 1
    recs[f].rows_dev, recs[f].n_rows, recs[f].row_stride = r.data_ptr(), r.size(0), r.stride(0) if r.size(0) > 1 else r.size(1)
    recs[f].dim, recs[f].pooling = r.size(1), _lib.POOLINGS[poolings[f]]
    recs[f].slices, recs[f].n_slices = sl, len(slices[f])
  _lib.call("mono_reduce_and_split_grad" if backward else "mono_reduce_and_split", dev.index, recs, F,
            ptr(bad_splits), bf16=dtype == torch.bfloat16, scale=scale, stream=stream(dev))


def _splits32(splits):
  s = splits.reshape(-1)
  return s if s.dtype == torch.int32 and s.is_contiguous() else s.to(torch.int32).contiguous()


def fused_reduce_and_split_gpu(splits: Sequence[torch.Tensor], embeddings: Sequence[torch.Tensor],
                               slice_dims: Sequence[Sequence[int]], *, pooling="sum", dtype: torch.dtype = torch.float32,
                               bad_splits: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
  """ref: fused_reduce_and_split_gpu (distribution_ops.py:838-872, MonolithFusedReduceAndSplitGPU).  Feature f's
  per-occurrence rows embeddings[f] ([n_f, D_f] float32) are pooled per sample by its row splits splits[f] ([B + 1])
  and cut into slices of slice_dims[f].  Returns the flat list of [B, s] slices, feature by feature, in `dtype`
  (float32, or bfloat16: the float32 result rounded once).  pooling: 'sum' (the reference op), 'mean'
  (ReduceMean's multiply), or one per feature.  bad_splits (int32 [1] on the device, optional) becomes 1 when some
  feature's splits are malformed (such samples pool as empty); no host round trip."""
  dtype = _tower_dtype(dtype, "fused_reduce_and_split_gpu's dtype")
  F = len(splits)
  if len(embeddings) != F or len(slice_dims) != F:
    raise ValueError("splits, embeddings and slice_dims must have the same length")
  sp = [_splits32(s) for s in splits]
  rows = [_rows2d(e, "embeddings[%d]" % f) for f, e in enumerate(embeddings)]
  outs = [[torch.empty(s.numel() - 1, d, dtype=dtype, device=s.device) for d in dims] for s, dims in zip(sp, slice_dims)]
  _reduce_split_call(False, sp, rows, outs, _poolings(pooling, F), bad_splits)
  return [t for o in outs for t in o]


def fused_reduce_and_split_gpu_grad(splits: Sequence[torch.Tensor], embeddings: Sequence[torch.Tensor],
                                    grads: Sequence[torch.Tensor], slice_dims: Sequence[Sequence[int]], *,
                                    pooling="sum", out: Optional[Sequence[torch.Tensor]] = None,
                                    bad_splits: Optional[torch.Tensor] = None,
                                    grad_scale: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
  """ref: MonolithFusedReduceAndSplitGPUGrad (reduce_op.cu.cc:478-680).  grads is the flat list of slice gradients
  (all float32 or all bfloat16, widened exactly).  Returns feature f's occurrence-row gradients [n_f, D_f] float32:
  sample b's slice gradients copied (SUM) or times ReduceMean's factor (MEAN) into each of b's rows.  out[f], when
  given, is written instead (a [n_f, D_f] view, e.g. of the flat gradient buffer raw_apply_gradients takes); rows
  no sample covers are left as they are.  embeddings only give the shapes (as in the reference gradient).

  grad_scale: a one-element float32 tensor on the splits' device (clip_ops.global_norm_scale's scale), read on the
  device: the result is bit for bit this call on every slice gradient multiplied by it in float32 first (a bfloat16
  gradient is widened before the multiply; MEAN's factor comes after it).  mono_reduce_and_split_grad[_bf16]_scaled."""
  sc = None if grad_scale is None else scale_ptr(
      grad_scale, splits[0].device if len(splits) else torch.device("cuda", torch.cuda.current_device()))
  F = len(splits)
  sp = [_splits32(s) for s in splits]
  shapes = [(e.size(0), e.size(1)) for e in embeddings]
  if out is None:
    out = [torch.empty(n, d, dtype=torch.float32, device=s.device) for (n, d), s in zip(shapes, sp)]
  rows = [_rows2d(o, "out[%d]" % f) for f, o in enumerate(out)]
  if [tuple(o.shape) for o in rows] != shapes:
    raise ValueError("out must have the shapes of embeddings")
  it = iter(grads)
  per = [[next(it) for _ in dims] for dims in slice_dims]
  if sum(len(d) for d in slice_dims) != len(grads):
    raise ValueError("grads must hold one tensor per slice")
  _reduce_split_call(True, sp, rows, per, _poolings(pooling, F), bad_splits, sc)
  return list(rows)


def _batch_size(id_dense_shape):
  if isinstance(id_dense_shape, int):
    return id_dense_shape
  return int(torch.as_tensor(id_dense_shape).reshape(-1)[0])


def _splits_from_indices(id_indices, B, sync):
  """Row splits [B + 1] (int32, on the device) of the non-decreasing sample indices in [0, B) the reference's
  callers pass (fused_value_rowids).  The reference CPU ops accept any order; these calls do not: with sync=True
  unsorted or out-of-range indices raise ValueError, with sync=False nothing is checked on the host (the kernel
  still reads and writes only inside the given buffers)."""
  idx = id_indices[:, 0] if id_indices.dim() == 2 else id_indices.reshape(-1)
  idx = idx.to(torch.int64).contiguous()
  if sync and idx.numel():
    bad = (idx[0] < 0) | (idx[-1] >= B)
    if idx.numel() > 1:
      bad = bad | (idx[1:] < idx[:-1]).any()
    if bool(bad):
      raise ValueError(f"id_indices must be non-decreasing and in [0, {B})")
  q = torch.arange(B + 1, dtype=torch.int64, device=idx.device)
  return torch.searchsorted(idx, q, out_int32=True)


def _reduce(id_indices, id_values, B, split_dims, pooling, dtype, sync):
  splits = _splits_from_indices(id_indices, B, sync)
  return fused_reduce_and_split_gpu([splits], [id_values], [split_dims], pooling=pooling, dtype=dtype)


def _reduce_grad(id_indices, grads, split_dims, pooling, sync, B=None, grad_scale=None):
  scale_ptr(grad_scale, id_indices.device)
  B = grads[0].size(0) if B is None else B
  splits = _splits_from_indices(id_indices, B, sync)
  out = torch.empty(id_indices.size(0), sum(split_dims), dtype=torch.float32, device=splits.device)
  return fused_reduce_and_split_gpu_grad([splits], [out], grads, [split_dims], pooling=pooling, out=[out],
                                         grad_scale=grad_scale)[0]


def reduce_sum(id_indices: torch.Tensor, id_values: torch.Tensor, id_dense_shape, *,
               dtype: torch.dtype = torch.float32, sync: bool = True) -> torch.Tensor:
  """ref: reduce_sum (distribution_ops.py:726-741, MonolithReduceSum): [B, D] with row b = +0.0 + the id_values rows
  whose index is b, in order.  B = id_dense_shape[0]; id_indices [n, 1] (or [n]), non-decreasing in [0, B)."""
  return _reduce(id_indices, id_values, _batch_size(id_dense_shape), [id_values.size(1)], "sum", dtype, sync)[0]


def reduce_mean(id_indices: torch.Tensor, id_values: torch.Tensor, id_dense_shape, *,
                dtype: torch.dtype = torch.float32, sync: bool = True) -> torch.Tensor:
  """ref: reduce_mean (distribution_ops.py:689-700, MonolithReduceMean): reduce_sum's rows times
  (float)(1.0 / (float)n); an empty row is NaN (0 * inf), as in the reference."""
  return _reduce(id_indices, id_values, _batch_size(id_dense_shape), [id_values.size(1)], "mean", dtype, sync)[0]


def reduce_sum_gradient(id_indices: torch.Tensor, grads: torch.Tensor, *, sync: bool = True,
                        grad_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
  """ref: MonolithReduceSumGradient (reduce_op.cc:124-148): row i is grads[id_indices[i]] ([n, D] float32).
  grad_scale: as fused_reduce_and_split_gpu_grad's, on id_indices' device: row i is grads[id_indices[i]] * scale."""
  return _reduce_grad(id_indices, [grads], [grads.size(1)], "sum", sync, grad_scale=grad_scale)


def reduce_mean_gradient(id_indices: torch.Tensor, grads: torch.Tensor, *, sync: bool = True,
                         grad_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
  """ref: MonolithReduceMeanGradient (reduce_op.cc:150-180): row i is grads[b] times the forward's factor for
  b = id_indices[i], counted per sample (the reference sizes its counter by the dim, reduce_op.cc:166).
  grad_scale: as reduce_sum_gradient's; row i is (grads[b] * scale) * factor."""
  return _reduce_grad(id_indices, [grads], [grads.size(1)], "mean", sync, grad_scale=grad_scale)


def fused_reduce_sum_and_split(id_indices: torch.Tensor, id_values: torch.Tensor, id_length, split_dims: Sequence[int],
                               *, dtype: torch.dtype = torch.float32, sync: bool = True) -> List[torch.Tensor]:
  """ref: fused_reduce_sum_and_split (distribution_ops.py:802-826, MonolithFusedReduceSumAndSplit): reduce_sum over
  id_length samples, cut into [id_length, split_dims[i]] tensors."""
  if sum(split_dims) != id_values.size(1):
    raise ValueError("split_dims must add up to id_values.size(1)")
  return _reduce(id_indices, id_values, _batch_size(id_length), list(split_dims), "sum", dtype, sync)


def fused_reduce_sum_and_split_gradient(id_indices: torch.Tensor, grads: Sequence[torch.Tensor],
                                        split_dims: Sequence[int], *, sync: bool = True,
                                        grad_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
  """ref: MonolithFusedReduceSumAndSplitGradient (reduce_op.cc:282-330): [n, sum(split_dims)] float32, row i the
  concatenated slice gradients of sample id_indices[i].  grad_scale: as reduce_sum_gradient's."""
  if [g.size(1) for g in grads] != list(split_dims):
    raise ValueError("grads must have the split_dims widths")
  return _reduce_grad(id_indices, list(grads), list(split_dims), "sum", sync, grad_scale=grad_scale)


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
    _lib.check(self._lib.mono_grouping_build(self._h, ptr(fids), M, num_shards, dim, ptr(uniq), ptr(offs), counts,
                                             C.byref(n_u), stream(self.device)))
    self.dim = dim
    self._keep = fids  # the grouping refers to positions of this tensor until the next build
    return uniq[:n_u.value], offs[:M], list(counts)

  def reduce(self, pooled_grad: torch.Tensor, out_rows: torch.Tensor, row_offsets: Optional[torch.Tensor] = None,
             pooling: str = "sum", grad_col: int = 0, grad_scale: Optional[torch.Tensor] = None):
    """grad_scale: a one-element float32 tensor on the grouping's device, read on the device when the reduce runs:
    the rows are bit for bit this call's on pooled_grad multiplied by it in float32 (mono_grouping_reduce_scaled)."""
    sp = scale_ptr(grad_scale, self.device)
    row_offsets, n_rows = _lib.row_offsets(row_offsets, self._keep.numel())
    _lib.call("mono_grouping_reduce", self._h, ptr(pooled_grad), pooled_grad.stride(0), grad_col, ptr(row_offsets),
              n_rows, _lib.POOLINGS[pooling], ptr(out_rows), scale=sp, stream=stream(self.device))
    return out_rows

  def reduce_push(self, pooled_grad: torch.Tensor, shard_sizes: Sequence[int], window: "PeerWindow", region_off: int,
                  dst_row_off: Sequence[int], row_offsets: Optional[torch.Tensor] = None, pooling: str = "sum",
                  grad_col: int = 0, grad_scale: Optional[torch.Tensor] = None):
    """reduce() whose output rows are stored into the owners' windows (fused gradient exchange).  grad_scale: as
    reduce()'s (mono_grouping_reduce_push_scaled)."""
    sp = scale_ptr(grad_scale, self.device)
    row_offsets, n_rows = _lib.row_offsets(row_offsets, self._keep.numel())
    n = window.world
    _lib.call("mono_grouping_reduce_push", self._h, ptr(pooled_grad), pooled_grad.stride(0), grad_col,
              ptr(row_offsets), n_rows, _lib.POOLINGS[pooling], (C.c_int64 * n)(*[int(x) for x in shard_sizes]),
              window._h, int(region_off), (C.c_int64 * n)(*[int(x) for x in dst_row_off]), scale=sp,
              stream=stream(self.device))

  # ---- several features (mono_pool_part arrays) of ONE table as one batch: the sharded step over parts ----
  def build_parts(self, table, parts_arr, n_parts: int, n_fids: int, num_shards: int, dim: int):
    """build() over the concatenated FIDs of the parts (mono_grouping_build_parts; `table` is the MultiHashTable the
    parts name, n_fids their total occurrence count)."""
    uniq = torch.empty(max(n_fids, 1), dtype=torch.int64, device=self.device)
    offs = torch.empty(max(n_fids, 1), dtype=torch.int32, device=self.device)
    counts = (C.c_int32 * num_shards)()
    n_u = C.c_int64(0)
    _lib.check(self._lib.mono_grouping_build_parts(self._h, table._h, parts_arr, n_parts, num_shards, ptr(uniq),
                                                   ptr(offs), counts, C.byref(n_u), stream(self.device)))
    self.dim = dim
    return uniq[:n_u.value], offs[:n_fids], list(counts)

  def reduce_parts(self, table, parts_arr, n_parts: int, bf16: bool, out_rows: torch.Tensor,
                   grad_scale: Optional[torch.Tensor] = None):
    """reduce() with the parts' rows as the gradients (mono_grouping_reduce_parts[_bf16][_scaled])."""
    sp = scale_ptr(grad_scale, self.device)
    _lib.call("mono_grouping_reduce_parts", self._h, table._h, parts_arr, n_parts, ptr(out_rows), bf16=bf16, scale=sp,
              stream=stream(self.device))
    return out_rows

  def reduce_push_parts(self, table, parts_arr, n_parts: int, bf16: bool, shard_sizes: Sequence[int],
                        window: "PeerWindow", region_off: int, dst_row_off: Sequence[int],
                        grad_scale: Optional[torch.Tensor] = None):
    """reduce_push() with the parts' rows as the gradients (mono_grouping_reduce_push_parts[_bf16][_scaled])."""
    sp = scale_ptr(grad_scale, self.device)
    n = window.world
    _lib.call("mono_grouping_reduce_push_parts", self._h, table._h, parts_arr, n_parts,
              (C.c_int64 * n)(*[int(x) for x in shard_sizes]), window._h, int(region_off),
              (C.c_int64 * n)(*[int(x) for x in dst_row_off]), bf16=bf16, scale=sp, stream=stream(self.device))


def gather_pool_parts(table, rows_in: torch.Tensor, occ_offsets: torch.Tensor, parts_arr, n_parts: int, bf16: bool):
  """The pooling of looked-up rows into the rows of the parts (mono_gather_pool_parts[_bf16]): occ_offsets are a
  parts grouping's row offsets (Grouping.build_parts), `table` the MultiHashTable the parts name."""
  _lib.call("mono_gather_pool_parts", table._h, ptr(rows_in), ptr(occ_offsets), parts_arr, n_parts, bf16=bf16,
            stream=stream(rows_in.device))


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
    _lib.check(self._lib.mono_peer_barrier(self._h, stream(self.device)))

  def put(self, region_off: int, dst_off: Sequence[int], src: torch.Tensor, src_off: Sequence[int],
          nbytes: Sequence[int]):
    """nbytes[r] bytes of src (+ src_off[r]) -> rank r's window at region_off + dst_off[r]."""
    n = self.world
    arr = lambda xs: (C.c_int64 * n)(*[int(x) for x in xs])
    _lib.check(self._lib.mono_peer_put(self._h, int(region_off), arr(dst_off), ptr(src), arr(src_off), arr(nbytes),
                                       stream(self.device)))


  def get(self, region_off: int, src_off: Sequence[int], dst: torch.Tensor, dst_off: Sequence[int],
          nbytes: Sequence[int]):
    """nbytes[r] bytes of rank r's window at region_off + src_off[r] -> dst (+ dst_off[r], bytes)."""
    n = self.world
    arr = lambda xs: (C.c_int64 * n)(*[int(x) for x in xs])
    _lib.check(self._lib.mono_peer_get(self._h, int(region_off), arr(src_off), ptr(dst), arr(dst_off), arr(nbytes),
                                       stream(self.device)))


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
  results rounded once to nearest even; the tasks' strides and columns then count bfloat16 elements).
  embeddings_list may also be all float16 (rows a transfer_float16 parameter server sent): the f16in kernels then
  widen every element exactly where they load it, so the outputs are bit for bit this call on the lists widened to
  float32 (mono_embedding_to_layout_f16in[_bf16])."""
  bf16 = _tower_dtype(dtype, "dtype") == torch.bfloat16
  f16_in = len(embeddings_list) > 0 and embeddings_list[0].dtype == torch.float16
  dev = _check_layout_inputs(fid_offset, feature_offset, nfl_offset, embeddings_list, "embeddings_list",
                             torch.float16 if f16_in else torch.float32)
  outs = [torch.zeros(*s, dtype=dtype, device=dev) for s in out_shapes]
  embs = [e.contiguous() for e in embeddings_list]
  ep, op = _ptr_table(embs, dev), _ptr_table(outs, dev)
  st = torch.tensor(list(emb_strides), dtype=torch.int32, device=dev)
  _lib.call("mono_embedding_to_layout_f16in" if f16_in else "mono_embedding_to_layout", dev.index, ptr(ep), ptr(st),
            len(embs), ptr(fid_offset), fid_offset.numel(), ptr(feature_offset), feature_offset.numel(),
            ptr(nfl_offset), nfl_offset.numel(), batch_size, _tasks_arr(tasks), len(tasks), ptr(op), bf16=bf16,
            stream=stream(dev))
  return outs


def fused_embedding_to_layout_grad(emb_sizes: Sequence[int], emb_strides: Sequence[int], fid_offset: torch.Tensor,
                                   feature_offset: torch.Tensor, nfl_offset: torch.Tensor, batch_size: int,
                                   tasks: Sequence[SliceTask], out_grads: Sequence[torch.Tensor],
                                   layout_tensors_grad_scale: Optional[torch.Tensor] = None,
                                   out: Optional[Sequence[torch.Tensor]] = None):
  """ref: MonolithEmbeddingToLayoutGradV* (fused_embedding_to_layout.cc:697-948).  The index tensors as in
  fused_embedding_to_layout; out_grads all float32 or all bfloat16 (widened exactly) on their device.  The
  returned embedding gradients are float32.  layout_tensors_grad_scale: a one-element float32 tensor on that device
  (the reference's `layout_tensors_grad_scale * grad`, distribution_ops.py:544-550): every gradient element is
  multiplied by it in float32 before the MEAN division (mono_embedding_to_layout_grad[_bf16]_scaled).
  out: zero-filled contiguous float32 tensors of emb_sizes elements on that device (e.g. views of one buffer) that
  receive the gradients and are returned, in place of fresh ones."""
  dtype = _tower_dtype(out_grads[0].dtype if len(out_grads) else torch.float32, "out_grads")
  if any(g.dtype != dtype for g in out_grads):
    raise ValueError(f"out_grads must be all torch.float32 or all torch.bfloat16, not {[g.dtype for g in out_grads]}")
  dev = _check_layout_inputs(fid_offset, feature_offset, nfl_offset, out_grads, "out_grads", dtype)
  sp = scale_ptr(layout_tensors_grad_scale, dev, "layout_tensors_grad_scale")
  if out is None:
    grads = [torch.zeros(n, dtype=torch.float32, device=dev) for n in emb_sizes]
  else:
    grads = list(out)
    if len(grads) != len(emb_sizes) or any(g.dtype != torch.float32 or g.device != dev or not g.is_contiguous() or
                                           g.numel() != int(n) for g, n in zip(grads, emb_sizes)):
      raise ValueError(f"out must be {len(emb_sizes)} contiguous float32 tensors on {dev} of emb_sizes elements")
  og = [g.contiguous() for g in out_grads]
  gp, op = _ptr_table(grads, dev), _ptr_table(og, dev)
  st = torch.tensor(list(emb_strides), dtype=torch.int32, device=dev)
  _lib.call("mono_embedding_to_layout_grad", dev.index, ptr(gp), ptr(st), len(grads), ptr(fid_offset),
            fid_offset.numel(), ptr(feature_offset), feature_offset.numel(), ptr(nfl_offset), nfl_offset.numel(),
            batch_size, _tasks_arr(tasks), len(tasks), ptr(op), bf16=dtype == torch.bfloat16, scale=sp,
            stream=stream(dev))
  return grads


# ---- async parameter-server worker path (ref: NT/distributed_ps.py:266-337, 430-516) --------------------------------
def _host_splits(splits, what):
  s = [int(x) for x in (splits.tolist() if isinstance(splits, torch.Tensor) else splits)]
  if not s or s[0] != 0 or any(b < a for a, b in zip(s, s[1:])):
    raise ValueError(f"{what} must start at 0 and not decrease")
  return s


@dataclasses.dataclass
class UniqueKeyWithValueAndOffset:
  """unique_key_with_value_and_offset's outputs.  unique_key = (values, row_splits): every table's distinct keys in
  first-occurrence order, row splits int64[K + 1] on the device.  value_offset = (values, row_splits): for every unique
  key the float offsets of all its occurrences in the value buffer, in occurrence order, and its int64 row splits over
  the unique keys.  value_buffer: float32[value_len], uninitialised (None without generate_buffer).  num_unique: U, or
  None with sync=False, when unique_key's values and value_offset's row splits are allocated for every key (M and
  M + 1 entries) and only the first U and U + 1 are written."""
  unique_key: Tuple[torch.Tensor, torch.Tensor]
  value_offset: Tuple[torch.Tensor, torch.Tensor]
  value_buffer: Optional[torch.Tensor]
  value_len: int
  num_unique: Optional[int]


def unique_key_with_value_and_offset(ids: torch.Tensor, key_split: Sequence[int], dims: Sequence[int],
                                     generate_buffer: bool = True, *, sync: bool = True) -> UniqueKeyWithValueAndOffset:
  """ref: distribution_ops.unique_key_with_value_and_offset / UniqueKeyWitValueAndOffsetOp (RT/ops/unique_mapping_ops.cc
  :51-124).  ids: int64 keys of K tables (CUDA), table k = ids[key_split[k]:key_split[k + 1]] (host row splits, as
  MultiHashTable.get_ragged_id gives them) with dims[k] floats per row.  Occurrence i of table k sits at float
  base_k + (i - key_split[k]) * dims[k] of the value buffer, base_k = sum of count_k' * dims[k'] over k' < k.
  sync=True reads the K + 1 unique row splits back (one synchronisation) to trim the outputs; sync=False makes no host
  round trip."""
  lib = _lib.load()
  splits = _host_splits(key_split, "key_split")
  K = len(splits) - 1
  if len(dims) != K:
    raise ValueError(f"dims has {len(dims)} entries for {K} tables")
  ids = ids.reshape(-1).to(torch.int64).contiguous()
  if splits[-1] != ids.numel():
    raise ValueError("key_split does not cover ids")
  M, dev = ids.numel(), ids.device
  i64 = dict(dtype=torch.int64, device=dev)
  uniq, uniq_split = torch.empty(max(M, 1), **i64), torch.empty(K + 1, **i64)
  off, off_split = torch.empty(max(M, 1), **i64), torch.empty(M + 1, **i64)
  value_len = C.c_int64(0)
  host = (C.c_int64 * (K + 1))() if sync else None
  _lib.check(lib.mono_unique_key_with_value_and_offset(
      dev.index, ptr(ids), (C.c_int64 * (K + 1))(*splits), K, (C.c_int32 * K)(*[int(d) for d in dims]), ptr(uniq),
      ptr(uniq_split), ptr(off), ptr(off_split), C.byref(value_len), host, stream(dev)))
  buf = torch.empty(value_len.value, dtype=torch.float32, device=dev) if generate_buffer else None
  U = host[K] if sync else None
  if sync:
    uniq, off_split = uniq[:U], off_split[:U + 1]
  else:
    uniq = uniq[:M]
  return UniqueKeyWithValueAndOffset((uniq, uniq_split), (off[:M], off_split), buf, value_len.value, U)


@dataclasses.dataclass
class RaggedSplit:
  """ragged_split_by_indices' outputs.  splits[s] = (values, row_splits) of split s (row splits int64[K + 1] on the
  device, starting at 0) and pos[s] the input index of each of its values; row_splits_host[s] the same row splits as
  Python ints.  All three are None with sync=False.  The flat fields hold the S splits concatenated split after
  split: values, positions, row_splits [S, K + 1], offsets [S + 1] (split s at offsets[s] .. offsets[s + 1]) and bad
  (int32[1], 1 for an index outside [0, S) or malformed row splits)."""
  splits: Optional[List[Tuple[torch.Tensor, torch.Tensor]]]
  pos: Optional[List[torch.Tensor]]
  row_splits_host: Optional[List[List[int]]]
  values: torch.Tensor
  positions: torch.Tensor
  row_splits: torch.Tensor
  offsets: torch.Tensor
  bad: torch.Tensor


def ragged_split_by_indices(indices: torch.Tensor, values: torch.Tensor, row_splits: torch.Tensor, num_splits: int, *,
                            sync: bool = True) -> RaggedSplit:
  """ref: distribution_ops.ragged_split_by_indices / RaggedSplitByIndicesOp (RT/ops/split_by_indices_op.cc:188-243):
  the ragged tensor (values, row_splits int64[K + 1], CUDA) split by indices[t] in [0, num_splits), stably.  values
  and indices may be longer than row_splits[K] (sync=False outputs of unique_key_with_value_and_offset); the rest is
  ignored.  sync=True reads every split's row splits back (one synchronisation), raises ValueError for an index outside
  [0, num_splits) or malformed row splits, and slices the splits; sync=False makes no host round trip."""
  lib = _lib.load()
  S = int(num_splits)
  dev = values.device
  values = values.reshape(-1).to(torch.int64).contiguous()
  indices = indices.reshape(-1).to(device=dev, dtype=torch.int64).contiguous()
  row_splits = row_splits.reshape(-1).to(device=dev, dtype=torch.int64).contiguous()
  if indices.numel() != values.numel():
    raise ValueError(f"Ragged tensor values size must match indices size. Got {values.numel()} v.s. {indices.numel()}")
  K, cap = row_splits.numel() - 1, values.numel()
  i64 = dict(dtype=torch.int64, device=dev)
  v_out, p_out = torch.empty(max(cap, 1), **i64), torch.empty(max(cap, 1), **i64)
  rs_out, offs = torch.empty(max(S, 0) * max(K + 1, 0), **i64), torch.empty(max(S, 0) + 1, **i64)
  bad = torch.zeros(1, dtype=torch.int32, device=dev)
  host = (C.c_int64 * (S * (K + 1)))() if sync and S > 0 and K > 0 else None
  _lib.check(lib.mono_ragged_split_by_indices(dev.index, ptr(indices), ptr(values), cap, ptr(row_splits), K, S,
                                              ptr(v_out), ptr(p_out), ptr(rs_out), ptr(offs), ptr(bad), host,
                                              stream(dev)), value_error=True)
  rs2 = rs_out.view(S, K + 1)
  out = RaggedSplit(None, None, None, v_out[:cap], p_out[:cap], rs2, offs, bad)
  if sync:
    h = [list(host[s * (K + 1):(s + 1) * (K + 1)]) for s in range(S)]
    starts = [0]
    for r in h:
      starts.append(starts[-1] + r[-1])
    out.row_splits_host = h
    out.splits = [(v_out[starts[s]:starts[s + 1]], rs2[s]) for s in range(S)]
    out.pos = [p_out[starts[s]:starts[s + 1]] for s in range(S)]
  return out


def split_by_indices(indices: torch.Tensor, tensor: torch.Tensor, num_splits: int) -> List[torch.Tensor]:
  """ref: distribution_ops.split_by_indices: the rows of `tensor` split by indices[i] in [0, num_splits), each split in
  input order.  One ragged split of the positions (a single list), then index_select by them.  Synchronises once."""
  n = indices.numel()
  dev = tensor.device
  positions = torch.arange(n, dtype=torch.int64, device=dev)
  r = ragged_split_by_indices(indices, positions, torch.tensor([0, n], dtype=torch.int64, device=dev), num_splits)
  return [tensor.index_select(0, p) for p in r.pos]


def _fill_call(grad, pos, pos_split, src, value_offset, dims, num_unique, dst, sync):
  splits = _host_splits(pos_split, "pos_split")
  K = len(splits) - 1
  if len(dims) != K:
    raise ValueError(f"dims has {len(dims)} entries for {K} tables")
  dev = src.device
  pos = pos.reshape(-1).to(device=dev, dtype=torch.int64).contiguous()
  if pos.numel() != splits[-1]:
    raise ValueError("pos_split does not cover pos")
  offs, offs_split = (t.reshape(-1).to(device=dev, dtype=torch.int64).contiguous() for t in value_offset)
  U = offs_split.numel() - 1 if num_unique is None else int(num_unique)
  # fp16 server rows are read as they are (the _f16 fill widens them exactly); anything else is widened here
  f16_src = not grad and src.dtype == torch.float16
  src = src.reshape(-1).to(torch.float16 if f16_src else torch.float32).contiguous()
  bad = torch.zeros(1, dtype=torch.int32, device=dev)
  c_split, c_dims = (C.c_int64 * (K + 1))(*splits), (C.c_int32 * K)(*[int(d) for d in dims])
  if grad:
    _lib.call("mono_fill_with_offset_map_grad_f16" if dst.dtype == torch.float16 else "mono_fill_with_offset_map_grad",
              dev.index, ptr(pos), c_split, K, c_dims, ptr(src), ptr(offs), ptr(offs_split), U, ptr(dst), ptr(bad),
              stream=stream(dev), value_error=True)
  else:
    _lib.call("mono_fill_with_offset_map_f16" if f16_src else "mono_fill_with_offset_map", dev.index, ptr(pos),
              c_split, K, c_dims, ptr(src), src.numel(), ptr(offs), ptr(offs_split), U, ptr(dst), ptr(bad),
              stream=stream(dev), value_error=True)
  if sync and int(bad.item()):
    raise ValueError(f"pos is bigger than offset size: a pos outside [0, {U})")
  return dst


def fill_with_offset_map(pos: torch.Tensor, pos_split: Sequence[int], value: torch.Tensor,
                         value_offset: Tuple[torch.Tensor, torch.Tensor], value_buffer: torch.Tensor,
                         dims: Sequence[int], *, num_unique: Optional[int] = None, sync: bool = True) -> torch.Tensor:
  """ref: distribution_ops.fill_with_offset_map / FillWithOffsetMapOp (RT/ops/unique_mapping_ops.cc:204-268): one
  server's rows `value` (row t of table k = pos_split row t, dims[k] floats, packed in row order) copied to every
  occurrence offset of the unique key pos[t] (value_offset = the unique op's (offsets, row splits)) in value_buffer,
  which is returned.  pos_split: host row splits.  num_unique defaults to value_offset's row splits length - 1.
  Raises ValueError when value is shorter than the rows need (a longer one is accepted); sync=True also checks that
  every pos lies in [0, num_unique) (one synchronisation); sync=False makes no host round trip.  A float16 value (rows
  sent as fp16, transfer_float16) is read as fp16 and widened exactly in the copy; another dtype is converted to
  float32 first."""
  if value_buffer.dtype != torch.float32 or not value_buffer.is_contiguous():
    raise ValueError("value_buffer must be a contiguous float32 tensor")
  return _fill_call(False, pos, pos_split, value, value_offset, dims, num_unique, value_buffer, sync)


def fill_with_offset_map_gradient(pos: torch.Tensor, pos_split: Sequence[int], grad: torch.Tensor,
                                  value_offset: Tuple[torch.Tensor, torch.Tensor], dims: Sequence[int], *,
                                  num_unique: Optional[int] = None, sync: bool = True,
                                  dtype: torch.dtype = torch.float32) -> torch.Tensor:
  """ref: distribution_ops.fill_with_offset_map_gradient / FillWithOffsetMapGradientOp (unique_mapping_ops.cc:284-329):
  row t of the result (packed like fill_with_offset_map's value) is +0.0 + grad[o_1 ..] + grad[o_2 ..] + ... in fp32
  over pos[t]'s occurrence offsets in occurrence order: the reference's bits at every run length.  sync as in
  fill_with_offset_map.  dtype=torch.float16 returns the same sums, each rounded once to fp16 (the gradients a
  transfer_float16 worker sends to its servers)."""
  if dtype not in (torch.float32, torch.float16):
    raise ValueError(f"fill_with_offset_map_gradient: dtype must be torch.float32 or torch.float16, not {dtype}")
  splits = _host_splits(pos_split, "pos_split")
  n_floats = sum((splits[k + 1] - splits[k]) * int(dims[k]) for k in range(len(splits) - 1))
  out = torch.empty(n_floats, dtype=dtype, device=grad.device)
  return _fill_call(True, pos, splits, grad, value_offset, dims, num_unique, out, sync)
