"""numpy restatement of the reference's per-slot parameter-server path, the one DistributedMultiTypeHashTable takes
with transfer_float16 (ref: NT/distributed_ps.py:340-412 lookup, :516-552 apply_gradients): per slot tf.unique
(first-occurrence order), floormod(id, num_ps) and a stable split_by_indices; every server's rows cast to fp16 and
back before map_id_to_embedding (RT/ops/map_id_to_embedding_op.cc:39-107), and every unique id's gradient summed by
map_id_to_embedding_gradient_back_prop (:109-146: memset to +0.0, then sequential fp32 +=, in occurrence order), then
cast to fp16 and back.

fp16 rounding is numpy's astype(np.float16): round to nearest even, beyond the fp16 range to +-inf, below half the
smallest fp16 subnormal to +-0, the sign of zero kept."""
import numpy as np


def f16_round(x):
  """f32(f16_rn(x)), elementwise"""
  with np.errstate(over="ignore", invalid="ignore"):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def unique_first(ids):
  """tf.unique: (distinct ids in first-occurrence order, idx with ids == unique[idx])"""
  ids = np.asarray(ids, np.int64).reshape(-1)
  u, first, inv = np.unique(ids, return_index=True, return_inverse=True)
  order = np.argsort(first, kind="stable")
  rank = np.empty(u.size, np.int64)
  rank[order] = np.arange(u.size)
  return u[order], rank[inv.reshape(-1)]


def split_by_indices(indices, values, num_splits):
  """distribution_ops.split_by_indices: the values with index s, in input order, for every s"""
  indices = np.asarray(indices, np.int64)
  return [values[indices == s] for s in range(num_splits)]


def map_id_to_embedding(split_ids, split_embeddings, ids):
  """MapIdToEmbeddingOp: the row of every id of `ids` (any shape) from the split that holds it; split s has rows
  split_embeddings[s] [n_s, dim] -> ids.shape + [dim]"""
  keys = np.concatenate([np.asarray(k, np.int64).reshape(-1) for k in split_ids])
  rows = np.concatenate([np.asarray(e, np.float32) for e in split_embeddings])
  order = np.argsort(keys, kind="stable")
  flat = np.asarray(ids, np.int64).reshape(-1)
  at = order[np.searchsorted(keys[order], flat)]
  assert np.array_equal(keys[at], flat), "an id is in no split"
  return rows[at].reshape(np.asarray(ids).shape + (rows.shape[1],))


def map_id_to_embedding_gradient(split_ids, ids, grads):
  """MapIdToEmbeddingGradientBackPropOp: per split, the rows of its ids = +0.0 + the gradients (ids.shape + [dim]) of
  their occurrences in `ids`, added one at a time in occurrence order in fp32"""
  flat = np.asarray(ids, np.int64).reshape(-1)
  grads = np.asarray(grads, np.float32)
  grads = grads.reshape(flat.size, grads.shape[-1])  # ids.shape + [dim]
  out = []
  with np.errstate(over="ignore", invalid="ignore"):
    for k in split_ids:
      k = np.asarray(k, np.int64).reshape(-1)
      acc = np.zeros((k.size, grads.shape[1]), np.float32)
      if k.size:
        order = np.argsort(k, kind="stable")
        j = np.searchsorted(k[order], flat)
        hit = (j < k.size) & (k[order][np.minimum(j, k.size - 1)] == flat)
        occ = np.nonzero(hit)[0]                 # the occurrences of this split's ids, in occurrence order
        row = order[j[occ]]
        # the r-th occurrence of every id is added in step r, so each id's adds stay in occurrence order
        by_row = np.argsort(row, kind="stable")
        new = np.concatenate([[True], row[by_row][1:] != row[by_row][:-1]]) if occ.size else np.zeros(0, bool)
        first = np.maximum.accumulate(np.where(new, np.arange(occ.size), 0)) if occ.size else np.zeros(0, np.int64)
        rank = np.empty(occ.size, np.int64)
        rank[by_row] = np.arange(occ.size) - first
        for r in range(int(rank.max()) + 1 if occ.size else 0):
          sel = rank == r
          acc[row[sel]] = acc[row[sel]] + grads[occ[sel]]
      out.append(acc)
  return out


def lookup(server_lookup, num_ps, slot_to_id):
  """The per-slot lookup: server_lookup(s, slot, ids) -> fp32 rows [n, dim] of server s (misses +0.0).
  -> slot -> [n, dim] as the worker sees them."""
  out = {}
  for slot, ids in slot_to_id.items():
    u, _ = unique_first(ids)
    split_ids = split_by_indices(np.mod(u, num_ps), u, num_ps)
    rows = [f16_round(server_lookup(s, slot, split_ids[s])) for s in range(num_ps)]
    out[slot] = map_id_to_embedding(split_ids, rows, ids)
  return out


def apply_gradients(num_ps, slot_to_id_and_grad):
  """The per-slot apply: -> per server s, slot -> (its unique ids, the fp32 gradients it applies: the summed
  gradients rounded to fp16 and widened back)"""
  per_ps = [dict() for _ in range(num_ps)]
  for slot, (ids, grad) in slot_to_id_and_grad.items():
    u, _ = unique_first(ids)
    split_ids = split_by_indices(np.mod(u, num_ps), u, num_ps)
    sums = map_id_to_embedding_gradient(split_ids, ids, grad)
    for s in range(num_ps):
      per_ps[s][slot] = (split_ids[s], f16_round(sums[s]))
  return per_ps
