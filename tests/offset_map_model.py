"""numpy restatement of the async parameter-server worker ops (ref: RT/ops/unique_mapping_ops.cc:51-124, 204-329;
RT/ops/split_by_indices_op.cc:188-243): the reference's loops, vectorised where the order they define allows it."""
import numpy as np


def unique_key_with_value_and_offset(keys, key_split, dims):
  """(unique_key, unique_key_split, value_offset, value_offset_split, value_len).  Per table, the distinct keys in
  first-occurrence order (keys equal when their bits are equal); for each, the float offsets of its occurrences in
  occurrence order, occurrence i of table j at base_j + (i - key_split[j]) * dims[j]."""
  keys = np.asarray(keys, np.int64)
  uniq, uks, vo, vos = [], [0], [], [np.zeros(1, np.int64)]
  base, n_vos = 0, 0
  for j in range(len(dims)):
    lo, hi = int(key_split[j]), int(key_split[j + 1])
    k = keys[lo:hi]
    offs = base + np.arange(hi - lo, dtype=np.int64) * int(dims[j])
    base += (hi - lo) * int(dims[j])
    if k.size == 0:
      uks.append(uks[-1])
      continue
    u, first, inv = np.unique(k, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")          # first-occurrence order
    ordinal = np.empty(u.size, np.int64)
    ordinal[order] = np.arange(u.size)
    occ_ord = ordinal[inv.reshape(-1)]
    grouped = np.argsort(occ_ord, kind="stable")      # occurrences grouped by ordinal, in occurrence order
    counts = np.bincount(occ_ord, minlength=u.size)
    uniq.append(u[order])
    uks.append(uks[-1] + u.size)
    vo.append(offs[grouped])
    vos.append(n_vos + np.cumsum(counts))
    n_vos += k.size
  cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)
  return (cat(uniq).astype(np.int64), np.asarray(uks, np.int64), cat(vo).astype(np.int64),
          cat(vos).astype(np.int64), base)


def ragged_split_by_indices(indices, values, num_split, S):
  """[(values_s, row_splits_s)], [pos_s]: stable split by indices; row splits per split over the K rows."""
  indices, values, num_split = (np.asarray(x, np.int64) for x in (indices, values, num_split))
  splits, pos = [], []
  for s in range(S):
    p = np.nonzero(indices == s)[0].astype(np.int64)
    rs = np.searchsorted(p, num_split, side="left").astype(np.int64)
    splits.append((values[p], rs))
    pos.append(p)
  return splits, pos


def _rows(pos_split, dims):
  """table and first float of every packed row"""
  table = np.repeat(np.arange(len(dims)), np.diff(np.asarray(pos_split, np.int64)))
  d = np.asarray(dims, np.int64)[table]
  return table, np.concatenate([[0], np.cumsum(d)[:-1]]).astype(np.int64) if d.size else np.zeros(0, np.int64), d


def fill_with_offset_map(pos, pos_split, value, value_offset, value_offset_split, dims, buffer):
  """buffer[o : o + dim] = value row t for every occurrence offset o of pos[t] (writes into buffer).  The rows' copies
  go to disjoint offsets, so their order does not matter."""
  _, start, d = _rows(pos_split, dims)
  value = np.asarray(value, np.float32)
  pos = np.asarray(pos, np.int64)
  if pos.size == 0:
    return buffer
  lo = value_offset_split[pos]
  n = value_offset_split[pos + 1] - lo
  t = np.repeat(np.arange(pos.size), n)                                  # the row of every occurrence
  first = np.concatenate([[0], np.cumsum(n)[:-1]])
  o = value_offset[np.repeat(lo - first, n) + np.arange(int(n.sum()))]  # its offset
  for dim in np.unique(d):
    sel = d[t] == dim
    cols = np.arange(dim)
    buffer[o[sel][:, None] + cols[None, :]] = value[start[t[sel]][:, None] + cols[None, :]]
  return buffer


def fill_with_offset_map_gradient(pos, pos_split, grad, value_offset, value_offset_split, dims):
  """row t = +0.0f + g[o_1 ..] + g[o_2 ..] + ... in float32, strictly in occurrence order (setZero, then +=)"""
  _, start, d = _rows(pos_split, dims)
  grad = np.asarray(grad, np.float32)
  pos = np.asarray(pos, np.int64)
  out = np.zeros(int(d.sum()), np.float32)
  lo = value_offset_split[pos] if pos.size else np.zeros(0, np.int64)
  n = value_offset_split[pos + 1] - lo if pos.size else np.zeros(0, np.int64)
  with np.errstate(over="ignore", invalid="ignore"):  # infinities and NaNs in the gradients are part of the contract
    for dim in np.unique(d):
      _sum_rows(out, grad, value_offset, start, lo, n, d, dim)
  return out


def _sum_rows(out, grad, value_offset, start, lo, n, d, dim):
  """the rows of width dim: the k-th occurrence of every key with more than k, for k = 0, 1, ..."""
  rows = np.nonzero(d == dim)[0]
  cols = np.arange(dim)
  acc = np.zeros((rows.size, dim), np.float32)
  for k in range(int(n[rows].max()) if rows.size else 0):
    live = rows[n[rows] > k]
    sel = np.searchsorted(rows, live)
    acc[sel] = acc[sel] + grad[value_offset[lo[live] + k][:, None] + cols[None, :]]
  out[start[rows][:, None] + cols[None, :]] = acc
