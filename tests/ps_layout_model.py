"""numpy restatement of PartitionedHashTable's parameter-server mode with the fused layout (ref: NT/distributed_ps.py
:1003-1460 without enable_gpu_emb): ShardingSparseFids version 5 (the version-3 outputs of tests/sharding_model.py plus
the sizes of parse_sparse_feature.cc:287-301, 329-336, 390-404 and parse_sparse_feature.h:837-893),
NormalizeMergedSplit (RT/ops/normalize_merged_split_op.cc:33-90), per-server dict tables with SGD and Adagrad, and the
fp16 casts of transfer_float16.  The layout forward and gradient themselves are the oracle's (tests/orc.py), which
tests/test_gpu_layout_paths.py pins on every layout and pooling."""
import numpy as np

from tests import orc
from tests import sharding_model as sm


def sharding_v5(feats, table_of, dims_sum, N, shared=(), unique=True, batch_size=None):
  """sharding_model.sharding's outputs plus the version-5 ones: fid_list_row_splits_size [K*N] (features of the table
  + 1), nfl_size, feature_size, fid_size, batch_size and emb_size [K*N] (floats of list (table k, shard n) at
  k * N + n), all int32."""
  out = sm.sharding(feats, table_of, dims_sum, N, shared, unique)
  names = sorted(feats)
  tables = sorted({table_of[n] for n in names})
  K = len(tables)
  if batch_size is None:
    rows = {feats[n][1].size - 1 for n in names if n not in set(shared)}
    assert len(rows) == 1
    batch_size = rows.pop()
  per_table = [sum(1 for n in names if table_of[n] == t) for t in tables]
  emb_len = np.asarray(out["fid_list_emb_row_length"]).reshape(N, K)
  out["fid_list_row_splits_size"] = np.asarray([per_table[k] + 1 for k in range(K) for _ in range(N)], np.int32)
  out["emb_size"] = emb_len.T.reshape(-1).astype(np.int32)
  out["nfl_size"] = np.asarray([len(names) + 1], np.int32)
  out["feature_size"] = np.asarray([out["feature_offset"].size], np.int32)
  out["fid_size"] = np.asarray([out["fid_offset"].size], np.int32)
  out["batch_size"] = np.asarray([batch_size], np.int32)
  return out


def normalize_merged_split(row_split, row_split_size):
  """The reference loop, line for line."""
  row_split = np.asarray(row_split, np.int64)
  sizes = np.asarray(row_split_size, np.int32)
  out = np.zeros(row_split.size + 1 - sizes.size, np.int64)
  offset = pre_size = output_idx = 0
  for i in range(sizes.size):
    lo = offset if i == 0 else offset + 1
    for j in range(lo, offset + int(sizes[i])):
      out[output_idx] = pre_size + row_split[j]
      output_idx += 1
    offset += int(sizes[i])
    pre_size += int(row_split[offset - 1])
  return out


def f16_round_trip(x):
  """f32(f16_rn(x)): what crosses between a transfer_float16 server and its worker."""
  return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


class DictTable:
  """One server's table: fid -> row (fp32, zeros-initialised), and the Adagrad accumulator.  apply() takes the ids in
  order, duplicates one after the other (the reference's per-id loop).  SGD: w -= lr * g.  Adagrad with no weight
  decay, BaselineAdagradOptimize (RT/hash_table/optimizer/avx_utils.h:29-38), the form the reference takes for rows
  shorter than 8 floats: norm += g * g; w -= lr / sqrt(norm) * g, all in fp32."""

  def __init__(self, dims, opt, lr, init_acc=0.1):
    self.dims, self.opt, self.lr, self.init_acc = dict(dims), opt, np.float32(lr), np.float32(init_acc)
    self.rows = {t: {} for t in dims}
    self.acc = {t: {} for t in dims}

  def lookup(self, table, ids):
    d = self.dims[table]
    return np.stack([self.rows[table].get(int(i), np.zeros(d, np.float32)) for i in ids]) if len(ids) else \
        np.zeros((0, d), np.float32)

  def apply(self, table, ids, grads):
    d = self.dims[table]
    for i, g in zip(ids, np.asarray(grads, np.float32).reshape(-1, d)):
      w = self.rows[table].setdefault(int(i), np.zeros(d, np.float32))
      if self.opt == "sgd":
        w -= self.lr * g
      else:
        assert d < 8, "the baseline Adagrad form is the reference's only below 8 floats"
        acc = self.acc[table].setdefault(int(i), np.full(d, self.init_acc, np.float32))
        acc += g * g
        w -= (self.lr / np.sqrt(acc)) * g


def ps_step(servers, feats, table_of, dims_sum, N, tasks, shapes, layout_grads=None, shared=(), unique=True,
            transfer_float16=False):
  """One PartitionedHashTablePS lookup (and apply when layout_grads is given) on dict tables.  Returns (layout
  tensors, sharding outputs)."""
  sh = sharding_v5(feats, table_of, dims_sum, N, shared, unique)
  tables = sorted({table_of[n] for n in feats})
  K = len(tables)
  B = int(sh["batch_size"][0])
  embs = []
  for k, t in enumerate(tables):
    for n in range(N):
      rows = servers[n].lookup(t, sh["fid_list"][k * N + n]).reshape(-1)
      embs.append(f16_round_trip(rows) if transfer_float16 else rows.astype(np.float32))
  fo, fe = sh["fid_offset"].view(np.uint64), sh["feature_offset"]
  nfl = sh["nfl_offset"].view(np.uint32)
  layouts = orc.embedding_to_layout(embs, [1] * (K * N), fo, fe, nfl, B, tasks, shapes)
  if layout_grads is not None:
    grads = orc.embedding_to_layout_grad([e.size for e in embs], [1] * (K * N), fo, fe, nfl, B, tasks, layout_grads)
    for k, t in enumerate(tables):
      for n in range(N):
        g = grads[k * N + n]
        servers[n].apply(t, sh["fid_list"][k * N + n], f16_round_trip(g) if transfer_float16 else g)
  return layouts, sh
