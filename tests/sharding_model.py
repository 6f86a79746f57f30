"""numpy restatement of ShardingSparseFids, versions 3 and 4, unique and non-unique (ref: parse_sparse_feature.cc:187-330,
parse_sparse_feature.h:714-920; the reference's Python model parse_sparse_feature_test.py:89-301, pinned on it by
tests/golden/ref_sharding_v4.npz).  Vectorised per feature, so it serves multi-million-FID batches too."""
import numpy as np


def _per_shard(v, N, unique):
  """-> (lists[n] of the feature's FIDs of shard n, ordinal of every occurrence inside its shard's list)"""
  shard = (v.view(np.uint64) % np.uint64(N)).astype(np.int64)
  if unique:
    _, first, inv = np.unique(v, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")         # distinct FIDs in first-occurrence order
    items, item_shard = v[first[order]], shard[first[order]]
    rank_of = np.empty(order.size, np.int64)
    rank_of[order] = np.arange(order.size)
    occ_item = rank_of[inv.reshape(-1)]
  else:
    items, item_shard, occ_item = v, shard, np.arange(v.size)
  perm = np.argsort(item_shard, kind="stable")
  counts = np.bincount(item_shard, minlength=N)
  start = np.concatenate([[0], np.cumsum(counts)])
  ordinal = np.empty(items.size, np.int64)
  ordinal[perm] = np.arange(items.size) - start[item_shard[perm]]
  lists = [items[perm[start[n]:start[n + 1]]] for n in range(N)]
  return lists, ordinal[occ_item], shard


def sharding(feats, table_of, dims_sum, N, shared=(), unique=True):
  """feats[name] = (fids int64[n], row_splits int64[rows + 1]).  Returns the version-3 outputs (fid_list as K*N arrays,
  index table * N + shard; fid_list_row_splits likewise), fid_offset uint64, feature_offset int32, nfl_offset uint32,
  and the version-4 ones: fid_list_fused (shard-major, table-minor), fid_list_row_splits_fused [shard][table][...],
  fid_list_table_row_length / fid_list_emb_row_length [N*K] and fid_list_shard_row_length [N] (int32)."""
  names = sorted(feats)
  tables = sorted({table_of[n] for n in names})
  K = len(tables)
  per = {n: _per_shard(np.asarray(feats[n][0], np.int64).reshape(-1), N, unique) for n in names}
  lists, rsplits, pre, emb_len = {}, {}, {}, {}
  for k, t in enumerate(tables):
    tf = [n for n in names if table_of[n] == t]
    for s in range(N):
      parts = [per[n][0][s] for n in tf]
      lists[k, s] = np.concatenate(parts) if parts else np.zeros(0, np.int64)
      rsplits[k, s] = np.concatenate([[0], np.cumsum([p.size for p in parts])]).astype(np.int64)
      emb = 0
      for n, p in zip(tf, parts):
        pre[n, s] = emb
        emb += p.size * int(dims_sum[n])
      emb_len[k, s] = emb
  fid_offset, feature_offset, nfl_offset, occ = [], [], [], 0
  for n in names:
    _, ordinal, shard = per[n]
    k = tables.index(table_of[n])
    base = np.array([pre[n, s] for s in range(N)], np.int64)
    local = ordinal * int(dims_sum[n]) + base[shard]
    fid_offset.append((((k * N + shard) << 32) | local).astype(np.int64).view(np.uint64))
    nfl_offset.append(len(feature_offset) | ((1 << 31) if n in shared else 0))
    rs = np.asarray(feats[n][1], np.int64).reshape(-1)
    feature_offset.extend((occ + rs[:-1]).tolist())
    occ += int(rs[-1])
  feature_offset.append(occ)
  nfl_offset.append(len(feature_offset))
  out = {"fid_list": [lists[k, s] for k in range(K) for s in range(N)],
         "fid_list_row_splits": [rsplits[k, s] for k in range(K) for s in range(N)],
         "fid_offset": np.concatenate(fid_offset) if fid_offset else np.zeros(0, np.uint64),
         "feature_offset": np.array(feature_offset, np.int32), "nfl_offset": np.array(nfl_offset, np.uint32),
         "table_names": tables, "feature_names": names}
  out["fid_list_fused"] = np.concatenate([lists[k, s] for s in range(N) for k in range(K)])
  out["fid_list_row_splits_fused"] = np.concatenate([rsplits[k, s] for s in range(N) for k in range(K)])
  out["fid_list_table_row_length"] = np.array([lists[k, s].size for s in range(N) for k in range(K)], np.int32)
  out["fid_list_shard_row_length"] = out["fid_list_table_row_length"].reshape(N, K).sum(1).astype(np.int32)
  out["fid_list_emb_row_length"] = np.array([emb_len[k, s] for s in range(N) for k in range(K)], np.int32)
  return out
