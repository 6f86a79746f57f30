"""Generates tests/golden/ref_sharding_v4.npz: ShardingSparseFids' version-3 and version-4 outputs, unique and
non-unique, computed by the REFERENCE's own Python model of the op.

monolith/native_training/data/parse_sparse_feature_test.py holds the model as methods of its test class:
`get_feature_cfg` (:89-139), `handle_feature` (:141-159, per-(feature, shard) lists of every occurrence and of the
distinct FIDs), `fill_row_split` (:73-80, the per-(table, shard) row splits, called before every feature and once per
table at the end, as its tests do at :720-748) and `get_offset_result` (:161-240).  They are lifted out with `ast`
(the module imports TensorFlow; nothing is copied into this repo) and run with version = 4.  The version-4 regrouping
of the lists (shard-major, table-minor) and the table / shard / embedding row lengths sit inside `diff_test` next to
TensorFlow code (:249-302), so they are restated below.  Inputs and outputs are stored as a fixture.

    MONOLITH_REF=<bytedance/monolith checkout> python tests/golden/make_sharding_v4_golden.py
"""
import ast
import logging
import os
import types
from collections import defaultdict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.environ.get("MONOLITH_REF", "."), "monolith/native_training/data/parse_sparse_feature_test.py")
WANTED = ("fid_v1_to_v2", "fill_row_split", "get_pre_output_offset", "get_feature_cfg", "handle_feature",
          "get_offset_result")


def reference_model():
  tree = ast.parse(open(REF).read())
  cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "DataOpsV2Test")
  fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in WANTED]
  assert len(fns) == len(WANTED)
  ns = {"defaultdict": defaultdict, "logging": logging, "print": lambda *a, **k: None}
  exec(compile(ast.Module(body=fns, type_ignores=[]), REF, "exec"), ns)
  model = types.SimpleNamespace(mask=(1 << 48) - 1, version=4)
  for name in WANTED:
    setattr(model, name, types.MethodType(ns[name], model))
  return model


def version4(table_name_sort, table_cfg, feature_cfg, N, lists, row_splits):
  """diff_test's version-4 regrouping (parse_sparse_feature_test.py:249-302) of one mode's per-(table, shard) lists"""
  K = len(table_name_sort)
  fused, fused_rs = [], []
  table_len, shard_len, emb_len = [0] * (N * K), [0] * N, [0] * (N * K)
  for s in range(N):
    for k, t in enumerate(table_name_sort):
      key = f"{t}:{s}"
      fused.extend(lists[key])
      fused_rs.extend(row_splits[key])
      table_len[s * K + k] = len(lists[key])
      shard_len[s] += len(lists[key])
      feats = table_cfg[t]["feature_list"]
      assert len(feats) + 1 == len(row_splits[key])
      emb_len[s * K + k] = sum(feature_cfg[f]["dims_sum"] * (row_splits[key][i + 1] - row_splits[key][i])
                               for i, f in enumerate(feats))
  return fused, fused_rs, table_len, shard_len, emb_len


CASES = [  # n_feat, n_tab, N, B, max FIDs per row, shared features, features without rows, features without FIDs
    dict(n_feat=5, n_tab=2, N=3, B=6, max_len=4, shared=(), no_rows=(), no_fids=()),
    dict(n_feat=9, n_tab=3, N=3, B=17, max_len=6, shared=(2, 7), no_rows=(4,), no_fids=(1,)),
    dict(n_feat=4, n_tab=4, N=1, B=5, max_len=3, shared=(), no_rows=(0,), no_fids=()),     # one feature per table
    dict(n_feat=12, n_tab=3, N=8, B=40, max_len=9, shared=(0,), no_rows=(11,), no_fids=(5,)),
    dict(n_feat=7, n_tab=5, N=8, B=23, max_len=5, shared=(3, 6), no_rows=(), no_fids=(2,)),
]


def main():
  model = reference_model()
  rng = np.random.default_rng(44)
  out = {}
  for ci, c in enumerate(CASES):
    N = c["N"]
    names = [f"f_{chr(97 + (5 * i) % 26)}{i}" for i in range(c["n_feat"])]          # not in sorted order on purpose
    cfgs = types.SimpleNamespace(feature_configs={
        n: types.SimpleNamespace(table=f"table_{(3 * i) % c['n_tab']}", slice_dims=list(rng.integers(1, 6, 3)))
        for i, n in enumerate(names)})
    feature_cfg, table_cfg, feature_name_sort, table_name_sort = model.get_feature_cfg(cfgs, N)
    shared = {names[i] for i in c["shared"]}
    flat, splits = {}, {}
    for fi, name in enumerate(names):
      rows = 0 if fi in c["no_rows"] else 1 if name in shared else c["B"]
      lens = np.zeros(rows, np.int64) if fi in c["no_fids"] else rng.integers(0, c["max_len"] + 1, rows)
      vals = ((np.int64(100 + fi) << 48) | rng.integers(0, 12, int(lens.sum()))).astype(np.int64)  # many repeats
      flat[name], splits[name] = vals, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    # the reference tests' flow: row splits before every feature, features in sorted-name order, then once per table
    fid_map_t, fid_map_unique_t, fid_map_unique_map = defaultdict(list), defaultdict(list), defaultdict(dict)
    fid_offset_map, fid_offset_map_unique = defaultdict(list), defaultdict(list)
    rs_t, rs_unique_t = defaultdict(list), defaultdict(list)
    for name in feature_name_sort:
      f_cfg = feature_cfg[name]
      t_cfg = table_cfg[f_cfg["table_name"]]
      model.fill_row_split(N, t_cfg, fid_map_t, rs_t)
      model.fill_row_split(N, t_cfg, fid_map_unique_t, rs_unique_t)
      for b in range(len(splits[name]) - 1):
        l1, l2 = [], []
        model.handle_feature([], [int(v) for v in flat[name][splits[name][b]:splits[name][b + 1]]], f_cfg, t_cfg, N,
                             l1, l2, fid_map_t, fid_map_unique_map, fid_map_unique_t)
        fid_offset_map[name].append(l1)
        fid_offset_map_unique[name].append(l2)
    for t in table_name_sort:
      model.fill_row_split(N, table_cfg[t], fid_map_t, rs_t)
      model.fill_row_split(N, table_cfg[t], fid_map_unique_t, rs_unique_t)
    nfl, feat_off, fid_off, fid_off_unique, tab_lists, tab_lists_unique = model.get_offset_result(
        feature_name_sort, table_name_sort, N, feature_cfg, table_cfg, fid_offset_map, fid_offset_map_unique,
        fid_map_t, fid_map_unique_t, shared)
    p = f"c{ci}_"
    out[p + "names"] = np.array(names)
    out[p + "tables"] = np.array([cfgs.feature_configs[n].table for n in names])
    out[p + "dims_sum"] = np.array([int(sum(cfgs.feature_configs[n].slice_dims)) for n in names], np.int64)
    out[p + "shared"] = np.array([n in shared for n in names])
    out[p + "N"] = np.int64(N)
    out[p + "n_tables"] = np.int64(len(table_name_sort))
    for n in names:
      out[p + "fids_" + n] = flat[n]
      out[p + "splits_" + n] = splits[n]
    out[p + "nfl_offset"] = np.array(nfl, np.uint32)
    out[p + "feature_offset"] = np.array(feat_off, np.int32)
    for mode, fo, lists, rs in (("unique", fid_off_unique, tab_lists_unique, rs_unique_t), ("all", fid_off, tab_lists,
                                                                                             rs_t)):
      q = p + mode + "_"
      out[q + "fid_offset"] = np.array(fo, np.uint64)
      for k, t in enumerate(table_name_sort):
        for s in range(N):
          out[q + f"list_{k}_{s}"] = np.array(lists[f"{t}:{s}"], np.int64)
          out[q + f"row_splits_{k}_{s}"] = np.array(rs[f"{t}:{s}"], np.int64)
      fused, fused_rs, tl, sl, el = version4(table_name_sort, table_cfg, feature_cfg, N, lists, rs)
      out[q + "fused"] = np.array(fused, np.int64)
      out[q + "fused_row_splits"] = np.array(fused_rs, np.int64)
      out[q + "table_row_length"] = np.array(tl, np.int32)
      out[q + "shard_row_length"] = np.array(sl, np.int32)
      out[q + "emb_row_length"] = np.array(el, np.int32)
  out["n_cases"] = np.int64(len(CASES))
  np.savez_compressed(os.path.join(HERE, "ref_sharding_v4.npz"), **out)
  print("wrote ref_sharding_v4.npz")


if __name__ == "__main__":
  main()
