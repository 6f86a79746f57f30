"""ReduceSum / ReduceMean / FusedReduceSumAndSplit / FusedReduceAndSplitGPU without a device: the numpy
restatement (tests/reduce_split_model.py) against the reference's own known answers (tests/golden/ref_reduce_split.json, from
distribution_ops_test.py:306-519) and against numpy scatter + split; ReduceMean's multiplier; the host-side argument
checks of mono_reduce_and_split[_grad][_bf16]."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

from tests import reduce_split_model as rsm

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ref_reduce_split.json")))


def splits_of(indices, B):
  """Row splits of non-decreasing sample indices (what fused_value_rowids gives)."""
  return np.searchsorted(np.asarray(indices, np.int64), np.arange(B + 1), side="left").astype(np.int32)


def rows(values, width):
  return np.asarray(values, np.float32).reshape(-1, width)


def mean_factor(n):
  """ReduceMeanOp's `float multiply = 1.0 / static_cast<float>(counter)` (reduce_op.cc:81), for one count."""
  return np.float32(1.0 / np.float64(np.float32(n)))


@pytest.mark.parametrize("op", ["reduce_sum", "reduce_mean"])
def test_reduce_known_answers(op):
  g = GOLDEN[op]
  v = rows(g["id_values"], 2)
  out = rsm.reduce_and_split([splits_of(g["id_indices"], g["batch_size"])], [v], [[2]], [op[7:]])[0][0]
  np.testing.assert_array_equal(out, g["expected"])


@pytest.mark.parametrize("op", ["reduce_sum_gradient", "reduce_mean_gradient"])
def test_reduce_gradient_known_answers(op):
  g = GOLDEN[op]
  pool = "sum" if op.startswith("reduce_sum") else "mean"
  sp = splits_of(g["id_indices"], g["batch_size"])
  got = rsm.reduce_and_split_grad([sp], [(len(g["id_indices"]), 2)], [[rows(g["loss_grad"], 2)]], [pool])[0]
  np.testing.assert_array_equal(got, g["expected"])


@pytest.mark.parametrize("case", range(3))
def test_fused_reduce_sum_and_split_known_answers(case):
  g = GOLDEN["fused_reduce_sum_and_split"][case]
  sp = splits_of(g["id_indices"], g["id_length"])
  outs = rsm.reduce_and_split([sp], [rows(g["id_values"], 3)], [g["split_dims"]], ["sum"])[0]
  assert len(outs) == len(g["expected"])
  for o, e in zip(outs, g["expected"]):
    np.testing.assert_array_equal(o, e)


def test_fused_reduce_sum_and_split_gradient_known_answer():
  g = GOLDEN["fused_reduce_sum_and_split_grad"]
  sp = splits_of(g["id_indices"], g["id_length"])
  ones = [np.ones((g["id_length"], d), np.float32) for d in g["split_dims"]]   # tf.gradients of the outputs
  got = rsm.reduce_and_split_grad([sp], [(3, 3)], [ones], ["sum"])[0]
  np.testing.assert_array_equal(got, g["expected"])


def test_fused_reduce_scatter_shapes():
  """fused_sorted_segment_sum's cases are SUM pools over sorted indices: one fused call, empty feature included."""
  cases = GOLDEN["fused_reduce_scatter"]
  sps = [splits_of(c["indices"], c["shape"][0]) for c in cases]
  vals = [rows(c["values"], c["shape"][1]) for c in cases]
  outs = rsm.reduce_and_split(sps, vals, [[c["shape"][1]] for c in cases], ["sum"] * len(cases))
  for o, c in zip(outs, cases):
    np.testing.assert_array_equal(o[0], c["expected"])


def test_102_features_against_numpy_scatter_and_split():
  """test_fused_reduce_and_split_gpu's shapes: dims 2i - 1, slices of l // 4 (1-column slices below 4), shuffled row
  lengths 0..255; random values, so the order of the adds shows."""
  rng = random.Random(7)
  nrng = np.random.default_rng(7)
  B, F = 256, 102
  lens = [2 * i - 1 for i in range(1, F + 1)]
  sdims = [[1] * l if l < 4 else [l // 4] * 3 + [l // 4 + l % 4] for l in lens]
  row_lens = list(range(B))
  rng.shuffle(row_lens)
  sp = np.concatenate([[0], np.cumsum(row_lens)]).astype(np.int32)
  rowids = np.repeat(np.arange(B), row_lens)
  embs = [nrng.standard_normal((sp[-1], l)).astype(np.float32) for l in lens]
  outs = rsm.reduce_and_split([sp] * F, embs, sdims, ["sum"] * F)
  for f in range(F):
    want = np.zeros((B, lens[f]), np.float32)
    for i, b in enumerate(rowids):   # sequential fp32 adds in occurrence order, from +0.0
      want[b] += embs[f][i]
    for o, w in zip(outs[f], np.split(want, np.cumsum(sdims[f])[:-1], axis=1)):
      np.testing.assert_array_equal(o.view(np.uint32), w.view(np.uint32))


def test_sum_starts_from_positive_zero_and_mean_of_empty_row_is_nan():
  v = np.array([[-0.0], [-0.0]], np.float32)
  s = rsm.reduce_and_split([[0, 2, 2]], [v], [[1]], ["sum"])[0][0]
  assert s.view(np.uint32).tolist() == [[0], [0]]          # +0.0 + -0.0 + -0.0 = +0.0
  m = rsm.reduce_and_split([[0, 2, 2]], [v], [[1]], ["mean"])[0][0]
  assert m[0, 0] == 0 and np.isnan(m[1, 0])                # 0 * (1 / 0)


def test_mean_factor_up_to_2_20_matches_the_c_expression():
  """The multiplier for n in 1 .. 2^20 is the double reciprocal of float(n) rounded to float: numpy's vectorised form
  against the literal C expression (ctypes float conversions around Python's double division) at the first and last
  4 096 counts and 20 000 random ones, and against the restatement's MEAN gradient."""
  n = np.arange(1, (1 << 20) + 1)
  fast = (1.0 / n.astype(np.float32).astype(np.float64)).astype(np.float32)
  for k in list(range(1, 4097)) + list(range(1 << 20, (1 << 20) - 4096, -1)) + list(nrange(n)):
    assert fast[k - 1] == np.float32(C.c_float(1.0 / C.c_float(k).value).value)
  # the restatement's MEAN gradient of a one-sample row with g = 1 is exactly the factor
  for k in (1, 3, 7, 1000, 4097, 65535, 1 << 20):
    got = rsm.reduce_and_split_grad([[0, k]], [(k, 1)], [[np.ones((1, 1), np.float32)]], ["mean"])[0]
    assert (got == fast[k - 1]).all() and mean_factor(k) == fast[k - 1]


def nrange(n):
  return np.random.default_rng(3).choice(n, 20000, replace=False) + 1


# ---- host-side argument checks: MONO_ERR_INVALID_ARGUMENT before the device is touched ---------------------------

def call(feats, fn="mono_reduce_and_split"):
  from monolith_b200 import _lib
  lib = _lib.load()
  keep, recs = [], (_lib.ReduceFeature * max(len(feats), 1))()
  for i, f in enumerate(feats):
    sl = (_lib.ReduceSlice * max(len(f.get("slices", [])), 1))()
    for j, (d, ptr, st) in enumerate(f.get("slices", [])):
      sl[j].dim, sl[j].out_dev, sl[j].stride = d, ptr, st
    keep.append(sl)
    recs[i].splits_dev, recs[i].batch_size = f.get("splits", 16), f.get("B", 4)
    recs[i].rows_dev, recs[i].n_rows, recs[i].row_stride = f.get("rows", 16), f.get("n", 8), f.get("stride", 4)
    recs[i].dim, recs[i].pooling = f.get("dim", 4), f.get("pooling", 0)
    recs[i].slices, recs[i].n_slices = (sl if "slices" in f else None), len(f.get("slices", []))
  return getattr(lib, fn)(0, recs, len(feats), None, None)


OK = dict(slices=[(4, 64, 4)])
BAD = {
    "different batch sizes": [OK, dict(OK, B=5)],
    "negative batch size": [dict(OK, B=-1)],
    "batch size over 2^31 - 2": [dict(OK, B=1 << 31)],
    "dim 0": [dict(OK, dim=0, slices=[(0, 64, 4)])],
    "negative n_rows": [dict(OK, n=-1)],
    "n_rows over 2^31 - 1": [dict(OK, n=1 << 31)],
    "row stride < dim": [dict(OK, stride=3)],
    "null splits": [dict(OK, splits=0)],
    "null rows": [dict(OK, rows=0)],
    "pooling FIRSTN": [dict(OK, pooling=2)],
    "no slices": [dict(OK, slices=[])],
    "slice dim 0": [dict(OK, slices=[(0, 64, 4), (4, 64, 4)])],
    "slice stride < slice dim": [dict(OK, slices=[(4, 64, 3)])],
    "null slice pointer": [dict(OK, slices=[(4, 0, 4)])],
    "slice dims short of dim": [dict(OK, slices=[(3, 64, 4)])],
    "slice dims over dim": [dict(OK, slices=[(3, 64, 4), (2, 64, 4)])],
    "features x batch over 2^33": [dict(OK, B=(1 << 31) - 2)] * 5,
}


@pytest.mark.parametrize("fn", ["mono_reduce_and_split", "mono_reduce_and_split_grad", "mono_reduce_and_split_bf16",
                                "mono_reduce_and_split_grad_bf16"])
@pytest.mark.parametrize("case", sorted(BAD))
def test_arguments_are_rejected_on_the_host(case, fn):
  assert call(BAD[case], fn) == -1   # MONO_ERR_INVALID_ARGUMENT


def test_negative_feature_count_is_rejected():
  from monolith_b200 import _lib
  assert _lib.load().mono_reduce_and_split(0, None, -1, None, None) == -1


def test_record_structs_match_the_header():
  from monolith_b200 import _lib
  assert C.sizeof(_lib.ReduceSlice) == 24
  assert C.sizeof(_lib.ReduceFeature) == 64
  assert [f for f, _ in _lib.ReduceFeature._fields_] == ["splits_dev", "batch_size", "rows_dev", "n_rows", "row_stride",
                                                         "dim", "pooling", "slices", "n_slices"]

