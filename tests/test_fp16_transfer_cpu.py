"""transfer_float16 of the async parameter-server table without a GPU: the three fp16 C entry points' declarations,
bindings and argument checks; the Python argument checks; and the per-slot model (tests/fp16_transfer_model.py)
pinned on the reference's own answers and shown equal, bit for bit, to the raw path (tests/offset_map_model.py)
followed by one fp16 rounding of the rows and of the gradient sums, which is what the engine computes."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from monolith_b200 import _lib, distribution_ops as dops
from monolith_b200.multi_hash_table_ops import MultiHashTable
from tests import fp16_transfer_model as fm
from tests import offset_map_model as om

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWINS = {"mono_mtable_lookup_f16": "mono_mtable_lookup",
         "mono_fill_with_offset_map_f16": "mono_fill_with_offset_map",
         "mono_fill_with_offset_map_grad_f16": "mono_fill_with_offset_map_grad"}
I64_MIN = np.iinfo(np.int64).min


def _declaration(header, name):
  m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", header)
  assert m, f"{name} is not declared"
  return [" ".join(a.split()) for a in m.group(1).split(",")]


def test_declarations_match_their_twins():
  header = open(os.path.join(ROOT, "include", "mono_emb.h")).read()
  for name, twin in TWINS.items():
    args, twin_args = _declaration(header, name), _declaration(header, twin)
    assert args == twin_args, (name, args, twin_args)  # the 16-bit rows pass through the twin's float pointer
    assert _lib.SIGNATURES[name] == _lib.SIGNATURES[twin]
    getattr(_lib.load(), name)
  assert "0x7FFF" in header


def test_abi_version_is_unchanged():
  assert _lib.load().mono_abi_version() == 1


# ---- the C entry points' argument checks: MONO_ERR_INVALID_ARGUMENT before the device is selected ----------------
_P = C.c_void_p(16)  # never dereferenced: every case below is rejected on the host


def _fill(split, dims, value_len=100, num_unique=4, grad=False):
  lib = _lib.load()
  K = len(dims)
  cs, cd = (C.c_int64 * len(split))(*split), (C.c_int32 * max(K, 1))(*dims)
  if grad:
    return lib.mono_fill_with_offset_map_grad_f16(0, _P, cs, K, cd, _P, _P, _P, num_unique, _P, None, None)
  return lib.mono_fill_with_offset_map_f16(0, _P, cs, K, cd, _P, value_len, _P, _P, num_unique, _P, None, None)


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("kw,what", [
    (dict(split=[0], dims=[]), "num_tables must be positive"),
    (dict(split=[1, 2], dims=[1]), "start at 0"),
    (dict(split=[0, 2, 1], dims=[1, 1]), "must not decrease"),
    (dict(split=[0, 2], dims=[0]), "dims must be positive"),
    (dict(split=[0, (1 << 30) + 1], dims=[1], value_len=1 << 31), "2^30 rows"),
    (dict(split=[0, 2], dims=[1], num_unique=-1), "num_unique"),
])
def test_f16_fill_rejects(kw, what, grad):
  assert _fill(grad=grad, **kw) == -1
  assert what in _lib.load().mono_last_error().decode()


def test_f16_fill_value_len_counts_fp16_elements():
  # 2 + 1 rows of dims 3 and 6: 10 fp16 elements where 12 are needed; 12 pass this check
  assert _fill([0, 2, 3], [3, 6], value_len=10) == -1
  assert "expected: 12, actual: 10" in _lib.load().mono_last_error().decode()
  assert _fill([0, 2, 3], [3, 6], value_len=12, num_unique=-1) == -1
  assert "num_unique" in _lib.load().mono_last_error().decode()


def test_f16_null_splits_are_rejected():
  lib = _lib.load()
  assert lib.mono_fill_with_offset_map_f16(0, _P, None, 1, (C.c_int32 * 1)(1), _P, 4, _P, _P, 1, _P, None, None) == -1
  assert lib.mono_fill_with_offset_map_grad_f16(0, _P, (C.c_int64 * 2)(0, 1), 1, None, _P, _P, _P, 1, _P, None,
                                                None) == -1


# ---- Python argument checks, before any device work -----------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float64, torch.int32])
def test_bad_dtypes_are_rejected(dtype):
  ids = torch.zeros(2, dtype=torch.int64)
  with pytest.raises(ValueError, match="dtype"):
    MultiHashTable.raw_lookup(object(), ids, [0, 2], dtype=dtype)  # refused before the table is touched
  with pytest.raises(ValueError, match="dtype"):
    dops.fill_with_offset_map_gradient(ids, [0, 2], torch.zeros(4), (ids, ids), [2], dtype=dtype)


@pytest.mark.parametrize("split", [[1, 2], [0, 2, 1], []])
def test_malformed_splits_are_rejected(split):
  ids = torch.zeros(2, dtype=torch.int64)
  with pytest.raises(ValueError, match="pos_split"):
    dops.fill_with_offset_map_gradient(ids, split, torch.zeros(4), (ids, ids), [2] * max(len(split) - 1, 1),
                                       dtype=torch.float16)
  with pytest.raises(ValueError, match="pos_split"):
    dops.fill_with_offset_map(ids, split, torch.zeros(4, dtype=torch.float16), (ids, ids), torch.zeros(4),
                              [2] * max(len(split) - 1, 1))


# ---- the model on the reference's answers ---------------------------------------------------------------------------
def test_map_id_to_embedding_reference_vectors():
  """ref: distribution_ops_test.py:128-141"""
  out = fm.map_id_to_embedding([[1], [2]], [np.array([[1, 1]]), np.array([[2, 2]])], np.array([[1], [2]]))
  assert out.tolist() == [[[1, 1]], [[2, 2]]]


def test_map_id_to_embedding_split_by_floormod():
  """ref: distribution_ops_test.py:143-162: 1000 ids split over 10 servers map back to their own rows"""
  ids = np.arange(1000, dtype=np.int64)
  emb = np.tile(np.arange(16, dtype=np.float32), (1000, 1))
  idx = np.mod(ids, 10)
  out = fm.map_id_to_embedding(fm.split_by_indices(idx, ids, 10), fm.split_by_indices(idx, emb, 10), ids)
  assert np.array_equal(out, emb)


def test_map_id_to_embedding_gradient_reference_vectors():
  """ref: distribution_ops_test.py:164-180: loss = target - output, so every occurrence's gradient is -1"""
  grads = fm.map_id_to_embedding_gradient([[1], [2]], np.array([1, 1, 2]), -np.ones((3, 2), np.float32))
  assert [g.tolist() for g in grads] == [[[-2, -2]], [[-1, -1]]]


class SgdServers:
  """num_ps servers of fp32 SGD tables (lr 1, zeros init): slot -> {id: row}"""

  def __init__(self, num_ps, dims, lr=1.0):
    self.t = [{s: {} for s in dims} for _ in range(num_ps)]
    self.dims, self.lr = dims, np.float32(lr)

  def lookup(self, s, slot, ids):
    d = self.dims[slot]
    return np.array([self.t[s][slot].get(int(i), np.zeros(d, np.float32)) for i in ids], np.float32).reshape(-1, d)

  def apply(self, per_ps):
    for s, slots in enumerate(per_ps):
      for slot, (ids, g) in slots.items():
        for i, row in zip(ids.tolist(), g):
          w = self.t[s][slot].get(i, np.zeros(self.dims[slot], np.float32))
          self.t[s][slot][i] = (w - self.lr * row).astype(np.float32)


def test_apply_gradients_float16_reference_answer():
  """ref: distributed_ps_test.py:376-413 (test_apply_gradients_float16, 2 servers, transfer_float16=True): loss1 =
  2 * values1, loss2 = 3 * values2, one SGD step at lr 1 from zeros"""
  srv = SgdServers(2, {"1": 1, "2": 2})
  ids = {"1": np.array([1, 2], np.int64), "2": np.array([3], np.int64)}
  grads = {"1": np.full((2, 1), 2, np.float32), "2": np.full((1, 2), 3, np.float32)}
  srv.apply(fm.apply_gradients(2, {k: (ids[k], grads[k]) for k in ids}))
  got = fm.lookup(srv.lookup, 2, ids)
  assert got["1"].tolist() == [[-2.0], [-2.0]]
  assert got["2"].tolist() == [[-3.0, -3.0]]


def test_f16_round_edges():
  x = np.array([65504, 65519.99, 65520, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, -0.0, 1e-45, np.inf, -1e9],
               np.float32)
  want = np.array([65504, 65504, np.inf, 2.0 ** -24, 0.0, 2.0 ** -24, -0.0, 0.0, np.inf, -np.inf], np.float32)
  got = fm.f16_round(x)
  assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist()
  assert np.isnan(fm.f16_round(np.array([np.nan], np.float32)))[0]


# ---- the per-slot model equals the raw path plus one rounding -------------------------------------------------------
def _same(got, want):
  got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
  assert got.shape == want.shape
  gn, wn = np.isnan(got), np.isnan(want)
  assert np.array_equal(gn, wn)
  assert np.array_equal(got[~gn].view(np.uint32), want[~wn].view(np.uint32))


def _rows(rng, n, d):
  x = (rng.standard_normal((n, d)) * rng.choice([1e-6, 1.0, 3e4], (n, 1))).astype(np.float32)
  sp = np.array([65504, 65519.99, 65520, -7e4, 2.0 ** -25, 3 * 2.0 ** -26, -0.0, 1e-42, np.inf, np.nan], np.float32)
  at = rng.random((n, d)) < 0.05
  x[at] = sp[rng.integers(0, sp.size, int(at.sum()))]
  return x


def _case(seed, S, with_specials=True):
  rng = np.random.default_rng(seed)
  dims = {"a": 1, "b": 3, "c": 16, "d": 5}
  names = sorted(dims)
  ids = {}
  for k in names:
    n = int(rng.integers(0, 400))
    v = rng.zipf(1.3, n).astype(np.int64) % 60 - 30
    if with_specials and n:
      v[rng.integers(0, n, 3)] = np.array([-1, I64_MIN, I64_MIN + 1], np.int64)
    ids[k] = v
  if seed % 3 == 0:
    ids["b"] = ids["b"][:0]
  store = [{k: {} for k in names} for _ in range(S)]
  for s in range(S):
    for k in names:
      keys = np.unique(ids[k])
      keys = keys[(np.mod(keys, S) == s) & (rng.random(keys.size) < 0.8)]  # the rest miss
      for key, row in zip(keys.tolist(), _rows(rng, keys.size, dims[k])):
        store[s][k][key] = row
  grads = {k: _rows(rng, ids[k].size, dims[k]) for k in names}
  return dims, names, ids, store, grads


@pytest.mark.parametrize("S", [1, 2, 3, 5])
@pytest.mark.parametrize("seed", range(4))
def test_per_slot_path_equals_raw_path_then_round(S, seed):
  dims, names, ids, store, grads = _case(seed * 10 + S, S)
  dl = [dims[k] for k in names]

  def server_lookup(s, slot, keys):
    z = np.zeros(dims[slot], np.float32)
    return np.array([store[s][slot].get(int(i), z) for i in keys], np.float32).reshape(-1, dims[slot])

  # the raw path: one unique over all tables, one split, each server's packed rows, one fill; then the rounding
  split = np.cumsum([0] + [ids[k].size for k in names])
  keys = np.concatenate([ids[k] for k in names])
  uk, uks, vo, vos, n = om.unique_key_with_value_and_offset(keys, split, dl)
  splits, pos = om.ragged_split_by_indices(np.mod(uk, S), uk, uks, S)
  buf = np.full(n, np.nan, np.float32)
  for s in range(S):
    v, rs = splits[s]
    rows = np.concatenate([server_lookup(s, k, v[rs[j]:rs[j + 1]]).reshape(-1) for j, k in enumerate(names)])
    om.fill_with_offset_map(pos[s], rs, fm.f16_round(rows), vo, vos, dl, buf)
  per_slot = fm.lookup(server_lookup, S, ids)
  off = 0
  for j, k in enumerate(names):
    c = ids[k].size * dims[k]
    _same(per_slot[k].reshape(-1), buf[off:off + c])
    off += c
  # gradients: the raw path's sums rounded once, per server and table
  flat = np.concatenate([grads[k].reshape(-1) for k in names])
  want = fm.apply_gradients(S, {k: (ids[k], grads[k]) for k in names})
  for s in range(S):
    v, rs = splits[s]
    g = fm.f16_round(om.fill_with_offset_map_gradient(pos[s], rs, flat, vo, vos, dl))
    at = 0
    for j, k in enumerate(names):
      got_ids, got_g = want[s][k]
      assert got_ids.tolist() == v[rs[j]:rs[j + 1]].tolist()
      c = (rs[j + 1] - rs[j]) * dims[k]
      _same(got_g.reshape(-1), g[at:at + c])
      at += c
