"""CPU checks of FIRSTN (sequence) parts in lookup_pool_parts / pool_backward_parts: PoolPart's rules, the record's
new field, and the two numpy restatements tests/test_gpu_seq_parts.py compares the device against: the forward's
placement of looked-up rows into [n_rows, L, dim], pinned on the reference's own numpy pooling oracle, and the
per-occurrence gradient terms of ScatterGrad's FIRSTN branch."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from monolith_b200 import PoolPart, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def firstn_place(rows, offs, L):
  """GatherEmb's FIRSTN branch (RT/ops/fused_embedding_to_layout.h:251-256) over looked-up rows: rows[m] is the
  row of occurrence m ([M, dim]), offs the CSR offsets (None: one occurrence per row).  -> [n_rows, L, dim], position
  j of row r = rows[offs[r] + j] for j < min(n_r, L), +0.0 elsewhere."""
  rows = np.asarray(rows, np.float32)
  M, D = rows.shape
  offs = np.arange(M + 1) if offs is None else np.asarray(offs, np.int64)
  out = np.zeros((offs.size - 1, L, D), np.float32)
  for r in range(offs.size - 1):
    n = min(int(offs[r + 1] - offs[r]), L)
    out[r, :n] = rows[offs[r]:offs[r] + n]
  return out


def firstn_terms(grad, offs, L, M):
  """ScatterGrad's FIRSTN branch (fused_embedding_to_layout.h:334-340) as per-occurrence terms: grad is
  [n_rows, L, dim]; occurrence m = offs[r] + j contributes grad[r, j] for j < L and nothing (a +0.0 row: the FID's
  gradient keeps its zero fill) beyond.  -> [M, dim], the terms of the equivalent one-FID-per-row SUM part."""
  grad = np.asarray(grad, np.float32)
  n_rows, _, D = grad.shape
  offs = np.arange(M + 1) if offs is None else np.asarray(offs, np.int64)
  assert offs.size == n_rows + 1 and offs[-1] == M
  terms = np.zeros((M, D), np.float32)
  for r in range(n_rows):
    n = min(int(offs[r + 1] - offs[r]), L)
    terms[offs[r]:offs[r] + n] = grad[r, :n]
  return terms


def test_pool_part_firstn_rules():
  f = torch.zeros(4, dtype=torch.int64)
  PoolPart("t", f, pooling="firstn", max_seq_len=1)
  PoolPart("t", f, pooling="firstn", max_seq_len=100, rows=torch.zeros(4, 800))
  for bad in (0, -3):
    with pytest.raises(ValueError):
      PoolPart("t", f, pooling="firstn", max_seq_len=bad)
  with pytest.raises(ValueError):
    PoolPart("t", f, pooling="firstn")
  for pooling in ("sum", "mean"):
    with pytest.raises(ValueError):
      PoolPart("t", f, pooling=pooling, max_seq_len=5)
  with pytest.raises(ValueError):
    PoolPart("t", f, pooling="firstn", max_seq_len=2.0)
  assert [x.name for x in __import__("dataclasses").fields(PoolPart)][-1] == "max_seq_len"


def test_max_seq_len_sits_in_the_trailing_padding():
  assert _lib.PoolPartC._fields_[-1] == ("max_seq_len", C.c_int32)
  assert _lib.PoolPartC.max_seq_len.offset == 68
  assert C.sizeof(_lib.PoolPartC) == 72
  assert _lib.POOL_FIRSTN == 2


def test_row_shape_rules():
  """_parts_arr's width rule, without a device: a FIRSTN part needs col + L * dim columns."""
  from monolith_b200.multi_hash_table_ops import MultiHashTable
  t = MultiHashTable.__new__(MultiHashTable)
  t._device = torch.device("cpu")
  t._table_names = ["t"]
  t._dims = [4]
  f = torch.arange(6, dtype=torch.int64)
  offs = torch.tensor([0, 2, 6], dtype=torch.int32)
  arr, _, outs = t._parts_arr([PoolPart("t", f, offs, "firstn", torch.zeros(2, 1 + 3 * 4), col=1, max_seq_len=3)],
                              forward=False)
  assert (arr[0].pooling, arr[0].max_seq_len, arr[0].n_rows, arr[0].stride, arr[0].col) == (2, 3, 2, 13, 1)
  with pytest.raises(ValueError):
    t._parts_arr([PoolPart("t", f, offs, "firstn", torch.zeros(2, 3 * 4), col=1, max_seq_len=3)], forward=False)
  with pytest.raises(ValueError):
    t._parts_arr([PoolPart("t", f, offs, "firstn", torch.zeros(1, 3 * 4), max_seq_len=3)], forward=False)
  arr, _, outs = t._parts_arr([PoolPart("t", f, offs, "firstn", max_seq_len=5),
                               PoolPart("t", f, offs, "sum", torch.zeros(2, 4))], forward=True)
  assert tuple(outs[0].shape) == (2, 20) and arr[0].max_seq_len == 5 and arr[1].max_seq_len == 0


def _golden_firstn_cases():
  z = np.load(os.path.join(ROOT, "tests", "golden", "ref_layout_pooling.npz"))
  cases = [i for i in range(int(z["n_cases"])) if int(z[f"c{i}_pooling"]) == 2]
  assert len(cases) == 2
  return [(z[f"c{i}_table"], z[f"c{i}_idx"], z[f"c{i}_offs"], int(z[f"c{i}_max_len"]), z[f"c{i}_expect"])
          for i in cases]


@pytest.mark.parametrize("case", range(2))
def test_placement_equals_the_reference_numpy_oracle(case):
  table, idx, offs, L, expect = _golden_firstn_cases()[case]
  got = firstn_place(table[idx], offs, L)
  np.testing.assert_array_equal(got.view(np.uint32), expect.astype(np.float32).view(np.uint32))
  assert (np.diff(offs) > L).any() and (np.diff(offs) < L).any()  # truncated and zero-padded rows both occur


def test_terms_restate_scatter_grad():
  """The reference's ScatterGrad loop, literally: for each row, seq_idx counts the row's FIDs and only
  seq_idx < L adds grad[r, seq_idx] into the FID's (zero-filled) gradient.  Summing firstn_terms per FID in
  occurrence order gives the same bits for runs this short."""
  rng = np.random.default_rng(3)
  L, D = 4, 8
  lens = rng.integers(0, 9, 60)
  offs = np.concatenate([[0], np.cumsum(lens)])
  M = int(offs[-1])
  fids = rng.integers(0, 40, M)
  grad = rng.standard_normal((lens.size, L, D)).astype(np.float32)
  want = {}
  for r in range(lens.size):
    seq_idx = 0
    for m in range(offs[r], offs[r + 1]):
      acc = want.setdefault(int(fids[m]), np.zeros(D, np.float32))
      if seq_idx < L:
        acc += grad[r, seq_idx]
      seq_idx += 1
  terms = firstn_terms(grad, offs, L, M)
  got = {}
  for m in range(M):
    got.setdefault(int(fids[m]), np.zeros(D, np.float32))
    got[int(fids[m])] += terms[m]
  assert got.keys() == want.keys()
  for k in want:
    np.testing.assert_array_equal(got[k].view(np.uint32), want[k].view(np.uint32))
  beyond = set(int(fids[m]) for r in range(lens.size) for m in range(offs[r] + L, offs[r + 1]))
  within = set(int(fids[m]) for r in range(lens.size) for m in range(offs[r], min(offs[r] + L, offs[r + 1])))
  assert beyond - within  # some FIDs occur only beyond L: they are in the id list with a zero gradient
  for k in beyond - within:
    assert not want[k].any()
