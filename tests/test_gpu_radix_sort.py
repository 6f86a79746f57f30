"""The backward's stable radix sort of (key, position) (csrc/bwd.cu: radix_hist/colscan/scatter_kernel), seen through
mono_scatter_grad_rows: the sort key is the destination row (offset / 4), a row of at most 64 occurrences is the
fp32 sum of its occurrences' gradients in occurrence order, so every row of the result pins which occurrences the
sort grouped under its key and, with order-sensitive gradients, the order it left them in.

The model is numpy's stable argsort of the keys.  Sizes: one item, a scatter tile (8192 items) minus one, a tile,
a tile plus one, and the C2 batch (2 097 152 occurrences); key widths of 1, 2 and 3 digit passes (11 bits each);
every value of every digit; all keys equal.
"""
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TILE = 8192
C2_M = 1 << 21
D = 4
SENTINEL = -1.5


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def _passes(rows):
  bits = 1
  while (1 << bits) < rows + 1:
    bits += 1
  return (bits + 10) // 11


def _model(keys, g, rows):
  """Each row's occurrences in stable key order, summed in that order in fp32 (runs of <= 64)."""
  order = np.argsort(keys, kind="stable")
  sk = keys[order]
  starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
  lens = np.diff(np.r_[starts, sk.size])
  assert lens.max() <= 64
  acc = np.zeros((starts.size, D), np.float32)
  for k in range(int(lens.max())):
    live = lens > k
    acc[live] += g[order[starts[live] + k]]
  out = np.full((rows, D), SENTINEL, np.float32)
  out[sk[starts]] = acc
  return out


def _run(keys, g, rows, dev):
  from monolith_b200 import distribution_ops as dops
  buf = torch.full((rows * D,), SENTINEL, device=dev)
  eo = torch.from_numpy((keys * D).astype(np.int32)).to(dev)
  dops.scatter_grad_rows(torch.from_numpy(g).to(dev), eo, D, buf)
  return buf.cpu().numpy().reshape(rows, D)


def _order_sensitive(rng, M):
  """Magnitudes 2^-10 .. 2^20, mixed signs: a reordered fp32 sum differs in its bits."""
  return (rng.choice([-1.0, 1.0], (M, D)) * np.exp2(rng.integers(-10, 21, (M, D))) *
          rng.uniform(1.0, 2.0, (M, D))).astype(np.float32)


# (M, rows): rows sets the key width; M / rows keeps every run short
CASES = [(1, 100), (TILE - 1, 2000), (TILE, 2000), (TILE + 1, 2000),
         (TILE - 1, 1 << 20), (TILE, 1 << 20), (TILE + 1, 1 << 20), (C2_M, 1 << 20),
         (TILE + 1, (1 << 22) + 5), (C2_M, (1 << 23) + 5)]


@pytest.mark.parametrize("M,rows", CASES, ids=lambda v: str(v))
def test_sort_matches_stable_argsort(M, rows, dev):
  rng = np.random.default_rng(zlib.crc32(f"{M}/{rows}".encode()))
  keys = rng.integers(0, rows, M).astype(np.int64)
  if M > 1:   # the first and last rows are used: the key width is the buffer's
    keys[0], keys[-1] = 0, rows - 1
  g = _order_sensitive(rng, M)
  got = _run(keys, g, rows, dev)
  want = _model(keys, g, rows)
  bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))
  assert bad.size == 0, f"{bad.size} rows differ ({_passes(rows)} passes), e.g. row {bad[0]}: {got[bad[0]]} vs {want[bad[0]]}"


def test_every_digit_value(dev):
  """Keys over 3 digits where each digit takes all 2048 values, the low digit cycling fastest."""
  M, rows = C2_M, 1 << 23
  i = np.arange(M, dtype=np.int64)
  keys = (i * 1031) % 2048 | ((i >> 10) * 523 % 2048) << 11 | (i & 1) << 22
  assert [np.unique((keys >> (11 * p)) & 2047).size for p in range(3)] == [2048, 2048, 2]
  assert _passes(rows) == 3
  rng = np.random.default_rng(7)
  g = _order_sensitive(rng, M)
  got = _run(keys, g, rows, dev)
  want = _model(keys, g, rows)
  assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("M", [TILE - 1, TILE, TILE + 1, 5 * TILE + 3])
def test_all_keys_equal(M, dev):
  """One run of M occurrences: integer gradients make every partial sum exact, so the row is their sum."""
  rng = np.random.default_rng(M)
  g = rng.integers(-3, 4, (M, D)).astype(np.float32)
  keys = np.full(M, 3, np.int64)
  got = _run(keys, g, 4000, dev)
  assert np.array_equal(got[3], g.astype(np.float64).sum(0).astype(np.float32))
  assert (np.delete(got, 3, 0) == SENTINEL).all()
