"""Runs of at most 8 occurrences (kApplyRun) are summed inside the fused backward's apply pass (csrc/bwd.cu
runs_apply_kernel); longer runs still come from the reduce kernels.  Every entry must equal the oracle fed the
documented sums (tests/reduce_order.py: a plain occurrence-order sum for runs <= 64, blocks + tree above), bit for
bit, on both sides of each threshold.

The table is SGD (lr 1) with rows initialised to -0.0, so an entry is -0.0 - sum: exact for a nonzero sum, and +0.0
or -0.0 exactly when the sum is -0.0 or +0.0.  Runs whose first term is -0.0, and runs of -0.0 only, therefore show
whether the sum starts from its first term (as the reduce does) or from +0.0.
"""
import zlib

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import table

pytestmark = pytest.mark.gpu

EDGE_LENS = [1, 2, 8, 9, 63, 64, 65, 129]
DIMS = [4, 32, 64, 128]   # G = 4, 8, 16, 32


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _fids(n, slot=5):
  return (np.int64(slot) << 48) | ((np.arange(n, dtype=np.int64) * 2654435761 + 777) & ((1 << 40) - 1))


def _cfg(D):
  from monolith_b200 import entry
  return {"t": table([(D, "sgd", {})], [1.0], capacity=64, init=entry.ConstantsInitializer(-0.0))}


def _run_of(rng, n_fill):
  """Run index of every occurrence: each edge length three times (random terms / -0.0 first term / -0.0 only)
  among short filler runs, occurrences at random positions."""
  lens = np.concatenate([np.repeat(EDGE_LENS, 3), rng.integers(1, 9, n_fill)]).astype(np.int64)
  lens = lens[rng.permutation(lens.size)]
  return lens, rng.permutation(np.repeat(np.arange(lens.size), lens))


def _first_occ(run_of, n_runs):
  first = np.full(n_runs, run_of.size, np.int64)
  np.minimum.at(first, run_of, np.arange(run_of.size))
  return first


def _neg_zero_rows(lens, run_of, row_of_occ):
  """Rows to set to -0.0: the first occurrence's row of the second run of each edge length, every row of the
  third one."""
  first = _first_occ(run_of, lens.size)
  rows = []
  for L in EDGE_LENS:
    runs = np.flatnonzero(lens == L)[:3]
    rows.append(row_of_occ[first[runs[1]]])
    rows.extend(row_of_occ[np.flatnonzero(run_of == runs[2])])
  return np.unique(np.asarray(rows))


def _csr(rng, M):
  rl = rng.integers(1, 5, M)
  rl = rl[np.cumsum(rl) <= M]
  rl = np.concatenate([rl, np.ones(M - int(rl.sum()), rl.dtype)])
  return np.concatenate([[0], np.cumsum(rl)]).astype(np.int32)


def _check(gpu, cfg, keys_of_occ, x, D, dev):
  """gpu entries == the oracle fed ro.call_sums of the per-occurrence rows x, bit for bit."""
  G = ro.pick_group(D)
  k, sums, length = ro.call_sums(x, keys_of_occ, G)
  assert set(EDGE_LENS) <= set(length.tolist())
  neg = np.signbit(sums).all(1) & (sums == 0).all(1)
  assert neg.any(), "no run sums to -0.0: the sign case is not exercised"
  cpu = orc.OracleMultiHashTable(cfg)
  cpu.apply_gradients({"t": (k, sums)}, req_time=9)
  got = gpu.lookup_entry("t", T(k, dev))["raw"].cpu().numpy()
  want = cpu.lookup_entry("t", k)
  bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))
  assert bad.size == 0, (f"{bad.size} entries differ, e.g. a run of {length[bad[0]]}: {got[bad[0]][:4]} vs "
                         f"{want[bad[0]][:4]}")


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("pooling", ["sum", "mean"])
def test_pool_backward_short_runs_bit_exact(pooling, D, dev):
  from monolith_b200 import MultiHashTable
  rng = np.random.default_rng(zlib.crc32(f"{pooling}/{D}".encode()))
  lens, run_of = _run_of(rng, 700)
  M = run_of.size
  u = _fids(lens.size)
  offs = _csr(rng, M) if pooling == "mean" else None
  R = M if offs is None else offs.size - 1
  row_of_occ = np.arange(M) if offs is None else np.repeat(np.arange(R), np.diff(offs))
  pg = rng.standard_normal((R, D)).astype(np.float32)
  pg[_neg_zero_rows(lens, run_of, row_of_occ)] = -0.0
  cfg = _cfg(D)
  gpu = MultiHashTable(cfg, device=dev)
  gpu.pool_backward("t", T(u[run_of], dev), T(pg, dev), None if offs is None else T(offs, dev), pooling, req_time=9)
  _check(gpu, cfg, u[run_of], ro.occurrence_rows(pg, M, offs, pooling), D, dev)


@pytest.mark.parametrize("D", DIMS)
def test_pool_backward_parts_short_runs_bit_exact(D, dev):
  """One table, three parts in one call: SUM rows, CSR MEAN rows and a FIRSTN sequence part (occurrences past
  max_seq_len add the +0.0 row); the FIDs of a run are spread over all three."""
  from monolith_b200 import MultiHashTable, PoolPart
  rng = np.random.default_rng(zlib.crc32(f"parts/{D}".encode()))
  lens, run_of = _run_of(rng, 900)
  M = run_of.size
  u = _fids(lens.size, slot=6)
  m1, m2 = M // 3, 2 * M // 3
  L = 3
  # part 1: one FID per row
  g1 = rng.standard_normal((m1, D)).astype(np.float32)
  # part 2: CSR MEAN
  o2 = _csr(rng, m2 - m1)
  g2 = rng.standard_normal((o2.size - 1, D)).astype(np.float32)
  # part 3: FIRSTN, rows of up to 5 FIDs, L positions of D floats per row
  rl = rng.integers(1, 6, M - m2)
  rl = rl[np.cumsum(rl) <= M - m2]
  rl = np.concatenate([rl, np.ones(M - m2 - int(rl.sum()), rl.dtype)])
  o3 = np.concatenate([[0], np.cumsum(rl)]).astype(np.int32)
  g3 = rng.standard_normal((o3.size - 1, L * D)).astype(np.float32)
  # -0.0 rows: the rows (or sequence positions) that feed the chosen occurrences
  zero_occ = set()
  first = _first_occ(run_of, lens.size)
  for Ln in EDGE_LENS:
    runs = np.flatnonzero(lens == Ln)[:3]
    zero_occ.add(int(first[runs[1]]))
    zero_occ.update(np.flatnonzero(run_of == runs[2]).tolist())
  row2 = np.repeat(np.arange(o2.size - 1), np.diff(o2))
  row3 = np.repeat(np.arange(o3.size - 1), np.diff(o3))
  pos3 = np.arange(M - m2) - o3[row3]
  for m in zero_occ:
    if m < m1:
      g1[m] = -0.0
    elif m < m2:
      g2[row2[m - m1]] = -0.0
    elif pos3[m - m2] < L:
      g3[row3[m - m2], pos3[m - m2] * D:(pos3[m - m2] + 1) * D] = -0.0
  x3 = np.zeros((M - m2, D), np.float32)
  inl = pos3 < L
  x3[inl] = g3.reshape(-1, L, D)[row3[inl], pos3[inl]]
  x = np.concatenate([g1, ro.occurrence_rows(g2, m2 - m1, o2, "mean"), x3])
  f = u[run_of]
  cfg = _cfg(D)
  gpu = MultiHashTable(cfg, device=dev)
  gpu.pool_backward_parts([PoolPart("t", T(f[:m1], dev), rows=T(g1, dev)),
                           PoolPart("t", T(f[m1:m2], dev), T(o2, dev), "mean", rows=T(g2, dev)),
                           PoolPart("t", T(f[m2:], dev), T(o3, dev), "firstn", rows=T(g3, dev), max_seq_len=L)],
                          req_time=9)
  _check(gpu, cfg, f, x, D, dev)
