"""The numpy restatement of the backward's summation order (tests/reduce_order.py) against the CPU oracle, exact
arithmetic, a literal one-run-at-a-time statement of the same rules, its own fp64 error bound, and the constants
of the CUDA sources it restates."""
import os
import re

import numpy as np
import pytest

from tests import orc
from tests import reduce_order as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "monolith_b200", "csrc")


def _literal_run_sum(x, G, np_):
  """The rules of reduce_order's docstring, one run, plain loops (no vectorisation)."""
  x = np.asarray(x, np.float32)
  L = x.shape[0]
  if L <= ro.SHORT_RUN:
    acc = x[0].copy()
    for r in x[1:]:
      acc = acc + r
    return acc
  b = []
  for s0 in range(0, L, ro.PIECE):
    acc = x[s0].copy()
    for r in x[s0 + 1:min(L, s0 + ro.PIECE)]:
      acc = acc + r
    b.append(acc)
  nblk = len(b)
  top, stride = 1, 1
  while np_ > top * ro.FINISH_MAX:
    top *= ro.TREE_FAN
    NG = 32 // G
    PER = ro.TREE_FAN // NG
    for k in range(0, nblk, ro.TREE_FAN * stride):
      if k + stride >= nblk:
        continue
      tot = None
      for g in range(NG):
        if k + g * PER * stride >= nblk:
          continue
        acc = np.zeros_like(b[0])
        for i in range(g * PER, (g + 1) * PER):
          if k + i * stride < nblk:
            acc = acc + b[k + i * stride]
        tot = acc if tot is None else tot + acc
      b[k] = tot
    stride *= ro.TREE_FAN
  acc = b[0].copy()
  for k in range(top, nblk, top):
    acc = acc + b[k]
  return acc


def test_tree_depth_by_call_size():
  assert ro.tree_top(ro.n_pieces(16384)) == (0, 1)
  assert ro.tree_top(ro.n_pieces(16385)) == (1, 128)
  assert ro.tree_top(ro.n_pieces(1 << 21)) == (1, 128)
  assert ro.tree_top(ro.n_pieces((1 << 21) + 1)) == (2, 16384)
  assert [ro.pick_group(d) for d in (4, 8, 12, 16, 20, 32, 36, 64, 100, 128)] == [4, 4, 4, 4, 8, 8, 16, 16, 32, 32]


@pytest.mark.parametrize("pooling", ["sum", "mean"])
@pytest.mark.parametrize("D", [4, 12, 36])
def test_short_runs_equal_the_oracle_scatter_bit_for_bit(D, pooling):
  """Runs of <= 64 occurrences: the model is the CPU reference's sequential ScatterGrad."""
  rng = np.random.default_rng(D)
  U = 400
  lens = rng.integers(1, 65, U)
  lens[:4] = [1, 2, 63, 64]
  u_of = rng.permutation(np.repeat(np.arange(U), lens))
  M = u_of.size
  if pooling == "mean":
    rl = rng.integers(1, 6, M)
    offs = np.concatenate([[0], np.cumsum(rl)])
    offs = offs[offs < M]
    offs = np.concatenate([offs, [M]]).astype(np.int32)
  else:
    offs = None
  R = M if offs is None else offs.size - 1
  pg = rng.standard_normal((R, D)).astype(np.float32)
  want = orc.gather_pool_grad(pg, (u_of * D).astype(np.int32), D, U * D, offs, pooling).reshape(U, D)
  x = ro.occurrence_rows(pg, M, offs, pooling)
  keys, sums, length = ro.call_sums(x, u_of, ro.pick_group(D))
  assert np.array_equal(keys, np.arange(U)) and np.array_equal(length, lens)
  np.testing.assert_array_equal(sums.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("L", [65, 96, 97, 4097, 16384])
def test_no_tree_level_is_a_sequential_sum_of_block_sums(L):
  rng = np.random.default_rng(L)
  x = rng.standard_normal((L, 8)).astype(np.float32)
  blocks = []
  for s in range(0, L, 32):
    acc = x[s].copy()
    for r in x[s + 1:s + 32]:
      acc += r
    blocks.append(acc)
  acc = blocks[0].copy()
  for bs in blocks[1:]:
    acc += bs
  for M in (L, 16384):   # every call size with 0 levels
    np.testing.assert_array_equal(ro.run_sum(x, 8, ro.n_pieces(M)).view(np.uint32), acc.view(np.uint32))


@pytest.mark.parametrize("G", [4, 8, 16, 32])
@pytest.mark.parametrize("L,M", [(65, 65), (4097, 16385), (5000, 1 << 21), (16385, 1 << 21),
                                 (70000, (1 << 21) + 1), (540000, (1 << 21) + 4097)])
def test_vectorised_model_equals_the_literal_rules(L, M, G):
  rng = np.random.default_rng(L + G)
  x = rng.standard_normal((L, 2)).astype(np.float32)
  np_ = ro.n_pieces(M)
  want = _literal_run_sum(x, G, np_)
  np.testing.assert_array_equal(ro.run_sum(x, G, np_).view(np.uint32), want.view(np.uint32))


def test_vectorised_model_over_many_runs_equals_one_run_at_a_time():
  rng = np.random.default_rng(9)
  lens = np.concatenate([rng.integers(1, 70, 300), [129, 4095, 4097, 20000, 17000]])
  keys = rng.permutation(np.repeat(np.arange(lens.size), lens))
  x = rng.standard_normal((keys.size, 3)).astype(np.float32)
  for M, G in ((keys.size, 8), ((1 << 21) + 33, 32)):
    k, sums, _ = ro.call_sums(x, keys, G, M=M)
    for j in range(lens.size):
      want = ro.run_sum(x[keys == k[j]], G, ro.n_pieces(M))
      np.testing.assert_array_equal(sums[j].view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("L", [1, 64, 65, 4097, 60000, 600000])
def test_integer_data_is_summed_exactly(L):
  rng = np.random.default_rng(L)
  x = rng.integers(-3, 4, (L, 4)).astype(np.float32)
  for M in (L, (1 << 21) + 1):
    for G in (4, 32):
      np.testing.assert_array_equal(ro.run_sum(x, G, ro.n_pieces(max(M, L))).astype(np.float64),
                                    x.astype(np.float64).sum(0))


@pytest.mark.parametrize("L", [2, 64, 65, 1000, 16385, 100000, 600000])
def test_random_data_within_the_fp64_bound(L):
  rng = np.random.default_rng(L + 1)
  x = (rng.standard_normal((L, 4)) + 0.5).astype(np.float32)
  exact = x.astype(np.float64).sum(0)
  for M in (L, 1 << 21, (1 << 21) + 1):
    M = max(M, L)
    for G in (4, 8, 16, 32):
      np_ = ro.n_pieces(M)
      err = np.abs(ro.run_sum(x, G, np_).astype(np.float64) - exact)
      bound = ro.error_bound(L, np_, G, np.abs(x.astype(np.float64)).sum(0))
      assert (err <= bound).all(), (M, G, err, bound)


def _src(name):
  with open(os.path.join(CSRC, name)) as f:
    return f.read()


def test_model_constants_match_the_cuda_sources():
  """A retune of the reduction fails here, by name, instead of as a bit mismatch on the GPU."""
  bwd = _src("bwd.cu")
  for name, val in (("kPiece", ro.PIECE), ("kShortRun", ro.SHORT_RUN), ("kTreeFan", ro.TREE_FAN),
                    ("kFinishMax", ro.FINISH_MAX)):
    m = re.search(r"constexpr\s+int\s+%s\s*=\s*(\d+)\s*;" % name, bwd)
    assert m, f"{name} not found in bwd.cu"
    assert int(m.group(1)) == val, f"bwd.cu {name} = {m.group(1)}, tests/reduce_order.py assumes {val}"
  # depth rule of launch_reduce
  assert re.search(r"while\s*\(\(uint64_t\)np\s*>\s*top\s*\*\s*kFinishMax\)\s*\{\s*(?://[^\n]*\s*)?top\s*\*=\s*kTreeFan;", bwd), \
      "launch_reduce's tree-depth rule changed"
  # pick_group
  ops = _src("ops.cu")
  m = re.search(r"int pick_group\(int max_dim\)\s*\{\s*int v = \(max_dim \+ 3\) / 4;\s*int g = 4;\s*"
                r"while \(g < v && g < 32\) g <<= 1;\s*return g;\s*\}", ops)
  assert m, "ops.cu pick_group changed: update reduce_order.pick_group"
  # round-to-nearest adds with no contraction: what np.float32 arithmetic reproduces
  assert "-fmad=false" in _src("build.sh") and "use_fast_math" not in _src("build.sh")
