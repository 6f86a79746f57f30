"""The fused layout op (fused_embedding_to_layout[_grad]: layout_fwd_kernel / layout_bwd_kernel) and the float-atomic
row scatter (gather_pool_grad: gather_pool_grad_kernel) against the CPU oracle, bit for bit, on every layout, pooling and
lane-group width; and the chain sharding_sparse_fids -> lookup of every (table, shard) list -> layout -> grad -> apply.

Conventions (those of test_gpu_forward_paths.py):
  * results are compared through uint32 views; NaN by class only in pooled (summed or divided) outputs, where the GPU's
    arithmetic returns its canonical NaN.  FIRSTN outputs only copy rows and keep every bit;
  * every call launches exactly one kernel (mono_kernel_launch_count); the profiler, when it recorded anything (records
    are lost whole at times, NOTES.md), must name exactly the instantiation the call is aimed at;
  * every call runs twice with identical bits, except the backward on random inputs, whose float atomics sum in an
    arbitrary order.
The backward sums with float atomics, so its exact comparisons use exact-sum inputs: terms k * 2^-6 with |k| <= 64,
MEAN rows of 1, 2, 4 or 8 FIDs and at most 2^15 terms per element, so every partial sum is exact in fp32 whatever the
order (tests/test_layout_paths_cpu.py pins the generator).  Random normal inputs are checked against an fp64 sum within
the order-free bound |got - exact| <= gamma(n - 1) * sum |t_i|.

The forward is called through the C ABI with sentinel-filled outputs: it writes exactly the elements its tasks cover
(include/mono_emb.h), so every element outside them must keep the sentinel's bits.  The last test requires the file to
have run all twelve instantiations.  The G rules are pinned against layout.cu in tests/test_layout_paths_cpu.py.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import orc
from tests.helpers import table
from tests.test_gpu_forward_paths import NAN_SENTINEL, T, assert_bits, assert_pooled, sweep_items, traced

pytestmark = pytest.mark.gpu

FAMILY = ("layout_fwd_kernel", "layout_bwd_kernel", "gather_pool_grad_kernel")
GS = (4, 8, 16, 32)
SEEN = set()
SUM, MEAN, FIRSTN = 0, 1, 2
U = 2.0 ** -24


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def layout_g(tasks):
  """layout.cu launch_layout: G = 4; while (G < max_dim && G < 32) G <<= 1."""
  g, m = 4, max(t.dim for t in tasks)
  while g < m and g < 32:
    g <<= 1
  return g


def scatter_g(dim):
  """layout.cu launch_gather_pool_grad: the smallest power of two >= dim, clamped to [4, 32]."""
  g = 4
  while g < dim and g < 32:
    g <<= 1
  return g


def one_launch(fn, expect, stable=True):
  """fn() -> list of numpy arrays, from exactly one kernel launch; the profiler's name, when it recorded one, is
  `expect`.  stable: a second run gives identical bits."""
  from monolith_b200 import _lib
  lib = _lib.load()
  for _ in range(10):
    n0 = lib.mono_kernel_launch_count()
    out, names = traced(fn, FAMILY)
    assert lib.mono_kernel_launch_count() - n0 == 1
    assert names <= {expect}, f"ran {sorted(names)}, aimed at {expect}"
    if names:
      SEEN.update(names)
      break
  if stable:
    for a, b in zip(out, fn()):
      np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32), err_msg="not bit-stable run to run")
  return out


def exact_terms(rng, shape):
  """k * 2^-6, |k| <= 64: sums of up to 2^15 such terms (each divided by 1, 2, 4 or 8) are exact in any order."""
  return (rng.integers(-64, 65, shape) * 2.0 ** -6).astype(np.float32)


def special_rows(rng, n):
  """Values with -0.0 rows, +-inf, subnormals, NaN with a payload and pairs whose sum overflows."""
  x = rng.standard_normal(n).astype(np.float32)
  pick = rng.integers(0, 40, n)
  x[pick == 0] = -0.0
  x[pick == 1] = np.inf
  x[pick == 2] = -np.inf
  x[pick == 3] = np.float32(1e-41) * rng.choice([-1, 1], int((pick == 3).sum()))
  x[pick == 4] = NAN_SENTINEL
  x[pick == 5] = np.float32(3e38)
  x[pick == 6] = np.float32(-3e38)
  return x


# ------------------------------------------------------------------------------------------------
# problems in the v3+ encoding: lists, features, tasks
# ------------------------------------------------------------------------------------------------
class Problem:
  """tables: [(row width W, lists)]; every list of a table holds n_rows rows of W floats padded to P >= W, read at
  stride 1 (fid_offset low word = float offset r * P) or at stride P (low word = row index r), alternating.
  feats: [(table, shared, per-row FID counts)]: one row if shared, B rows otherwise, none for a feature without rows.
  hot: a feature index whose FIDs all land on one row of its table's first list."""

  def __init__(self, rng, B, tables, feats, n_rows=48, values=None, hot=None):
    self.B = B
    self.lists = []                      # (table, W, P, stride)
    for ti, (W, nl) in enumerate(tables):
      for j in range(nl):
        P = W + (j % 3)
        self.lists.append((ti, W, P, P if (len(self.lists) % 2) else 1))
    self.n_rows = n_rows
    self.embs = []
    for (ti, W, P, st) in self.lists:
      e = np.full((n_rows, P), NAN_SENTINEL, np.float32)   # padding is never read
      e[:, :W] = (values or (lambda n: rng.standard_normal(n).astype(np.float32)))(n_rows * W).reshape(n_rows, W)
      self.embs.append(e.reshape(-1))
    self.strides = [st for (_, _, _, st) in self.lists]
    fo, fe, nfl = [], [], []
    self.rows_of = []                    # per feature: list of (per row) lists of (list, row)
    for fi, (ti, shared, lens) in enumerate(feats):
      nfl.append(len(fe) | ((1 << 31) if shared else 0))
      mine = [li for li, l in enumerate(self.lists) if l[0] == ti]
      rows = []
      for n in lens:
        fe.append(len(fo))
        r = []
        for _ in range(int(n)):
          li = mine[0] if fi == hot else int(rng.choice(mine))
          row = 3 if fi == hot else int(rng.integers(0, n_rows))
          P, st = self.lists[li][2], self.lists[li][3]
          fo.append((li << 32) | (row if st > 1 else row * P))
          r.append((li, row))
        rows.append(r)
      self.rows_of.append(rows)
    nfl.append(len(fe) + 1)
    fe.append(len(fo))
    self.fo = np.array(fo, np.uint64)
    self.fe = np.array(fe, np.int32)
    self.nfl = np.array(nfl, np.uint32)
    self.feats = feats

  def sizes(self):
    return [e.size for e in self.embs]

  def elem(self, li, row):
    """float offset of row `row` of list li"""
    return row * self.lists[li][2]


def chunk_slices(rng, W, d):
  return int(rng.integers(0, W - d + 1))


def build_tasks(rng, prob, dims, L, sum_feats, mean_feats, seq_feats, shared_feats):
  """Every layout as tasks over slice dims `dims`; returns (tasks, out shapes as [B, row stride]).  ADDN members
  and the other layouts' tasks are interleaved in the task list."""
  from monolith_b200.distribution_ops import SliceTask
  W = {fi: [l[1] for l in prob.lists if l[0] == prob.feats[fi][0]][0] for fi in range(len(prob.feats))}
  tasks, shapes = [], []
  pool = sum_feats + mean_feats

  def sl(fi, d):
    return chunk_slices(rng, W[fi], d)

  def pooling(fi):
    return MEAN if fi in mean_feats or fi == shared_feats[-1] else SUM

  # CONCAT with gaps: one slice per dim, 1-2 unwritten floats between slices and 3 after
  ot, col = len(shapes), 1
  for i, d in enumerate(dims):
    fi = pool[i % len(pool)]
    tasks.append(SliceTask(fi, sl(fi, d), d, pooling(fi), 0, ot, -1, col, 0))
    col += d + 1 + (i % 2)
  for t in tasks:
    t.out_row_stride = col + 3
  shapes.append(col + 3)
  # STACK [B, 3, d] over the largest dim (shared members included)
  d = max(dims)
  ot = len(shapes)
  for s, fi in enumerate([pool[0], shared_feats[0], pool[-1]]):
    tasks.append(SliceTask(fi, sl(fi, d), d, pooling(fi), 0, ot, 3 * d, s * d, 0))
  shapes.append(3 * d)
  # STACK FIRSTN [B, 2, L, d]: a per-sample sequence and a shared one
  ot = len(shapes)
  for s, fi in enumerate([seq_feats[0], shared_feats[-1]]):
    tasks.append(SliceTask(fi, sl(fi, d), d, FIRSTN, L, ot, 2 * L * d, s * L * d, 0))
  shapes.append(2 * L * d)
  # ADDN chains of 2..5 members per dim: MEAN members and a shared member (its via_tmp branch)
  for i, d in enumerate(dims):
    ot = len(shapes)
    members = [pool[(i + j) % len(pool)] for j in range(2 + i % 4)]
    members[1] = shared_feats[i % len(shared_feats)]
    for fi in members:
      tasks.append(SliceTask(fi, sl(fi, d), d, pooling(fi), 0, ot, d, 0, 1))
    shapes.append(d)
  # NONE: a pooled slice and a FIRSTN [B, L, d]
  d = min(dims)
  ot = len(shapes)
  tasks.append(SliceTask(mean_feats[0], sl(mean_feats[0], d), d, MEAN, 0, ot, d, 0, 0))
  shapes.append(d)
  ot = len(shapes)
  tasks.append(SliceTask(seq_feats[-1], sl(seq_feats[-1], d), d, FIRSTN, L, ot, L * d, 0, 0))
  shapes.append(L * d)
  order = rng.permutation(len(tasks))
  return [tasks[i] for i in order], [(prob.B, s) for s in shapes]


def standard_problem(rng, B, dims, L, n_tables=3, n_shards=5, values=None, exact=False, hot=False):
  """3 tables x 5 shards (15 lists) and nine features: SUM, MEAN (rows of 1, 2, 4 or 8 FIDs when `exact`), two
  FIRSTN sequences (rows empty, shorter than L, L, up to 2L), two shared features (SUM / MEAN), a feature without rows,
  rows without FIDs."""
  W = max(dims) + 3
  tables = [(W, n_shards)] * n_tables
  mean_lens = lambda n: rng.choice([1, 2, 4, 8] if exact else [0, 1, 2, 3, 5], n)
  seq = np.concatenate([[0, L - 1, L, 2 * L], rng.integers(0, 2 * L + 1, max(B - 4, 0))])[:B]
  feats = [
      (0, False, rng.integers(0, 5, B)),                    # 0 SUM, rows without FIDs
      (1, False, mean_lens(B)),                             # 1 MEAN
      (2, False, rng.permutation(seq)),                     # 2 FIRSTN
      (0, True, [int(rng.integers(1, 6))]),                 # 3 shared SUM / FIRSTN
      (1, True, mean_lens(1)),                              # 4 shared MEAN
      (2, False, []),                                       # 5 no rows at all
      (1, False, rng.integers(0, 4, B) if not hot else np.full(B, 16)),   # 6 SUM (hot: one FID, 16 per row)
      (2, False, mean_lens(B)),                             # 7 MEAN
      (0, False, seq),                                      # 8 FIRSTN
  ]
  prob = Problem(rng, B, tables, feats, values=values, hot=6 if hot else None)
  tasks, shapes = build_tasks(rng, prob, dims, L, [0, 5, 6], [1, 7], [2, 8], [3, 4])
  return prob, tasks, shapes


# ------------------------------------------------------------------------------------------------
# calls
# ------------------------------------------------------------------------------------------------
def c_tasks(tasks):
  from monolith_b200 import distribution_ops as dops
  return dops._tasks_arr(tasks)


def raw_layout(dev, prob, tasks, bufs, outs, backward):
  """The C ABI call on caller-filled buffers (the Python wrapper zero-fills them)."""
  from monolith_b200 import _lib
  lib = _lib.load()
  P = lambda t: C.c_void_p(t.data_ptr())
  bp = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=dev)
  op = torch.tensor([o.data_ptr() for o in outs], dtype=torch.int64, device=dev)
  st = T(np.array(prob.strides, np.int32), dev)
  fo, fe, nf = T(prob.fo.view(np.int64), dev), T(prob.fe, dev), T(prob.nfl.view(np.int32), dev)
  stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
  fn = lib.mono_embedding_to_layout_grad if backward else lib.mono_embedding_to_layout
  _lib.check(fn(dev.index, P(bp), P(st), len(bufs), P(fo), fo.numel(), P(fe), fe.numel(), P(nf), nf.numel(), prob.B,
                c_tasks(tasks), len(tasks), P(op), stream))


def covered(tasks, shapes):
  """Masks of the output elements the tasks cover."""
  masks = [np.zeros(s, bool) for s in shapes]
  for t in tasks:
    w = t.dim * (t.max_seq_len if t.pooling == FIRSTN else 1)
    masks[t.out_tensor][:, t.out_col:t.out_col + w] = True
  return masks


def check_forward(dev, prob, tasks, shapes):
  want = orc.embedding_to_layout(prob.embs, prob.strides, prob.fo, prob.fe, prob.nfl, prob.B, tasks, shapes)
  embs = [T(e, dev) for e in prob.embs]

  def f():
    outs = [torch.full(s, float(NAN_SENTINEL), device=dev) for s in shapes]
    raw_layout(dev, prob, tasks, embs, outs, backward=False)
    return [o.cpu().numpy() for o in outs]
  got = one_launch(f, f"layout_fwd_kernel<{layout_g(tasks)}>")
  seq = {t.out_tensor for t in tasks if t.pooling == FIRSTN}
  for i, (g, w, m) in enumerate(zip(got, want, covered(tasks, shapes))):
    (assert_bits if i in seq else assert_pooled)(g[m], w[m])
    assert_bits(g[~m], np.full((~m).sum(), NAN_SENTINEL, np.float32))
  return got


def layout_grad(dev, prob, tasks, ograds, fill=0.0, stable=True):
  og = [T(g, dev) for g in ograds]

  def f():
    bufs = [torch.full((n,), fill, device=dev) for n in prob.sizes()]
    raw_layout(dev, prob, tasks, bufs, og, backward=True)
    return [b.cpu().numpy() for b in bufs]
  return one_launch(f, f"layout_bwd_kernel<{layout_g(tasks)}>", stable)


def terms_model(prob, tasks, ograds):
  """ScatterGrad as fp64 sums of the fp32 terms: -> per buffer (sum, sum of |t|, number of terms)."""
  out = [(np.zeros(n), np.zeros(n), np.zeros(n, np.int64)) for n in prob.sizes()]
  for t in tasks:
    rows = prob.rows_of[t.nfl_idx]
    if not rows:
      continue
    shared = prob.feats[t.nfl_idx][1]
    g = ograds[t.out_tensor].reshape(prob.B, -1)
    for b in range(prob.B):
      occ = rows[0 if shared else b]
      for f, (li, row) in enumerate(occ):
        if t.pooling == FIRSTN and f >= t.max_seq_len:
          break
        gc = t.out_col + (f * t.dim if t.pooling == FIRSTN else 0)
        x = g[b, gc:gc + t.dim]
        if t.pooling == MEAN:
          x = (x / np.float32(len(occ))).astype(np.float32)
        e = prob.elem(li, row) + t.slice_start
        s, a, n = out[li]
        s[e:e + t.dim] += x
        a[e:e + t.dim] += np.abs(x.astype(np.float64))
        n[e:e + t.dim] += 1
  return out


def within_bound(got, model):
  s, a, n = model
  gamma = np.where(n > 1, (n - 1) * U / (1 - (n - 1) * U), 0.0)
  err = np.abs(got.astype(np.float64) - s)
  bad = err > gamma * a
  assert not bad.any(), f"{bad.sum()} elements beyond the order-free bound, first at {np.flatnonzero(bad)[:5]}"


# ------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------
DIM_SETS = [(1, 3, 4), (1, 5, 8), (3, 9, 16), (1, 17, 32, 4), (33, 64, 5), (100, 257, 1)]


@pytest.mark.parametrize("B", [1, 37, 256])
@pytest.mark.parametrize("dims", DIM_SETS, ids=lambda d: "-".join(map(str, d)))
def test_forward_every_layout(dims, B, dev):
  rng = np.random.default_rng(B * 1000 + sum(dims))
  prob, tasks, shapes = standard_problem(rng, B, dims, L=3 if max(dims) < 64 else 2)
  check_forward(dev, prob, tasks, shapes)


@pytest.mark.parametrize("dims", [(1, 3, 4), (3, 9, 16), (33, 64, 5)], ids=lambda d: "-".join(map(str, d)))
def test_forward_special_values(dims, dev):
  rng = np.random.default_rng(7 + sum(dims))
  prob, tasks, shapes = standard_problem(rng, 37, dims, L=3, values=lambda n: special_rows(rng, n))
  check_forward(dev, prob, tasks, shapes)


def test_forward_one_fid_rows_keep_nan_payloads(dev):
  """SUM over one FID copies the row: every bit, NaN payloads included."""
  from monolith_b200.distribution_ops import SliceTask
  rng = np.random.default_rng(5)
  B = 64
  prob = Problem(rng, B, [(8, 2)], [(0, False, np.ones(B, int))], values=lambda n: special_rows(rng, n))
  tasks = [SliceTask(0, 1, 7, SUM, 0, 0, 7, 0, 0)]
  got = check_forward(dev, prob, tasks, [(B, 7)])
  want = orc.embedding_to_layout(prob.embs, prob.strides, prob.fo, prob.fe, prob.nfl, B, tasks, [(B, 7)])
  assert np.isnan(want[0]).any()
  assert_bits(got[0], want[0])


def test_forward_more_chains_than_one_sweep(dev):
  """chains x B beyond one grid-stride sweep of G-lane groups: every unit is still written once."""
  rng = np.random.default_rng(9)
  dims = (1, 17, 32, 4)
  B = sweep_items(32) // 12 + 5
  prob, tasks, shapes = standard_problem(rng, B, dims, L=2, n_tables=3, n_shards=2)
  chains = len({(t.out_tensor, t.out_col) if t.accumulate else id(t) for t in tasks})
  assert chains * B > sweep_items(layout_g(tasks))
  check_forward(dev, prob, tasks, shapes)


# ------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 37, 256])
@pytest.mark.parametrize("dims", DIM_SETS, ids=lambda d: "-".join(map(str, d)))
def test_backward_exact_sums(dims, B, dev):
  rng = np.random.default_rng(B * 7 + sum(dims))
  prob, tasks, shapes = standard_problem(rng, B, dims, L=3, exact=True, hot=B == 256)
  ograds = [exact_terms(rng, s) for s in shapes]
  want = orc.embedding_to_layout_grad(prob.sizes(), prob.strides, prob.fo, prob.fe, prob.nfl, B, tasks, ograds)
  got = layout_grad(dev, prob, tasks, ograds)
  model = terms_model(prob, tasks, ograds)
  assert max(int(n.max()) for _, _, n in model) <= 1 << 15
  if B == 256:
    assert max(int(n.max()) for _, _, n in model) >= 4096      # the hot FID
  for g, w, (s, _, n) in zip(got, want, model):
    assert_bits(g, w)
    np.testing.assert_array_equal(g, s)                         # the fp64 model, exact here
    assert_bits(g[n == 0], np.zeros((n == 0).sum(), np.float32))   # rows nobody refers to: +0.0


@pytest.mark.parametrize("dims", [(1, 5, 8), (1, 17, 32, 4), (100, 257, 1)], ids=lambda d: "-".join(map(str, d)))
def test_backward_random_within_order_free_bound(dims, dev):
  rng = np.random.default_rng(31 + sum(dims))
  prob, tasks, shapes = standard_problem(rng, 64, dims, L=3)
  ograds = [rng.standard_normal(s).astype(np.float32) for s in shapes]
  got = layout_grad(dev, prob, tasks, ograds, stable=False)
  for g, m in zip(got, terms_model(prob, tasks, ograds)):
    within_bound(g, m)


def test_backward_addn_members_and_firstn_tail(dev):
  """Every ADDN member receives the same row gradient; FIRSTN positions >= L add nothing; the call accumulates into
  what the buffers hold (they must arrive zero-filled: here they hold 0.5 and keep it where nothing refers)."""
  from monolith_b200.distribution_ops import SliceTask
  rng = np.random.default_rng(3)
  B, d, L = 40, 6, 2
  prob = Problem(rng, B, [(d, 1), (d, 1), (d, 1)],
                 [(0, False, np.ones(B, int)), (1, False, np.ones(B, int)), (2, False, np.full(B, 2 * L))], n_rows=4096)
  tasks = [SliceTask(0, 0, d, SUM, 0, 0, d, 0, 1), SliceTask(2, 0, d, FIRSTN, L, 1, L * d, 0, 0),
           SliceTask(1, 0, d, SUM, 0, 0, d, 0, 1)]
  og = [exact_terms(rng, (B, d)), exact_terms(rng, (B, L * d))]
  got = layout_grad(dev, prob, tasks, og, fill=0.5)
  want = orc.embedding_to_layout_grad(prob.sizes(), prob.strides, prob.fo, prob.fe, prob.nfl, B, tasks, og)
  for g, w in zip(got, want):
    assert_bits(g, w + np.float32(0.5))
  model = terms_model(prob, tasks, og)
  once = lambda li, row: model[li][2][prob.elem(li, row)] == 1
  n_same = 0
  for b in range(B):
    (l0, r0), = prob.rows_of[0][b]
    (l1, r1), = prob.rows_of[1][b]
    if once(l0, r0) and once(l1, r1):
      np.testing.assert_array_equal(got[l0][prob.elem(l0, r0):][:d], og[0][b] + np.float32(0.5))
      np.testing.assert_array_equal(got[l1][prob.elem(l1, r1):][:d], og[0][b] + np.float32(0.5))
      n_same += 1
  assert n_same > B // 2
  head = {occ for row in prob.rows_of[2] for occ in row[:L]}
  tail = {occ for row in prob.rows_of[2] for occ in row[L:]} - head
  assert len(tail) > B // 2
  for li, row in tail:
    assert_bits(got[li][prob.elem(li, row):][:d], np.full(d, 0.5, np.float32))


# ------------------------------------------------------------------------------------------------
# gather_pool_grad
# ------------------------------------------------------------------------------------------------
SCATTER_DIMS = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 64, 100, 129, 255, 256, 300]


def g_scatter(dev, pg, eo, dim, total, offs, pooling, col, stable=True):
  from monolith_b200 import distribution_ops as dops
  pgd, eod, od = T(pg, dev), T(eo, dev), None if offs is None else T(offs, dev)
  return one_launch(lambda: [dops.gather_pool_grad(pgd, eod, dim, total, od, pooling, grad_col=col).cpu().numpy()],
                    f"gather_pool_grad_kernel<{scatter_g(dim)}>", stable)[0]


@pytest.mark.parametrize("dim", SCATTER_DIMS)
def test_gather_pool_grad_exact_sums(dim, dev):
  """Rows behind a dim-5 table (offsets not multiples of 4), a hot row with thousands of occurrences, gradient rows
  at grad_stride > dim and grad_col > 0, CSR SUM / MEAN (rows of 0, 1, 2, 4 or 8) and one occurrence per row."""
  rng = np.random.default_rng(dim)
  n_u, base = 300, 5 * 7
  total = base + n_u * dim + 3
  n_rows = 2000
  lens = rng.choice([0, 1, 2, 4, 8], n_rows)
  offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  u = rng.integers(0, n_u, int(offs[-1]))
  u[rng.random(u.size) < 0.4] = 17                                # hot row
  eo = (base + u * dim).astype(np.int32)
  col = 3
  pg = exact_terms(rng, (n_rows, col + dim + 2))
  sub = np.ascontiguousarray(pg[:, col:col + dim])
  assert (eo == base + 17 * dim).sum() >= 1000
  for pooling in ("sum", "mean"):
    got = g_scatter(dev, pg, eo, dim, total, offs, pooling, col)
    assert_bits(got, orc.gather_pool_grad(sub, eo, dim, total, offs, pooling))
  eo1 = eo[:n_rows]
  got = g_scatter(dev, pg, eo1, dim, total, None, "sum", col)
  assert_bits(got, orc.gather_pool_grad(sub, eo1, dim, total, None, "sum"))


@pytest.mark.parametrize("dim", [3, 8, 16, 100])
def test_gather_pool_grad_random_within_order_free_bound(dim, dev):
  rng = np.random.default_rng(50 + dim)
  n_rows, n_u = 3000, 200
  lens = rng.integers(0, 6, n_rows)
  offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  u = rng.integers(0, n_u, int(offs[-1]))
  u[rng.random(u.size) < 0.3] = 5
  eo = (u * dim + 1).astype(np.int32)
  total = n_u * dim + 1
  pg = rng.standard_normal((n_rows, dim)).astype(np.float32)
  got = g_scatter(dev, pg, eo, dim, total, offs, "mean", 0, stable=False)
  s, a, n = np.zeros(total), np.zeros(total), np.zeros(total, np.int64)
  for r in range(n_rows):
    k = int(lens[r])
    if k:
      x = (pg[r] / np.float32(k)).astype(np.float32).astype(np.float64)
      for e in eo[offs[r]:offs[r + 1]]:
        s[e:e + dim] += x
        a[e:e + dim] += np.abs(x)
        n[e:e + dim] += 1
  within_bound(got, (s, a, n))


# ------------------------------------------------------------------------------------------------
# the chain: sharding_sparse_fids -> lookup per (table, shard) list -> layout -> grad -> apply
# ------------------------------------------------------------------------------------------------
CHAIN_TABLES = {"ta": 4, "tb": 8, "tc": 24}   # dims pool_backward_parts serves; rows laid out in slices of 1, 3, 4, 16
CHAIN_SLICES = {"ta": [(0, 1), (1, 3)], "tb": [(0, 4), (4, 4)], "tc": [(0, 1), (1, 4), (5, 16), (21, 3)]}
CHAIN_FEATS = {  # name: (table, pooling, shared)
    "fa_sum": ("ta", "sum", False), "fb_mean": ("tb", "mean", False), "fc_sum": ("tc", "sum", False),
    "fc_seq": ("tc", "firstn", False), "fu_shared": ("tb", "sum", True), "fv_shared_mean": ("tc", "mean", True)}
CHAIN_L = 3


def _chain_features(rng, B):
  feats = {}
  for slot, (name, (t, pooling, shared)) in enumerate(sorted(CHAIN_FEATS.items())):
    n_rows = 1 if shared else B
    if pooling == "mean":
      lens = rng.choice([1, 2, 4, 8], n_rows)
    elif pooling == "firstn":
      lens = rng.integers(0, 2 * CHAIN_L + 1, n_rows)
    else:
      lens = rng.integers(0, 5, n_rows)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fids = (np.int64(slot + 1) << 48) | rng.integers(0, 40, int(rs[-1])).astype(np.int64)
    feats[name] = (fids, rs)
  return feats


def _chain_tasks(names, B):
  """CONCAT [B, C] of every pooled feature, each row as its table's slices, and NONE FIRSTN [B, L, 24]."""
  from monolith_b200.distribution_ops import SliceTask
  tasks, col, cols = [], 0, {}
  for name in names:
    t, pooling, _ = CHAIN_FEATS[name]
    if pooling == "firstn":
      continue
    cols[name] = col
    for s0, d in CHAIN_SLICES[t]:
      tasks.append(SliceTask(names.index(name), s0, d, {"sum": SUM, "mean": MEAN}[pooling], 0, 0, -1, col + s0, 0))
    col += CHAIN_TABLES[t]
  for tk in tasks:
    tk.out_row_stride = col
  d = CHAIN_TABLES["tc"]
  tasks.append(SliceTask(names.index("fc_seq"), 0, d, FIRSTN, CHAIN_L, 1, CHAIN_L * d, 0, 0))
  return tasks, [(B, col), (B, CHAIN_L * d)], cols


@pytest.mark.parametrize("N", [1, 2, 5])
def test_chain_sharding_lookup_layout_grad_apply(N, dev):
  from monolith_b200 import MultiHashTable, PoolPart
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(100 + N)
  B = 37
  cfg = lambda: {t: table([(d, "adagrad", {})], [0.25], capacity=4096) for t, d in CHAIN_TABLES.items()}
  gpu, twin, o = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev), orc.OracleMultiHashTable(cfg())
  feats = _chain_features(rng, B)
  # every FID gets a row of its own first (lookups never insert)
  for t, d in CHAIN_TABLES.items():
    ids = np.unique(np.concatenate([f for n, (f, _) in feats.items() if CHAIN_FEATS[n][0] == t]))
    vals = rng.standard_normal((ids.size, d)).astype(np.float32)
    for tb in (gpu, twin):
      tb.assign({t: (T(ids, dev), T(vals, dev))}, req_time=10, ids_unique=True)
    o.assign({t: (ids, vals)}, req_time=10)
  feature_table = {n: v[0] for n, v in CHAIN_FEATS.items()}
  dims_sum = {n: CHAIN_TABLES[v[0]] for n, v in CHAIN_FEATS.items()}
  shared = [n for n, v in CHAIN_FEATS.items() if v[2]]
  r = dops.sharding_sparse_fids({n: (T(f, dev), T(rs, dev)) for n, (f, rs) in feats.items()}, feature_table,
                                dims_sum, N, shared)
  tables, names = r["table_names"], r["feature_names"]
  embs = []
  for k, t in enumerate(tables):
    for n in range(N):
      ids = r["fid_list"][k * N + n]
      embs.append(gpu.lookup({t: ids})[t].reshape(-1) if ids.numel() else torch.zeros(1, device=dev))
  tasks, shapes, cols = _chain_tasks(names, B)
  outs = dops.fused_embedding_to_layout(embs, [1] * len(embs), r["fid_offset"], r["feature_offset"], r["nfl_offset"],
                                        B, tasks, shapes)
  concat, seq = [x.cpu().numpy() for x in outs]
  # forward == the oracle's lookup_pool of each feature read from the raw features, without sharding
  parts = []
  for name in names:
    t, pooling, sh = CHAIN_FEATS[name]
    f, rs = feats[name]
    d = CHAIN_TABLES[t]
    if pooling == "firstn":
      rows = o.lookup({t: f})[t] if f.size else np.zeros((0, d), np.float32)
      want = np.zeros((B, CHAIN_L, d), np.float32)
      for b in range(B):
        m = min(int(rs[b + 1] - rs[b]), CHAIN_L)
        want[b, :m] = rows[rs[b]:rs[b] + m]
      assert_bits(seq, want.reshape(B, -1))
      parts.append(PoolPart(t, T(f, dev), T(rs.astype(np.int32), dev), "firstn", max_seq_len=CHAIN_L))
      continue
    want = o.lookup_pool(t, f, rs.astype(np.int32), pooling)
    if sh:
      want = np.repeat(want, B, axis=0)
    assert_bits(concat[:, cols[name]:cols[name] + d], want)
    ff = np.tile(f, B) if sh else f
    rr = (np.arange(B + 1) * f.size if sh else rs).astype(np.int32)
    parts.append(PoolPart(t, T(ff, dev), T(rr, dev), pooling))
  # == the engine's own lookup_pool_parts over the same features
  got_parts = [x.cpu().numpy() for x in gpu.lookup_pool_parts(parts)]
  for name, part, g in zip(names, parts, got_parts):
    if part.pooling == "firstn":
      assert_bits(seq, g)
    else:
      assert_bits(concat[:, cols[name]:cols[name] + CHAIN_TABLES[part.slot]], g)
  # backward with exact-sum gradients: layout grad, then one apply per table over the table's lists
  og = [exact_terms(rng, s) for s in shapes]
  grads = dops.fused_embedding_to_layout_grad([e.numel() for e in embs], [1] * len(embs), r["fid_offset"],
                                              r["feature_offset"], r["nfl_offset"], B, tasks, [T(g, dev) for g in og])
  np_lists = [x.cpu().numpy() for x in r["fid_list"]]
  want_g = orc.embedding_to_layout_grad([max(x.size * CHAIN_TABLES[tables[i // N]], 1) for i, x in enumerate(np_lists)],
                                        [1] * len(embs), r["fid_offset"].cpu().numpy().view(np.uint64),
                                        r["feature_offset"].cpu().numpy(), r["nfl_offset"].cpu().numpy().view(np.uint32),
                                        B, tasks, og)
  for g, w in zip(grads, want_g):
    assert_bits(g.cpu().numpy(), w)
  for k, t in enumerate(tables):
    d = CHAIN_TABLES[t]
    ids = np.concatenate(np_lists[k * N:(k + 1) * N])
    gk = np.concatenate([want_g[k * N + n][:np_lists[k * N + n].size * d] for n in range(N)]).reshape(-1, d)
    gg = torch.cat([grads[k * N + n][:np_lists[k * N + n].size * d] for n in range(N)]).reshape(-1, d)
    gpu.apply_gradients({t: (T(ids, dev), gg)}, req_time=20, ids_unique=True)
    o.apply_gradients({t: (ids, gk)}, req_time=20)
  # twin: pool_backward_parts over the raw features (a shared feature as B rows of its one FID list)
  bparts = []
  for name, part in zip(names, parts):
    if part.pooling == "firstn":
      bparts.append(PoolPart(part.slot, part.fids, part.row_offsets, "firstn", rows=T(og[1], dev),
                             max_seq_len=CHAIN_L))
    else:
      bparts.append(PoolPart(part.slot, part.fids, part.row_offsets, part.pooling, rows=T(og[0], dev), col=cols[name]))
  twin.pool_backward_parts(bparts, req_time=20)
  for t in tables:
    keys = o.keys(t)
    want = o.lookup_entry(t, keys)
    assert_bits(gpu.lookup_entry(t, T(keys, dev))["raw"].cpu().numpy(), want)
    assert_bits(twin.lookup_entry(t, T(keys, dev))["raw"].cpu().numpy(), want)
    assert gpu.size(t) == twin.size(t) == o.size(t)
  assert r["nfl_offset"].dtype == torch.int32


# ------------------------------------------------------------------------------------------------
def test_every_layout_instantiation_ran():
  want = {f"{k}<{g}>" for k in FAMILY for g in GS}
  assert SEEN == want, f"missing {sorted(want - SEEN)}, unexpected {sorted(SEEN - want)}"
