"""bf16 tower-side tensors in the fused layout op, the gather calls and PartitionedHashTable, bit for bit.

Forward: every bf16 element equals the fp32 call's element .to(torch.bfloat16) (round to nearest even, pinned in
test_bf16_parts_cpu.py), NaN by isnan; elements no task covers keep their bits.  Backward: the fp32 results of the
bf16 call equal the fp32 call on the gradients widened exactly to fp32.  The layout backward and the atomic scatter
sum with float atomics, so their exact comparisons use exact-sum inputs (tests/test_gpu_layout_paths.py's
exact_terms, k * 2^-6 with |k| <= 64, which bf16 holds exactly).

Every call pins its launch count with mono_kernel_launch_count(); the profiler, when it recorded anything (records
are lost whole at times, NOTES.md), must name the instantiation the call is aimed at.  The last test requires the
file to have run all twenty bf16 layout / gather kernels and the bf16 reduce instantiations the scatter picks.

PartitionedHashTable at world 1 runs in the suite's own process (a one-rank NCCL group, destroyed afterwards), not in
a spawned one: a CUDA process spawned from the suite's process made torch.profiler lose every kernel record of later
files' profiled cases (NOTES.md).  World 2 needs a process per GPU and runs only where two GPUs are present.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from tests import orc
from tests.helpers import table
from tests.test_gpu_forward_paths import T, pick_group, traced
from tests.test_gpu_layout_paths import (CHAIN_FEATS, CHAIN_L, CHAIN_TABLES, DIM_SETS, FIRSTN, SCATTER_DIMS, Problem,
                                         _chain_features, _chain_tasks, covered, exact_terms, layout_g, scatter_g,
                                         special_rows, standard_problem, terms_model, within_bound)

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GS = (4, 8, 16, 32)
FAMILY = ("bf16_layout_fwd_kernel", "bf16_layout_bwd_kernel", "bf16_gather_rows_kernel", "bf16_gather_pool_kernel",
          "bf16_gather_pool_grad_kernel", "bf16_seg_reduce_kernel")
SEEN = set()
SENTINEL = 0x7FAB                      # a bf16 NaN with a payload: never the value of a covered element
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def lib():
  from monolith_b200 import _lib
  return _lib.load()


def launches(fn, expect, n=1, stable=True):
  """fn() -> list of tensors, from exactly n kernel launches; the profiler's names of FAMILY, when it recorded any,
  are `expect`.  stable: a second run gives identical bits."""
  expect = {expect} if isinstance(expect, str) else set(expect)
  for _ in range(10):
    torch.cuda.synchronize()
    n0 = lib().mono_kernel_launch_count()
    out, names = traced(fn, FAMILY)
    assert lib().mono_kernel_launch_count() - n0 == n
    assert names <= expect, f"ran {sorted(names)}, aimed at {sorted(expect)}"
    if names:
      assert names == expect
      SEEN.update(names)
      break
  if stable:
    for a, b in zip(out, fn()):
      assert torch.equal(a.view(torch.int16 if a.dtype == BF else torch.int32),
                         b.view(torch.int16 if b.dtype == BF else torch.int32)), "not bit-stable run to run"
  return out


def assert_bf16(got, want):
  """bf16 tensors equal bit for bit, NaN positions by isnan (the payload is not specified)."""
  gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
  assert torch.equal(gn, wn)
  g, w = got.view(torch.int16).clone(), want.view(torch.int16).clone()
  g[gn] = 0
  w[wn] = 0
  mism = (g != w).nonzero()
  assert mism.numel() == 0, f"{mism.shape[0]} elements differ, first at {mism[0].tolist()}"


def assert_f32(got, want):
  assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def bf16_full(shape, dev):
  return torch.full(shape, SENTINEL, dtype=torch.int16, device=dev).view(BF)


# ------------------------------------------------------------------------------------------------
# layout
# ------------------------------------------------------------------------------------------------
def raw_layout(dev, prob, tasks, bufs, outs, backward, bf16):
  from monolith_b200 import _lib
  from monolith_b200 import distribution_ops as dops
  L = lib()
  P = lambda t: C.c_void_p(t.data_ptr())
  bp = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=dev)
  op = torch.tensor([o.data_ptr() for o in outs], dtype=torch.int64, device=dev)
  st = T(np.array(prob.strides, np.int32), dev)
  fo, fe, nf = T(prob.fo.view(np.int64), dev), T(prob.fe, dev), T(prob.nfl.view(np.int32), dev)
  stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
  name = "mono_embedding_to_layout" + ("_grad" if backward else "") + ("_bf16" if bf16 else "")
  _lib.check(getattr(L, name)(dev.index, P(bp), P(st), len(bufs), P(fo), fo.numel(), P(fe), fe.numel(), P(nf),
                              nf.numel(), prob.B, dops._tasks_arr(tasks), len(tasks), P(op), stream))


def check_forward(dev, prob, tasks, shapes):
  embs = [T(e, dev) for e in prob.embs]
  f32 = [torch.zeros(s, device=dev) for s in shapes]
  raw_layout(dev, prob, tasks, embs, f32, False, False)

  def f():
    outs = [bf16_full(s, dev) for s in shapes]
    raw_layout(dev, prob, tasks, embs, outs, False, True)
    return outs
  got = launches(f, f"bf16_layout_fwd_kernel<{layout_g(tasks)}>")
  for g, w, m in zip(got, f32, covered(tasks, shapes)):
    m = torch.from_numpy(m).to(dev)
    assert_bf16(g[m], w[m].to(BF))
    assert (g.view(torch.int16)[~m] == SENTINEL).all()


@pytest.mark.parametrize("B", [1, 37, 256])
@pytest.mark.parametrize("dims", DIM_SETS, ids=lambda d: "-".join(map(str, d)))
def test_layout_forward_every_layout(dims, B, dev):
  rng = np.random.default_rng(B * 1000 + sum(dims) + 1)
  prob, tasks, shapes = standard_problem(rng, B, dims, L=3 if max(dims) < 64 else 2)
  check_forward(dev, prob, tasks, shapes)


@pytest.mark.parametrize("dims", [(1, 3, 4), (3, 9, 16), (33, 64, 5)], ids=lambda d: "-".join(map(str, d)))
def test_layout_forward_special_values(dims, dev):
  rng = np.random.default_rng(8 + sum(dims))
  prob, tasks, shapes = standard_problem(rng, 37, dims, L=3, values=lambda n: special_rows(rng, n))
  check_forward(dev, prob, tasks, shapes)


def layout_grad(dev, prob, tasks, og, bf16, stable=True):
  def f():
    bufs = [torch.zeros(n, device=dev) for n in prob.sizes()]
    raw_layout(dev, prob, tasks, bufs, og, True, bf16)
    return bufs
  if not bf16:
    return f()
  return launches(f, f"bf16_layout_bwd_kernel<{layout_g(tasks)}>", stable=stable)


@pytest.mark.parametrize("B", [1, 37, 256])
@pytest.mark.parametrize("dims", DIM_SETS, ids=lambda d: "-".join(map(str, d)))
def test_layout_backward_exact_sums(dims, B, dev):
  rng = np.random.default_rng(B * 7 + sum(dims) + 1)
  prob, tasks, shapes = standard_problem(rng, B, dims, L=3, exact=True, hot=B == 256)
  og = [exact_terms(rng, s) for s in shapes]
  og_bf = [T(g, dev).to(BF) for g in og]
  assert all(torch.equal(b.float().cpu(), torch.from_numpy(g)) for b, g in zip(og_bf, og))   # exact in bf16
  got = layout_grad(dev, prob, tasks, og_bf, True)
  f32 = layout_grad(dev, prob, tasks, [b.float() for b in og_bf], False)
  want = orc.embedding_to_layout_grad(prob.sizes(), prob.strides, prob.fo, prob.fe, prob.nfl, B, tasks, og)
  for g, f, w in zip(got, f32, want):
    assert_f32(g, f)
    assert_f32(g.cpu(), torch.from_numpy(w))


@pytest.mark.parametrize("dims", [(1, 5, 8), (1, 17, 32, 4), (100, 257, 1)], ids=lambda d: "-".join(map(str, d)))
def test_layout_backward_random_within_order_free_bound(dims, dev):
  rng = np.random.default_rng(32 + sum(dims))
  prob, tasks, shapes = standard_problem(rng, 64, dims, L=3)
  og_bf = [T(rng.standard_normal(s).astype(np.float32), dev).to(BF) for s in shapes]
  got = layout_grad(dev, prob, tasks, og_bf, True, stable=False)
  for g, m in zip(got, terms_model(prob, tasks, [b.float().cpu().numpy() for b in og_bf])):
    within_bound(g.cpu().numpy(), m)


# ------------------------------------------------------------------------------------------------
# gather_pool
# ------------------------------------------------------------------------------------------------
def k_gather(dim, csr, rows_ok):
  g = pick_group(dim)
  if not csr and rows_ok and dim % 4 == 0 and dim <= 4 * g:
    return f"bf16_gather_rows_kernel<{g}>"
  return f"bf16_gather_pool_kernel<{g}>"


@pytest.mark.parametrize("dim", SCATTER_DIMS)
def test_gather_pool_equals_fp32_rounded(dim, dev):
  """A fused buffer behind a dim-5 table (rows at offsets that are not multiples of 4) and an aligned one; one
  occurrence per row and CSR SUM / MEAN rows (0, 1, 2, 3 or 8 occurrences); packed output, and odd column and
  stride; NaN / inf / subnormal values."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(dim + 7)
  n_u, n_rows = 200, 700
  for base in (0, 5 * 9):
    fused = T(np.concatenate([rng.standard_normal(base).astype(np.float32), special_rows(rng, n_u * dim + 3)]), dev)
    lens = rng.choice([0, 1, 2, 3, 8], n_rows)
    offs = T(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32), dev)
    eo = T((base + rng.integers(0, n_u, int(lens.sum())) * dim).astype(np.int32), dev)
    eo1 = eo[:n_rows]
    for ro, pooling, e in ((None, "sum", eo1), (offs, "sum", eo), (offs, "mean", eo)):
      for col, stride in ((0, dim), (3, dim + 6 + (dim % 2 == 0))):
        want = torch.zeros(n_rows, stride, device=dev)
        dops.gather_pool(fused, e, dim, ro, pooling, out=want, out_col=col)
        aligned = col % 4 == 0 and stride % 4 == 0    # the row copy loads rows at any float offset

        def f():
          out = bf16_full((n_rows, stride), dev)
          dops.gather_pool(fused, e, dim, ro, pooling, out=out, out_col=col)
          return [out]
        got, = launches(f, k_gather(dim, ro is not None, aligned))
        assert_bf16(got[:, col:col + dim], want[:, col:col + dim].to(BF))
        assert (got.view(torch.int16)[:, :col] == SENTINEL).all()
        assert (got.view(torch.int16)[:, col + dim:] == SENTINEL).all()
  # dtype= allocates bf16 rows when no out is given
  got = dops.gather_pool(fused, eo1, dim, dtype=BF)
  assert got.dtype == BF and got.shape == (n_rows, dim)


# ------------------------------------------------------------------------------------------------
# gather_pool_grad (float atomics) and scatter_grad_rows (sort-based)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", SCATTER_DIMS)
def test_gather_pool_grad_equals_fp32_on_widened(dim, dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(dim + 11)
  n_u, base, n_rows = 300, 5 * 7, 2000
  total = base + n_u * dim + 3
  lens = rng.choice([0, 1, 2, 4, 8], n_rows)
  offs = T(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32), dev)
  u = rng.integers(0, n_u, int(lens.sum()))
  u[rng.random(u.size) < 0.4] = 17
  eo = T((base + u * dim).astype(np.int32), dev)
  col = 3
  pg = T(exact_terms(rng, (n_rows, col + dim + 2)), dev).to(BF)
  for ro, pooling, e in ((offs, "sum", eo), (offs, "mean", eo), (None, "sum", eo[:n_rows])):
    want = dops.gather_pool_grad(pg.float(), e, dim, total, ro, pooling, grad_col=col)
    got, = launches(lambda: [dops.gather_pool_grad(pg, e, dim, total, ro, pooling, grad_col=col)],
                    f"bf16_gather_pool_grad_kernel<{scatter_g(dim)}>")
    assert got.dtype == torch.float32
    assert_f32(got, want)


def scatter_case(rng, dim, n_rows, lens_choice, hot_share):
  lens = rng.choice(lens_choice, n_rows)
  offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  M = int(offs[-1])
  n_u = max(M // 3, 8)
  u = rng.integers(0, n_u, M)
  u[rng.random(M) < hot_share] = 5
  return offs, (u * dim).astype(np.int32), n_u * dim


@pytest.mark.parametrize("dim", [4, 8, 12, 16, 32, 64, 100, 128])
def test_scatter_grad_rows_equals_fp32_on_widened(dim, dev):
  """Run lengths 1..129 (short runs, a block boundary, the tree), SUM and MEAN, one occurrence per row, and
  M > 16 384 occurrences with a hot row (tree depth 1).  Random bf16 gradients: the sums are not exact, so this pins
  the association too."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(dim + 13)
  G = pick_group(dim)
  cases = []
  for L in (1, 2, 8, 9, 31, 32, 33, 64, 65, 129):   # one destination row per run length
    n_rows = 4 * L
    offs = np.arange(0, n_rows + 1, dtype=np.int32)
    eo = np.repeat(np.arange(4, dtype=np.int32) * dim, L)
    cases.append((offs, rng.permutation(eo), 4 * dim))
  cases.append(scatter_case(rng, dim, 9000, [1, 2, 3], 0.3))           # M > 16384: one tree level, a hot row
  for offs, eo, total in cases:
    n_rows = offs.size - 1
    col = 4
    pg = T(rng.standard_normal((n_rows, col + dim + 4)).astype(np.float32), dev).to(BF)
    od, ed = T(offs, dev), T(eo, dev)
    for ro, pooling in ((od, "sum"), (od, "mean"), (None, "sum")):
      e = ed if ro is not None else ed[:n_rows]
      if ro is None and e.numel() != n_rows:
        continue
      n0 = lib().mono_kernel_launch_count()
      want = dops.scatter_grad_rows(pg.float(), e, dim, torch.full((total,), -1.5, device=dev), ro, pooling,
                                    grad_col=col)
      n_fp32 = lib().mono_kernel_launch_count() - n0
      got, = launches(lambda: [dops.scatter_grad_rows(pg, e, dim, torch.full((total,), -1.5, device=dev), ro,
                                                      pooling, grad_col=col)],
                      f"bf16_seg_reduce_kernel<{G},1,true>", n=n_fp32)
      assert_f32(got, want)


def test_scatter_grad_rows_rejects_unaligned_bf16_rows(dev):
  from monolith_b200 import _lib
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(3)
  eo = T((rng.integers(0, 10, 64) * 8).astype(np.int32), dev)
  pg = T(rng.standard_normal((64, 20)).astype(np.float32), dev).to(BF)
  for kw in ({"dim": 6, "pg": pg[:, :6]}, {"dim": 8, "pg": pg[:, :8], "grad_col": 2},
             {"dim": 8, "pg": pg.reshape(-1)[1:1 + 64 * 8].reshape(64, 8)},     # 2-byte aligned rows
             {"dim": 8, "pg": pg.reshape(-1)[:64 * 18].reshape(64, 18)[:, :8]},  # stride 18
             {"dim": 132, "pg": torch.zeros(64, 132, device=dev, dtype=BF)}):
    buf = torch.full((10 * 132,), 0.25, device=dev)
    n0 = lib().mono_kernel_launch_count()
    with pytest.raises(_lib.MonoError, match="InvalidArgument"):
      dops.scatter_grad_rows(kw["pg"], eo, kw["dim"], buf, grad_col=kw.get("grad_col", 0))
    assert lib().mono_kernel_launch_count() == n0
    assert (buf == 0.25).all()


# ------------------------------------------------------------------------------------------------
# the chain: sharding_sparse_fids -> lookup -> bf16 layout -> bf16 grad -> apply
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2, 5])
def test_chain_in_bf16(N, dev):
  from monolith_b200 import MultiHashTable, PoolPart
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(200 + N)
  B = 37
  cfg = lambda: {t: table([(d, "adagrad", {})], [0.25], capacity=4096) for t, d in CHAIN_TABLES.items()}
  gpu, ref, twin = (MultiHashTable(cfg(), device=dev) for _ in range(3))
  feats = _chain_features(rng, B)
  for t, d in CHAIN_TABLES.items():
    ids = np.unique(np.concatenate([f for n, (f, _) in feats.items() if CHAIN_FEATS[n][0] == t]))
    vals = rng.standard_normal((ids.size, d)).astype(np.float32)
    for tb in (gpu, ref, twin):
      tb.assign({t: (T(ids, dev), T(vals, dev))}, req_time=10, ids_unique=True)
  r = dops.sharding_sparse_fids({n: (T(f, dev), T(rs, dev)) for n, (f, rs) in feats.items()},
                                {n: v[0] for n, v in CHAIN_FEATS.items()},
                                {n: CHAIN_TABLES[v[0]] for n, v in CHAIN_FEATS.items()}, N,
                                [n for n, v in CHAIN_FEATS.items() if v[2]])
  tables, names = r["table_names"], r["feature_names"]
  embs = []
  for k, t in enumerate(tables):
    for n in range(N):
      ids = r["fid_list"][k * N + n]
      embs.append(gpu.lookup({t: ids})[t].reshape(-1) if ids.numel() else torch.zeros(1, device=dev))
  tasks, shapes, cols = _chain_tasks(names, B)
  idx = (r["fid_offset"], r["feature_offset"], r["nfl_offset"])
  f32 = dops.fused_embedding_to_layout(embs, [1] * len(embs), *idx, B, tasks, shapes)
  bf = dops.fused_embedding_to_layout(embs, [1] * len(embs), *idx, B, tasks, shapes, dtype=BF)
  for g, w in zip(bf, f32):
    assert g.dtype == BF
    assert_bf16(g, w.to(BF))
  og = [T(exact_terms(rng, s), dev).to(BF) for s in shapes]
  sizes = [e.numel() for e in embs]
  g_bf = dops.fused_embedding_to_layout_grad(sizes, [1] * len(embs), *idx, B, tasks, og)
  g_32 = dops.fused_embedding_to_layout_grad(sizes, [1] * len(embs), *idx, B, tasks, [g.float() for g in og])
  for a, b in zip(g_bf, g_32):
    assert a.dtype == torch.float32
    assert_f32(a, b)
  np_lists = [x.cpu().numpy() for x in r["fid_list"]]
  for k, t in enumerate(tables):
    d = CHAIN_TABLES[t]
    ids = T(np.concatenate(np_lists[k * N:(k + 1) * N]), dev)
    for tb, gr in ((gpu, g_bf), (ref, g_32)):
      gg = torch.cat([gr[k * N + n][:np_lists[k * N + n].size * d] for n in range(N)]).reshape(-1, d)
      tb.apply_gradients({t: (ids, gg)}, req_time=20, ids_unique=True)
  # twin: the bf16 parts backward over the raw features on the same bf16 rows
  bparts = []
  for name in names:
    t, pooling, sh = CHAIN_FEATS[name]
    f, rs = feats[name]
    if pooling == "firstn":
      bparts.append(PoolPart(t, T(f, dev), T(rs.astype(np.int32), dev), "firstn", rows=og[1], max_seq_len=CHAIN_L))
      continue
    ff = np.tile(f, B) if sh else f
    rr = (np.arange(B + 1) * f.size if sh else rs).astype(np.int32)
    bparts.append(PoolPart(t, T(ff, dev), T(rr, dev), pooling, rows=og[0], col=cols[name]))
  twin.pool_backward_parts(bparts, req_time=20)
  for t in tables:
    ids, raw = next(iter(ref.export(t, chunk=1 << 14)))
    want = ref.lookup_entry(t, ids)["raw"]
    assert_f32(gpu.lookup_entry(t, ids)["raw"], want)
    assert_f32(twin.lookup_entry(t, ids)["raw"], want)


# ------------------------------------------------------------------------------------------------
# PartitionedHashTable: bf16 lookup and apply_gradients in spawned NCCL processes
# ------------------------------------------------------------------------------------------------
TABLE_SETS = {"vec": {"a": 8, "b": 16}, "dim6": {"a": 8, "b": 6}}


def _pht_batch(rank, step, dims):
  rng = np.random.default_rng(100 * step + rank)
  fa = (np.int64(1) << 48) | rng.integers(0, 300, 900).astype(np.int64)
  fa[rng.random(fa.size) < 0.2] = (np.int64(1) << 48) | 7           # a hot FID
  lens = rng.choice([1, 2, 4, 8], 200)
  offs_b = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  fb = (np.int64(2) << 48) | rng.integers(0, 300, int(offs_b[-1])).astype(np.int64)
  ga = exact_terms(rng, (fa.size, dims["a"]))
  gb = exact_terms(rng, (200, dims["b"]))
  if dims["b"] % 4 == 0:           # the sort-based scatter is deterministic: random bf16 gradients
    ga = rng.standard_normal(ga.shape).astype(np.float32)
    gb = rng.standard_normal(gb.shape).astype(np.float32)
  return fa, fb, offs_b, ga, gb


def _pht_run(rank, world, set_name):
  """Three steps of bf16 lookup / apply_gradients against a twin's fp32 ones on the widened gradients (the process
  group of `world` ranks is up)."""
  from monolith_b200 import MultiHashTable
  from monolith_b200.distributed_ps import PartitionedHashTable
  dev = torch.device("cuda", rank)
  dims = TABLE_SETS[set_name]
  cfg = lambda: {t: table([(d, "adagrad", {})], [0.1], capacity=8192) for t, d in dims.items()}
  tb, tw = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
  pb, pw = PartitionedHashTable(tb, world, rank), PartitionedHashTable(tw, world, rank)
  t = lambda x: torch.from_numpy(x).to(dev)
  for step in range(3):
    fa, fb, offs_b, ga, gb = _pht_batch(rank, step, dims)
    kw = dict(row_offsets={"b": t(offs_b)}, pooling={"b": "mean"})
    bf, ctx_b = pb.lookup({"a": t(fa), "b": t(fb)}, dtype=BF, **kw)
    f32, ctx_w = pw.lookup({"a": t(fa), "b": t(fb)}, **kw)
    for n in ("a", "b"):
      assert bf[n].dtype == BF and bf[n].shape == f32[n].shape
      assert_bf16(bf[n], f32[n].to(BF))
    gbf = {"a": t(ga).to(BF), "b": t(gb).to(BF)}
    pb.apply_gradients(ctx_b, gbf, req_time=10 + step)
    pw.apply_gradients(ctx_w, {n: g.float() for n, g in gbf.items()}, req_time=10 + step)
  for n in dims:
    got = [(i.cpu().numpy(), r.cpu().numpy()) for i, r in tb.export(n, chunk=1 << 14)]
    want = [(i.cpu().numpy(), r.cpu().numpy()) for i, r in tw.export(n, chunk=1 << 14)]
    gi, gr = np.concatenate([g[0] for g in got]), np.concatenate([g[1] for g in got])
    wi, wr = np.concatenate([w[0] for w in want]), np.concatenate([w[1] for w in want])
    go, wo = np.argsort(gi), np.argsort(wi)
    np.testing.assert_array_equal(gi[go], wi[wo])
    np.testing.assert_array_equal(gr[go].view(np.uint32), wr[wo].view(np.uint32))
    assert gi.size > 100
  tb.close()
  tw.close()


def _pht_worker(rank, world, port, q, set_name):
  try:
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    _pht_run(rank, world, set_name)
    q.put((rank, "OK", ""))
    dist.barrier()
    dist.destroy_process_group()
  except Exception:
    import traceback
    q.put((rank, "ERROR", traceback.format_exc()))
    raise


@pytest.mark.parametrize("set_name", sorted(TABLE_SETS))
@pytest.mark.parametrize("world", [1, 2])
def test_partitioned_hash_table_bf16(world, set_name, dev):
  """bf16 lookup == fp32 lookup rounded; after bf16 apply_gradients, every exported entry equals a twin's fp32 run on
  the widened gradients.  "vec": every dim a multiple of 4 (the sort-based scatter); "dim6": a dim-6 table, so every
  table takes the float-atomic kernel (exact-sum gradients)."""
  if torch.cuda.device_count() < world:
    pytest.skip(f"needs {world} GPUs")
  import torch.distributed as dist
  if world == 1:   # a one-rank NCCL group in this process (see the module docstring)
    assert not dist.is_initialized()
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1, device_id=dev)
    try:
      _pht_run(0, 1, set_name)
    finally:
      dist.destroy_process_group()
    return
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = 29500 + (os.getpid() % 150) + 2 * world + (set_name == "vec")
  procs = [ctx.Process(target=_pht_worker, args=(r, world, port, q, set_name)) for r in range(world)]
  for p in procs:
    p.start()
  got = [q.get(timeout=300) for _ in range(world)]
  for p in procs:
    p.join(timeout=60)
  for g in got:
    assert g[1] == "OK", g[2]
  for p in procs:
    assert p.exitcode == 0


# ------------------------------------------------------------------------------------------------
def test_every_bf16_instantiation_ran():
  want = {f"{k}<{g}>" for k in FAMILY[:5] for g in GS} | {f"bf16_seg_reduce_kernel<{g},1,true>" for g in GS}
  assert SEEN == want, f"missing {sorted(want - SEEN)}, unexpected {sorted(SEEN - want)}"
