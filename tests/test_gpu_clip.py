"""Clip by global norm on the device.

mono_global_norm against the numpy restatement of its documented order (tests/global_norm_model.py), bit for bit:
0, 1 and 4096 tensors, chunk-boundary sizes, mixed fp32 / bf16, unaligned starts, special values, a tensor above 2^31
elements; two launches, run-to-run identical bits, no wait on a busy stream.

The scaled backward calls against their unscaled twins on rows pre-multiplied in fp32 with torch / numpy, bit for bit
where the twin is deterministic (pool_backward_parts on every optimizer and lane-group width, SUM / MEAN / FIRSTN, tree
depths 0 and 1; scatter_grad_rows), on exact-sum inputs where it adds with float atomics (embedding_to_layout_grad,
gather_pool_grad).  Every scaled call launches what its twin launches, and the last test checks that every scaled_
instantiation ran.  The chain tests clip the torch way and the fused way and compare the tables.
"""
import copy
import socket
import time
import zlib

import numpy as np
import pytest
import torch

from tests import global_norm_model as gm
from tests.test_gpu_apply_paths import assert_same, table_set
from tests.test_gpu_forward_paths import traced
from tests.test_gpu_layout_paths import exact_terms, layout_g, scatter_g, standard_problem
from tests.test_gpu_parts_apply_paths import capacity, knob_setting, matrix_calls, mixed_calls
from tests.test_parts_apply_paths_cpu import BF16_DIMS, FP32_DIMS, GS, OPTS, call_launches

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FAMILY = ("scaled_seg_reduce_kernel", "scaled_bf16_seg_reduce_kernel", "scaled_runs_apply_kernel",
          "scaled_bf16_runs_apply_kernel", "scaled_gather_pool_grad_kernel", "scaled_bf16_gather_pool_grad_kernel",
          "scaled_layout_bwd_kernel", "scaled_bf16_layout_bwd_kernel")
SEEN = set()
SEG_KNOBS = [{}, {"seg_vpl": 2}, {"seg_ahead": 0}, {"seg_vpl": 2, "seg_ahead": 0}]


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def bits(x):
  return np.asarray(x, np.float32).view(np.uint32)


def launches(fn):
  from monolith_b200 import _lib
  lib = _lib.load()
  torch.cuda.synchronize()
  n0 = lib.mono_kernel_launch_count()
  out = fn()
  torch.cuda.synchronize()
  return out, lib.mono_kernel_launch_count() - n0


def scaled_traced(fn):
  out, seen = traced(fn, FAMILY)
  SEEN.update(seen)
  return out


# ------------------------------------------------------------------------------------------------
# 1. the norm
# ------------------------------------------------------------------------------------------------
def host(t):
  return t.float().cpu().numpy() if t.dtype == BF else t.cpu().numpy()


def check_norm(tensors, clip=1.0):
  from monolith_b200 import clip_ops
  (scale, norm), n = launches(lambda: clip_ops.global_norm_scale(tensors, clip))
  elements = sum(t.numel() for t in tensors)
  assert n == (2 if elements else 1), "kernel launches"
  want = gm.norm([host(t) for t in tensors])
  with np.errstate(all="ignore"):
    want_scale = gm.scale(want, clip)
  got = norm.item()
  if np.isnan(want):
    assert np.isnan(got)
  else:
    assert bits(got) == bits(want), (got, want)
  assert bits(scale.item()) == bits(want_scale), (scale.item(), want_scale)
  again = clip_ops.global_norm(tensors)
  assert bits(again.item()) == bits(got) or (np.isnan(got) and np.isnan(again.item())), "not run-to-run stable"
  return got


def randn(rng, n, dtype, dev, mag=1.0):
  return (torch.from_numpy(rng.standard_normal(n).astype(np.float32) * mag)).to(dev).to(dtype)


def test_no_tensors_and_only_empty_ones(dev):
  assert bits(check_norm([])) == 0
  assert bits(check_norm([torch.zeros(0, device=dev), torch.zeros(0, dtype=BF, device=dev)])) == 0


@pytest.mark.parametrize("n", [0, 1, 8191, 8192, 8193, 3 * 8192 + 17, 1 << 20])
@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_one_tensor_sizes(n, dtype, dev):
  rng = np.random.default_rng(n)
  check_norm([randn(rng, n, dtype, dev, 30.0)], clip=5.0)


def test_4096_mixed_tensors(dev):
  rng = np.random.default_rng(4096)
  ts = []
  for i in range(4096):
    n = int(rng.choice([0, 1, 7, 300, 8192, 8193, 20000]))
    ts.append(randn(rng, n, BF if i % 3 == 0 else torch.float32, dev, float(rng.choice([1e-3, 1.0, 50.0]))))
  check_norm(ts, clip=100.0)


def test_unaligned_starts_and_mixed_dtypes(dev):
  """bf16 slices starting 2, 6 and 10 bytes past a 16-byte boundary, an fp32 slice 4 bytes past one, full chunks."""
  rng = np.random.default_rng(7)
  b = randn(rng, 5 * 8192 + 64, BF, dev)
  f = randn(rng, 3 * 8192 + 64, torch.float32, dev)
  ts = [b[1:1 + 2 * 8192 + 9], f[1:1 + 2 * 8192], b[3:3 + 8192], b[5:5 + 8193], f[:8192], b[:8192]]
  assert ts[0].data_ptr() % 16 == 2 and ts[1].data_ptr() % 16 == 4
  check_norm(ts, clip=10.0)


@pytest.mark.parametrize("case", ["zeros", "subnormal", "near sqrt(FLT_MAX)", "inf", "nan", "tiny clip"])
def test_special_values(case, dev):
  rng = np.random.default_rng(zlib.crc32(case.encode()))
  base = rng.standard_normal(3 * 8192 + 5).astype(np.float32)
  base[::7] = -0.0
  base[1::7] = 0.0
  base[2::11] = np.float32(1e-45)
  base[3::11] = -np.float32(1e-40)
  if case == "zeros":
    base[:] = -0.0
  elif case == "subnormal":
    base[:] = np.float32(1e-45) * rng.integers(1, 1000, base.size)
  elif case == "near sqrt(FLT_MAX)":
    base[::5] = np.float32(1.8e19)
  elif case == "inf":
    base[100] = np.inf
  elif case == "nan":
    base[8192 + 3] = np.nan
  bf = torch.from_numpy(base).to(BF).to(dev)
  got = check_norm([T(base, dev), bf[1:]], clip=1e-30 if case == "tiny clip" else 1000.0)
  if case == "zeros":
    assert bits(got) == 0
  if case == "near sqrt(FLT_MAX)":
    assert np.isinf(got)


def test_a_tensor_above_2_31_elements(dev):
  """One bf16 tensor of 2^31 + 8193 ones after a small fp32 one: every partial is an exact integer, so the sum is
  exact in any order and checks the 64-bit element and chunk indexing."""
  from monolith_b200 import clip_ops
  free, _ = torch.cuda.mem_get_info(dev)
  n = (1 << 31) + 8193
  assert free > 3 * n, "not enough device memory for the 2^31-element case"
  big = torch.ones(n, dtype=BF, device=dev)
  small = torch.tensor([1.0, 2.0, 3.0], device=dev)
  norm = clip_ops.global_norm([small, big]).item()
  assert bits(norm) == bits(np.sqrt(np.float32(float(n + 14)), dtype=np.float32))
  del big
  torch.cuda.empty_cache()


def test_call_on_a_busy_stream_returns_without_waiting(dev):
  from monolith_b200 import clip_ops
  rng = np.random.default_rng(3)
  ts = [randn(rng, 100000, torch.float32, dev)]
  clip_ops.global_norm_scale(ts, 1.0)        # warm: modules loaded
  torch.cuda.synchronize()
  torch.cuda._sleep(int(3e9))                 # about 1.5 s of device time on the current stream
  t0 = time.perf_counter()
  scale, norm = clip_ops.global_norm_scale(ts, 1.0)
  dt = time.perf_counter() - t0
  torch.cuda.synchronize()
  assert dt < 0.5, f"the call waited for the stream ({dt:.3f} s)"
  assert bits(norm.item()) == bits(gm.norm([host(t) for t in ts]))


def test_python_checks(dev):
  from monolith_b200 import clip_ops
  with pytest.raises(ValueError):
    clip_ops.global_norm([torch.zeros(4, 4, device=dev).t()])        # not contiguous
  with pytest.raises(ValueError):
    clip_ops.global_norm([torch.zeros(4, dtype=torch.float16, device=dev)])
  with pytest.raises(ValueError):
    clip_ops.global_norm_scale([torch.zeros(4, device=dev)], float("inf"))
  with pytest.raises(ValueError):
    clip_ops.scale_ptr(torch.ones(2, device=dev), dev)
  with pytest.raises(ValueError):
    clip_ops.scale_ptr(torch.ones(1, dtype=torch.float64, device=dev), dev)
  x = torch.ones(3, device=dev)
  out, norm = clip_ops.clip_by_global_norm([x], 1000.0)
  assert out[0] is not x and torch.equal(out[0], x) and norm.dim() == 0


# ------------------------------------------------------------------------------------------------
# 2. scaled pool_backward_parts: bit for bit the unscaled call on pre-multiplied rows
# ------------------------------------------------------------------------------------------------
def scale_values(calls, dev):
  """1.0, +0.0, a subnormal, clip / norm of the first call's rows, a random float."""
  from monolith_b200 import clip_ops
  g = T(calls[0].grad, dev)
  norm = clip_ops.global_norm([g]).item()
  s, _ = clip_ops.global_norm_scale([g], norm / 3.0)
  return {"one": 1.0, "zero": 0.0, "subnormal": float(np.float32(3e-41)), "clip": s.item(), "random": 0.8437156}


def premultiplied(calls, s):
  """The calls with fp32 rows g * s (bf16 rows widened first): what the scaled call must equal."""
  out = []
  for c in calls:
    d = copy.copy(c)
    d.grad = (np.asarray(c.grad, np.float32) * np.float32(s)).astype(np.float32)
    d.bf16, d.offset8 = False, False
    out.append(d)
  return out


def replay(tabs, calls, dev, scale=None, knobs=None):
  """-> (entries by table, sizes, launches per call)."""
  from monolith_b200 import MultiHashTable
  cfg = {n: v[0] for n, v in tabs.items()}
  names = sorted(tabs)
  every = {n: np.unique(np.concatenate([np.zeros(0, np.int64)] + [p.fids for c in calls for p in c.parts
                                                                   if p.slot == n])) for n in names}

  def run():
    gpu = MultiHashTable(cfg, device=dev)
    lib = gpu._lib
    sc = None if scale is None else torch.tensor([scale], dtype=torch.float32, device=dev)
    n_launch = []
    for c in calls:
      if c.evict:
        for n in names:
          gpu.evict(n, c.ts)
      dp = c.device_parts(dev)
      torch.cuda.synchronize()
      n0 = lib.mono_kernel_launch_count()
      gpu.pool_backward_parts(dp, req_time=c.ts, grad_scale=sc)
      torch.cuda.synchronize()
      n_launch.append(lib.mono_kernel_launch_count() - n0)
    ent = {n: gpu.lookup_entry(n, T(every[n], dev))["raw"].cpu().numpy() for n in names}
    return ent, [gpu.size(n) for n in names], n_launch

  with knob_setting(knobs or {}):
    return scaled_traced(run) if scale is not None else run()


def check_scaled(tabs, calls, dev, s, knobs=None):
  ent, size, n_launch = replay(tabs, calls, dev, scale=s, knobs=knobs)
  want, want_size, want_launch = replay(tabs, premultiplied(calls, s), dev, knobs=knobs)
  assert n_launch == want_launch == [call_launches(list(c.per_table().values())) for c in calls]
  assert size == want_size
  for n in sorted(tabs):
    assert_same(ent[n], want[n], f"table {n}, scale {s!r}")


MATRIX = [("fp32", d) for d in FP32_DIMS] + [("bf16", d) for d in BF16_DIMS]
SCALE_NAMES = ["one", "zero", "subnormal", "clip", "random"]


@pytest.mark.parametrize("dtype,dim", MATRIX, ids=lambda v: str(v))
def test_parts_every_optimizer_and_width(dtype, dim, dev):
  """table_set(dim): the 20 single-optimizer tables and two multi-segment ones, SUM / MEAN / FIRSTN parts, evictions;
  one scale per width, cycling through the five."""
  tabs = capacity(table_set(dim), 8192)
  calls = matrix_calls(zlib.crc32(f"clip/{dtype}/{dim}".encode()), tabs, dtype == "bf16", steps=3)
  name = SCALE_NAMES[MATRIX.index((dtype, dim)) % len(SCALE_NAMES)]
  check_scaled(tabs, calls, dev, scale_values(calls, dev)[name])


@pytest.mark.parametrize("name", SCALE_NAMES)
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_parts_mixed_widths_tree_depth_1(dtype, name, dev):
  tabs, calls = mixed_calls(dtype == "bf16")
  check_scaled(tabs, calls, dev, scale_values(calls, dev)[name])


@pytest.mark.parametrize("knobs", SEG_KNOBS[1:], ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()))
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_parts_reduce_variants(dtype, knobs, dev):
  tabs, calls = mixed_calls(dtype == "bf16")
  check_scaled(tabs, calls, dev, 0.8437156, knobs=knobs)


# ------------------------------------------------------------------------------------------------
# 3. scatter_grad_rows (deterministic) and the atomic calls
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knobs", SEG_KNOBS, ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()) or "default")
@pytest.mark.parametrize("dim", [4, 20, 36, 100])
@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_scatter_grad_rows(dtype, dim, knobs, dev):
  """SUM over one occurrence per row (the PLAIN reduce) and CSR MEAN, a hot row over 64 occurrences, scales 0.75 and
  a random one: bit for bit the unscaled call on the fp32 rows times the scale."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(dim + (dtype == BF))
  n_u, n_rows = 500, 3000
  lens = rng.integers(0, 5, n_rows)
  offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  u = rng.integers(0, n_u, int(offs[-1]))
  u[rng.random(u.size) < 0.1] = 7
  eo = (u * dim).astype(np.int32)
  pg = torch.from_numpy((rng.standard_normal((n_rows, dim)) * 3).astype(np.float32)).to(dtype).to(dev)
  wide = pg.float()
  for s in (0.75, 0.8437156):
    sc = torch.tensor([s], dtype=torch.float32, device=dev)
    for pooling, ro, eoc in (("sum", None, eo[:n_rows]), ("mean", T(offs, dev), eo)):
      e = T(eoc, dev)
      with knob_setting(knobs):
        got, n = launches(lambda: scaled_traced(lambda: dops.scatter_grad_rows(
            pg, e, dim, torch.zeros(n_u * dim, device=dev), ro, pooling, scale=sc)))
        want, n_want = launches(lambda: dops.scatter_grad_rows(wide * sc, e, dim, torch.zeros(n_u * dim, device=dev),
                                                               ro, pooling))
      assert n == n_want
      assert_same(got.cpu().numpy(), want.cpu().numpy(), f"{pooling}, scale {s}")


@pytest.mark.parametrize("dim", [3, 8, 16, 100])
@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_gather_pool_grad_exact_sums(dtype, dim, dev):
  """k * 2^-6 terms (|k| <= 64, rows of 0-8 occurrences) and scales of at most 3 significant bits: every product and
  partial sum is exact, so the float atomics give one answer in any order."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(100 + dim)
  n_u, n_rows = 300, 2000
  offs = np.concatenate([[0], np.cumsum(rng.choice([0, 1, 2, 4, 8], n_rows))]).astype(np.int32)
  eo = T((rng.integers(0, n_u, int(offs[-1])) * dim).astype(np.int32), dev)
  pg = T(exact_terms(rng, (n_rows, dim)), dev).to(dtype)
  for s in (0.75, 0.625, 0.125):
    sc = torch.tensor([s], dtype=torch.float32, device=dev)
    for pooling in ("sum", "mean"):
      got, n = launches(lambda: scaled_traced(lambda: dops.gather_pool_grad(pg, eo, dim, n_u * dim, T(offs, dev),
                                                                            pooling, scale=sc)))
      want = dops.gather_pool_grad(pg.float() * sc, eo, dim, n_u * dim, T(offs, dev), pooling)
      assert n == 1
      assert_same(got.cpu().numpy(), want.cpu().numpy(), f"{pooling}, scale {s}")
  assert scatter_g(dim) in GS


LAYOUT_DIMS = [(1, 3, 4), (5, 8, 2), (9, 16, 1), (17, 100, 5)]


@pytest.mark.parametrize("dims", LAYOUT_DIMS, ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("dtype", [torch.float32, BF])
def test_layout_grad_exact_sums(dtype, dims, dev):
  """The layout problem of the existing layout tests (SUM, MEAN over rows of 1, 2, 4 or 8, FIRSTN, shared features)
  with k * 2^-6 gradients: the scaled call equals the unscaled call on the gradients times the scale."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(sum(dims) + 7 * (dtype == BF))
  prob, tasks, shapes = standard_problem(rng, 37, dims, L=3, exact=True)
  og = [T(exact_terms(rng, s), dev).to(dtype) for s in shapes]
  args = (prob.sizes(), prob.strides, T(prob.fo.view(np.int64), dev), T(prob.fe, dev),
          T(prob.nfl.view(np.int32), dev), prob.B, tasks)
  for s in (0.75, 0.625, 0.125):
    sc = torch.tensor([s], dtype=torch.float32, device=dev)
    got, n = launches(lambda: scaled_traced(lambda: dops.fused_embedding_to_layout_grad(
        *args, og, layout_tensors_grad_scale=sc)))
    want, n_want = launches(lambda: dops.fused_embedding_to_layout_grad(*args, [g.float() * sc for g in og]))
    assert n == n_want == 1
    for a, b in zip(got, want):
      assert_same(a.cpu().numpy(), b.cpu().numpy(), f"scale {s}")
  assert layout_g(tasks) in GS
  with pytest.raises(ValueError):
    dops.fused_embedding_to_layout_grad(*args, og, layout_tensors_grad_scale=torch.ones(1, device=dev).double())


# ------------------------------------------------------------------------------------------------
# 4. the chain: clip the torch way + unscaled backward == global_norm_scale + scaled backward
# ------------------------------------------------------------------------------------------------
def part_rows(c, rows, dev):
  from monolith_b200 import PoolPart
  return [PoolPart(p.slot, T(p.fids, dev), None if p.offs is None else T(p.offs, dev), p.pooling, rows, p.col,
                   max_seq_len=p.L) for p in c.parts]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_chain_parts(dtype, dev):
  from monolith_b200 import MultiHashTable, clip_ops
  tabs, calls = mixed_calls(dtype == "bf16")
  cfg = {n: v[0] for n, v in tabs.items()}
  torch_way, fused = MultiHashTable(cfg, device=dev), MultiHashTable(cfg, device=dev)
  for c in calls:
    g = T(c.grad, dev)
    if dtype == "bf16":
      g = g.to(BF)
    dense = torch.from_numpy(np.random.default_rng(c.ts).standard_normal(5000).astype(np.float32)).to(dev)
    clip = float(clip_ops.global_norm([g, dense]).item()) / 4.0   # the norm exceeds clip_norm: the scale is used
    # torch: norm, scale, multiply every layout gradient (in fp32), unscaled backward
    norm = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(t.float().double()) for t in (g, dense)]))
    s_torch = torch.where(norm.float() > clip, clip / norm.float(), torch.ones((), device=dev))
    s_dev, _ = clip_ops.global_norm_scale([g, dense], clip)
    assert bits(s_torch.item()) == bits(s_dev.item()) or abs(s_torch.item() / s_dev.item() - 1) < 1e-6
    torch_way.pool_backward_parts(part_rows(c, g.float() * s_dev, dev), req_time=c.ts)
    fused.pool_backward_parts(part_rows(c, g, dev), req_time=c.ts, grad_scale=s_dev)
  for n in sorted(tabs):
    ids = torch.from_numpy(np.unique(np.concatenate([p.fids for c in calls for p in c.parts if p.slot == n]))).to(dev)
    assert_same(fused.lookup_entry(n, ids)["raw"].cpu().numpy(), torch_way.lookup_entry(n, ids)["raw"].cpu().numpy(),
                f"table {n}")


def test_chain_partitioned_hash_table_world_1(dev):
  import os
  import torch.distributed as dist
  from monolith_b200 import MultiHashTable, clip_ops
  from monolith_b200.distributed_ps import PartitionedHashTable
  from tests.helpers import table
  with socket.socket() as sk:
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
  os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
  dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
  try:
    cfg = lambda: {"a": table([(8, "adagrad", {})], [0.1]), "b": table([(4, "ftrl", {}), (4, "sgd", {})], [0.05, 0.2])}
    ta, tb = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
    pa, pb = PartitionedHashTable(ta, 1, 0), PartitionedHashTable(tb, 1, 0)
    for step in range(3):
      rng = np.random.default_rng(step)
      fa = T((np.int64(1) << 48) | rng.integers(0, 60, 900), dev)
      offs = np.concatenate([[0], np.cumsum(rng.integers(0, 4, 400))]).astype(np.int32)
      fb = T((np.int64(2) << 48) | rng.integers(0, 25, int(offs[-1])), dev)
      ga = T(rng.standard_normal((900, 8)).astype(np.float32) * 40, dev)
      gb = T(rng.standard_normal((400, 8)).astype(np.float32) * 40, dev).to(BF)
      kw = dict(row_offsets={"b": T(offs, dev)}, pooling={"b": "mean"})
      _, ca = pa.lookup({"a": fa, "b": fb}, **kw)
      _, cb = pb.lookup({"a": fa, "b": fb}, **kw)
      s, norm = clip_ops.global_norm_scale([ga, gb], 100.0)
      assert s.item() < 1.0
      pa.apply_gradients(ca, {"a": ga * s, "b": gb.float() * s}, req_time=10 + step)
      pb.apply_gradients(cb, {"a": ga, "b": gb}, req_time=10 + step, grad_scale=s)
    for n in ("a", "b"):
      ea, eb = dict(), dict()
      for t, e in ((ta, ea), (tb, eb)):
        for ids, raw in t.export(n, chunk=1 << 14):
          for i, r in zip(ids.cpu().numpy(), raw.cpu().numpy()):
            e[int(i)] = r
      assert sorted(ea) == sorted(eb)
      for k in ea:
        assert_same(eb[k], ea[k], f"table {n}")
  finally:
    dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------
# 5. census: keep last
# ------------------------------------------------------------------------------------------------
def test_every_scaled_instantiation_ran():
  """The union of what this file's cases recorded (run the file whole)."""
  seg = lambda prefix, plain: {f"{prefix}<{g},1,{p}{a}>" for g in GS for p in plain for a in ("true", "false")} | \
      {f"{prefix}<{g},2,{p}{a}>" for g in (4, 8, 16) for p in plain for a in ("true", "false")}
  want = {
      "scaled_runs_apply_kernel<": {f"scaled_runs_apply_kernel<{g},{o}>" for g in GS for o in OPTS},
      "scaled_bf16_runs_apply_kernel<": {f"scaled_bf16_runs_apply_kernel<{g},{o}>" for g in GS for o in OPTS},
      "scaled_seg_reduce_kernel<": seg("scaled_seg_reduce_kernel", ("true,", "false,")),
      "scaled_bf16_seg_reduce_kernel<": seg("scaled_bf16_seg_reduce_kernel", ("",)),
      "scaled_gather_pool_grad_kernel<": {f"scaled_gather_pool_grad_kernel<{g}>" for g in GS},
      "scaled_bf16_gather_pool_grad_kernel<": {f"scaled_bf16_gather_pool_grad_kernel<{g}>" for g in GS},
      "scaled_layout_bwd_kernel<": {f"scaled_layout_bwd_kernel<{g}>" for g in GS},
      "scaled_bf16_layout_bwd_kernel<": {f"scaled_bf16_layout_bwd_kernel<{g}>" for g in GS},
  }
  assert SEEN, "no kernel was recorded: the census is the union of this file's other tests"
  for prefix, names in want.items():
    got = {s for s in SEEN if s.startswith(prefix)}
    assert got == names, f"{prefix}: never ran {sorted(names - got)}; ran but not listed {sorted(got - names)}"
