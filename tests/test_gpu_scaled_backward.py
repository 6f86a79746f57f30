"""The clip scale in the one-table fused backward, the ReduceSum / ReduceMean gradients and the sharded step.

Every new _scaled call against its unscaled twin on gradient rows pre-multiplied by the scale in fp32 (on the device,
bf16 rows widened first), bit for bit through uint32 views (a NaN only has to meet a NaN): scales 1, 0.5, 0.3, +0.0, a
subnormal and +inf, and a NaN gradient element.  A scaled call launches as many kernels as its twin, the scaled_ twins
of the twin's kernels; a NULL scale is the unscaled call; a scaled call does not wait for a busy stream.  The chain
test runs the reference's default ReduceSum training step both ways and compares the tables.  The last test checks
that every new scaled_ reduce_split instantiation ran.
"""
import time
import zlib

import numpy as np
import pytest
import torch

from tests.helpers import table
from tests.test_gpu_apply_paths import assert_same
from tests.test_gpu_forward_paths import traced

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GS = (4, 8, 16, 32)
SCALES = {"one": 1.0, "half": 0.5, "p3": 0.3, "zero": 0.0, "subnormal": float(np.float32(3e-41)), "inf": float("inf")}
# the kernels that load gradient rows, and their scaled_ twins
FAMILY = ("seg_reduce_kernel", "scaled_seg_reduce_kernel", "runs_apply_kernel", "scaled_runs_apply_kernel",
          "reduce_split_bwd_kernel", "bf16_reduce_split_bwd_kernel", "scaled_reduce_split_bwd_kernel",
          "scaled_bf16_reduce_split_bwd_kernel")
SEEN = set()


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def scale_t(s, dev):
  return torch.tensor([s], dtype=torch.float32, device=dev)


def premul(g, s):
  """g * s in fp32 on the device (bf16 widened exactly first): the rows the twin gets."""
  return g.float() * scale_t(s, g.device)


def launch_count():
  from monolith_b200 import _lib
  return _lib.load().mono_kernel_launch_count()


def unscaled_name(n, widened=False):
  """The kernel the twin runs in place of scaled_ kernel n; widened: the twin is the fp32 call on the widened rows of
  a bf16 call, so scaled_bf16_X is the twin's X."""
  if not n.startswith("scaled_"):
    return None
  n = n[len("scaled_"):]
  return n[len("bf16_"):] if widened and n.startswith("bf16_") else n


def compare(scaled_fn, twin_fn, tries=5, widened=False):
  """Runs both (each builds its own state) -> (scaled outputs, twin outputs).  The scaled run must launch as many
  kernels as the twin (mono_kernel_launch_count), the scaled_ twins of its kernels (unscaled_name).

  torch.profiler now and then loses a batch of device records, and in a long process (the whole GPU suite) it may
  return no kernel record at all for many traces in a row (NOTES.md).  A lost record can only make a kernel MISSING,
  so a pair whose name sets differ by such a loss is traced again; when one side still recorded nothing, the launch
  counts stand for the names."""
  for _ in range(tries):
    torch.cuda.synchronize()
    n0 = launch_count()
    got, names = traced(scaled_fn, FAMILY)
    torch.cuda.synchronize()
    n1 = launch_count()
    want, twin_names = traced(twin_fn, FAMILY)
    torch.cuda.synchronize()
    n2 = launch_count()
    assert n1 - n0 == n2 - n1, f"{n1 - n0} launches, the twin {n2 - n1}"
    assert all(n.startswith("scaled_") for n in names) and not any(n.startswith("scaled_") for n in twin_names), \
        (sorted(names), sorted(twin_names))
    mapped = {unscaled_name(n, widened) for n in names}
    if mapped == twin_names:
      break
    assert mapped < twin_names or twin_names < mapped, f"ran {sorted(names)}, the twin {sorted(twin_names)}"
  if names and twin_names:
    assert mapped == twin_names, f"ran {sorted(names)}, the twin {sorted(twin_names)}"
  SEEN.update(names)
  return got, want


def assert_all(got, want, what):
  assert len(got) == len(want)
  for i, (a, b) in enumerate(zip(got, want)):
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    if a.dtype.kind == "f":
      assert_same(a, b, f"{what} [{i}]")
    else:
      np.testing.assert_array_equal(a, b, err_msg=f"{what} [{i}]")


# ------------------------------------------------------------------------------------------------
# 1. the one-table fused backward: MultiHashTable.pool_backward
# ------------------------------------------------------------------------------------------------
# the four optimizers with a register-resident apply and one that takes the generic one (opt_sel -1)
POOL_OPTS = [("sgd", "sgd", {}, 0.05), ("adagrad", "adagrad", {"initial_accumulator_value": 0.1}, 0.05),
             ("ftrl", "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01}, 0.05),
             ("adam", "adam", {}, 0.01), ("amsgrad", "amsgrad", {"use_nesterov": True}, 0.01)]
T0, T1 = 1000, 1000 + 2 * 86400      # FIDs of slot 3 expire after one day: evicting at T1 frees their rows


def pool_tabs(dim):
  from monolith_b200 import entry
  kw = dict(capacity=64, init=entry.RandomUniformInitializer(-0.1, 0.1), init_seed=7, slot_expire_times={3: 1})
  return {name: table([(dim, opt, params)], [lr], **kw) for name, opt, params, lr in POOL_OPTS}


def pool_calls(seed, dim, mean):
  """Three steps: fresh rows; resident and fresh rows with a run of over 2^14 occurrences (tree depth 1); after an
  eviction of slot 3, new FIDs in the freed rows.  Runs of 1-8, 9-64 and over 64 occurrences in every step; one NaN
  gradient element in the first."""
  rng = np.random.default_rng(seed)
  calls = []
  for step, (n_rows, hot) in enumerate([(900, 150), (9000, 17000), (900, 100)]):
    base = 3000 * step
    u = np.concatenate([rng.integers(0, 400, n_rows), np.full(hot, 7), np.repeat(np.arange(20, 26), 30)])
    slot = np.where(np.arange(u.size) % 3 == 0, 3, 5)
    sig = np.where(slot == 3, u + base, u)
    fids = ((slot.astype(np.int64) << 48) | sig.astype(np.int64))
    rng.shuffle(fids)
    if mean:
      lens = rng.integers(0, 6, fids.size)
      offs = np.concatenate([[0], np.cumsum(lens)])
      offs = offs[offs < fids.size]
      offs = np.concatenate([offs, [fids.size]]).astype(np.int32)
      rows = offs.size - 1
    else:
      offs, rows = None, fids.size
    g = (rng.standard_normal((rows, dim)) * 3).astype(np.float32)
    if step == 0:
      g[rows // 2, dim - 1] = np.nan
    calls.append((fids, offs, g, T0 + step if step < 2 else T1 + 1, step == 2))
  return calls


def pool_run(tabs, calls, dev, s, twin):
  from monolith_b200 import MultiHashTable
  gpu = MultiHashTable(tabs, device=dev)
  sc = scale_t(s, dev)
  for fids, offs, g, ts, evict in calls:
    if evict:
      for n in tabs:
        gpu.evict(n, T1)
    gt = T(g, dev)
    for n in sorted(tabs):
      if twin:
        gpu.pool_backward(n, T(fids, dev), premul(gt, s), None if offs is None else T(offs, dev),
                          "mean" if offs is not None else "sum", req_time=ts)
      else:
        gpu.pool_backward(n, T(fids, dev), gt, None if offs is None else T(offs, dev),
                          "mean" if offs is not None else "sum", req_time=ts, grad_scale=sc)
  every = T(np.unique(np.concatenate([c[0] for c in calls])), dev)
  return [gpu.lookup_entry(n, every)["raw"] for n in sorted(tabs)] + [np.array([gpu.size(n) for n in sorted(tabs)])]


@pytest.mark.parametrize("scale", list(SCALES))
@pytest.mark.parametrize("pooling", ["sum", "mean"])
@pytest.mark.parametrize("dim", [4, 20, 64, 128])
def test_pool_backward(dim, pooling, scale, dev):
  """dims 4, 20, 64, 128: lane groups 4, 8, 16, 32; SUM one FID per row (the PLAIN reduce) and CSR MEAN; every
  entry (weights, optimizer state, found flag, timestamp) of the five tables and their sizes."""
  tabs = pool_tabs(dim)
  calls = pool_calls(zlib.crc32(f"pool/{dim}/{pooling}".encode()), dim, pooling == "mean")
  s = SCALES[scale]
  got, want = compare(lambda: pool_run(tabs, calls, dev, s, False), lambda: pool_run(tabs, calls, dev, s, True))
  assert_all(got, want, f"dim {dim}, {pooling}, scale {scale}")


# ------------------------------------------------------------------------------------------------
# 2. the ReduceSum / ReduceMean gradients: mono_reduce_and_split_grad[_bf16]_scaled
# ------------------------------------------------------------------------------------------------
# per feature: its slice dims (whole rows and odd slices; widest slices 1-16, 17-32, 33-64 and over 64 take lane
# groups 4, 8, 16, 32; multiples of 4 at 16-byte columns take the vector path)
FEATURES = [[1], [3], [16], [4, 8, 4], [17], [5, 7, 25], [33], [64], [1, 63], [100], [257], [1, 128, 127, 1],
            [128, 128, 1]]


def rs_problem(rng, B, dtype, dev, n_feats=None):
  feats = FEATURES if n_feats is None else FEATURES[:n_feats]
  splits, embs, grads = [], [], []
  for dims in feats:
    lens = rng.integers(0, 4, B)
    lens[rng.random(B) < 0.2] = 0                       # empty rows
    sp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    splits.append(T(sp, dev))
    embs.append(torch.empty(int(sp[-1]), sum(dims), device=dev))
    for d in dims:
      g = (rng.standard_normal((B, d)) * 2).astype(np.float32)
      grads.append(T(g, dev).to(dtype))
  grads[len(grads) // 2].view(-1)[0] = float("nan")
  return feats, splits, embs, grads


@pytest.mark.parametrize("B", [1, 37, 65536])
@pytest.mark.parametrize("pooling", ["sum", "mean"])
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_reduce_and_split_grad(dtype, pooling, B, dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(B + 2 * (pooling == "mean") + (dtype == BF))
  feats, splits, embs, grads = rs_problem(rng, B, dtype, dev, n_feats=None if B < 65536 else 8)
  for name, s in SCALES.items():
    sc = scale_t(s, dev)
    got, want = compare(
        lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, grads, feats, pooling=pooling, grad_scale=sc),
        lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, [premul(g, s) for g in grads], feats,
                                                     pooling=pooling), widened=dtype == BF)
    assert_all(got, want, f"{pooling}, B {B}, scale {name}")


@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
def test_reduce_gradient_wrappers(dtype, dev):
  """reduce_sum_gradient, reduce_mean_gradient and fused_reduce_sum_and_split_gradient pass the scale through."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(5)
  B, n = 300, 1000
  idx = T(np.sort(rng.integers(0, B, n))[:, None].astype(np.int64), dev)
  g = T(rng.standard_normal((B, 24)).astype(np.float32), dev).to(dtype)
  parts = [g[:, :5], g[:, 5:]]
  for s in (0.3, float("inf")):
    sc = scale_t(s, dev)
    for fn in (dops.reduce_sum_gradient, dops.reduce_mean_gradient):
      got, want = compare(lambda: [fn(idx, g, grad_scale=sc)], lambda: [fn(idx, premul(g, s))], widened=dtype == BF)
      assert_all(got, want, f"{fn.__name__}, scale {s}")
    got, want = compare(lambda: [dops.fused_reduce_sum_and_split_gradient(idx, [p.contiguous() for p in parts],
                                                                          [5, 19], grad_scale=sc)],
                        lambda: [dops.fused_reduce_sum_and_split_gradient(idx, [premul(p, s) for p in parts],
                                                                          [5, 19])], widened=dtype == BF)
    assert_all(got, want, f"fused_reduce_sum_and_split_gradient, scale {s}")


# ------------------------------------------------------------------------------------------------
# 3. Grouping.reduce / reduce_push
# ------------------------------------------------------------------------------------------------
def grouping_case(rng, D, mean, dev):
  u = np.concatenate([rng.integers(0, 500, 4000), np.full(300, 9)])
  fids = T((np.int64(5) << 48) | u.astype(np.int64), dev)
  if mean:
    offs = np.concatenate([[0], np.cumsum(rng.integers(0, 5, 2000))]).astype(np.int32)
    offs = np.minimum(offs, u.size)
    offs[-1] = u.size
    ro, rows = T(offs, dev), offs.size - 1
  else:
    ro, rows = None, u.size
  pg = T(rng.standard_normal((rows, D)).astype(np.float32), dev)
  pg[1, 0] = float("nan")
  return fids, ro, pg


@pytest.mark.parametrize("pooling", ["sum", "mean"])
@pytest.mark.parametrize("D", [4, 20, 64, 128])
def test_grouping_reduce_and_push(D, pooling, dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(D + (pooling == "mean"))
  fids, ro, pg = grouping_case(rng, D, pooling == "mean", dev)
  grp = dops.Grouping(dev)
  uniq, _, sizes = grp.build(fids, 1, D)
  U = uniq.numel()
  win = dops.PeerWindow(dev, 1, 0, U * D * 4)
  try:
    for name, s in SCALES.items():
      sc = scale_t(s, dev)
      got, want = compare(lambda: [grp.reduce(pg, torch.empty(U * D, device=dev), ro, pooling, grad_scale=sc)],
                          lambda: [grp.reduce(premul(pg, s), torch.empty(U * D, device=dev), ro, pooling)])
      assert_all(got, want, f"reduce, scale {name}")

      def push(g, scale):
        grp.reduce_push(g, sizes, win, 0, [0], ro, pooling, grad_scale=scale)
        return [win.view(0, U * D, torch.float32).clone()]
      got, want = compare(lambda: push(pg, sc), lambda: push(premul(pg, s), None))
      assert_all(got, want, f"reduce_push, scale {name}")
  finally:
    torch.cuda.synchronize()
    win.close()


# ------------------------------------------------------------------------------------------------
# 4. ShardedStep.step at world 1 in every exchange
# ------------------------------------------------------------------------------------------------
def _one_rank_group(dev):
  import torch.distributed as dist
  assert not dist.is_initialized()
  dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1, device_id=dev)


def step_batches(D, mean):
  rng = np.random.default_rng(3 + mean)
  out = []
  for step in range(3):
    n = 5000 + 700 * step
    u = rng.integers(0, 800, n)
    u[rng.random(n) < 0.2] = 3                          # a hot FID: a run of ~1 000 occurrences
    fids = (np.int64(5) << 48) | u.astype(np.int64)
    if mean:
      offs = np.concatenate([[0], np.cumsum(rng.integers(0, 5, n))]).astype(np.int32)
      offs = np.minimum(offs, n)
      offs = offs[: int(np.searchsorted(offs, n)) + 1]
      rows = offs.size - 1
    else:
      offs, rows = None, n
    g = (rng.standard_normal((rows, D)) * 4).astype(np.float32)
    out.append((fids, offs, g))
  return out


def step_run(exchange, D, batches, dev, s, twin, in_callable=False):
  """-> forward outputs and the exported table (sorted by FID)."""
  from monolith_b200 import MultiHashTable, clip_ops
  from monolith_b200.distributed_ps import ShardedStep
  tab = MultiHashTable({"t": table([(D, "adagrad", {"initial_accumulator_value": 0.1})], [0.1])}, device=dev)
  st = ShardedStep(tab, "t", D, 1, 0, dev, exchange=exchange)
  outs = []
  try:
    for step, (fids, offs, g) in enumerate(batches):
      gt = T(g, dev)
      ro = None if offs is None else T(offs, dev)
      out = torch.empty(gt.shape[0], D, device=dev)
      pooling = "mean" if offs is not None else "sum"
      if in_callable:
        # the scale comes from a norm over the forward output and the gradient, inside the callable: the step has
        # to read the buffer on the device, after the callable filled it
        buf = torch.full((1,), float("nan"), device=dev)

        def grad():
          sc, _ = clip_ops.global_norm_scale([out, gt], 50.0)
          if twin:
            return gt * sc
          buf.copy_(sc.reshape(1))
          return gt
        st.step(T(fids, dev), grad, out, 20 + step, ro, pooling, grad_scale=None if twin else buf)
      elif twin:
        st.step(T(fids, dev), premul(gt, s), out, 20 + step, ro, pooling)
      else:
        st.step(T(fids, dev), gt, out, 20 + step, ro, pooling, grad_scale=scale_t(s, dev))
      outs.append(out.clone())
    torch.cuda.synchronize()
  finally:
    if exchange == "direct":
      st.close_direct()
    elif st.window is not None:
      torch.cuda.synchronize()
      st.window.close()
  ks, rows = [], []
  for ids, raw in tab.export("t", chunk=1 << 14):
    ks.append(ids.cpu().numpy())
    rows.append(raw.cpu().numpy())
  ks, rows = np.concatenate(ks), np.concatenate(rows)
  o = np.argsort(ks)
  return outs + [ks[o], rows[o]]


EXCHANGES = ["direct", "peer-push", "peer-pull", "nccl"]


@pytest.mark.parametrize("pooling", ["sum", "mean"])
@pytest.mark.parametrize("exchange", EXCHANGES)
def test_sharded_step_world_1(exchange, pooling, dev, monkeypatch):
  if exchange.startswith("peer-"):
    monkeypatch.setenv("MONO_PEER_BULK", exchange.split("-")[1])
  ex = exchange.split("-")[0]
  D = 16
  batches = step_batches(D, pooling == "mean")
  import torch.distributed as dist
  _one_rank_group(dev)
  try:
    for name in (["half", "p3", "inf"] if pooling == "sum" else ["zero", "subnormal", "one"]):
      s = SCALES[name]
      got, want = compare(lambda: step_run(ex, D, batches, dev, s, False), lambda: step_run(ex, D, batches, dev, s, True))
      assert_all(got, want, f"{exchange}, {pooling}, scale {name}")
    got, want = compare(lambda: step_run(ex, D, batches, dev, None, False, in_callable=True),
                        lambda: step_run(ex, D, batches, dev, None, True, in_callable=True))
    assert_all(got, want, f"{exchange}, {pooling}, scale written inside the callable")
  finally:
    dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------
# 5. NULL scale, no host synchronisation, argument checks
# ------------------------------------------------------------------------------------------------
def test_null_scale_is_the_unscaled_call(dev, monkeypatch):
  """Each unscaled entry point routed through its _scaled twin with grad_scale_dev = NULL: the same bits and the
  same kernels as the unscaled call."""
  from monolith_b200 import _lib, distribution_ops as dops
  lib = _lib.load()
  rng = np.random.default_rng(9)
  D = 20
  tabs = pool_tabs(D)
  calls = pool_calls(11, D, True)[:1]
  feats, splits, embs, grads = rs_problem(rng, 37, torch.float32, dev)
  _, _, _, bgrads = rs_problem(np.random.default_rng(9), 37, BF, dev)
  fids, ro, pg = grouping_case(rng, D, True, dev)

  def run_all():
    torch.cuda.synchronize()
    out = pool_run(tabs, [(f, o, g, ts, e) for f, o, g, ts, e in calls], dev, 1.0, True)
    out += dops.fused_reduce_and_split_gpu_grad(splits, embs, grads, feats, pooling="mean")
    out += dops.fused_reduce_and_split_gpu_grad(splits, embs, bgrads, feats, pooling="sum")
    grp = dops.Grouping(dev)
    uniq = grp.build(fids, 1, D)[0]       # the order of the distinct FIDs is the engine's: compare in FID order
    rows = grp.reduce(pg, torch.empty(uniq.numel() * D, device=dev), ro, "mean").view(-1, D)
    out.append(rows[torch.argsort(uniq)])
    torch.cuda.synchronize()
    return out

  null = {"mono_mtable_pool_backward": "mono_mtable_pool_backward_scaled",
          "mono_reduce_and_split_grad": "mono_reduce_and_split_grad_scaled",
          "mono_reduce_and_split_grad_bf16": "mono_reduce_and_split_grad_bf16_scaled",
          "mono_grouping_reduce": "mono_grouping_reduce_scaled"}
  for _ in range(5):   # a trace that lost records is taken again (see compare)
    n0 = launch_count()
    want, want_names = traced(run_all, FAMILY)
    n1 = launch_count()
    with monkeypatch.context() as m:
      for plain, scaled in null.items():
        m.setattr(lib, plain, lambda *a, _fn=getattr(lib, scaled): _fn(*a[:-1], None, a[-1]))
      got, names = traced(run_all, FAMILY)
    assert launch_count() - n1 == n1 - n0
    if names == want_names:
      break
  assert not any(n.startswith("scaled_") for n in names | want_names), (sorted(names), sorted(want_names))
  if names and want_names:   # else a trace recorded nothing (see compare)
    assert names == want_names, (sorted(names), sorted(want_names))
  assert_all(got, want, "NULL scale")


def test_no_host_sync(dev):
  """A scaled call queued behind ~50 ms of device sleep returns while the stream is still busy."""
  from monolith_b200 import MultiHashTable, distribution_ops as dops
  rng = np.random.default_rng(4)
  D = 16
  feats, splits, embs, grads = rs_problem(rng, 4096, torch.float32, dev, n_feats=4)
  fids, ro, pg = grouping_case(rng, D, False, dev)
  grp = dops.Grouping(dev)
  U = grp.build(fids, 1, D)[0].numel()
  gpu = MultiHashTable({"t": table([(D, "adagrad", {})], [0.1], capacity=1 << 14)}, device=dev)
  sc = scale_t(0.5, dev)
  calls = {
      "pool_backward": lambda: gpu.pool_backward("t", fids, pg, None, "sum", req_time=5, grad_scale=sc),
      "reduce_and_split_grad": lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, grads, feats,
                                                                            grad_scale=sc),
      "grouping_reduce": lambda: grp.reduce(pg, torch.empty(U * D, device=dev), None, "sum", grad_scale=sc),
  }
  for name, fn in calls.items():
    fn()                                     # warm: modules loaded, table grown
    torch.cuda.synchronize()
    torch.cuda._sleep(int(1e8))              # about 50 ms of device time on the current stream
    t0 = time.perf_counter()
    fn()
    busy = not torch.cuda.current_stream(dev).query()
    dt = time.perf_counter() - t0
    torch.cuda.synchronize()
    assert busy, f"{name} returned after the stream drained ({dt * 1e3:.1f} ms): it waited"


def test_bad_scales_are_refused(dev):
  from monolith_b200 import MultiHashTable, distribution_ops as dops
  gpu = MultiHashTable({"t": table([(8, "sgd", {})], [0.1])}, device=dev)
  fids = T(np.arange(10, dtype=np.int64), dev)
  pg = torch.zeros(10, 8, device=dev)
  idx = T(np.arange(10, dtype=np.int64)[:, None], dev)
  bad = [torch.ones(1, dtype=torch.float64, device=dev), torch.ones(2, device=dev), torch.ones(1), 0.5]
  for b in bad:
    with pytest.raises(ValueError):
      gpu.pool_backward("t", fids, pg, grad_scale=b)
    with pytest.raises(ValueError):
      dops.reduce_sum_gradient(idx, pg, grad_scale=b)
  assert gpu.size("t") == 0


# ------------------------------------------------------------------------------------------------
# 6. the reference's default chain: lookup -> reduce_sum -> grads -> global norm -> scaled gradient -> apply
# ------------------------------------------------------------------------------------------------
def test_reduce_sum_chain(dev):
  """Clip by global norm with the ReduceSum combiner: the fused way (reduce_sum_gradient(grad_scale=)) and the
  torch way (grads multiplied by the scale, then the unscaled calls) leave bit-identical tables."""
  from monolith_b200 import MultiHashTable, clip_ops, distribution_ops as dops
  cfg = lambda: {"a": table([(8, "adagrad", {"initial_accumulator_value": 0.1})], [0.1]),
                 "b": table([(4, "ftrl", {}), (4, "sgd", {})], [0.05, 0.2])}
  fused, torch_way = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
  for step in range(4):
    rng = np.random.default_rng(step)
    B = 512
    ids, idx = {}, {}
    for n, slot in (("a", 1), ("b", 2)):
      k = np.sort(rng.integers(0, B, 3000))
      idx[n] = T(k[:, None].astype(np.int64), dev)
      ids[n] = T((np.int64(slot) << 48) | rng.integers(0, 700, k.size).astype(np.int64), dev)
    dense = T(rng.standard_normal(5000).astype(np.float32), dev)
    for tab, way in ((fused, "fused"), (torch_way, "torch")):
      emb = tab.lookup(ids)
      pooled = {n: dops.reduce_sum(idx[n], emb[n], B) for n in ids}
      pg = {n: torch.from_numpy(rng.standard_normal((B, 8)).astype(np.float32) * 60).to(dev) for n in ids} \
          if way == "fused" else pg
      s, _ = clip_ops.global_norm_scale([dense] + [pg[n] for n in sorted(pg)], 100.0)
      if way == "fused":
        assert s.item() < 1.0
        rows = {n: dops.reduce_sum_gradient(idx[n], pg[n], grad_scale=s) for n in ids}
      else:
        rows = {n: dops.reduce_sum_gradient(idx[n], pg[n] * s) for n in ids}
      split = [0, ids["a"].numel(), ids["a"].numel() + ids["b"].numel()]
      tab.raw_apply_gradients(torch.cat([ids["a"], ids["b"]]), split,
                              torch.cat([rows["a"].reshape(-1), rows["b"].reshape(-1)]), req_time=10 + step,
                              enable_dedup=True)
  for n in ("a", "b"):
    ea, eb = {}, {}
    for t, e in ((fused, ea), (torch_way, eb)):
      for i, raw in t.export(n, chunk=1 << 14):
        for k, r in zip(i.cpu().numpy(), raw.cpu().numpy()):
          e[int(k)] = r
    assert sorted(ea) == sorted(eb)
    for k in ea:
      assert_same(ea[k], eb[k], f"table {n}")


# ------------------------------------------------------------------------------------------------
# 7. census: keep last
# ------------------------------------------------------------------------------------------------
def test_every_scaled_reduce_split_instantiation_ran(dev):
  """The union of what this file's cases recorded (run the file whole).  An instantiation whose every trace was lost
  (compare then stands on launch counts) is traced again here, at all four widths in both dtypes, until the profiler
  records it; one that never runs fails after twenty traces."""
  from monolith_b200 import distribution_ops as dops
  want = {f"{p}<{g}>" for p in ("scaled_reduce_split_bwd_kernel", "scaled_bf16_reduce_split_bwd_kernel") for g in GS}
  rng = np.random.default_rng(1)
  sc = scale_t(0.5, dev)
  for _ in range(20):
    if want <= SEEN:
      break
    for dtype in (torch.float32, BF):
      feats, splits, embs, grads = rs_problem(rng, 37, dtype, dev)
      SEEN.update(traced(lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, grads, feats, grad_scale=sc),
                         FAMILY)[1])
  got = {s for s in SEEN if "reduce_split" in s}
  assert got == want, f"never ran {sorted(want - got)}; ran but not listed {sorted(got - want)}"
