"""Every optimizer, on every path that applies it to a row, against the CPU oracle bit for bit.

The device has four implementations of one optimizer step on one row: apply_row's float4 fast path (one segment,
SGD / Adagrad / FTRL / Adam, dim % 4 == 0, 16-byte aligned gradient), apply_row's generic path (everything else,
GroupAdaGrad one lane per segment), and the fused backward's bwd_apply<G, OPT> (registers) and bwd_apply<G, -1>
(staged through scratch into the generic apply_row).  They are reached from apply_gradients (unique ids, duplicate
rounds, dedup sum), fused_apply_gradient (shard groups, per-shard accumulation), mono_mtable_optimize_host,
pool_backward and the world-1 ShardedStep ("direct" = csrc/xstep.cu, "peer").

Every case runs one MultiHashTable holding one table per configuration below, so one call reaches every
optimizer branch at the same lane-group width G.  The row histories mix fresh and resident FIDs in each call,
evict a subset and insert new FIDs that take the freed rows (stale state must be overwritten by each path's own
initialisation).  The oracle gets the same gradient sums: as given, or for the fused backward and the sharded step
the sums of tests/reduce_order.py.  Every entry (weights, optimizer state, found flag, timestamp), size() and the
forward output of the sharded step are compared through uint32 views (assert_same).  Each case also asserts,
through torch.profiler, the apply kernels it launched, and the last test checks the file ran all of them.
The rules the cases are aimed with (opt_sel, the fast-path condition, pick_group, the state sizes) are pinned against
the sources in tests/test_apply_paths_cpu.py.
"""
import zlib

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import table
from tests.test_gpu_forward_paths import run as _run

pytestmark = pytest.mark.gpu

# (table name, optimizer, params, learning rate): every branch of every optimizer at least once
CONFIGS = [
    ("sgd", "sgd", {}, 0.05),
    ("adagrad", "adagrad", {"initial_accumulator_value": 0.1}, 0.05),
    ("adagrad_wd", "adagrad", {"initial_accumulator_value": 0.5, "weight_decay_factor": 0.01}, 0.05),
    ("ftrl", "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01}, 0.05),
    ("ftrl_l1_0", "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.0, "l2": 0.01}, 0.05),
    ("adam", "adam", {}, 0.01),
    ("adam_nesterov_wd", "adam", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.01),
    ("adam_fast", "adam", {"beta1": 0.5, "beta2": 0.25}, 0.01),
    ("momentum_wd", "momentum", {"weight_decay_factor": 0.01}, 0.02),
    ("momentum_nesterov_wd", "momentum", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.02),
    ("rmsprop_wd", "rmsprop", {"learning_rate": 0.02, "weight_decay_factor": 0.01}, 0.05),
    ("rmspropv2_wd", "rmspropv2", {"weight_decay_factor": 0.01}, 0.02),
    ("adadelta_wd", "adadelta", {"weight_decay_factor": 0.01, "averaging_ratio": 0.8, "epsilon": 1e-6}, 0.5),
    ("amsgrad", "amsgrad", {}, 0.01),
    ("amsgrad_nesterov_wd", "amsgrad", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.01),
    ("amsgrad_fast", "amsgrad", {"beta1": 0.5, "beta2": 0.25}, 0.01),
    ("moving_average", "moving_average", {"momentum": 0.8}, 0.0),
    ("group_adagrad", "group_adagrad", {"l2": 0.05, "beta": 1.0, "initial_accumulator_value": 0.1,
                                        "weight_decay_factor": 0.01}, 0.05),
    ("group_adagrad_l2_0", "group_adagrad", {"l2": 0.0, "beta": 0.5, "initial_accumulator_value": 0.1}, 0.05),
    ("group_adagrad_l2_big", "group_adagrad", {"l2": 1e3, "beta": 1.0, "initial_accumulator_value": 0.1}, 0.05),
]
# multi-segment tables: a learning rate per segment, 16 columns (the backward needs dim % 4 == 0)
MULTI = [
    ("mix_a", [(1, "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01}),
               (7, "amsgrad", {"use_nesterov": True, "weight_decay_factor": 0.01}),
               (4, "group_adagrad", {"l2": 0.05, "beta": 1.0, "weight_decay_factor": 0.01}),
               (4, "momentum", {"use_nesterov": True, "weight_decay_factor": 0.01})], [0.05, 0.01, 0.05, 0.02]),
    ("mix_b", [(3, "adam", {}), (5, "rmsprop", {"learning_rate": 0.02, "weight_decay_factor": 0.01}),
               (4, "adadelta", {"weight_decay_factor": 0.01, "averaging_ratio": 0.8, "epsilon": 1e-6}),
               (4, "moving_average", {"momentum": 0.8})], [0.01, 0.0, 0.5, 0.0]),
]
MULTI_DIM = 16
# the special-value case adds a GroupAdaGrad table whose l2 equals the norm of a (3, 4, 0, ...) gradient on a zero row
L2_EDGE = ("group_adagrad_l2_5", "group_adagrad", {"l2": 5.0, "beta": 1.0, "initial_accumulator_value": 0.1}, 0.05)
OPT_CODE = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 3}   # MONO_OPT_*: the four with a register-resident apply

GS = (4, 8, 16, 32)
FAMILY = ("upsert_apply_kernel", "runs_apply_kernel", "dup_accumulate_kernel")
INVENTORY = frozenset(
    [f"runs_apply_kernel<{g},{o}>" for g in GS for o in (0, 1, 2, 3, -1)] +
    [f"upsert_apply_kernel<{g},0>" for g in GS] +          # kOpOptimize
    [f"upsert_apply_kernel<{g},1>" for g in GS] +          # kOpAssign: the special-value case writes its weights
    [f"dup_accumulate_kernel<{g}>" for g in GS])
SEEN = set()

UPSERT_DIMS = [1, 3, 4, 8, 12, 17, 20, 32, 36, 64, 100, 128, 200, 260]
POOL_DIMS = [4, 8, 12, 20, 32, 36, 64, 100, 128]
# path -> dims; every path meets every lane-group width it accepts, and together they meet every width of its list
PATH_DIMS = {
    "unique": UPSERT_DIMS,
    "dup": [1, 17, 36, 128],
    "dedup": [3, 20, 64, 200],
    "fused_n1": [4, 32, 36, 260],
    "fused_n3": [8, 17, 64, 100],
    "fused_acc_n1": [12, 20, 36, 128],
    "fused_acc_n3": [1, 32, 64, 200],
    "host": [12, 17, 36, 100],
    "pool_sum": [4, 12, 20, 36, 100],
    "pool_mean": [8, 32, 64, 128],
    "direct": [4, 8, 20, 64, 128],
    "peer": [12, 32, 36, 100],
}
UPSERT_PATHS = ("unique", "dup", "dedup", "fused_n1", "fused_n3", "fused_acc_n1", "fused_acc_n3", "host")
BWD_PATHS = ("pool_sum", "pool_mean", "direct", "peer")

T0, T1 = 1000, 1000 + 2 * 86400      # FIDs of slot 3 expire after one day: evicting at T1 frees exactly those rows
SPECIAL_G = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x7F7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000],
                     np.uint32).view(np.float32)
SPECIAL_G = np.concatenate([SPECIAL_G, np.float32([3e38, -3e38])])   # 3e38^2 = inf


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def pick_group(d):
  return ro.pick_group(d)


def opt_sel(segs):
  """bwd.cu: the register-resident apply for a single SGD / Adagrad / FTRL / Adam segment, else -1."""
  return OPT_CODE.get(segs[0][1], -1) if len(segs) == 1 else -1


def assert_same(got, want, what):
  """Bit for bit through uint32 views, signed zeros included; where one side holds a NaN the other must hold a NaN
  (the GPU's arithmetic returns its canonical NaN, x86 keeps an operand's payload)."""
  g, w = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
  assert g.shape == w.shape, f"{what}: shape {g.shape} vs {w.shape}"
  gn, wn = np.isnan(g), np.isnan(w)
  bad = (gn != wn) | (~gn & (g.view(np.uint32) != w.view(np.uint32)))
  if bad.any():
    r = np.argwhere(bad)[0]
    raise AssertionError(f"{what}: {int(bad.sum())} values differ, first at {tuple(r)}: "
                         f"{g[tuple(r)]!r} ({g.view(np.uint32)[tuple(r)]:#010x}) vs "
                         f"{w[tuple(r)]!r} ({w.view(np.uint32)[tuple(r)]:#010x})")


# ------------------------------------------------------------------------------------------------
# tables
# ------------------------------------------------------------------------------------------------
def table_set(dim, zeros=False, extra=()):
  """name -> (config, dim, segments).  zeros: zero initializer (the special-value case writes exact weights)."""
  from monolith_b200 import entry
  init = entry.ZerosInitializer() if zeros else entry.RandomUniformInitializer(-0.1, 0.1)
  kw = dict(capacity=64, init=init, init_seed=7, slot_expire_times={3: 1})
  out = {}
  for name, opt, params, lr in list(CONFIGS) + list(extra):
    segs = [(dim, opt, params)]
    out[name] = (table(segs, [lr], **kw), dim, segs)
  for name, segs, lrs in MULTI:
    out[name] = (table(segs, lrs, **kw), MULTI_DIM, segs)
  return out


def fid(slot, sig):
  return (np.asarray(slot, np.int64) << np.int64(48)) | np.asarray(sig, np.int64)


# ------------------------------------------------------------------------------------------------
# row histories
# ------------------------------------------------------------------------------------------------
def _grads(rng, shape, special):
  g = (rng.standard_normal(shape) * rng.choice([1.0, 1e-3, 30.0], (shape[0], 1))).astype(np.float32)
  if special:
    m = rng.random(shape) < 0.3
    g[m] = SPECIAL_G[rng.integers(0, SPECIAL_G.size, int(m.sum()))]
  return g


def make_history(seed, tabs, path, n=96, steps=5, special=False, evict=True, keep_all=False):
  """Steps of (req_time, evict_first, {name: call data}).  Each step about half fresh FIDs (slots 3 and 4) and
  half resident ones; before step 3 the slot-3 FIDs are evicted, and steps 3 and 4 insert new FIDs into the freed
  rows next to some of the evicted FIDs, now fresh again.  `special`: the last step also brings, to every table,
  fresh FIDs with all-zero gradients and fresh FIDs whose gradient is (3, 4, 0, ...).  `keep_all`: every resident
  FID in every step, and two new ones per step after the first."""
  rng = np.random.default_rng(seed)
  N = 3 if path.endswith("n3") else 1
  dup = path in ("dup", "dedup") or path.startswith("fused_acc") or path in BWD_PATHS
  hist, next_sig = [], {k: 1 for k in tabs}
  resident = {k: np.zeros(0, np.int64) for k in tabs}
  evicted = {k: np.zeros(0, np.int64) for k in tabs}
  for s in range(steps):
    ts = T0 if (s < 3 or not evict) else T1
    ev = evict and s == 3
    calls = {}
    for name, (_, D, _) in tabs.items():
      if ev:
        slot3 = (resident[name] >> 48) == 3
        evicted[name], resident[name] = resident[name][slot3], resident[name][~slot3]
      n_new = (2 if keep_all else n // 2) if s else n
      new = fid(rng.choice([3, 4], n_new), np.arange(next_sig[name], next_sig[name] + n_new))
      next_sig[name] += n_new
      old = resident[name] if keep_all else rng.permutation(resident[name])[:n - n_new]
      back = rng.permutation(evicted[name])[:n // 8] if s >= 3 else np.zeros(0, np.int64)
      evicted[name] = np.setdiff1d(evicted[name], back)
      u = rng.permutation(np.concatenate([new, old, back]))
      resident[name] = np.union1d(resident[name], u)
      edge = np.zeros(0, np.int64)
      if special and s == steps - 1:
        edge = fid(5, np.arange(next_sig[name], next_sig[name] + 8))
        next_sig[name] += 8
        resident[name] = np.union1d(resident[name], edge)
      calls[name] = _call(rng, path, N, dup, u, edge, D, special)
    hist.append((ts, ev, calls))
  return hist


def _edge_grads(edge, D):
  """First half: all-zero gradients; second half: (3, 4, 0, ...), whose norm is exactly 5."""
  g = np.zeros((edge.size, D), np.float32)
  g[edge.size // 2:, 0] = 3.0
  if D > 1:
    g[edge.size // 2:, 1] = 4.0
  return g


def _call(rng, path, N, dup, u, edge, D, special):
  if path in BWD_PATHS:
    # occurrences: every FID 1..4 times and one hot FID 70 times (a > 64 run: the block reduction); the edge FIDs
    # once each, at the end, as one-FID rows
    reps = rng.integers(1, 5, u.size)
    reps[0] = 70
    fids = rng.permutation(np.repeat(u, reps))
    M = fids.size
    if path.endswith("mean") or (path in ("direct", "peer") and D % 8 == 0):
      lens = rng.integers(1, 5, M)
      lens = lens[np.cumsum(lens) <= M]
      lens = np.concatenate([lens, np.ones(M - int(lens.sum()), np.int64)])
      offs = np.concatenate([[0], np.cumsum(lens)])
      pooling = "mean"
    else:
      offs, pooling = None, "sum"
    pg = _grads(rng, (M if offs is None else offs.size - 1, D), special)
    if special:   # zero rows of the pooled gradient too
      pg[rng.random(pg.shape[0]) < 0.05] = 0.0
    if edge.size:
      fids = np.concatenate([fids, edge])
      pg = np.concatenate([pg, _edge_grads(edge, D)])
      if offs is not None:
        offs = np.concatenate([offs, offs[-1] + 1 + np.arange(edge.size)])
    return dict(fids=fids, pg=pg, offs=None if offs is None else offs.astype(np.int32), pooling=pooling)
  if N == 1:
    ids = np.repeat(u, rng.integers(1, 4, u.size)) if dup else u
    ids = rng.permutation(ids)
    g = _grads(rng, (ids.size, D), special)
    ids, g = np.concatenate([ids, edge]), np.concatenate([g, _edge_grads(edge, D)])
    return dict(shards=[(ids, g)])
  # three shards: a FID is in one to three of them (unique inside a shard unless accumulating)
  shards = []
  first = rng.integers(0, N, u.size)
  for s in range(N):
    sel = u[(first == s) | (rng.random(u.size) < 0.35)]
    ids = rng.permutation(np.repeat(sel, rng.integers(1, 3, sel.size)) if dup else sel)
    g = _grads(rng, (ids.size, D), special)
    if s == N - 1:
      ids, g = np.concatenate([ids, edge]), np.concatenate([g, _edge_grads(edge, D)])
    shards.append((ids, g))
  return dict(shards=shards)


# ------------------------------------------------------------------------------------------------
# paths: one step on the device, the same step on the oracle
# ------------------------------------------------------------------------------------------------
def _fused_flat(names, calls):
  N = len(calls[names[0]]["shards"])
  ids, g, ss = [], [], []
  for s in range(N):
    for n in names:
      i, x = calls[n]["shards"][s]
      ids.append(i)
      g.append(x.reshape(-1))
      ss.append(i.size)
  return np.concatenate(ids), np.concatenate(g), ss, N


def _model_sums(c, D):
  M = c["fids"].size
  x = ro.occurrence_rows(c["pg"], M, c["offs"], c["pooling"])
  with np.errstate(all="ignore"):
    keys, sums, _ = ro.call_sums(x, c["fids"], ro.pick_group(D))
  return keys, sums


def cpu_step(path, cpu, tabs, ts, calls):
  names = sorted(calls)
  if path in BWD_PATHS:
    fwd = {}
    for n in names:
      c = calls[n]
      if path in ("direct", "peer"):
        fwd[n] = cpu.lookup_pool(n, c["fids"], c["offs"], c["pooling"])
      keys, sums = _model_sums(c, tabs[n][1])
      cpu.apply_gradients({n: (keys, sums)}, req_time=ts)
    return fwd
  if path.startswith("fused"):
    ids, g, ss, N = _fused_flat(names, calls)
    cpu.fused_apply_gradient(ids, ss, g, N, req_time=ts, enable_grad_accumulation=path.startswith("fused_acc"))
    return {}
  d = {n: calls[n]["shards"][0] for n in names}
  cpu.apply_gradients(d, req_time=ts, enable_dedup=(path == "dedup"))
  return {}


class GpuPath:
  def __init__(self, path, dev, tabs):
    self.path, self.dev, self.tabs = path, dev, tabs
    self.steps = {}

  def close(self):
    for st in self.steps.values():
      st.close_direct()

  def step(self, gpu, ts, calls):
    from monolith_b200 import _lib
    from monolith_b200.distributed_ps import ShardedStep
    path, dev, names = self.path, self.dev, sorted(calls)
    if path in ("pool_sum", "pool_mean"):
      for n in names:
        c = calls[n]
        gpu.pool_backward(n, T(c["fids"], dev), T(c["pg"], dev), None if c["offs"] is None else T(c["offs"], dev),
                          c["pooling"], req_time=ts)
      return {}
    if path in ("direct", "peer"):
      fwd = {}
      for n in names:
        c, D = calls[n], self.tabs[n][1]
        if n not in self.steps:
          self.steps[n] = ShardedStep(gpu, n, D, 1, 0, dev, exchange=path)
        out = torch.empty(c["pg"].shape[0], D, device=dev)
        self.steps[n].step(T(c["fids"], dev), T(c["pg"], dev), out, ts,
                           None if c["offs"] is None else T(c["offs"], dev), c["pooling"])
        fwd[n] = out
      return fwd
    if path.startswith("fused"):
      ids, g, ss, N = _fused_flat(names, calls)
      _, _, ko, eo = gpu.fused_offsets(ss, N)
      ti = T(ids, dev)
      gpu.fused_apply_gradient(ti, ti, ss, T(g, dev), ko, eo, 0, ts, N,
                               enable_grad_accumulation=path.startswith("fused_acc"))
      return {}
    d = {n: calls[n]["shards"][0] for n in names}
    if path == "host":
      ids = np.ascontiguousarray(np.concatenate([d[n][0] for n in names]), np.int64)
      split = np.cumsum([0] + [d[n][0].size for n in names]).astype(np.int64)
      g = np.ascontiguousarray(np.concatenate([d[n][1].reshape(-1) for n in names]), np.float32)
      lr = np.asarray(gpu.learning_rates(), np.float32)
      _lib.check(_lib.load().mono_mtable_optimize_host(gpu.handle, orc.p(ids), orc.p(split), orc.p(g), orc.p(lr),
                                                       ts, 0, _lib.FLAG_IDS_UNIQUE))
      return {}
    gpu.apply_gradients({n: (T(d[n][0], dev), T(d[n][1], dev)) for n in names}, req_time=ts,
                        ids_unique=(path == "unique"), enable_dedup=(path == "dedup"))
    return {}


def expected_kernels(path, tabs, special):
  dims = {n: v[1] for n, v in tabs.items()}
  G = pick_group(max(dims.values()))                         # one call over every table: the widest sets G
  if path in ("pool_sum", "pool_mean"):
    k = {f"runs_apply_kernel<{pick_group(dims[n])},{opt_sel(tabs[n][2])}>" for n in tabs}
  elif path in ("direct", "peer"):
    k = {f"upsert_apply_kernel<{pick_group(dims[n])},0>" for n in tabs}
  else:
    k = {f"upsert_apply_kernel<{G},0>"}
    if path == "dedup" or path.startswith("fused_acc"):
      k.add(f"dup_accumulate_kernel<{G}>")
  if special:
    k.add(f"upsert_apply_kernel<{G},1>")
  return k


def special_weights(rng, n, D):
  """Random rows, a quarter of them -0.0, a quarter subnormals of both signs."""
  w = rng.standard_normal((n, D)).astype(np.float32)
  q = n // 4
  w[:q] = -0.0
  den = rng.integers(1, 1 << 23, (q, D)).astype(np.uint32) | (rng.integers(0, 2, (q, D)).astype(np.uint32) << 31)
  w[q:2 * q] = den.view(np.float32)
  return w


def check_case(path, dim, dev, seed, special=False, steps=5, n=96, evict=True, tabs=None, keep_all=False):
  from monolith_b200 import MultiHashTable
  tabs = tabs or table_set(dim, zeros=special, extra=(L2_EDGE,) if special else ())
  cfg = {n_: v[0] for n_, v in tabs.items()}
  hist = make_history(seed, tabs, path, n=n, steps=steps, special=special, evict=evict, keep_all=keep_all)
  names = sorted(tabs)
  pre = {}
  if special:   # the first step's FIDs start from written weights
    rng = np.random.default_rng(seed + 1)
    for nm in names:
      c = hist[0][2][nm]
      u = np.unique(c["fids"] if "fids" in c else np.concatenate([i for i, _ in c["shards"]]))
      pre[nm] = (u, special_weights(rng, u.size, tabs[nm][1]))
  every = {}
  for _, _, calls in hist:
    for nm, c in calls.items():
      f = c["fids"] if "fids" in c else np.concatenate([i for i, _ in c["shards"]])
      every[nm] = np.union1d(every.get(nm, np.zeros(0, np.int64)), f)
  # the oracle
  cpu = orc.OracleMultiHashTable(cfg)
  if pre:
    cpu.assign(pre, req_time=T0)
  want_fwd = []
  for ts, ev, calls in hist:
    if ev:
      for nm in names:
        cpu.evict(nm, ts)
    want_fwd.append(cpu_step(path, cpu, tabs, ts, calls))
  want = [cpu.lookup_entry(nm, every[nm]) for nm in names]
  want_size = np.array([cpu.size(nm) for nm in names], np.int64)
  if evict:
    assert any((e[:, -2] == 0).any() for e in want), "no FID was left evicted"

  def replay():
    gpu = MultiHashTable(cfg, device=dev)
    gp = GpuPath(path, dev, tabs)
    try:
      if pre:
        gpu.assign({nm: (T(u, dev), T(w, dev)) for nm, (u, w) in pre.items()}, req_time=T0, ids_unique=True)
      fwd = []
      for ts, ev, calls in hist:
        if ev:
          for nm in names:
            gpu.evict(nm, ts)
        f = gp.step(gpu, ts, calls)
        fwd += [f[nm].cpu().numpy() for nm in names if nm in f]
      ent = [gpu.lookup_entry(nm, T(every[nm], dev))["raw"].cpu().numpy() for nm in names]
      size = np.array([gpu.size(nm) for nm in names], np.int64)
      torch.cuda.synchronize()
      return tuple(ent) + tuple(fwd) + (size,)
    finally:
      gp.close()

  out = _run(replay, expected_kernels(path, tabs, special), FAMILY, SEEN)
  ent, size = out[:len(names)], out[-1]
  np.testing.assert_array_equal(size, want_size, err_msg=f"{path} dim {dim}: size()")
  for nm, g, w in zip(names, ent, want):
    assert_same(g, w, f"{path} dim {dim} table {nm}")
  fwd = out[len(names):-1]
  want_f = [wf[nm] for wf in want_fwd for nm in names if nm in wf]
  assert len(fwd) == len(want_f)
  for i, (g, w) in enumerate(zip(fwd, want_f)):
    assert_same(g, w, f"{path} dim {dim}: forward output {i}")
  return want, names


CASES = [(p, d) for p in UPSERT_PATHS + BWD_PATHS for d in PATH_DIMS[p]]


@pytest.mark.parametrize("path,dim", CASES, ids=lambda v: str(v))
def test_every_optimizer_on_every_path(path, dim, dev):
  check_case(path, dim, dev, zlib.crc32(f"{path}/{dim}".encode()))


SPECIAL_CASES = [(p, 12) for p in UPSERT_PATHS + BWD_PATHS] + [("unique", 260), ("fused_n3", 20), ("direct", 64),
                                                               ("pool_sum", 128)]


@pytest.mark.parametrize("path,dim", SPECIAL_CASES, ids=lambda v: str(v))
def test_special_values(path, dim, dev):
  """Gradient columns of +-0, +-smallest subnormal, FLT_MAX, 3e38 (its square overflows), +-inf and NaN, weights
  written as -0.0 and subnormals; in the last step fresh FIDs with all-zero gradients (GroupAdaGrad with l2 = 0:
  0 / 0; FTRL with l1 = 0: |z| = 0) and with (3, 4, 0, ...) (a GroupAdaGrad norm exactly at l2 = 5)."""
  want, names = check_case(path, dim, dev, zlib.crc32(f"special/{path}/{dim}".encode()), special=True, steps=3,
                           evict=False)
  e = want[names.index(L2_EDGE[0])]
  edge = e[-4:, :2]                                       # the last FIDs of slot 5: norm 5 = l2, coefficient -0
  assert (edge.view(np.uint32) == 0x80000000).all(), "the l2 edge case did not land on its boundary"


@pytest.mark.parametrize("path,dim", [("unique", 8), ("pool_sum", 8)], ids=lambda v: str(v))
def test_beta_powers_run_into_subnormals_and_zero(path, dim, dev):
  """Adam and AMSGrad with beta1 = 0.5, beta2 = 0.25 for 160 steps: the per-row powers 0.5^k and 0.25^k pass
  through the subnormals (0.5^127 .. 0.5^149) and become 0; two FIDs join at every step and stay, so every exponent
  is held by some row at the end."""
  from monolith_b200 import entry
  kw = dict(capacity=64, init=entry.RandomUniformInitializer(-0.1, 0.1), init_seed=7)
  tabs = {}
  for name, opt, params, lr in CONFIGS:
    if name in ("adam_fast", "amsgrad_fast"):
      tabs[name] = (table([(dim, opt, params)], [lr], **kw), dim, [(dim, opt, params)])
  want, names = check_case(path, dim, dev, 160 + dim, steps=160, n=200, evict=False, tabs=tabs, keep_all=True)
  for nm, e in zip(names, want):
    po = (2 if nm.startswith("adam") else 3) * dim
    b1 = e[:, dim + po]
    assert (b1 == 0).any() and ((b1 != 0) & (np.abs(b1) < np.finfo(np.float32).tiny)).any(), nm


@pytest.mark.parametrize("path", ["unique", "dup"])
def test_misaligned_gradient_gives_the_same_bits(path, dev):
  """One update from a 16-byte aligned gradient buffer (apply_row's float4 path where it applies) and from a view
  one float later (the generic path): bit-identical tables, equal to the oracle."""
  from monolith_b200 import MultiHashTable
  for dim in (4, 36, 260):
    tabs = table_set(dim)
    cfg = {n: v[0] for n, v in tabs.items()}
    names = sorted(tabs)
    hist = make_history(zlib.crc32(f"align/{path}/{dim}".encode()), tabs, path, steps=2, evict=False)
    cpu = orc.OracleMultiHashTable(cfg)
    for ts, _, calls in hist:
      cpu_step(path, cpu, tabs, ts, calls)
    every = {n: np.unique(np.concatenate([c[n]["shards"][0][0] for _, _, c in hist])) for n in names}

    def replay(shift):
      def f():
        gpu = MultiHashTable(cfg, device=dev)
        for ts, _, calls in hist:
          ids = np.concatenate([calls[n]["shards"][0][0] for n in names])
          split = [int(x) for x in np.cumsum([0] + [calls[n]["shards"][0][0].size for n in names])]
          g = np.concatenate([calls[n]["shards"][0][1].reshape(-1) for n in names])
          buf = torch.zeros(g.size + 4, device=dev)
          view = buf[shift:shift + g.size]
          view.copy_(T(g, dev))
          assert (view.data_ptr() % 16 == 0) == (shift == 0)
          gpu.raw_apply_gradients(T(ids, dev), split, view, req_time=ts, ids_unique=(path == "unique"))
        torch.cuda.synchronize()
        return tuple(gpu.lookup_entry(n, T(every[n], dev))["raw"].cpu().numpy() for n in names)
      return f

    G = pick_group(max(v[1] for v in tabs.values()))
    a = _run(replay(0), f"upsert_apply_kernel<{G},0>", FAMILY, SEEN)
    b = _run(replay(1), f"upsert_apply_kernel<{G},0>", FAMILY, SEEN)
    for n, x, y in zip(names, a, b):
      np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32), err_msg=f"{path} dim {dim} table {n}")
      assert_same(x, cpu.lookup_entry(n, every[n]), f"{path} dim {dim} table {n}")


def test_case_matrix_covers_every_dim_and_width():
  """Each path meets every lane-group width it accepts; each of the four implementations meets every dim it
  accepts (the fast path and bwd_apply<G, OPT> only take dim % 4 == 0, the fused backward only dim <= 128)."""
  for p, dims in PATH_DIMS.items():
    accepted = UPSERT_DIMS if p in UPSERT_PATHS else POOL_DIMS
    assert set(dims) <= set(accepted)
    assert {pick_group(d) for d in dims} == {pick_group(d) for d in accepted}, p
  upsert = {d for p in UPSERT_PATHS for d in PATH_DIMS[p]}
  bwd = {d for p in ("pool_sum", "pool_mean") for d in PATH_DIMS[p]}
  assert upsert == set(UPSERT_DIMS)                                   # generic apply_row: every dim
  assert {d for d in upsert if d % 4 == 0} == {d for d in UPSERT_DIMS if d % 4 == 0}   # float4 apply_row
  assert bwd == set(POOL_DIMS)                                        # bwd_apply<G, OPT> and <G, -1>
  assert any(opt_sel([(1, c[1], {})]) >= 0 for c in CONFIGS) and any(opt_sel([(1, c[1], {})]) < 0 for c in CONFIGS)


# ------------------------------------------------------------------------------------------------
# inventory: keep last
# ------------------------------------------------------------------------------------------------
def test_every_apply_instantiation_ran_and_no_other():
  """The union of what the cases above ran (run this file whole: the inventory is collected from them)."""
  assert SEEN, "no apply kernel was recorded: the inventory is the union of this file's other tests"
  missing, extra = sorted(INVENTORY - SEEN), sorted(SEEN - INVENTORY)
  assert not missing and not extra, f"never ran: {missing}; ran but not listed: {extra}"
