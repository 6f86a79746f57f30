"""The many-feature fused backward (mono_mtable_pool_backward_parts and its bf16 form) against the CPU oracle, bit
for bit, on every optimizer, lane-group width, reduce variant and row dtype.

Every case replays steps of pool_backward_parts on a MultiHashTable and the same steps on orc.OracleMultiHashTable,
fed per table with reduce_order's sums of the table's per-occurrence terms (tests/test_parts_apply_paths_cpu.py:
the parts in part order, then occurrence order; SUM the row, CSR MEAN row / n, FIRSTN position j's slice or +0.0
past L; bf16 rows widened exactly).  Every entry (weights, optimizer state, found flag, timestamp) and size() are
compared through uint32 views (assert_same).  All parts of a call take their rows from column slices of ONE shared
[B, W] gradient tensor (columns = 0 mod 4, W = 4 mod 8, so rows alternate between 16- and 8-byte alignment in bf16;
odd steps also start the bf16 tensor 8 bytes past a 16-byte boundary).

Each call's kernel launches are counted (mono_kernel_launch_count) and must equal the pipeline's count; the reduce
and apply instantiations torch.profiler recorded must be the ones the dispatch picks (the profiler loses whole
batches of records in a long process, so names are required only when it recorded them, NOTES.md).  The last test
checks the file launched every bf16 reduce and apply instantiation, and every fp32 apply under a parts call.
"""
import contextlib
import zlib

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import table
from tests.test_gpu_apply_paths import L2_EDGE, T0, assert_same, fid, make_history, special_weights, table_set
from tests.test_gpu_forward_paths import traced
from tests.test_gpu_reduce_order import KNOBS
from tests.test_parts_apply_paths_cpu import (BF16_DIMS, BOUNDARY_LENS, FP32_DIMS, GS, OPTS, SEQ_L, Part,
                                              apply_kernel, bf16_widen, call_launches, opt_sel, seg_kernel,
                                              table_sums)

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FAMILY = ("runs_apply_kernel", "bf16_runs_apply_kernel", "seg_reduce_kernel", "bf16_seg_reduce_kernel")
SEEN = set()
BF16_SPECIAL = np.array([0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x7F7F, 0xFF7F, 0x7F80, 0xFF80, 0x7FC0, 0x7F81],
                        np.uint32)
BF16_SPECIAL = (BF16_SPECIAL << 16).view(np.float32)    # exact fp32 values of the bf16 patterns (NaN payload kept)


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


# ------------------------------------------------------------------------------------------------
# one call: parts in column slices of one shared gradient array
# ------------------------------------------------------------------------------------------------
class Call:
  """One pool_backward_parts call: its parts (column slices assigned here) and the shared gradient array, already
  rounded to bf16 (and widened back) for a bf16 call."""

  def __init__(self, rng, parts, dims, bf16, ts, evict=False, offset8=False, fill=None):
    self.parts, self.bf16, self.ts, self.evict, self.offset8 = parts, bf16, ts, evict, offset8
    col = 0
    for p in parts:
      p.col = col + 4 * int(rng.integers(0, 2))
      col = p.col + p.width(dims[p.slot])
    W = col + 4
    W += 4 if W % 8 == 0 else 0
    B = max(p.n_rows() for p in parts) + 3
    g = (rng.standard_normal((B, W)) * rng.choice([1.0, 1e-3, 30.0], (B, 1))).astype(np.float32)
    if fill is not None:
      fill(g)
    self.grad = bf16_widen(g) if bf16 else g

  def device_parts(self, dev):
    from monolith_b200 import PoolPart
    if self.bf16:
      h = torch.from_numpy(self.grad).to(BF)
      buf = torch.empty(h.numel() + 8, dtype=BF, device=dev)
      k = 4 if self.offset8 else 0
      rows = buf[k:k + h.numel()].view(h.shape)
      rows.copy_(h.to(dev))
      assert rows.data_ptr() % 16 == (8 if self.offset8 else 0)
    else:
      rows = T(self.grad, dev)
    return [PoolPart(p.slot, T(p.fids, dev), None if p.offs is None else T(p.offs, dev), p.pooling, rows, p.col,
                     max_seq_len=p.L) for p in self.parts]

  def per_table(self):
    out = {}
    for p in self.parts:
      out[p.slot] = out.get(p.slot, 0) + p.fids.size
    return out


def expected_kernels(calls, tabs, knobs):
  sv, sa = knobs.get("seg_vpl", 1), knobs.get("seg_ahead", 1)
  k = set()
  for c in calls:
    for n in c.per_table():
      D, segs = tabs[n][1], tabs[n][2]
      G = ro.pick_group(D)
      k |= {seg_kernel(G, c.bf16, sv, sa), apply_kernel(G, opt_sel(segs), c.bf16)}
  return k


@contextlib.contextmanager
def knob_setting(setting):
  from monolith_b200 import _lib
  lib = _lib.load()
  names = sorted({k for s in KNOBS for k in s})
  old = {k: lib.mono_get_option(k.encode()) for k in names}
  try:
    for k in names:
      assert lib.mono_set_option(k.encode(), setting.get(k, old[k])) == 0
    yield
  finally:
    for k in names:
      lib.mono_set_option(k.encode(), old[k])


def check_calls(tabs, calls, dev, pre=None, knobs=None, tries=4):
  """Replay `calls` on the device and on the oracle; every entry of every FID the calls named, and size(), bit for
  bit.  -> the oracle's entries by table."""
  from monolith_b200 import MultiHashTable
  knobs = knobs or {}
  cfg = {n: v[0] for n, v in tabs.items()}
  names = sorted(tabs)
  dims = {n: v[1] for n, v in tabs.items()}
  every = {n: np.unique(np.concatenate([np.zeros(0, np.int64)] + [p.fids for c in calls for p in c.parts
                                                                   if p.slot == n])) for n in names}
  cpu = orc.OracleMultiHashTable(cfg)
  if pre:
    cpu.assign(pre, req_time=T0)
  for c in calls:
    if c.evict:
      for n in names:
        cpu.evict(n, c.ts)
    for n in c.per_table():
      u, sums, _ = table_sums(c.grad, c.parts, n, dims[n])
      cpu.apply_gradients({n: (u, sums)}, req_time=c.ts)
  want = {n: cpu.lookup_entry(n, every[n]) for n in names}
  want_size = [cpu.size(n) for n in names]
  want_launches = [call_launches(list(c.per_table().values())) for c in calls]
  expect = expected_kernels(calls, tabs, knobs)

  def replay():
    gpu = MultiHashTable(cfg, device=dev)
    lib = gpu._lib
    if pre:
      gpu.assign({n: (T(u, dev), T(w, dev)) for n, (u, w) in pre.items()}, req_time=T0, ids_unique=True)
    launches = []
    for c in calls:
      if c.evict:
        for n in names:
          gpu.evict(n, c.ts)
      dp = c.device_parts(dev)
      torch.cuda.synchronize()
      n0 = lib.mono_kernel_launch_count()
      gpu.pool_backward_parts(dp, req_time=c.ts)
      torch.cuda.synchronize()
      launches.append(lib.mono_kernel_launch_count() - n0)
    ent = {n: gpu.lookup_entry(n, T(every[n], dev))["raw"].cpu().numpy() for n in names}
    return ent, [gpu.size(n) for n in names], launches

  with knob_setting(knobs):
    for _ in range(tries):
      (ent, size, launches), seen = traced(replay, FAMILY)
      assert seen <= expect, f"ran {sorted(seen - expect)}, aimed at {sorted(expect)}"
      SEEN.update(seen)
      if seen == expect:
        break
  assert launches == want_launches, "kernel launches per call"
  assert size == want_size, "size()"
  for n in names:
    assert_same(ent[n], want[n], f"table {n}")
  return want


def capacity(tabs, n):
  """Tables that never grow during a case: growth launches kernels of its own."""
  for cfg, _, _ in tabs.values():
    cfg.table_config.initial_capacity = n
  return tabs


# ------------------------------------------------------------------------------------------------
# 1. optimizer x width matrix
# ------------------------------------------------------------------------------------------------
KINDS = [("sum", "mean", "firstn"), ("sum", "firstn"), ("mean", "firstn"), ("sum", "mean")]


def csr(rng, M, hi=5):
  lens = rng.integers(1, hi, M)
  lens = lens[np.cumsum(lens) <= M]
  lens = np.concatenate([lens, np.ones(M - int(lens.sum()), np.int64)])
  return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def firstn_part(rng, slot, chunk, beyond, L=SEQ_L):
  """Rows of 0 .. L + 3 FIDs holding `chunk` in order; the `beyond` FIDs only at positions >= L."""
  k = -(-beyond.size // 3) + 1
  lens = [L + 3] * k
  total = chunk.size + beyond.size
  while sum(lens) < total:
    lens.append(min(int(rng.integers(0, L + 4)), total - sum(lens)))
  offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  row = np.repeat(np.arange(len(lens)), lens)
  pos = np.arange(total) - offs[:-1][row]
  at = rng.choice(np.flatnonzero(pos >= L), beyond.size, replace=False)
  fids = np.empty(total, np.int64)
  m = np.zeros(total, bool)
  m[at] = True
  fids[at] = beyond
  fids[~m] = chunk
  return Part(slot, fids, offs, "firstn", L)


def table_parts(rng, slot, u, kinds, hot_len=70, extra=(), rest_hi=5):
  """One table's parts over its distinct FIDs u: a hot FID (> 64 occurrences, spread over the parts), runs of exactly
  8, 9, 64 and 65 (plus `extra` lengths), the rest 1 .. rest_hi - 1; with a FIRSTN part two FIDs occur only past L."""
  u = rng.permutation(u)
  fixed = [hot_len, 8, 9, 64, 65] + list(extra)
  beyond = u[:2] if "firstn" in kinds else np.zeros(0, np.int64)
  main = u[beyond.size:]
  lens = np.concatenate([fixed, rng.integers(1, rest_hi, main.size - len(fixed))])
  occ = rng.permutation(np.repeat(main, lens))
  cuts = np.sort(rng.choice(np.arange(occ.size // 5, occ.size - occ.size // 5), len(kinds) - 1, replace=False))
  parts = []
  for kind, chunk in zip(kinds, np.split(occ, cuts)):
    if kind == "sum":
      parts.append(Part(slot, chunk))
    elif kind == "mean":
      parts.append(Part(slot, chunk, csr(rng, chunk.size), "mean"))
    else:
      parts.append(firstn_part(rng, slot, chunk, beyond))
  hot = main[0]
  assert sum(bool((p.fids == hot).any()) for p in parts) >= 2, "the hot FID is not split across parts"
  return parts


def matrix_calls(seed, tabs, bf16, special=False, steps=5):
  """make_history's FIDs (fresh and resident FIDs, slot-3 FIDs evicted before step 3, rows reused after), each step
  ONE call over every table with 2-3 parts per table.  special: gradients partly bf16 special values, and the last
  step brings 8 fresh slot-5 FIDs per table as one-FID SUM rows, all-zero and (3, 4, 0, ...)."""
  hist = make_history(seed, tabs, "pool_sum", n=96, steps=steps, evict=not special)
  rng = np.random.default_rng(seed + 1)
  dims = {n: v[1] for n, v in tabs.items()}
  calls = []
  for s, (ts, ev, hc) in enumerate(hist):
    parts, edges = [], []
    for i, n in enumerate(sorted(tabs)):
      parts += table_parts(rng, n, np.unique(hc[n]["fids"]), KINDS[(i + s) % len(KINDS)])
      if special and s == steps - 1:
        e = Part(n, fid(5, np.arange(1 << 20, (1 << 20) + 8) + 16 * i))
        parts.append(e)
        edges.append(e)

    def fill(g, parts=parts, edges=edges):
      if special:
        m = rng.random(g.shape) < 0.3
        g[m] = BF16_SPECIAL[rng.integers(0, BF16_SPECIAL.size, int(m.sum()))]
      for e in edges:   # after the parts' columns are known
        D = dims[e.slot]
        g[:e.n_rows(), e.col:e.col + D] = 0.0
        g[4:e.n_rows(), e.col] = 3.0
        g[4:e.n_rows(), e.col + 1] = 4.0
    calls.append(Call(rng, parts, dims, bf16, ts, evict=ev, offset8=bf16 and s % 2 == 1, fill=fill))
  return calls


MATRIX = [("fp32", d) for d in FP32_DIMS] + [("bf16", d) for d in BF16_DIMS]


@pytest.mark.parametrize("dtype,dim", MATRIX, ids=lambda v: str(v))
def test_every_optimizer_and_width(dtype, dim, dev):
  """table_set(dim): the 20 single-optimizer configs and the two multi-segment tables, one call per step over all 22."""
  tabs = capacity(table_set(dim), 8192)
  calls = matrix_calls(zlib.crc32(f"matrix/{dtype}/{dim}".encode()), tabs, dtype == "bf16")
  want = check_calls(tabs, calls, dev)
  assert any((e[:, -2] == 0).any() for e in want.values()), "no FID was left evicted"


@pytest.mark.parametrize("dim", [12, 100])
def test_bf16_special_values(dim, dev):
  """bf16 gradient values +-0, +-smallest subnormal, the largest subnormal, +-largest finite, +-inf, quiet NaN and a
  NaN with payload; weights written as -0.0 and subnormals; in the last step fresh FIDs with all-zero gradients and
  with (3, 4, 0, ...) (a GroupAdaGrad norm exactly at l2 = 5)."""
  tabs = capacity(table_set(dim, zeros=True, extra=(L2_EDGE,)), 8192)
  seed = zlib.crc32(f"special/{dim}".encode())
  calls = matrix_calls(seed, tabs, True, special=True, steps=3)
  rng = np.random.default_rng(seed + 2)
  pre = {}
  for n in sorted(tabs):
    u = np.unique(np.concatenate([p.fids for p in calls[0].parts if p.slot == n]))
    pre[n] = (u, special_weights(rng, u.size, tabs[n][1]))
  want = check_calls(tabs, calls, dev, pre=pre)
  e = want[L2_EDGE[0]]
  edge = e[-4:, :2]                                       # the last slot-5 FIDs: norm 5 = l2, coefficient -0
  assert (edge.view(np.uint32) == 0x80000000).all(), "the l2 edge case did not land on its boundary"
  g = np.concatenate([c.grad.ravel() for c in calls])
  assert np.isnan(g).any() and np.isinf(g).any() and (g.view(np.uint32) == 0x00010000).any()


# ------------------------------------------------------------------------------------------------
# 2. mixed widths in one call, one table at tree depth 1
# ------------------------------------------------------------------------------------------------
MIXED = [("m004", 4, "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01}, 0.05),
         ("m020", 20, "adam", {}, 0.01),
         ("m036", 36, "momentum", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.02),
         ("m100", 100, "adagrad", {"initial_accumulator_value": 0.1}, 0.05)]
DEEP = "m036"


def mixed_tabs():
  from monolith_b200 import entry
  out = {}
  for i, (n, D, opt, params, lr) in enumerate(MIXED):
    segs = [(D, opt, params)]
    out[n] = (table(segs, [lr], capacity=1 << 17, init=entry.RandomUniformInitializer(-0.1, 0.1), init_seed=i + 1),
              D, segs)
  return out


def mixed_calls(bf16):
  tabs = mixed_tabs()
  rng = np.random.default_rng(29 + bf16)
  dims = {n: v[1] for n, v in tabs.items()}
  calls = []
  for s in range(2):
    parts = []
    for i, (n, D, _, _, _) in enumerate(MIXED):
      nu = 3000 if n == DEEP else 120
      u = fid(4, np.arange(s * nu // 2, s * nu // 2 + nu) + 1)   # step 1: half resident, half fresh
      if n == DEEP:
        parts += table_parts(rng, n, u, KINDS[0], hot_len=4097, extra=(1000, 129), rest_hi=9)
      else:
        parts += table_parts(rng, n, u, KINDS[(i + s) % len(KINDS)])
    c = Call(rng, parts, dims, bf16, 100 + s, offset8=bf16 and s == 1)
    per = c.per_table()
    assert ro.tree_top(ro.n_pieces(per[DEEP]))[0] == 1
    assert all(ro.tree_top(ro.n_pieces(m))[0] == 0 for n, m in per.items() if n != DEEP)
    calls.append(c)
  return tabs, calls


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_mixed_widths_and_depths_in_one_call(dtype, dev):
  tabs, calls = mixed_calls(dtype == "bf16")
  check_calls(tabs, calls, dev)


# ------------------------------------------------------------------------------------------------
# 3. table boundaries inside a piece
# ------------------------------------------------------------------------------------------------
# one FID per table, so a table's sorted range is that one run; names sort in chain order.  After table A (a run of
# L_A) come runs long | short | long | 9-64 | long | short (8) | 9-64 (9) | long (65): every boundary class
CHAIN = [97, 5, 70, 40, 129, 8, 9, 65]
CHAIN_DIMS = [4, 20, 36, 100, 8, 64, 128, 12, 32]       # G = 4 8 16 32 4 16 32 4 8


def chain_tabs(opt):
  from monolith_b200 import entry
  out = {}
  for i, D in enumerate(CHAIN_DIMS):
    if opt == "sgd":
      segs, lr, ini = [(D, "sgd", {})], 1.0, entry.ConstantsInitializer(-0.0)
    else:
      segs, lr, ini = [(D, "adagrad", {"initial_accumulator_value": 0.1})], 0.05, \
          entry.RandomUniformInitializer(-0.1, 0.1)
    out[f"c{i}"] = (table(segs, [lr], capacity=1 << 16, init=ini, init_seed=i + 1), D, segs)
  return out


def boundary_calls(bf16, lens_a=BOUNDARY_LENS):
  """One call per L_A, fresh FIDs in every call.  Long runs are split over a one-FID SUM part and a CSR MEAN part;
  per (call, table) the run's terms are random, start with -0.0, or are all -0.0."""
  rng = np.random.default_rng(31 + bf16)
  dims = {f"c{i}": D for i, D in enumerate(CHAIN_DIMS)}
  calls = []
  for ci, LA in enumerate(lens_a):
    parts, zero = [], []
    for i, L in enumerate([LA] + CHAIN):
      n = f"c{i}"
      f = np.full(L, fid(6, 1000 * ci + i + 1), np.int64)
      if L > 8:
        k = L // 2 + int(rng.integers(-2, 3))
        parts += [Part(n, f[:k]), Part(n, f[k:], csr(rng, L - k), "mean")]
      else:
        parts.append(Part(n, f))
      mode = (ci + i) % 3
      if mode:
        zero.append((n, mode))

    def fill(g, parts=parts, zero=zero):
      for n, mode in zero:
        ps = [p for p in parts if p.slot == n]
        if mode == 1:
          r, col = ps[0].cell(0, dims[n])
          g[r, col:col + dims[n]] = -0.0
        else:
          for p in ps:
            g[:p.n_rows(), p.col:p.col + p.width(dims[n])] = -0.0
    c = Call(rng, parts, dims, bf16, 200 + ci, offset8=bf16 and ci % 2 == 1, fill=fill)
    calls.append(c)
  return calls


@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_table_boundaries_inside_a_piece(dtype, opt, dev):
  tabs = chain_tabs(opt)
  calls = boundary_calls(dtype == "bf16")
  want = check_calls(tabs, calls, dev)
  if opt == "sgd":   # a row is -0.0 - sum: the all -0.0 runs give +0.0, the others -(sum)
    pz = sum(int((e[:, 0].view(np.uint32) == 0).sum()) for e in want.values())
    assert pz > 0, "no run summed to -0.0"


# ------------------------------------------------------------------------------------------------
# 4. bf16 run-length edges
# ------------------------------------------------------------------------------------------------
EDGE_LENS = [1, 2, 8, 9, 63, 64, 65, 129]


@pytest.mark.parametrize("D", [4, 32, 64, 128])
def test_bf16_run_length_edges(D, dev):
  """SGD lr 1 from -0.0: each edge length three times (random terms, -0.0 first term, -0.0 only) among short runs,
  spread over a SUM, a CSR MEAN and a FIRSTN part; one more FID occurs in the FIRSTN part once at a -0.0 position and
  once past L: its sum is -0.0 + (+0.0) = +0.0, so its row is -0.0."""
  from monolith_b200 import entry
  rng = np.random.default_rng(zlib.crc32(f"bf16 edges/{D}".encode()))
  tabs = {"t": (table([(D, "sgd", {})], [1.0], capacity=4096, init=entry.ConstantsInitializer(-0.0)), D,
                [(D, "sgd", {})])}
  lens = np.concatenate([np.repeat(EDGE_LENS, 3), rng.integers(1, 9, 700)]).astype(np.int64)
  u = fid(7, np.arange(lens.size) + 1)
  special = fid(7, 1 << 30)
  run_of = rng.permutation(np.repeat(np.arange(lens.size), lens))
  occ = u[run_of]
  M = occ.size
  m1, m2 = M // 3, 2 * M // 3
  sp = Part("t", occ[:m1])
  mp = Part("t", occ[m1:m2], csr(rng, m2 - m1), "mean")
  fp = firstn_part(rng, "t", occ[m2:], np.zeros(0, np.int64), L=3)
  # the special FID: a last row [special (-0.0), two one-occurrence FIDs, special (past L)]
  row = np.array([special, special + 1, special + 2, special])
  fp = Part("t", np.concatenate([fp.fids, row]), np.concatenate([fp.offs, [fp.offs[-1] + 4]]), "firstn", 3)
  parts = [sp, mp, fp]
  # the occurrences whose term is -0.0: the special FID's first, the first of each second run, every one of each third
  flat = np.concatenate([p.fids for p in parts])
  zero_occ = [M]
  first = {}
  for i, f in enumerate(flat[:M]):
    first.setdefault(f, i)
  for L in EDGE_LENS:
    runs = np.flatnonzero(lens == L)[:3]
    zero_occ.append(first[u[runs[1]]])
    zero_occ.extend(np.flatnonzero(flat[:M] == u[runs[2]]).tolist())

  def fill(g):
    for i in zero_occ:
      for p, b in zip(parts, np.cumsum([0] + [p.fids.size for p in parts])[:-1]):
        if b <= i < b + p.fids.size:
          c = p.cell(i - b, D)
          if c is not None:
            g[c[0], c[1]:c[1] + D] = -0.0
  calls = [Call(rng, parts, {"t": D}, True, 9, offset8=True, fill=fill)]
  _, sums, length = table_sums(calls[0].grad, parts, "t", D)
  assert set(EDGE_LENS) <= set(length.tolist())
  k = np.flatnonzero(np.unique(flat) == special)[0]
  assert (sums[k].view(np.uint32) == 0).all(), "the FIRSTN -0.0 + past-L FID does not sum to +0.0"
  assert (np.signbit(sums).all(1) & (sums == 0).all(1)).any(), "no run sums to -0.0"
  want = check_calls(tabs, calls, dev)
  assert (want["t"][k, :D].view(np.uint32) == 0x80000000).all()


# ------------------------------------------------------------------------------------------------
# 5. tree depth 2 in bf16
# ------------------------------------------------------------------------------------------------
def test_bf16_tree_depth_2(dev):
  """> 2^21 occurrences of a dim-4 table, runs of > 524 288 (two tree levels), over a SUM and a CSR MEAN part."""
  from monolith_b200 import entry
  rng = np.random.default_rng(37)
  lens = [17, 600000, 5, 524289, 65, 530001, 129, 4097, 33]
  fill_n = (1 << 21) + 4097 - sum(lens)
  short = rng.integers(1, 9, fill_n // 2)
  short = short[np.cumsum(short) <= fill_n]
  lens = np.asarray(lens + list(short) + [1] * (fill_n - int(short.sum())), np.int64)
  u = fid(8, np.arange(lens.size) + 1)
  occ = u[rng.permutation(np.repeat(np.arange(lens.size), lens))]
  M = occ.size
  assert ro.tree_top(ro.n_pieces(M))[0] == 2
  k = M // 2
  parts = [Part("d", occ[:k]), Part("d", occ[k:], csr(rng, M - k), "mean")]
  segs = [(4, "adagrad", {"initial_accumulator_value": 0.1})]
  tabs = {"d": (table(segs, [0.05], capacity=1 << 22, init=entry.RandomUniformInitializer(-0.1, 0.1), init_seed=3),
                4, segs)}
  check_calls(tabs, [Call(rng, parts, {"d": 4}, True, 11, offset8=True)], dev, tries=2)


# ------------------------------------------------------------------------------------------------
# 6. knobs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting", KNOBS, ids=lambda s: ",".join(f"{k}={v}" for k, v in s.items()))
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_knobs_give_the_same_bits(dtype, setting, dev):
  """The mixed-width call and the boundary chain under every reduce / claim / apply option: the oracle's bits, which
  are those of the default options (the cases above)."""
  bf16 = dtype == "bf16"
  tabs, calls = mixed_calls(bf16)
  check_calls(tabs, calls, dev, knobs=setting)
  check_calls(chain_tabs("sgd"), boundary_calls(bf16, [95, 96, 4097, 16385]), dev, knobs=setting)


# ------------------------------------------------------------------------------------------------
# 7. census: keep last
# ------------------------------------------------------------------------------------------------
def test_every_parts_instantiation_ran():
  """The union of what the cases above recorded (run this file whole)."""
  assert SEEN, "no kernel was recorded: the census is the union of this file's other tests"
  bf16_apply = {apply_kernel(g, o, True) for g in GS for o in OPTS}
  bf16_seg = ({f"bf16_seg_reduce_kernel<{g},1,{a}>" for g in GS for a in ("true", "false")} |
              {f"bf16_seg_reduce_kernel<{g},2,{a}>" for g in (4, 8, 16) for a in ("true", "false")})
  fp32_apply = {apply_kernel(g, o, False) for g in GS for o in OPTS}
  for what, want, prefix in (("bf16 apply", bf16_apply, "bf16_runs_apply_kernel<"),
                             ("bf16 reduce", bf16_seg, "bf16_seg_reduce_kernel<"),
                             ("fp32 apply", fp32_apply, "runs_apply_kernel<")):
    got = {s for s in SEEN if s.startswith(prefix)}
    assert got == want, f"{what}: never ran {sorted(want - got)}; ran but not listed {sorted(got - want)}"
