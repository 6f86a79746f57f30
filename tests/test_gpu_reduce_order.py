"""The sparse backward's gradient reduction (csrc/bwd.cu: seg_reduce_kernel, tree_level_kernel, long_finish_kernel)
pinned bit for bit at every run length, row width and tree depth.

Each case goes through three gates:
  (a) exact    integer-valued gradients in [-3, 3] (never 0; MEAN rows have power-of-two lengths), so every partial
               sum is exact in fp32: the result equals the fp64 sum whatever the order.  Catches any dropped or doubled
               occurrence.
  (b) order    random normal gradients: the result is bit-equal to tests/reduce_order.py, the documented summation
               order (run length, lane group G = pick_group(dim), tree depth from the call's occurrence count).
  (c) accuracy the same result is within the model's fp64 error bound.
"""
import zlib

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import table

pytestmark = pytest.mark.gpu

DIMS = [4, 8, 12, 16, 20, 32, 36, 64, 100, 128]
SENTINEL = -7.25


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _grads(rng, shape, gate):
  """(a): nonzero integers in [-3, 3]; (b)/(c): standard normal."""
  if gate == "exact":
    return (rng.integers(1, 4, shape) * rng.choice([-1, 1], shape)).astype(np.float32)
  return rng.standard_normal(shape).astype(np.float32)


def _row_offsets(rng, M, gate):
  """CSR rows covering M occurrences; power-of-two lengths for the exact gate (x / 2^k stays exact)."""
  rl = rng.choice([1, 2, 4] if gate == "exact" else [1, 2, 3, 4, 5, 7], M)
  rl = rl[np.cumsum(rl) <= M]
  rl = np.concatenate([rl, np.ones(M - int(rl.sum()), rl.dtype)])
  return np.concatenate([[0], np.cumsum(rl)]).astype(np.int32)


def _occurrences(rng, lens):
  """Run index of every occurrence: run j has lens[j] occurrences at random positions."""
  return rng.permutation(np.repeat(np.arange(len(lens)), lens))


def _exact_and_abs(x, run_of, n_runs):
  """fp64 sums and sums of |x| per run."""
  x64 = x.astype(np.float64)
  s = np.zeros((n_runs,) + x.shape[1:])
  a = np.zeros((n_runs,) + x.shape[1:])
  order = np.argsort(run_of, kind="stable")
  heads = np.flatnonzero(np.concatenate([[True], np.diff(run_of[order]) != 0]))
  s[run_of[order][heads]] = np.add.reduceat(x64[order], heads, axis=0)
  a[run_of[order][heads]] = np.add.reduceat(np.abs(x64[order]), heads, axis=0)
  return s, a


def _check_bound(got, exact, abs_sum, lens, M, G):
  np_ = ro.n_pieces(M)
  ls, inv = np.unique(lens, return_inverse=True)
  gamma = np.array([ro.error_bound(int(L), np_, G, 1.0) for L in ls])
  bound = gamma[inv][:, None] * abs_sum
  err = np.abs(got.astype(np.float64) - exact)
  bad = np.argwhere(err > bound)
  assert bad.size == 0, f"{len(bad)} elements outside the fp64 bound, first: run {bad[0]} (len {lens[bad[0][0]]})"


def _bits_equal(got, want, lens, what):
  gb, wb = got.view(np.uint32), want.view(np.uint32)
  bad = np.flatnonzero((gb != wb).reshape(gb.shape[0], -1).any(1))
  assert bad.size == 0, (f"{what}: {bad.size} runs differ from the model, e.g. run {bad[0]} of length {lens[bad[0]]}: "
                         f"{got[bad[0]][:4]} vs {want[bad[0]][:4]}")


def _sort_passes(total_floats):
  bits = 1
  while (1 << bits) < (total_floats >> 2) + 1:
    bits += 1
  return max(1, (bits + 10) // 11)


# ------------------------------------------------------------------------------------------------
# mono_scatter_grad_rows: the sort key is the destination row, so run order and alignment are the test's
# ------------------------------------------------------------------------------------------------
def _boundary_lengths(G):
  per = ro.TREE_FAN * G // 32                          # tree members per lane group
  return [1, 2, 31, 32, 33, 63, 64, 65, 66, 95, 96, 97, 127, 128, 129,
          32 * per - 1, 32 * per, 32 * per + 1, 4095, 4096, 4097]


def _scatter_lens(case, D, rng):
  G = ro.pick_group(D)
  if case == "depth0":                                 # <= 16384 occurrences: no tree level, 1-pass sort
    lens = [1, 2, 31, 32, 33, 63, 64, 65, 66, 95, 96, 97, 127, 128, 129, 4095, 4096, 4097]
  elif case == "depth1":                               # one tree level, 2-pass sort
    lens = _boundary_lengths(G) + [16383, 16384, 16385] + list(rng.integers(1, 9, 3000))
  elif case == "offsets":                              # long runs starting at every offset mod 32
    lens, at = [], 0
    for o in range(32):
      filler = (o - at) % 32
      if filler:
        lens.append(filler)
        at += filler
      L = 65 + 37 * o
      lens.append(L)
      at += L
    lens += list(rng.integers(1, 5, 500))
  else:                                                # depth2: > 2^21 occurrences, runs of > 524 288
    lens = [17, 600000, 5, 524289, 65, 530001, 129, 4097, 33]
    fill = (1 << 21) + 4097 - sum(lens)
    short = rng.integers(1, 9, fill // 2)
    short = short[np.cumsum(short) <= fill]
    lens += list(short) + [1] * (fill - int(short.sum()))
  return np.asarray(lens, np.int64)


SCATTER_CASES = ([(c, D, p) for c in ("depth0", "depth1", "offsets") for D in DIMS for p in ("sum", "mean")] +
                 [("depth2", 4, "sum"), ("depth2", 20, "sum"), ("depth2", 4, "mean")])


@pytest.mark.parametrize("case,D,pooling", SCATTER_CASES, ids=lambda v: str(v))
def test_scatter_grad_rows_matches_the_model(case, D, pooling, dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(zlib.crc32(f"{case}/{D}/{pooling}".encode()))
  G = ro.pick_group(D)
  lens = _scatter_lens(case, D, rng)
  U = lens.size
  grad_col = 4 if case in ("offsets", "depth2") else 0        # a column slice of a wider gradient buffer
  # destination rows ascending (= run order) with unreferenced rows between them; the buffer size picks the sort depth
  total_rows = {"depth0": 2 * U, "depth1": 4 * U, "offsets": (1 << 24) // D + 8, "depth2": U + 8}[case]
  want_passes = {"depth0": 1, "depth1": 2, "offsets": 3, "depth2": 2}[case]
  assert _sort_passes(total_rows * D) == want_passes
  dest = np.sort(rng.choice(total_rows, U, replace=False))
  run_of = _occurrences(rng, lens)
  M = run_of.size
  eo = (dest[run_of] * D).astype(np.int32)
  unref = np.ones(total_rows, bool)
  unref[dest] = False
  for gate in ("exact", "order"):
    offs = _row_offsets(rng, M, gate) if pooling == "mean" else None
    R = M if offs is None else offs.size - 1
    wide = _grads(rng, (R, D + 2 * grad_col), gate)
    pg = wide[:, grad_col:grad_col + D]
    x = ro.occurrence_rows(pg, M, offs, pooling)
    outs = []
    for rep in range(2 if gate == "order" else 1):
      buf = torch.full((total_rows * D,), SENTINEL, device=dev)
      dops.scatter_grad_rows(T(wide, dev), T(eo, dev), D, buf, None if offs is None else T(offs, dev), pooling,
                             grad_col=grad_col)
      outs.append(buf.cpu().numpy().reshape(total_rows, D))
    out = outs[0]
    assert (out[unref] == SENTINEL).all(), "a row no occurrence refers to was written"
    got = out[dest]
    exact, abs_sum = _exact_and_abs(x, run_of, U)
    if gate == "exact":
      np.testing.assert_array_equal(got.astype(np.float64), exact)
      continue
    keys, want, length = ro.call_sums(x, run_of, G)
    assert np.array_equal(length, lens)
    _bits_equal(got, want, lens, f"scatter {case} D={D} {pooling}")
    _check_bound(got, exact, abs_sum, lens, M, G)
    np.testing.assert_array_equal(outs[1].view(np.uint32), out.view(np.uint32))   # a second call: same bits


# ------------------------------------------------------------------------------------------------
# mono_mtable_pool_backward: SGD lr 1 on a zero-initialised table makes every row minus its FID's summed gradient
# ------------------------------------------------------------------------------------------------
def _fid_lens(rng, M):
  if M >= (1 << 21):
    hot = [600000, 70000, 4097, 129, 65]
  elif M >= 16384:
    hot = [M // 4, 4097, 1000, 129, 65]
  elif M >= 512:
    hot = [M // 3, 97, 65]
  else:
    hot = [max(1, M // 2)]
  fill = M - sum(hot)
  short = rng.integers(1, 9, max(fill, 0) // 2 + 1)
  short = short[np.cumsum(short) <= fill]
  lens = np.asarray(hot + list(short) + [1] * (fill - int(short.sum())), np.int64)
  assert lens.sum() == M
  return lens


def _fids(n, slot=3):
  # distinct 40-bit signatures (odd multiplier mod 2^40 is a bijection)
  return (np.int64(slot) << 48) | ((np.arange(n, dtype=np.int64) * 2654435761 + 12345) & ((1 << 40) - 1))


POOL_SIZES = [(1, 36), (31, 20), (32, 100), (33, 12), (512, 36), (513, 20), (1024, 100), (1025, 4),
              (16384, 36), (16385, 20), (1 << 21, 4), ((1 << 21) + 4097, 8)]


@pytest.mark.parametrize("M,D", POOL_SIZES, ids=lambda v: str(v))
def test_pool_backward_sgd_row_is_minus_the_model_sum(M, D, dev):
  from monolith_b200 import MultiHashTable
  rng = np.random.default_rng(M * 7 + D)
  G = ro.pick_group(D)
  lens = _fid_lens(rng, M)
  run_of = _occurrences(rng, lens)
  u = _fids(lens.size)
  fids = u[run_of]
  for gate in ("exact", "order"):
    t = MultiHashTable({"t": table([(D, "sgd", {})], [1.0], capacity=lens.size)}, device=dev)
    pg = _grads(rng, (M, D), gate)
    t.pool_backward("t", T(fids, dev), T(pg, dev), None, "sum", req_time=5)
    got = -t.lookup({"t": T(u, dev)})["t"].cpu().numpy()
    assert t.size("t") == u.size
    exact, abs_sum = _exact_and_abs(pg, run_of, u.size)
    if gate == "exact":
      np.testing.assert_array_equal(got.astype(np.float64), exact)
      continue
    _, want, length = ro.call_sums(pg, run_of, G)
    assert np.array_equal(length, lens)
    _bits_equal(got, want, lens, f"pool_backward M={M} D={D}")
    _check_bound(got, exact, abs_sum, lens, M, G)


OPT_TABLES = [
    ("adagrad36", [(36, "adagrad", {"initial_accumulator_value": 0.1, "weight_decay_factor": 0.01})], [0.05]),
    ("ftrl20", [(20, "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01})], [0.05]),
    ("adam100", [(100, "adam", {})], [0.01]),
    ("multiseg16", [(4, "ftrl", {}), (12, "adagrad", {"weight_decay_factor": 0.01})], [0.1, 0.05]),
]


@pytest.mark.parametrize("M", [16000, 200000])
@pytest.mark.parametrize("case", OPT_TABLES, ids=lambda c: c[0])
def test_pool_backward_optimizer_entries_bit_exact(case, M, dev):
  """The oracle fed the model's per-FID sums: every entry (row, optimizer state, timestamps) bit for bit, hot
  FIDs included; two steps, so fresh and existing rows both go through the fused apply."""
  from monolith_b200 import MultiHashTable, entry
  _, segs, lrs = case
  D = sum(s[0] for s in segs)
  G = ro.pick_group(D)
  rng = np.random.default_rng(M + D)
  cfg = {"t": table(segs, lrs, capacity=256, init=entry.RandomUniformInitializer(-0.1, 0.1), init_seed=5)}
  gpu, cpu = MultiHashTable(cfg, device=dev), orc.OracleMultiHashTable(cfg)
  vocab = _fids(M)
  for step in range(2):
    lens = _fid_lens(rng, M)
    run_of = _occurrences(rng, lens)
    u = vocab[rng.choice(M, lens.size, replace=False)]
    fids = u[run_of]
    pg = rng.standard_normal((M, D)).astype(np.float32)
    gpu.pool_backward("t", T(fids, dev), T(pg, dev), None, "sum", req_time=10 + step)
    _, sums, _ = ro.call_sums(pg, run_of, G)
    cpu.apply_gradients({"t": (u, sums)}, req_time=10 + step)
  keys = cpu.keys("t")
  assert gpu.size("t") == keys.size
  got = gpu.lookup_entry("t", T(keys, dev))["raw"].cpu().numpy()
  want = cpu.lookup_entry("t", keys)
  bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)).any(1))
  assert bad.size == 0, f"{bad.size} entries differ, e.g. {keys[bad[0]]:#x}: {got[bad[0]][:4]} vs {want[bad[0]][:4]}"


# ------------------------------------------------------------------------------------------------
# owner grouping: reduce and reduce_push
# ------------------------------------------------------------------------------------------------
def _grouping_batch(rng, M):
  lens = np.concatenate([[20000, 4097, 1025, 513, 129, 97, 65], rng.integers(1, 9, 6000)])
  lens = lens[np.cumsum(lens) <= M]
  lens = np.concatenate([lens, np.ones(M - int(lens.sum()), np.int64)])
  run_of = _occurrences(rng, lens)
  return rng.integers(-2**62, 2**62, lens.size)[run_of]


@pytest.mark.parametrize("N", [1, 3, 8])
def test_grouping_reduce_matches_the_model(N, dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(100 + N)
  D, M = 36, 120000
  G = ro.pick_group(D)
  fids = _grouping_batch(rng, M)
  g = dops.Grouping(dev)
  uniq, offs, _ = g.build(T(fids, dev), N, D)
  u, o = uniq.cpu().numpy(), offs.cpu().numpy()
  run_of = o // D                                           # bucketed index of every occurrence's FID
  lens = np.bincount(run_of, minlength=u.size)
  assert lens.max() == 20000
  for gate in ("exact", "order"):
    pg = _grads(rng, (M, D), gate)
    got = g.reduce(T(pg, dev), torch.empty(u.size * D, device=dev)).cpu().numpy().reshape(-1, D)
    exact, abs_sum = _exact_and_abs(pg, run_of, u.size)
    if gate == "exact":
      np.testing.assert_array_equal(got.astype(np.float64), exact)
      continue
    _, want, _ = ro.call_sums(pg, run_of, G)
    _bits_equal(got, want, lens, f"grouping N={N}")
    _check_bound(got, exact, abs_sum, lens, M, G)


@pytest.mark.parametrize("pooling", ["sum", "mean"])
def test_grouping_reduce_push_long_runs_equal_reduce(pooling, dev):
  """reduce_push on a world-1 peer window stores the same bits as reduce, hot FIDs included."""
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(8)
  D, M = 20, 60000
  fids = _grouping_batch(rng, M)
  g = dops.Grouping(dev)
  uniq, offs, sizes = g.build(T(fids, dev), 1, D)
  U = uniq.numel()
  ro_ = _row_offsets(rng, M, "order") if pooling == "mean" else None
  R = M if ro_ is None else ro_.size - 1
  pg = T(rng.standard_normal((R, D + 8)).astype(np.float32), dev)
  ro_t = None if ro_ is None else T(ro_, dev)
  want = g.reduce(pg, torch.empty(U * D, device=dev), ro_t, pooling, grad_col=4).cpu().numpy()
  run_of = offs.cpu().numpy() // D
  x = ro.occurrence_rows(pg.cpu().numpy()[:, 4:4 + D], M, ro_, pooling)
  _, model, _ = ro.call_sums(x, run_of, ro.pick_group(D))
  _bits_equal(want.reshape(-1, D), model, np.bincount(run_of), "grouping reduce")
  w = dops.PeerWindow(dev, 1, 0, 1 << 23)
  try:
    g.reduce_push(pg, sizes, w, 1 << 20, [3], ro_t, pooling, grad_col=4)
    w.barrier()
    got = w.view((1 << 20) + 3 * D * 4, U * D, torch.float32).cpu().numpy()
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
  finally:
    w.close()


# ------------------------------------------------------------------------------------------------
# every knob setting gives the same bits
# ------------------------------------------------------------------------------------------------
KNOBS = [{"seg_vpl": 2}, {"seg_ahead": 0}, {"claim_pf": 1}, {"claim_dual": 1}, {"apply_pf": 1},
         {"seg_vpl": 2, "seg_ahead": 0, "claim_pf": 1, "claim_dual": 1, "apply_pf": 1}]


@pytest.mark.parametrize("D", [20, 36, 100])
def test_backward_knobs_give_identical_bits(D, dev):
  from monolith_b200 import MultiHashTable, _lib, distribution_ops as dops, entry
  lib = _lib.load()
  rng = np.random.default_rng(D)
  M = 60000
  lens = np.concatenate([[1, 2, 31, 32, 33, 63, 64, 65, 66, 97, 129, 4096, 4097, 20000], rng.integers(1, 9, 6000)])
  lens = lens[np.cumsum(lens) <= M]
  lens = np.concatenate([lens, np.ones(M - int(lens.sum()), np.int64)])
  run_of = _occurrences(rng, lens)
  u = _fids(lens.size, slot=4)
  fids = u[run_of]
  pg = rng.standard_normal((M, D)).astype(np.float32)
  offs = _row_offsets(rng, M, "order")
  pgw = rng.standard_normal((offs.size - 1, D + 8)).astype(np.float32)
  eo = (run_of * D).astype(np.int32)
  cfg = {"t": table([(D, "adagrad", {"initial_accumulator_value": 0.1})], [0.05],
                    init=entry.RandomUniformInitializer(-0.1, 0.1), init_seed=2)}

  def run():
    t = MultiHashTable(cfg, device=dev)
    for step in range(2):
      t.pool_backward("t", T(fids, dev), T(pg, dev), None, "sum", req_time=3 + step)
    entries = t.lookup_entry("t", T(u, dev))["raw"].cpu().numpy()
    buf = torch.full((lens.size * D,), SENTINEL, device=dev)
    sc = dops.scatter_grad_rows(T(pgw, dev), T(eo, dev), D, buf, T(offs, dev), "mean", grad_col=4).cpu().numpy()
    g = dops.Grouping(dev)
    uniq, _, _ = g.build(T(fids, dev), 3, D)
    red = g.reduce(T(pg, dev), torch.empty(uniq.numel() * D, device=dev)).cpu().numpy().reshape(-1, D)
    uq = uniq.cpu().numpy()   # the order inside a shard is the claim set's slot order: compare per FID
    by_fid = np.argsort(uq)
    return [entries.view(np.uint32), sc.view(np.uint32), uq[by_fid], red[by_fid].view(np.uint32)]

  base = run()
  x = ro.occurrence_rows(pgw[:, 4:4 + D], M, offs, "mean")
  _, model, _ = ro.call_sums(x, run_of, ro.pick_group(D))
  _bits_equal(base[1].view(np.float32).reshape(-1, D), model, lens, "scatter (default knobs)")
  names = sorted({k for s in KNOBS for k in s})
  old = {k: lib.mono_get_option(k.encode()) for k in names}
  try:
    for setting in KNOBS:
      for k in names:
        assert lib.mono_set_option(k.encode(), setting.get(k, old[k])) == 0
      for what, a, b in zip(("pool_backward entries", "scatter", "grouping uniq", "grouping reduce"), base, run()):
        assert np.array_equal(a, b), f"{setting}: {what} differs from the default knobs"
  finally:
    for k in names:
      lib.mono_set_option(k.encode(), old[k])
