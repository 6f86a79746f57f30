"""mono_mtable_pool_backward_parts: the fused backward over many features (parts) of several tables in one call.

Every comparison goes through uint32 views.  The reference point is the single-table pool_backward: the parts of one
table with one pooling must give exactly the bits of one pool_backward over their concatenated FIDs, stacked gradient
rows and rebased row offsets; mixed pooling is checked against the oracle fed tests/reduce_order.py's sums.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _cfg():
  from monolith_b200 import entry
  ini = entry.RandomUniformInitializer(-0.1, 0.1)
  return {
      "a8": table([(8, "adagrad", {"initial_accumulator_value": 0.1})], [0.05], capacity=4096, init=ini, init_seed=3),
      "b32": table([(32, "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01})], [0.05],
                   capacity=4096, init=ini, init_seed=4),
      "c128": table([(128, "adam", {})], [0.01], capacity=4096, init=ini, init_seed=5),
      "d16": table([(4, "ftrl", {}), (12, "adagrad", {"weight_decay_factor": 0.01})], [0.1, 0.05], capacity=4096,
                   init=[ini, ini], init_seed=6),
  }


def _fids(n, slot):
  return (np.int64(slot) << 48) | (np.arange(1, n + 1, dtype=np.int64) * 7919)


class Part:
  """One feature in host form: FIDs, CSR offsets (or None), pooling, gradient rows and the column they start at."""

  def __init__(self, slot, fids, offs, pooling, rows, col):
    self.slot, self.fids, self.offs, self.pooling, self.rows, self.col = slot, fids, offs, pooling, rows, col

  def n_rows(self):
    return self.fids.size if self.offs is None else self.offs.size - 1

  def to_pool_part(self, dev):
    from monolith_b200 import PoolPart
    return PoolPart(self.slot, T(self.fids, dev), None if self.offs is None else T(self.offs, dev), self.pooling,
                    T(self.rows, dev), self.col)

  def terms(self, D):
    """Per occurrence: the gradient row, divided by the row's n for a CSR MEAN part."""
    g = self.rows[:, self.col:self.col + D]
    if self.offs is None:
      return g.copy()
    n = np.diff(self.offs)
    row = np.repeat(np.arange(n.size), n)
    t = g[row]
    if self.pooling == "mean":
      t = (t / n[row].astype(np.float32)[:, None]).astype(np.float32)
    return t


def _make_part(rng, slot, D, fids, csr, pooling, wide):
  if csr:
    lens = rng.integers(1, 5, size=fids.size)
    lens = lens[:int(np.searchsorted(np.cumsum(lens), fids.size)) + 1]
    lens[-1] -= lens.sum() - fids.size
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  else:
    offs = None
  n_rows = fids.size if offs is None else offs.size - 1
  col = 4 if wide else 0
  rows = np.full((n_rows, D + (12 if wide else 0)), -7.25, np.float32)
  rows[:, col:col + D] = rng.standard_normal((n_rows, D)).astype(np.float32)
  return Part(slot, fids, offs, pooling, rows, col)


def _concat_single(t, slot, parts, dev, req_time):
  """The same batch as ONE pool_backward on table `slot`: FIDs concatenated, rows stacked, offsets rebased."""
  D = t.get_table_dim_sizes()[t.table_names.index(slot)]
  fids = np.concatenate([p.fids for p in parts])
  rows = np.concatenate([p.rows[:, p.col:p.col + D] for p in parts]).astype(np.float32)
  pooling = parts[0].pooling
  if all(p.offs is None for p in parts):
    offs = None
  else:
    lens = np.concatenate([np.ones(p.fids.size, np.int64) if p.offs is None else np.diff(p.offs) for p in parts])
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  t.pool_backward(slot, T(fids, dev), T(rows, dev), None if offs is None else T(offs, dev), pooling,
                  req_time=req_time)


def _entries(t, slot, keys, dev):
  return t.lookup_entry(slot, T(keys, dev))["raw"].cpu().numpy().view(np.uint32)


def _history(t, dev):
  """Same earlier history on both copies: a step, an eviction, and a step that reuses the freed rows."""
  rng = np.random.default_rng(11)
  for slot, D, s in (("a8", 8, 1), ("b32", 32, 2), ("c128", 128, 3), ("d16", 16, 4)):
    f = _fids(300, s)
    t.pool_backward(slot, T(f, dev), T(rng.standard_normal((300, D)).astype(np.float32), dev), req_time=5)
    t.pool_backward(slot, T(f[:100], dev), T(rng.standard_normal((100, D)).astype(np.float32), dev), req_time=9)
    t.evict(slot, 6)  # FIDs 100..299 go, their rows return to the free list
    nf = _fids(500, s)[400:]
    t.pool_backward(slot, T(nf, dev), T(rng.standard_normal((100, D)).astype(np.float32), dev), req_time=10)


def _step_parts(rng, dims, hot=True):
  """2-3 parts per table; the parts of a table share FIDs, bring new ones, and one hot FID (> 64 occurrences)
  is split across two parts."""
  parts = []
  for s, (slot, D) in enumerate(dims, start=1):
    pool = _fids(700, s)  # 0..99 resident, 100..299 evicted, 400..499 resident, the rest new
    pooling = "mean" if slot == "b32" else "sum"
    n_parts = 3 if slot in ("a8", "c128") else 2
    for i in range(n_parts):
      n = int(rng.integers(150, 400))
      f = pool[rng.integers(0, 700, n)]
      if hot and i < 2:
        f[rng.choice(n, 40, replace=False)] = pool[0]  # 80 occurrences of pool[0] across parts 0 and 1
      csr = pooling == "mean" or i == 1
      parts.append(_make_part(rng, slot, D, f, csr, pooling, wide=(i == 0)))
  return parts


DIMS = [("a8", 8), ("b32", 32), ("c128", 128), ("d16", 16)]


def _launches(lib):
  return lib.mono_kernel_launch_count()


def test_parts_equal_concatenated_single_table_calls(dev):
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  _history(ta, dev)
  _history(tb, dev)
  rng = np.random.default_rng(5)
  for step in range(2):
    parts = _step_parts(rng, DIMS)
    torch.cuda.synchronize()
    n0 = _launches(ta._lib)
    ta.pool_backward_parts([p.to_pool_part(dev) for p in parts], req_time=20 + step)
    torch.cuda.synchronize()
    n_parts_call = _launches(ta._lib) - n0
    n0 = _launches(tb._lib)
    for slot, _ in DIMS:
      _concat_single(tb, slot, [p for p in parts if p.slot == slot], dev, 20 + step)
    torch.cuda.synchronize()
    n_single = _launches(tb._lib) - n0
    # 1 occurrence map + claim + miss + finalize + 3 per radix pass + 3 run list, then reduce / finish / apply per table
    M = sum(p.fids.size for p in parts)
    per = {slot: sum(p.fids.size for p in parts if p.slot == slot) for slot, _ in DIMS}
    cap = sum(max(1024, 1 << int(np.ceil(np.log2(2 * m)))) for m in per.values())
    passes = max(1, -(-int(np.ceil(np.log2(cap))) // 11))
    assert M < 16384
    assert n_parts_call == 4 + 3 * passes + 3 + 3 * len(DIMS)
    assert n_parts_call < n_single
  for s, (slot, _) in enumerate(DIMS, start=1):
    keys = _fids(700, s)
    assert ta.size(slot) == tb.size(slot)
    np.testing.assert_array_equal(_entries(ta, slot, keys, dev), _entries(tb, slot, keys, dev))


def test_one_part_equals_pool_backward(dev):
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  rng = np.random.default_rng(7)
  for step in range(2):
    f = _fids(300, 2)[rng.integers(0, 300, 1000)]
    p = _make_part(rng, "b32", 32, f, True, "mean", wide=True)
    ta.pool_backward_parts([p.to_pool_part(dev)], req_time=3 + step)
    tb.pool_backward("b32", T(p.fids, dev), T(p.rows[:, 4:36], dev), T(p.offs, dev), "mean", req_time=3 + step)
  keys = _fids(300, 2)
  assert ta.size("b32") == tb.size("b32")
  np.testing.assert_array_equal(_entries(ta, "b32", keys, dev), _entries(tb, "b32", keys, dev))


def test_two_identical_runs_give_identical_bits(dev):
  from monolith_b200 import MultiHashTable
  out = []
  for _ in range(2):
    t = MultiHashTable(_cfg(), device=dev)
    rng = np.random.default_rng(9)
    for step in range(2):
      t.pool_backward_parts([p.to_pool_part(dev) for p in _step_parts(rng, DIMS)], req_time=30 + step)
    out.append([_entries(t, slot, _fids(700, s), dev) for s, (slot, _) in enumerate(DIMS, start=1)])
  for a, b in zip(*out):
    np.testing.assert_array_equal(a, b)


def test_mixed_pooling_and_tree_depths_match_the_oracle(dev):
  """Table `zbig` gets > 16384 occurrences (tree depth 1) from a SUM and a CSR MEAN part; the other table a few (depth
  0).  `zbig` sorts last, so its sorted range starts inside a piece of `small`'s.  Every entry must equal the oracle's, which is fed reduce_order's sums over the table's terms in part order."""
  from monolith_b200 import MultiHashTable, entry
  ini = entry.RandomUniformInitializer(-0.1, 0.1)
  cfg = {"zbig": table([(36, "adagrad", {"initial_accumulator_value": 0.1})], [0.05], capacity=4096, init=ini,
                      init_seed=1),
         "small": table([(20, "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01})],
                        [0.05], capacity=4096, init=ini, init_seed=2)}
  gpu, cpu = MultiHashTable(cfg, device=dev), orc.OracleMultiHashTable(cfg)
  rng = np.random.default_rng(13)
  vb, vs = _fids(3000, 1), _fids(200, 2)
  for step in range(2):
    fb1 = vb[rng.integers(0, 3000, 12000)]
    fb1[rng.choice(12000, 300, replace=False)] = vb[0]
    fb2 = vb[rng.integers(0, 3000, 9000)]
    fb2[rng.choice(9000, 200, replace=False)] = vb[0]  # 500 occurrences of vb[0]: blocks and the tree
    p1 = _make_part(rng, "zbig", 36, fb1, False, "sum", wide=True)
    p2 = _make_part(rng, "zbig", 36, fb2, True, "mean", wide=False)
    p3 = _make_part(rng, "small", 20, vs[rng.integers(0, 200, 300)], True, "mean", wide=False)
    gpu.pool_backward_parts([p1.to_pool_part(dev), p3.to_pool_part(dev), p2.to_pool_part(dev)], req_time=40 + step)
    for slot, D, ps in (("zbig", 36, [p1, p2]), ("small", 20, [p3])):
      terms = np.concatenate([p.terms(D) for p in ps])
      keys = np.concatenate([p.fids for p in ps])
      u, sums, length = ro.call_sums(terms, keys, ro.pick_group(D))
      assert (slot != "zbig") or ro.tree_top(ro.n_pieces(keys.size))[0] == 1
      cpu.apply_gradients({slot: (u, sums)}, req_time=40 + step)
      exact = np.zeros((u.size, D))
      np.add.at(exact, np.searchsorted(u, keys), terms.astype(np.float64))
      abs_sum = np.zeros((u.size, D))
      np.add.at(abs_sum, np.searchsorted(u, keys), np.abs(terms.astype(np.float64)))
      for i in np.flatnonzero(length > 64):
        bound = ro.error_bound(int(length[i]), ro.n_pieces(keys.size), ro.pick_group(D), abs_sum[i])
        assert np.all(np.abs(sums[i].astype(np.float64) - exact[i]) <= bound)
  for slot in ("zbig", "small"):
    keys = cpu.keys(slot)
    assert gpu.size(slot) == keys.size
    got = _entries(gpu, slot, keys, dev)
    want = cpu.lookup_entry(slot, keys).view(np.uint32)
    np.testing.assert_array_equal(got, want)


def test_admission_filter_counts_a_fid_once_per_call(dev):
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  for t in (ta, tb):
    t.set_hash_filter("a8", 1 << 16, 2)
  rng = np.random.default_rng(17)
  f = _fids(50, 1)
  for step in range(3):
    parts = [_make_part(rng, "a8", 8, f[:30].copy(), False, "sum", wide=False),
             _make_part(rng, "a8", 8, f[20:].copy(), True, "sum", wide=True)]
    ta.pool_backward_parts([p.to_pool_part(dev) for p in parts], req_time=50 + step)
    _concat_single(tb, "a8", parts, dev, 50 + step)
    assert ta.size("a8") == tb.size("a8")
    if step == 0:
      assert ta.size("a8") == 0  # every FID seen twice in the call, counted once: below the threshold
  np.testing.assert_array_equal(_entries(ta, "a8", f, dev), _entries(tb, "a8", f, dev))


def test_errors_leave_every_table_unchanged(dev):
  from monolith_b200 import MultiHashTable, _lib
  from monolith_b200._lib import MonoError, PoolPartC
  cfg = _cfg()
  cfg["e1"] = table([(1, "sgd", {})], [0.1], capacity=4096)
  t = MultiHashTable(cfg, device=dev)
  rng = np.random.default_rng(19)
  t.pool_backward_parts([p.to_pool_part(dev) for p in _step_parts(rng, DIMS, hot=False)], req_time=60)
  names = t.table_names
  before = {slot: (t.size(slot), _entries(t, slot, _fids(700, s), dev)) for s, (slot, _) in enumerate(DIMS, start=1)}
  f = T(_fids(64, 1), dev)
  g = torch.zeros(64, 136, dtype=torch.float32, device=dev)
  lr = t.learning_rates()
  lr_arr = (C.c_float * len(lr))(*lr)

  def call(**over):
    good = dict(table=names.index("a8"), fids_dev=f.data_ptr(), n_fids=64, row_offsets_dev=None, n_rows=64,
                pooling=_lib.POOL_SUM, rows_dev=g.data_ptr(), stride=136, col=0)
    good.update(over)
    arr = (PoolPartC * 2)(PoolPartC(**dict(good, table=names.index("b32"))), PoolPartC(**good))
    return t._lib.mono_mtable_pool_backward_parts(t.handle, arr, 2, lr_arr, 61, 0,
                                                  C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))

  assert call() == 0 and t.size("a8") >= 0  # the good call itself works
  before = {slot: (t.size(slot), _entries(t, slot, _fids(700, s), dev)) for s, (slot, _) in enumerate(DIMS, start=1)}
  cases = {
      "bad table": dict(table=len(names)),
      "negative table": dict(table=-1),
      "dim % 4": dict(table=names.index("e1")),
      "misaligned column": dict(col=1),
      "misaligned stride": dict(stride=135),
      "pooling": dict(pooling=_lib.POOL_FIRSTN),
      "over 2^30 occurrences": dict(n_fids=(1 << 30), n_rows=(1 << 30)),
  }
  for what, over in cases.items():
    assert call(**over) == -1, what
  with pytest.raises(MonoError, match="InvalidArgument"):
    t.pool_backward_parts([_make_part(rng, "e1", 1, _fids(8, 9), False, "sum", False).to_pool_part(dev)])
  torch.cuda.synchronize()
  for s, (slot, _) in enumerate(DIMS, start=1):
    assert t.size(slot) == before[slot][0]
    np.testing.assert_array_equal(_entries(t, slot, _fids(700, s), dev), before[slot][1])
  assert t.size("e1") == 0


# ------------------------------------------------------------------------------------------------
# forward: lookup_pool_parts
# ------------------------------------------------------------------------------------------------
FWD_DIMS = [1, 3, 8, 12, 32, 100, 128, 256, 512]


def test_forward_parts_match_lookup_pool_and_launch_once_per_kernel(dev):
  from monolith_b200 import MultiHashTable, PoolPart
  from tests.helpers import sgd_table
  from tests.test_gpu_forward_paths import traced
  names = [f"f{d:03d}" for d in FWD_DIMS]
  t = MultiHashTable({n: sgd_table(d, capacity=4096) for n, d in zip(names, FWD_DIMS)}, device=dev)
  rng = np.random.default_rng(23)
  for s_, (n, d) in enumerate(zip(names, FWD_DIMS), start=1):
    ids = _fids(500, s_)
    t.assign({n: (T(ids, dev), T(rng.standard_normal((500, d)).astype(np.float32), dev))})
  B = 64
  shared_w = 8 + 32 + 12 + 3
  specs = []  # (slot, fids, offs, pooling, buffer key, col)
  for s_, (n, d) in enumerate(zip(names, FWD_DIMS), start=1):
    pool = _fids(600, s_)  # 500..599 absent
    f = pool[rng.integers(0, 600, 3 * B)]
    lens = rng.integers(0, 6, B)
    lens[-1] += 3 * B - lens.sum() if lens.sum() < 3 * B else 0
    offs = np.minimum(np.concatenate([[0], np.cumsum(lens)]), 3 * B).astype(np.int32)
    specs.append((n, f, offs, "mean" if s_ % 2 else "sum", None, 0))
    specs.append((n, f[:B], None, "sum" if s_ % 2 else "mean", None, 0))
  for n, d in (("f032", 32), ("f128", 128)):  # packed rows: the TMA lookup serves these
    s_ = names.index(n) + 1
    specs.append((n, _fids(600, s_)[rng.integers(0, 600, B)], None, "sum", "exact", 0))
  col = 0
  for n, d in (("f008", 8), ("f032", 32), ("f012", 12), ("f003", 3)):  # disjoint columns of one tensor
    s_ = names.index(n) + 1
    f = _fids(600, s_)[rng.integers(0, 600, 2 * B)]
    specs.append((n, f, np.arange(0, 2 * B + 1, 2, dtype=np.int32), "mean", "shared", col))
    col += d

  def buffers():
    bufs = {"shared": torch.full((B, shared_w), -7.25, device=dev)}
    outs = []
    for n, f, offs, pooling, key, c in specs:
      d = FWD_DIMS[names.index(n)]
      outs.append(bufs["shared"] if key == "shared" else torch.full((B, d + (0 if key else 4)), -7.25, device=dev))
    return bufs, outs

  def parts(outs):
    return [PoolPart(n, T(f, dev), None if offs is None else T(offs, dev), pooling, outs[i],
                     c if key else 1 if FWD_DIMS[names.index(n)] % 4 else 0)
            for i, (n, f, offs, pooling, key, c) in enumerate(specs)]

  # reference: one lookup_pool per part, same output layout
  _, ref = buffers()

  def single():
    for p in parts(ref):
      t.lookup_pool(p.slot, p.fids, p.row_offsets, p.pooling, out=p.rows, out_col=p.col)

  _, want_names = traced(single)
  _, got = buffers()
  torch.cuda.synchronize()
  n0 = t._lib.mono_kernel_launch_count()
  t.lookup_pool_parts(parts(got))
  torch.cuda.synchronize()
  assert t._lib.mono_kernel_launch_count() - n0 == len(want_names)
  assert len(want_names) < len(specs)
  for a, b in zip(got, ref):
    np.testing.assert_array_equal(a.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32))
  _, again = buffers()
  _, got_names = traced(lambda: t.lookup_pool_parts(parts(again)))
  assert got_names == want_names
  for a, b in zip(again, ref):
    np.testing.assert_array_equal(a.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32))


def test_forward_parts_errors(dev):
  from monolith_b200 import MultiHashTable, PoolPart
  t = MultiHashTable(_cfg(), device=dev)
  f = T(_fids(8, 1), dev)
  with pytest.raises(KeyError):
    t.lookup_pool_parts([PoolPart("nope", f)])
  arr = (__import__("monolith_b200")._lib.PoolPartC * 1)()
  arr[0].table, arr[0].n_fids, arr[0].n_rows, arr[0].pooling = 99, 0, 0, 0
  assert t._lib.mono_mtable_lookup_pool_parts(t.handle, arr, 1, None) == -1
  arr[0].table, arr[0].pooling = 0, 2
  assert t._lib.mono_mtable_lookup_pool_parts(t.handle, arr, 1, None) == -1
  assert t._lib.mono_mtable_lookup_pool_parts(t.handle, arr, 1025, None) == -1
