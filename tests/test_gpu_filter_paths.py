"""The counting admission filter on every path that consults it, cell for cell against the oracle.

After every call `FWorld.check` compares each filtered table's whole cell array (MultiHashTable.hash_filter_cells)
with the oracle's, and then everything tests/test_gpu_write_paths.py's World.check compares (entries bit for bit,
export, counters).  The device and the oracle use the same mix64 cell layout, so the arrays must be equal wherever no
two FIDs of one call contend for a probe window: the cases build their FIDs (tests/filter_place.py) with pairwise
distinct start cells, or send the FIDs whose order matters one call at a time.  Gradients are small integers, so
every sum is exact in any order.  The rules the cases are aimed with are pinned in tests/test_filter_paths_cpu.py.
"""
import collections

import numpy as np
import pytest
import torch

from tests import filter_place as fp
from tests import orc
from tests import reduce_order as ro
from tests.helpers import table
from tests.test_gpu_forward_paths import _canon
from tests.test_gpu_write_paths import T, World

pytestmark = pytest.mark.gpu

I64 = np.iinfo(np.int64)
D = 8
T0 = 10 ** 6


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def cfg(names=("t",), capacity=1024):
  return {n: table([(D, "adagrad", {})], [0.1], capacity=capacity) for n in names}


def grads(rng, n):
  return rng.integers(-3, 4, (n, D)).astype(np.float32)


class FWorld(World):
  """World with admission filters: filters = {name: (capacity, default threshold, {slot: threshold})}."""

  def __init__(self, dev, filters, names=("t",), capacity=1024):
    super().__init__(dev, cfg(names, capacity), capacity)
    self.filters = {}
    for n, f in filters.items():
      self.set_filter(n, *f)

  def set_filter(self, n, capacity, thr, slot_thr=None):
    self.gpu.set_hash_filter(n, capacity, thr, slot_thr)
    self.cpu.set_hash_filter(n, capacity, thr, slot_thr)
    self.filters[n] = (capacity, thr, slot_thr)

  def cells(self, n):
    return self.gpu.hash_filter_cells(n)

  def check(self, **kw):
    for n in self.filters:
      np.testing.assert_array_equal(self.gpu.hash_filter_cells(n), self.cpu.hash_filter_cells(n),
                                    err_msg=f"table {n}: filter cells")
    super().check(**kw)

  def present(self, n, keys):
    got = self.gpu.contains(n, T(np.asarray(keys, np.int64), self.dev)).cpu().numpy()
    np.testing.assert_array_equal(got, self.cpu.contains(n, keys))
    return got

  def opt(self, n, keys, ts, rng, **kw):
    keys = np.asarray(keys, np.int64)
    self.optimize({n: (keys, grads(rng, keys.size))}, ts, **kw)

  def fused_call(self, n, shards, ts, rng, unique=True, accumulate=False):
    """shards: [keys] of table n (the only table)."""
    N = len(shards)
    ss = [len(s) for s in shards]
    ids = np.concatenate([np.asarray(s, np.int64) for s in shards])
    g = grads(rng, ids.size).reshape(-1)
    self.note({n: ids})
    _, _, ko, eo = self.gpu.fused_offsets(ss, N)
    ti = T(ids, self.dev)
    self.gpu.fused_apply_gradient(ti, ti, ss, T(g, self.dev), ko, eo, 0, ts, N, enable_grad_accumulation=accumulate,
                                  ids_unique=unique)
    self.cpu.fused_apply_gradient(ids, ss, g, N, req_time=ts, enable_grad_accumulation=accumulate)


def slot_keys(total, cells, slots, rng, sig=None):
  """One FID per cell, starting its probe there, in FID slot slots[i]."""
  return np.concatenate([fp.keys(total, c, 1, rng, sig=sig, slot=s) for c, s in zip(cells, slots)])


# ------------------------------------------------------------------------------------------------
# cell-level cases
# ------------------------------------------------------------------------------------------------
def test_counts_thresholds_and_saturation(dev):
  """Counts 0..15 and saturation; thresholds 1, 15, 16 (never admitted) and 0 (admitted at once, nothing counted), and
  the default 2; one call per count, the numpy filter replayed next to it."""
  rng = np.random.default_rng(1)
  cap = 1000
  total = fp.total_for(cap)
  thr = {1: 1, 2: 15, 3: 16, 4: 0}
  slots = np.repeat([1, 2, 3, 4, 5], 3)
  keys = slot_keys(total, rng.choice(total, slots.size, replace=False), slots, rng)
  w = FWorld(dev, {"t": (cap, 2, thr)})
  model, admitted = fp.Filter(cap), set()
  for call in range(20):
    w.opt("t", keys, T0 + call, rng, unique=True)
    for k, s in zip(keys.tolist(), slots.tolist()):
      if k not in admitted and not model.should_be_filtered(k, 1, thr.get(s, 2)):
        admitted.add(k)
    w.check()
    np.testing.assert_array_equal(w.cells("t"), model.cells)
    want = {1: call >= 1, 2: call >= 15, 3: False, 4: True, 5: call >= 2}
    np.testing.assert_array_equal(w.present("t", keys), [want[s] for s in slots.tolist()])
  for k in keys[slots == 3].tolist():
    assert model.get(k) == 15
  assert not model.cells[[int(fp.start_cell(k, total)) for k in keys[slots == 4]]].any()


def test_dedup_count_above_15(dev):
  """The dedup path hands the filter 1 + occ_extra occurrences: 20 clamps to 15 (admitted on the next call at
  threshold 15, never at 16); 3 occurrences at threshold 3 admit on the next call."""
  rng = np.random.default_rng(2)
  cap = 500
  total = fp.total_for(cap)
  keys = slot_keys(total, rng.choice(total, 3, replace=False), [1, 2, 3], rng)
  w = FWorld(dev, {"t": (cap, 3, {1: 15, 2: 16})})
  ids = np.concatenate([np.repeat(keys[:2], 20), np.repeat(keys[2:], 3)])
  rng.shuffle(ids)
  w.opt("t", ids, T0, rng, unique=False, dedup=True)
  w.check()
  assert not w.present("t", keys).any()
  c = w.cells("t")
  assert sorted(int(v) & 15 for v in c[c != 0]) == [3, 15, 15]
  w.opt("t", keys, T0 + 1, rng, unique=False, dedup=True)
  w.check()
  np.testing.assert_array_equal(w.present("t", keys), [True, False, True])


def test_full_window_and_spill_cells(dev):
  """64 FIDs holding the 64 cells of one window: a 65th FID starting there finds no cell, add returns 15 and it is
  admitted at once (threshold 15) with the cells unchanged.  Windows that start at the last cell run on into the 64
  spill cells past total."""
  rng = np.random.default_rng(3)
  cap = 200
  total = fp.total_for(cap)
  c0 = 100
  crowd = np.concatenate([fp.keys(total, c0 + i, 1, rng, sig=1 + i, slot=1) for i in range(64)])
  w = FWorld(dev, {"t": (cap, 3, {2: 15})})
  w.opt("t", crowd, T0, rng)
  w.check()
  before = w.cells("t")
  assert (before[c0:c0 + 64] != 0).all()
  newcomer = fp.keys(total, c0, 1, rng, sig=500, slot=2)
  w.opt("t", newcomer, T0 + 1, rng)
  w.check()
  np.testing.assert_array_equal(w.cells("t"), before)
  assert w.present("t", newcomer).all()
  # the last start cell: one FID per call (their order decides their cells)
  tail = np.concatenate([fp.keys(total, total - 1, 1, rng, sig=700 + i, slot=1) for i in range(4)])
  for i, k in enumerate(tail):
    w.opt("t", [k], T0 + 2 + i, rng)
    w.check()
  c = w.cells("t")
  assert (c[total - 1:total + 3] >> 4).tolist() == [700, 701, 702, 703]


def test_two_fids_share_one_counter(dev):
  """x and y share a start cell and a signature, so one counter: x (threshold 1) counts 2, then y (threshold 3) sees 2
  and is filtered, and is admitted on its second call."""
  rng = np.random.default_rng(4)
  cap = 300
  total = fp.total_for(cap)
  x = fp.keys(total, 77, 1, rng, sig=0x123, slot=1)
  y = fp.keys(total, 77, 1, rng, sig=0x123, slot=2)
  w = FWorld(dev, {"t": (cap, 2, {1: 1, 2: 3})})
  for call, (k, want) in enumerate([(x, False), (x, True), (y, False), (y, True)]):
    w.opt("t", k, T0 + call, rng)
    w.check()
    assert w.present("t", k)[0] == want, call
  assert int(w.cells("t")[77]) == (0x123 << 4) | 4


def test_signature_zero_negative_and_extreme_fids_many_slots(dev):
  rng = np.random.default_rng(5)
  cap = 100_000
  total = fp.total_for(cap)
  keys = np.concatenate([np.asarray([I64.min, I64.max, -1, 0, 1, I64.min + 1], np.int64),
                         -rng.integers(1, 1 << 62, 40, dtype=np.int64),
                         fp.keys(total, 5, 1, rng, sig=0), fp.keys(total, 9, 1, rng, sig=0, slot=0x7FFF)])
  starts = fp.start_cell(keys, total)
  assert np.unique(starts).size == keys.size
  slots = np.unique(((keys.view(np.uint64) >> np.uint64(48)) & np.uint64(0x7FFF)).astype(np.int64))
  thr = {int(s): int(rng.integers(0, 17)) for s in slots}
  thr.update({int(s): 3 for s in range(100, 140)})     # 40 more slots nobody uses
  w = FWorld(dev, {"t": (cap, 2, thr)})
  for call in range(17):
    w.opt("t", keys, T0 + call, rng)
    w.check()


@pytest.mark.parametrize("cap", [1, 2, 3, 1_000_003])
def test_capacities(cap, dev):
  """total = 1, 3, 4 and 1 500 004 cells; one FID per call, so the order of the adds is the oracle's."""
  rng = np.random.default_rng(cap)
  keys = rng.integers(I64.min, I64.max, 8, dtype=np.int64)
  w = FWorld(dev, {"t": (cap, 2, None)})
  assert w.cells("t").size == fp.n_cells(cap)
  for rep in range(3):
    for i, k in enumerate(keys):
      w.opt("t", [k], T0 + 10 * rep + i, rng)
      w.check()


def test_set_hash_filter_twice_resets(dev):
  rng = np.random.default_rng(6)
  cap = 1000
  total = fp.total_for(cap)
  keys = fp.distinct_start_keys(total, rng.choice(total, 50, replace=False), rng)
  w = FWorld(dev, {"t": (cap, 3, None)})
  for call in range(2):
    w.opt("t", keys[:30], T0 + call, rng)
    w.check()
  w.set_filter("t", cap, 3, None)
  assert not w.cells("t").any()
  for call in range(3):
    w.opt("t", keys, T0 + 10 + call, rng)
    w.check()


def test_two_filtered_tables_in_one_call(dev):
  rng = np.random.default_rng(7)
  w = FWorld(dev, {"a": (500, 2, None), "b": (700, 3, None)}, names=("a", "b"))
  ka = fp.distinct_start_keys(fp.total_for(500), rng.choice(fp.total_for(500), 80, replace=False), rng)
  kb = fp.distinct_start_keys(fp.total_for(700), rng.choice(fp.total_for(700), 80, replace=False), rng)
  for call in range(4):
    w.optimize({"a": (ka, grads(rng, ka.size)), "b": (kb, grads(rng, kb.size))}, T0 + call)
    w.check()


def test_concurrent_adds_to_both_halves_of_words(dev):
  """8000 FIDs in one call, every one with its own start cell and 4000 pairs in the two 16-bit halves of one word
  (the 32-bit CAS): the cells must equal the oracle's exactly, on the unique and the dedup path."""
  rng = np.random.default_rng(8)
  cap = 20_000
  total = fp.total_for(cap)
  words = rng.choice(total // 2, 4000, replace=False)
  keys = fp.distinct_start_keys(total, np.concatenate([2 * words, 2 * words + 1]), rng)
  w = FWorld(dev, {"t": (cap, 3, None)}, capacity=1 << 14)
  for call in range(3):
    w.opt("t", keys[rng.random(keys.size) < 0.8], T0 + call, rng)
    w.check()
  for call in range(2):
    ids = np.repeat(keys, rng.integers(1, 5, keys.size))
    rng.shuffle(ids)
    w.opt("t", ids, T0 + 5 + call, rng, unique=False, dedup=True)
    w.check()


# ------------------------------------------------------------------------------------------------
# every inserter on one scripted history
# ------------------------------------------------------------------------------------------------
PATHS = ["optimize-unique", "optimize-dup", "optimize-dedup", "assign-unique", "assign-dup", "assign_add-unique",
         "assign_add-dup", "fused-n1", "fused-n3-unique", "fused-n3-dup", "fused-n3-accumulate", "optimize_host",
         "pool_backward-sum", "pool_backward-csr_mean", "parts-fp32", "parts-bf16", "parts-two-features",
         "xstep-direct", "xstep-peer"]


def _host_optimize(w, keys, ts, rng):
  from monolith_b200 import _lib
  keys = np.ascontiguousarray(keys, np.int64)
  g = grads(rng, keys.size)
  w.note({"t": keys})
  split = np.asarray([0, keys.size], np.int64)
  lr = np.asarray(w.gpu.learning_rates(), np.float32)
  _lib.check(_lib.load().mono_mtable_optimize_host(w.gpu.handle, orc.p(keys), orc.p(split), orc.p(g.reshape(-1)),
                                                   orc.p(lr), ts, 0, _lib.FLAG_IDS_UNIQUE))
  w.cpu.apply_gradients({"t": (keys, g)}, req_time=ts)


def _pool_backward_mean(w, fids, ts, rng):
  lens = rng.integers(0, 4, fids.size)
  offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  offs = offs[offs <= fids.size]
  offs[-1] = fids.size
  pg = grads(rng, offs.size - 1)
  w.note({"t": fids})
  w.gpu.pool_backward("t", T(fids, w.dev), T(pg, w.dev), T(offs, w.dev), "mean", req_time=ts)
  x = ro.occurrence_rows(pg, fids.size, offs, "mean")
  u, ug, _ = ro.call_sums(x, fids, ro.pick_group(D))
  w.cpu.apply_gradients({"t": (u, ug)}, req_time=ts)


def _parts(w, parts, ts, dtype):
  from monolith_b200 import PoolPart
  w.note({"t": np.concatenate([f for f, _ in parts])})
  w.gpu.pool_backward_parts([PoolPart("t", T(f, w.dev), None, "sum", T(g, w.dev).to(dtype)) for f, g in parts],
                            req_time=ts)
  w.cpu.apply_gradients({"t": w._sums(np.concatenate([f for f, _ in parts]), np.concatenate([g for _, g in parts]))},
                        req_time=ts)


def _xstep(w, fids, ts, rng, exchange):
  from monolith_b200.distributed_ps import ShardedStep
  g = grads(rng, fids.size)
  w.note({"t": fids})
  st = ShardedStep(w.gpu, "t", D, 1, 0, w.dev, exchange=exchange)
  try:
    out = torch.empty(fids.size, D, device=w.dev)
    st.step(T(fids, w.dev), T(g, w.dev), out, ts, None, "sum")
    torch.cuda.synchronize()
  finally:
    if exchange == "direct":
      st.close_direct()
  w._cpu_sums("t", fids, g, ts)


@pytest.mark.parametrize("path", PATHS)
def test_path_matrix(path, dev):
  """120 FIDs with their own start cells in two FID slots (thresholds 2 and 3), six calls of one inserter with random
  subsets, repeats where the path takes them; cells and entries after every call."""
  rng = np.random.default_rng(zlib_crc(path))
  cap = 2000
  total = fp.total_for(cap)
  keys = slot_keys(total, rng.choice(total, 120, replace=False), np.repeat([1, 2], 60), rng)
  w = FWorld(dev, {"t": (cap, 2, {2: 3})})
  for call in range(6):
    ts = T0 + call
    sub = keys[rng.random(keys.size) < 0.7]
    dup = np.repeat(sub, rng.integers(1, 4, sub.size))
    rng.shuffle(dup)
    kind, _, var = path.partition("-")
    if kind in ("optimize", "assign", "assign_add"):
      ids = dup if var == "dup" or var == "dedup" else sub
      if kind == "optimize":
        w.opt("t", ids, ts, rng, unique=var == "unique", dedup=var == "dedup")
      else:
        w.assign({"t": (ids, grads(rng, ids.size))}, ts, unique=var == "unique", add=kind == "assign_add")
    elif kind == "fused":
      N = 1 if var == "n1" else 3
      shards = [keys[rng.random(keys.size) < 0.6] for _ in range(N)]
      if var == "n3-dup":
        shards = [np.repeat(s, rng.integers(1, 3, s.size)) for s in shards]
      w.fused_call("t", shards, ts, rng, unique=var in ("n1", "n3-unique"), accumulate=var == "n3-accumulate")
    elif kind == "optimize_host":
      _host_optimize(w, sub, ts, rng)
    elif kind == "pool_backward":
      if var == "sum":
        w.pool_backward("t", dup, grads(rng, dup.size), ts)
      else:
        _pool_backward_mean(w, dup, ts, rng)
    elif kind == "parts":
      half = dup.size // 2
      if var == "two-features":
        _parts(w, [(dup[:half], grads(rng, half)), (dup[half:], grads(rng, dup.size - half))], ts, torch.float32)
      else:
        _parts(w, [(dup, grads(rng, dup.size))], ts, torch.bfloat16 if var == "bf16" else torch.float32)
    else:
      _xstep(w, dup, ts, rng, var)
    w.check()
  assert w.present("t", keys).any()


def zlib_crc(s):
  import zlib
  return zlib.crc32(s.encode())


# ------------------------------------------------------------------------------------------------
# what leaves the filter alone
# ------------------------------------------------------------------------------------------------
def test_readers_restore_and_reinitialize_leave_the_cells(dev):
  rng = np.random.default_rng(9)
  cap = 1000
  total = fp.total_for(cap)
  keys = fp.distinct_start_keys(total, rng.choice(total, 60, replace=False), rng)
  w = FWorld(dev, {"t": (cap, 2, None)})
  for call in range(2):
    w.opt("t", keys[:40], T0 + call, rng)
  w.check()
  before = w.cells("t")
  tk = T(keys, dev)
  w.gpu.lookup({"t": tk})
  w.gpu.lookup_pool("t", tk, None, "sum")
  w.gpu.contains("t", tk)
  w.gpu.lookup_entry("t", tk)
  w.export("t")
  w.reinit("t", keys[30:50], T0 + 5)                   # inserts the absent ones without asking the filter
  rows = w.gpu.lookup_entry("t", T(keys[30:40], dev))["raw"].cpu().numpy()
  w.restore("t", keys[50:60], rows)
  torch.cuda.synchronize()
  np.testing.assert_array_equal(w.cells("t"), before)
  w.check()


def test_eviction_and_growth_leave_the_cells(dev):
  """Eviction removes entries, not counts: an evicted FID is admitted again at once.  Growth (rehash and row growth
  from a 16-row table) leaves the filter alone."""
  rng = np.random.default_rng(10)
  cap = 5000
  total = fp.total_for(cap)
  keys = fp.distinct_start_keys(total, rng.choice(total, 3000, replace=False), rng)
  w = FWorld(dev, {"t": (cap, 2, None)}, capacity=16)
  for call in range(3):
    w.opt("t", keys, T0 + call, rng)
    w.check()
  assert w.present("t", keys).all()
  before = w.cells("t")
  w.evict("t", T0 + 2 + 36500 * 86400)                 # the default expiry: every entry goes
  w.check()
  np.testing.assert_array_equal(w.cells("t"), before)
  assert not w.present("t", keys).any()
  w.opt("t", keys[:100], T0 + 3 + 36500 * 86400, rng)
  w.check()
  assert w.present("t", keys[:100]).all()


# ------------------------------------------------------------------------------------------------
# the defects these cases found
# ------------------------------------------------------------------------------------------------
def test_defect1_fused_shards_count_once_per_shard(dev):
  """Threshold 2, a new FID in shards 0, 1 and 2 of one fused optimize (ids unique per shard): the reference's
  per-shard BatchOptimize filters it twice and inserts it with shard 2's gradient; the filter counts 3."""
  rng = np.random.default_rng(11)
  cap = 300
  total = fp.total_for(cap)
  k = fp.keys(total, 10, 1, rng, slot=1)
  w = FWorld(dev, {"t": (cap, 2, None)})
  w.fused_call("t", [k, k, k], T0, rng)
  assert w.present("t", k).all()
  w.check()
  assert int(w.cells("t")[10]) & 15 == 3


@pytest.mark.parametrize("op", ["optimize", "assign"])
def test_defect2_optimize_duplicates_count_every_occurrence(op, dev):
  """x (threshold 1) four times in one non-unique call: every occurrence of an id absent at call start counts, so
  the shared counter reads 4, and y (same cell and signature, threshold 3) is admitted on its first call."""
  rng = np.random.default_rng(12)
  cap = 300
  total = fp.total_for(cap)
  x = fp.keys(total, 33, 1, rng, sig=0x321, slot=1)
  y = fp.keys(total, 33, 1, rng, sig=0x321, slot=2)
  w = FWorld(dev, {"t": (cap, 2, {1: 1, 2: 3})})
  ids = np.repeat(x, 4)
  if op == "optimize":
    w.opt("t", ids, T0, rng, unique=False)
  else:
    w.assign({"t": (ids, grads(rng, 4))}, T0, unique=False)
  assert w.present("t", x).all()
  w.opt("t", y, T0 + 1, rng) if op == "optimize" else w.assign({"t": (y, grads(rng, 1))}, T0 + 1)
  assert w.present("t", y).all(), "the shared counter missed occurrences of x after it was admitted"
  w.check()
  assert int(w.cells("t")[33]) == (0x321 << 4) | 5


# ------------------------------------------------------------------------------------------------
# launches: filter-less calls keep theirs
# ------------------------------------------------------------------------------------------------
FAMILY = ("resolve_hit_kernel", "miss_split_kernel", "absent_at_start_kernel", "dup_split_kernel")


def _launches(fn):
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  return collections.Counter(c.split("<")[0] for c in (_canon(e.name, FAMILY) for e in prof.events()) if c)


@pytest.mark.parametrize("filtered", [False, True])
def test_launches_with_and_without_a_filter(filtered, dev):
  """A fused optimize of 3 unique shards: one grouped resolve without a filter, one resolve per shard with one.  A
  duplicate optimize: the absent-at-start pass only with a filter."""
  rng = np.random.default_rng(13)
  w = FWorld(dev, {"t": (1000, 2, None)} if filtered else {})
  keys = fp.distinct_start_keys(fp.total_for(1000), rng.choice(fp.total_for(1000), 300, replace=False), rng)
  c = _launches(lambda: w.fused_call("t", [keys[:200], keys[100:], keys[50:250]], T0, rng))
  assert (c["resolve_hit_kernel"], c["miss_split_kernel"]) == ((3, 0) if filtered else (1, 1)), c
  ids = np.repeat(keys[:50], 3)
  c = _launches(lambda: w.opt("t", ids, T0 + 1, rng, unique=False))
  assert c["absent_at_start_kernel"] == (1 if filtered else 0) and c["dup_split_kernel"] == 3, c
  w.check()
