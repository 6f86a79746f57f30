"""FIRSTN (sequence) parts of lookup_pool_parts and pool_backward_parts, bit for bit.

Forward: every position equals tests/test_seq_parts_cpu.firstn_place over the oracle's rows (the placement is pinned
there on the reference's numpy pooling oracle), with the exact lookup_seq_kernel instantiation checked through
torch.profiler.  Backward: a FIRSTN part must give exactly the bits of the one-FID-per-row SUM part whose gradient
rows are test_seq_parts_cpu.firstn_terms (ScatterGrad's FIRSTN branch), and the oracle fed reduce_order's sums.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import sgd_table, table
from tests.test_gpu_forward_paths import assert_bits, basic, k_lookup, k_pool, pick_group, queries, traced
from tests.test_gpu_pool_parts import DIMS, _cfg, _entries, _fids, _history
from tests.test_seq_parts_cpu import firstn_place, firstn_terms

pytestmark = pytest.mark.gpu

SEQ = ("lookup_seq_kernel",)
SEEN = set()


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def k_seq(d, confirm):
  return f"lookup_seq_kernel<{pick_group(d)},{'true' if confirm else 'false'}>"


def run_one(lib, fn, expect):
  """fn() -> numpy arrays, from exactly one kernel launch (the engine's launch counter), which torch.profiler must
  name `expect`; run twice, identical bits.  In a long process the profiler at times records no kernel in many
  traces in a row (records are lost whole, never invented): the case is traced up to ten times, any kernel other
  than `expect` fails at once, and a case whose traces all came back empty rests on the launch counter (the final
  test still requires every instantiation to have been named)."""
  for _ in range(10):
    torch.cuda.synchronize()
    n0 = lib.mono_kernel_launch_count()
    out, names = traced(fn, SEQ)
    assert lib.mono_kernel_launch_count() - n0 == 1
    assert names <= {expect}, f"ran {sorted(names)}, aimed at {expect}"
    if names:
      SEEN.add(expect)
      break
  for a, b in zip(out, fn()):
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32), err_msg="not bit-stable run to run")
  return out


def seq_offs(rng, n_rows, L):
  """Row lengths 0 .. L + 8: empty, short, exactly L and truncated rows."""
  lens = rng.integers(0, L + 9, n_rows)
  lens[:4] = [0, L, L + 8, 1][:min(4, n_rows)]
  return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


# ------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [1, 5, 64])
@pytest.mark.parametrize("dim", [1, 3, 8, 12, 16, 32, 64, 100, 128, 256, 512])
def test_forward_places_the_oracle_rows(dim, L, dev):
  from monolith_b200 import PoolPart
  p, keys, absent, rng = basic(dev, dim, seed=L)
  n_rows = 300 if L < 64 else 60
  offs = seq_offs(rng, n_rows, L)
  fids = queries(rng, keys, absent, int(offs[-1]))
  col = 3 if dim % 4 else 4
  width = col + L * dim + 5
  want = np.full((n_rows, width), -7.25, np.float32)
  want[:, col:col + L * dim] = firstn_place(p.cpu.lookup({"t": fids})["t"], offs, L).reshape(n_rows, -1)
  one = queries(rng, keys, absent, n_rows)  # without offsets: one FID per row, positions 1.. are zeros
  want1 = firstn_place(p.cpu.lookup({"t": one})["t"], None, L).reshape(n_rows, -1)

  def call():
    out = torch.full((n_rows, width), -7.25, device=dev)
    outs = p.gpu.lookup_pool_parts([PoolPart("t", T(fids, dev), T(offs, dev), "firstn", out, col, max_seq_len=L),
                                    PoolPart("t", T(one, dev), pooling="firstn", max_seq_len=L)])
    return tuple(o.cpu().numpy() for o in outs)

  got = run_one(p.gpu._lib, call, k_seq(dim, False))
  assert_bits(got[0], want)   # sentinel columns untouched
  assert_bits(got[1], want1)
  side = torch.cuda.Stream(dev)

  def on_side():
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
      r = call()
    torch.cuda.current_stream(dev).wait_stream(side)
    return r

  got = run_one(p.gpu._lib, on_side, k_seq(dim, True))
  assert_bits(got[0], want)
  assert_bits(got[1], want1)


def test_mixed_forward_call_equals_each_part_alone(dev):
  from monolith_b200 import MultiHashTable, PoolPart
  dims = {"s16": 16, "s32": 32, "s3": 3}
  t = MultiHashTable({n: sgd_table(d, capacity=4096) for n, d in dims.items()}, device=dev)
  rng = np.random.default_rng(31)
  for s, (n, d) in enumerate(dims.items(), start=1):
    t.assign({n: (T(_fids(500, s), dev), T(rng.standard_normal((500, d)).astype(np.float32), dev))})
  B = 128
  specs = []
  for s, (n, d) in enumerate(dims.items(), start=1):
    pool = _fids(600, s)
    offs = seq_offs(rng, B, 20)
    specs.append((n, pool[rng.integers(0, 600, int(offs[-1]))], offs, "firstn", 20))
    specs.append((n, pool[rng.integers(0, 600, B)], None, "sum", 0))
    offs2 = seq_offs(rng, B, 3)
    specs.append((n, pool[rng.integers(0, 600, int(offs2[-1]))], offs2, "mean", 0))
  specs.append(("s32", _fids(600, 2)[rng.integers(0, 600, 2 * B)], None, "firstn", 7))

  def parts():
    return [PoolPart(n, T(f, dev), None if o is None else T(o, dev), pl, max_seq_len=L) for n, f, o, pl, L in specs]

  # the instantiation of each part (test_gpu_forward_paths' dispatch rules): one launch per distinct one
  plans = {k_seq(dims[n], False) if pl == "firstn" else k_lookup(dims[n]) if o is None else k_pool(dims[n])
           for n, f, o, pl, L in specs}
  alone = [t.lookup_pool_parts([p])[0].cpu().numpy() for p in parts()]
  torch.cuda.synchronize()
  n0 = t._lib.mono_kernel_launch_count()
  got = t.lookup_pool_parts(parts())
  torch.cuda.synchronize()
  assert t._lib.mono_kernel_launch_count() - n0 == len(plans) < len(specs)
  for a, b in zip(got, alone):
    assert_bits(a.cpu().numpy(), b)


# ------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------
def seq_batch(rng, pool, n_rows, L, D, hot=None, beyond=None, wide=False):
  """FIDs, offsets and [n_rows, L*D] gradients (col 4 of a wider buffer when `wide`) of a FIRSTN part; `hot` gets
  > 64 occurrences inside sequences, `beyond` FIDs occur only at positions >= L."""
  offs = seq_offs(rng, n_rows, L)
  fids = pool[rng.integers(0, pool.size, int(offs[-1]))]
  lens = np.diff(offs)
  pos = np.arange(fids.size) - np.repeat(offs[:-1], lens)
  if beyond is not None:
    fids[np.isin(fids, beyond)] = pool[0]
    at = np.flatnonzero(pos >= L)
    fids[at[:beyond.size * 3]] = np.resize(beyond, min(at.size, beyond.size * 3))
  if hot is not None:
    at = np.flatnonzero(pos < L)
    fids[rng.choice(at, 80, replace=False)] = hot
  col = 4 if wide else 0
  g = np.full((n_rows, col + L * D + (8 if wide else 0)), -7.25, np.float32)
  g[:, col:col + L * D] = rng.standard_normal((n_rows, L * D)).astype(np.float32)
  return fids, offs, g, col


def firstn_part(slot, fids, offs, g, col, L, dev):
  from monolith_b200 import PoolPart
  return PoolPart(slot, T(fids, dev), T(offs, dev), "firstn", T(g, dev), col, max_seq_len=L)


def sum_part(slot, fids, terms, dev):
  from monolith_b200 import PoolPart
  return PoolPart(slot, T(fids, dev), None, "sum", T(terms, dev))


def seq_terms(fids, offs, g, col, L, D):
  return firstn_terms(g[:, col:col + L * D].reshape(-1, L, D), offs, L, fids.size)


def test_backward_equals_the_materialised_sum_part(dev):
  """Per table of test_gpu_pool_parts._cfg (Adagrad, FTRL, Adam, multi-segment), after its eviction history: one
  FIRSTN part with a hot FID and FIDs only beyond L, plus a SUM part of the same table in the same call."""
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  _history(ta, dev)
  _history(tb, dev)
  rng = np.random.default_rng(37)
  L = 5
  for step in range(2):
    pa, pb, beyond_all = [], [], {}
    for s, (slot, D) in enumerate(DIMS, start=1):
      pool = _fids(700, s)
      beyond = _fids(900, s)[800 + 10 * step:810 + 10 * step]   # new FIDs, never within the first L positions
      fids, offs, g, col = seq_batch(rng, pool, 200, L, D, hot=pool[1], beyond=beyond, wide=(s % 2 == 0))
      assert np.isin(beyond, fids).all()
      sf = pool[rng.integers(0, 700, 150)]
      sg = rng.standard_normal((150, D)).astype(np.float32)
      pa += [firstn_part(slot, fids, offs, g, col, L, dev), sum_part(slot, sf, sg, dev)]
      pb += [sum_part(slot, fids, seq_terms(fids, offs, g, col, L, D), dev), sum_part(slot, sf, sg, dev)]
      beyond_all[slot] = beyond
    ta.pool_backward_parts(pa, req_time=70 + step)
    tb.pool_backward_parts(pb, req_time=70 + step)
    for slot, b in beyond_all.items():
      assert ta.contains(slot, T(b, dev)).all()
  for s, (slot, _) in enumerate(DIMS, start=1):
    keys = np.concatenate([_fids(700, s), _fids(900, s)[800:]])
    assert ta.size(slot) == tb.size(slot)
    np.testing.assert_array_equal(_entries(ta, slot, keys, dev), _entries(tb, slot, keys, dev))


def test_backward_matches_the_oracle_at_tree_depth_1(dev):
  """> 16384 occurrences of one table (FIRSTN + SUM): the oracle gets reduce_order's sums over the terms; FIDs that
  occur only beyond L must be found with ts = req_time and the values of a zero-gradient step."""
  from monolith_b200 import MultiHashTable, entry
  ini = entry.RandomUniformInitializer(-0.1, 0.1)
  cfg = {"seq": table([(36, "adagrad", {"initial_accumulator_value": 0.1})], [0.05], capacity=4096, init=ini,
                      init_seed=1)}
  gpu, cpu = MultiHashTable(cfg, device=dev), orc.OracleMultiHashTable(cfg)
  rng = np.random.default_rng(41)
  D, L = 36, 12
  pool = _fids(3000, 1)
  for step in range(2):
    beyond = _fids(4000, 1)[3500 + 20 * step:3520 + 20 * step]
    fids, offs, g, col = seq_batch(rng, pool, 1500, L, D, hot=pool[2], beyond=beyond, wide=True)
    sf = pool[rng.integers(0, 3000, 4000)]
    sg = rng.standard_normal((4000, D)).astype(np.float32)
    gpu.pool_backward_parts([firstn_part("seq", fids, offs, g, col, L, dev), sum_part("seq", sf, sg, dev)],
                            req_time=80 + step)
    keys = np.concatenate([fids, sf])
    terms = np.concatenate([seq_terms(fids, offs, g, col, L, D), sg])
    assert keys.size > 16384 and ro.tree_top(ro.n_pieces(keys.size))[0] == 1
    u, sums, _ = ro.call_sums(terms, keys, ro.pick_group(D))
    cpu.apply_gradients({"seq": (u, sums)}, req_time=80 + step)
    assert gpu.contains("seq", T(beyond, dev)).all()
  keys = cpu.keys("seq")
  assert gpu.size("seq") == keys.size
  np.testing.assert_array_equal(_entries(gpu, "seq", keys, dev), cpu.lookup_entry("seq", keys).view(np.uint32))


def test_admission_filter_counts_a_fid_seen_only_beyond_L(dev):
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  for t in (ta, tb):
    t.set_hash_filter("a8", 1 << 16, 2)
  rng = np.random.default_rng(43)
  pool, beyond = _fids(40, 1), _fids(60, 1)[50:]
  L = 3
  for step in range(3):
    fids, offs, g, col = seq_batch(rng, pool, 60, L, 8, beyond=beyond)
    assert all((fids == b).sum() >= 2 for b in beyond)   # several occurrences, one count per call
    ta.pool_backward_parts([firstn_part("a8", fids, offs, g, col, L, dev)], req_time=90 + step)
    tb.pool_backward_parts([sum_part("a8", fids, seq_terms(fids, offs, g, col, L, 8), dev)], req_time=90 + step)
    assert ta.size("a8") == tb.size("a8")
    present = ta.contains("a8", T(beyond, dev)).cpu().numpy()
    if step == 0:
      assert not present.any()   # seen in one call: counted once, below the threshold
  assert present.all()
  keys = np.concatenate([pool, beyond])
  np.testing.assert_array_equal(_entries(ta, "a8", keys, dev), _entries(tb, "a8", keys, dev))


def test_errors_leave_every_table_unchanged(dev):
  from monolith_b200 import MultiHashTable, PoolPart, _lib
  from monolith_b200._lib import PoolPartC
  cfg = _cfg()
  cfg["e1"] = table([(1, "sgd", {})], [0.1], capacity=4096)
  cfg["e132"] = table([(132, "sgd", {})], [0.1], capacity=4096)
  t = MultiHashTable(cfg, device=dev)
  rng = np.random.default_rng(47)
  fids, offs, g, col = seq_batch(rng, _fids(300, 1), 64, 4, 8)
  t.pool_backward_parts([firstn_part("a8", fids, offs, g, col, 4, dev)], req_time=100)
  names = t.table_names
  f, o = T(fids, dev), T(offs, dev)
  gd = torch.zeros(64, 4 * 132 + 8, dtype=torch.float32, device=dev)
  lr = t.learning_rates()
  lr_arr = (C.c_float * len(lr))(*lr)
  stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

  def arr(**over):
    good = dict(table=names.index("a8"), fids_dev=f.data_ptr(), n_fids=fids.size, row_offsets_dev=o.data_ptr(),
                n_rows=64, pooling=_lib.POOL_FIRSTN, rows_dev=gd.data_ptr(), stride=gd.shape[1], col=0, max_seq_len=4)
    good.update(over)
    return (PoolPartC * 2)(PoolPartC(**dict(good, table=names.index("b32"), pooling=_lib.POOL_SUM, max_seq_len=0,
                                            row_offsets_dev=None, n_fids=64)), PoolPartC(**good))

  def bwd(**over):
    return t._lib.mono_mtable_pool_backward_parts(t.handle, arr(**over), 2, lr_arr, 101, 0, stream)

  def fwd(**over):
    return t._lib.mono_mtable_lookup_pool_parts(t.handle, arr(**over), 2, stream)

  before = {n: (t.size(n), _entries(t, n, _fids(300, s), dev)) for s, n in enumerate(names, start=1)}
  big = dict(n_rows=1 << 20, n_fids=1 << 20, row_offsets_dev=None, max_seq_len=1 << 12)  # 2^32 slots
  cases = {"max_seq_len 0": dict(max_seq_len=0), "max_seq_len < 0": dict(max_seq_len=-2), "n_rows * L": big}
  for what, over in cases.items():
    assert bwd(**over) == -1, what
    assert fwd(**over) == -1, what
  for what, over in {"dim % 4": dict(table=names.index("e1")), "dim > 128": dict(table=names.index("e132")),
                     "misaligned column": dict(col=1), "misaligned stride": dict(stride=gd.shape[1] - 1)}.items():
    assert bwd(**over) == -1, what
  torch.cuda.synchronize()
  for s, n in enumerate(names, start=1):
    assert t.size(n) == before[n][0], n
    np.testing.assert_array_equal(_entries(t, n, _fids(300, s), dev), before[n][1])
  # max_seq_len is not read for SUM / MEAN parts
  outs = []
  for junk in (0, 12345):
    tt = MultiHashTable(_cfg(), device=dev)
    _history(tt, dev)
    r = np.random.default_rng(5)
    sf = T(_fids(300, 2)[r.integers(0, 300, 256)], dev)
    sg = T(r.standard_normal((256, 32)).astype(np.float32), dev)
    out = torch.empty(256, 32, device=dev)
    kw = dict(table=tt.table_names.index("b32"), fids_dev=sf.data_ptr(), n_fids=256, row_offsets_dev=None, n_rows=256,
              pooling=_lib.POOL_SUM, stride=32, col=0, max_seq_len=junk)
    lr2 = tt.learning_rates()
    assert tt._lib.mono_mtable_lookup_pool_parts(tt.handle, (PoolPartC * 1)(PoolPartC(rows_dev=out.data_ptr(), **kw)),
                                                 1, stream) == 0
    assert tt._lib.mono_mtable_pool_backward_parts(tt.handle, (PoolPartC * 1)(PoolPartC(rows_dev=sg.data_ptr(), **kw)),
                                                   1, (C.c_float * len(lr2))(*lr2), 110, 0, stream) == 0
    torch.cuda.synchronize()
    outs.append((out.cpu().numpy().view(np.uint32), _entries(tt, "b32", _fids(700, 2), dev)))
  for x, y in zip(*outs):
    np.testing.assert_array_equal(x, y)


def test_every_seq_instantiation_ran():
  """Runs last in this file: the forward cases above launched all 8 lookup_seq_kernel instantiations."""
  assert SEEN == {f"lookup_seq_kernel<{g},{c}>" for g in (4, 8, 16, 32) for c in ("false", "true")}
