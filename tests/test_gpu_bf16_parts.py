"""bf16 rows in lookup_pool_parts / pool_backward_parts (the *_parts_bf16 calls), bit for bit.

Forward: every bf16 output equals the fp32 call's output .to(torch.bfloat16) (round to nearest even, pinned in
test_bf16_parts_cpu.py), NaN positions compared with isnan; the kernels each call launches are the stated bf16
instantiations.  Backward: on twin tables, the bf16 call must give exactly the bits of the fp32 call on the rows
widened to float32.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.helpers import sgd_table, table
from tests.test_gpu_forward_paths import basic, pick_group, queries, traced
from tests.test_gpu_pool_parts import DIMS, _cfg, _entries, _fids, _history, _step_parts
from tests.test_gpu_seq_parts import seq_batch, seq_offs

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FWD = ("bf16_lookup_kernel", "bf16_pool_staged_kernel", "bf16_pool_kernel", "bf16_seq_kernel")
GS = (4, 8, 16, 32)
POOL_VARIANTS = ((4, 1, 4), (8, 1, 4), (16, 1, 4), (32, 1, 4), (32, 2, 2), (32, 4, 1))
SEEN = set()
FWD_DIMS = [1, 3, 8, 12, 32, 64, 100, 128, 256, 512]


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def tf(c):
  return "true" if c else "false"


def kb_lookup(d, confirm):
  return f"bf16_lookup_kernel<{pick_group(d)},{tf(confirm)}>"


def kb_seq(d, confirm):
  return f"bf16_seq_kernel<{pick_group(d)},{tf(confirm)}>"


def kb_pool(d, staged_ok):
  g = pick_group(d)
  if staged_ok and d % 4 == 0 and d <= 128:
    return f"bf16_pool_staged_kernel<{g}>"
  nv = -(-d // (4 * g))
  v = (g, 1, 4) if g < 32 else {1: (32, 1, 4), 2: (32, 2, 2)}.get(nv, (32, 4, 1))
  return "bf16_pool_kernel<%d,%d,%d>" % v


def assert_bf16_bits(got, want):
  """bf16 tensors equal bit for bit, NaN positions by isnan (the payload is not specified)."""
  gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
  assert torch.equal(gn, wn)
  g, w = got.view(torch.int16).clone(), want.view(torch.int16).clone()
  g[gn] = 0
  w[wn] = 0
  mism = (g != w).nonzero()
  assert mism.numel() == 0, f"{mism.shape[0]} elements differ, first at {mism[0].tolist()}"


def run_fwd(lib, fn, expect):
  """fn() -> outputs, from exactly len(expect) kernel launches; the profiler, when it recorded anything (records are
  lost whole at times, see NOTES.md), must name exactly `expect`.  Run twice: identical bits."""
  for _ in range(10):
    torch.cuda.synchronize()
    n0 = lib.mono_kernel_launch_count()
    out, names = traced(fn, FWD)
    assert lib.mono_kernel_launch_count() - n0 == len(expect)
    assert names <= expect, f"ran {sorted(names)}, aimed at {sorted(expect)}"
    if names:
      assert names == expect
      SEEN.update(names)
      break
  for a, b in zip(out, fn()):
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "not bit-stable run to run"
  return out


# ------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [1, 5, 64])
@pytest.mark.parametrize("dim", FWD_DIMS)
def test_forward_equals_fp32_rounded(dim, L, dev):
  """One call per stream: a one-FID part into a new tensor, a CSR SUM part and a one-FID part in disjoint columns of
  one 4-aligned tensor, a CSR MEAN part and a one-FID part at odd stride and column (scalar stores), and a FIRSTN part;
  absent FIDs throughout, sentinel columns around every part."""
  from monolith_b200 import PoolPart
  p, keys, absent, rng = basic(dev, dim, seed=L + 100)
  t = p.gpu
  n = 300 if L < 64 else 60
  one = queries(rng, keys, absent, n)
  offs = seq_offs(rng, n, 6)
  csr = queries(rng, keys, absent, int(offs[-1]))
  offs_s = seq_offs(rng, n, L)
  seq = queries(rng, keys, absent, int(offs_s[-1]))
  ca = 4
  cb = ca + ((dim + 3) // 4) * 4 + 4
  wa = cb + dim + 8                       # multiple of 4 when dim is
  wa += (-wa) % 4
  cc, wb = 3, 3 + 2 * dim + 6             # odd column; odd stride
  wb += 1 - wb % 2
  cd = cc + dim + 1
  cs = 4 if dim % 4 == 0 else 3           # FIRSTN: vector stores when dim % 4 == 0, scalar ones otherwise

  def call(dtype):
    a = torch.full((n, wa), -7.25, device=dev, dtype=dtype)
    b = torch.full((n, wb), -7.25, device=dev, dtype=dtype)
    s = torch.full((n, cs + L * dim + cs), -7.25, device=dev, dtype=dtype)
    parts = [PoolPart("t", T(one, dev)),
             PoolPart("t", T(csr, dev), T(offs, dev), "sum", a, ca), PoolPart("t", T(one, dev), rows=a, col=cb),
             PoolPart("t", T(csr, dev), T(offs, dev), "mean", b, cc), PoolPart("t", T(one, dev), rows=b, col=cd),
             PoolPart("t", T(seq, dev), T(offs_s, dev), "firstn", s, cs, max_seq_len=L)]
    outs = t.lookup_pool_parts(parts, dtype=dtype)
    return (outs[0], a, b, s)

  want = [o.to(BF) for o in call(torch.float32)]
  for confirm in (False, True):
    staged_ok = dim % 4 == 0
    expect = {kb_lookup(dim, confirm), kb_pool(dim, staged_ok), kb_pool(dim, False), kb_seq(dim, confirm)}
    if not confirm:
      got = run_fwd(t._lib, lambda: call(BF), expect)
    else:
      side = torch.cuda.Stream(dev)

      def on_side():
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
          r = call(BF)
        torch.cuda.current_stream(dev).wait_stream(side)
        return r
      got = run_fwd(t._lib, on_side, expect)
    for g, w in zip(got, want):
      assert g.dtype == BF
      assert_bf16_bits(g, w)


def test_forward_edge_values(dev):
  """Rows whose values, sums and means land on bf16 ties, overflow to inf, are subnormal, -0.0, inf or NaN."""
  from monolith_b200 import MultiHashTable, PoolPart
  u = lambda x: np.uint32(x).view(np.float32)  # noqa: E731
  edges = np.array([u(0x3F808000), u(0x3F818000), u(0x3F808001), np.finfo(np.float32).max, u(0x7F7F8000),
                    u(0x7F7F7FFF), u(0x00000001), u(0x00018000), u(0x00010000), -0.0, np.inf, -np.inf, np.nan,
                    u(0xBF808000), 1.0, u(0x3B800000)], np.float32)  # the last: 2^-8, so 1 + it is a tie
  dims = {"e8": 8, "e3": 3, "e36": 36}
  t = MultiHashTable({n: sgd_table(d, capacity=4096) for n, d in dims.items()}, device=dev)
  rng = np.random.default_rng(3)
  keys = {}
  for s, (n, d) in enumerate(dims.items(), start=1):
    k = _fids(64, s)
    v = edges[rng.integers(0, edges.size, (64, d))]
    v[:edges.size, 0] = edges
    t.assign({n: (T(k, dev), T(v, dev))})
    keys[n] = k
  parts_spec = []
  for n in dims:
    k = keys[n]
    f = k[rng.integers(0, 64, 512)]
    offs = np.concatenate([[0], np.cumsum(rng.integers(0, 4, 200))]).astype(np.int32)
    fc = k[rng.integers(0, 64, int(offs[-1]))]
    parts_spec += [(n, f, None, "sum", 0), (n, fc, offs, "sum", 0), (n, fc, offs, "mean", 0),
                   (n, fc, offs, "firstn", 3)]

  def call(dtype):
    return t.lookup_pool_parts([PoolPart(n, T(f, dev), None if o is None else T(o, dev), pl, max_seq_len=L)
                                for n, f, o, pl, L in parts_spec], dtype=dtype)

  want = [o.to(BF) for o in call(torch.float32)]
  got = call(BF)
  for g, w in zip(got, want):
    assert_bf16_bits(g, w)
  assert any(torch.isinf(g.float()).any() for g in got) and any(torch.isnan(g.float()).any() for g in got)


def test_forward_errors_match_the_fp32_call(dev):
  from monolith_b200 import MultiHashTable, _lib
  from monolith_b200._lib import PoolPartC
  t = MultiHashTable({"big": sgd_table(520, capacity=1024), "s": sgd_table(8, capacity=1024)}, device=dev)
  f = T(_fids(8, 1), dev)
  out = torch.empty(8, 520, dtype=BF, device=dev)
  stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
  for over in (dict(table=t.table_names.index("big")), dict(table=7), dict(pooling=9),
               dict(pooling=_lib.POOL_FIRSTN, max_seq_len=0)):
    kw = dict(table=t.table_names.index("s"), fids_dev=f.data_ptr(), n_fids=8, row_offsets_dev=None, n_rows=8,
              pooling=_lib.POOL_SUM, rows_dev=out.data_ptr(), stride=520, col=0, max_seq_len=0)
    kw.update(over)
    arr = (PoolPartC * 1)(PoolPartC(**kw))
    assert t._lib.mono_mtable_lookup_pool_parts_bf16(t.handle, arr, 1, stream) == -1
    assert t._lib.mono_mtable_lookup_pool_parts(t.handle, arr, 1, stream) == -1


# ------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------
def bf16_rows(x, dev, offset8=False):
  """Host fp32 rows -> device bf16 rows (rounded); offset8: the tensor's base is 8- but not 16-byte aligned."""
  r = torch.from_numpy(np.ascontiguousarray(x)).to(dev).to(BF)
  if not offset8:
    return r
  buf = torch.empty(r.numel() + 8, dtype=BF, device=dev)
  v = buf[4:4 + r.numel()].view(r.shape)
  v.copy_(r)
  assert v.data_ptr() % 16 == 8
  return v


def twin_step(ta, tb, specs, dev, req_time):
  """specs: (slot, fids, offs, pooling, fp32 rows, col, L).  ta gets bf16 rows, tb the same rows widened to fp32;
  -> (launches of the bf16 call, launches of the fp32 call)."""
  from monolith_b200 import PoolPart
  pa, pb = [], []
  for i, (slot, f, o, pl, rows, col, L) in enumerate(specs):
    r16 = bf16_rows(rows, dev, offset8=(i % 3 == 1))
    o_ = None if o is None else T(o, dev)
    pa.append(PoolPart(slot, T(f, dev), o_, pl, r16, col, max_seq_len=L))
    pb.append(PoolPart(slot, T(f, dev), o_, pl, r16.float(), col, max_seq_len=L))
  n = []
  for t, p in ((ta, pa), (tb, pb)):
    torch.cuda.synchronize()
    n0 = t._lib.mono_kernel_launch_count()
    t.pool_backward_parts(p, req_time=req_time)
    torch.cuda.synchronize()
    n.append(t._lib.mono_kernel_launch_count() - n0)
  return n


def assert_twins(ta, tb, slots_keys, dev):
  for slot, keys in slots_keys:
    assert ta.size(slot) == tb.size(slot), slot
    np.testing.assert_array_equal(_entries(ta, slot, keys, dev), _entries(tb, slot, keys, dev), err_msg=slot)


def step_specs(rng, step):
  """_step_parts (hot FID split across parts: a run > 64; CSR MEAN on b32; Adagrad, FTRL, Adam, a multi-segment
  table) plus, per table, a warm FID with 20 occurrences (a 9-64 run) and a FIRSTN part with FIDs only beyond L."""
  specs = []
  for p in _step_parts(rng, DIMS):
    specs.append((p.slot, p.fids, p.offs, p.pooling, p.rows, p.col, 0))
  for s, (slot, D) in enumerate(DIMS, start=1):
    pool = _fids(700, s)
    f = pool[rng.integers(0, 700, 100)]
    f[:20] = pool[5]
    specs.append((slot, f, None, "sum", rng.standard_normal((100, D)).astype(np.float32), 0, 0))
    beyond = _fids(900, s)[800 + 10 * step:810 + 10 * step]
    fids, offs, g, col = seq_batch(rng, pool, 120, 5, D, hot=pool[1], beyond=beyond, wide=(s % 2 == 0))
    specs.append((slot, fids, offs, "firstn", g, col, 5))
  return specs


def test_backward_equals_fp32_on_widened_rows(dev):
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  _history(ta, dev)   # an eviction, then rows reused
  _history(tb, dev)
  rng = np.random.default_rng(61)
  for step in range(2):
    na, nb = twin_step(ta, tb, step_specs(rng, step), dev, 40 + step)
    assert na == nb
  assert_twins(ta, tb, [(slot, np.concatenate([_fids(700, s), _fids(900, s)[800:]]))
                        for s, (slot, _) in enumerate(DIMS, start=1)], dev)


def test_backward_at_tree_depth_1(dev):
  """> 16384 occurrences of one table (tree depth 1), SUM + CSR MEAN + FIRSTN, a FID with > 64 occurrences."""
  from monolith_b200 import MultiHashTable, entry
  ini = entry.RandomUniformInitializer(-0.1, 0.1)
  cfg = {"z": table([(36, "adagrad", {"initial_accumulator_value": 0.1})], [0.05], capacity=4096, init=ini,
                    init_seed=1),
         "y": table([(8, "adam", {})], [0.01], capacity=4096, init=ini, init_seed=2)}
  ta, tb = MultiHashTable(cfg, device=dev), MultiHashTable(cfg, device=dev)
  rng = np.random.default_rng(67)
  pool = _fids(3000, 1)
  for step in range(2):
    f = pool[rng.integers(0, 3000, 9000)]
    f[rng.choice(9000, 300, replace=False)] = pool[3]
    offs = np.concatenate([[0], np.cumsum(rng.integers(1, 5, 3000))]).astype(np.int32)
    fc = pool[rng.integers(0, 3000, int(offs[-1]))]
    fs, os_, g, col = seq_batch(rng, pool, 300, 8, 36, hot=pool[2], wide=True)
    small = _fids(50, 2)[rng.integers(0, 50, 200)]
    specs = [("z", f, None, "sum", rng.standard_normal((9000, 36)).astype(np.float32), 0, 0),
             ("y", small, None, "sum", rng.standard_normal((200, 8)).astype(np.float32), 0, 0),
             ("z", fc, offs, "mean", rng.standard_normal((3000, 40)).astype(np.float32), 4, 0),
             ("z", fs, os_, "firstn", g, col, 8)]
    assert 9000 + int(offs[-1]) + fs.size > 16384
    na, nb = twin_step(ta, tb, specs, dev, 50 + step)
    assert na == nb
  assert_twins(ta, tb, [("z", pool), ("y", _fids(50, 2))], dev)


def test_backward_with_admission_filter(dev):
  from monolith_b200 import MultiHashTable
  ta, tb = MultiHashTable(_cfg(), device=dev), MultiHashTable(_cfg(), device=dev)
  for t in (ta, tb):
    t.set_hash_filter("a8", 1 << 16, 2)
  rng = np.random.default_rng(71)
  pool, beyond = _fids(40, 1), _fids(60, 1)[50:]
  for step in range(3):
    fids, offs, g, col = seq_batch(rng, pool, 60, 3, 8, beyond=beyond)
    f = pool[rng.integers(0, 40, 80)]
    specs = [("a8", fids, offs, "firstn", g, col, 3),
             ("a8", f, None, "sum", rng.standard_normal((80, 8)).astype(np.float32), 0, 0)]
    twin_step(ta, tb, specs, dev, 60 + step)
    assert ta.size("a8") == tb.size("a8")
  assert_twins(ta, tb, [("a8", np.concatenate([pool, beyond]))], dev)


def test_backward_two_runs_identical_bits(dev):
  from monolith_b200 import MultiHashTable, PoolPart
  out = []
  for _ in range(2):
    t = MultiHashTable(_cfg(), device=dev)
    rng = np.random.default_rng(73)
    for step in range(2):
      t.pool_backward_parts([PoolPart(slot, T(f, dev), None if o is None else T(o, dev), pl, bf16_rows(r, dev), c,
                                      max_seq_len=L) for slot, f, o, pl, r, c, L in step_specs(rng, step)],
                            req_time=80 + step)
    out.append([_entries(t, slot, _fids(900, s), dev) for s, (slot, _) in enumerate(DIMS, start=1)])
  for a, b in zip(*out):
    np.testing.assert_array_equal(a, b)


def test_backward_misaligned_rows_are_invalid_and_change_nothing(dev):
  from monolith_b200 import MultiHashTable, _lib
  from monolith_b200._lib import PoolPartC
  t = MultiHashTable(_cfg(), device=dev)
  _history(t, dev)
  names = t.table_names
  f = T(_fids(300, 1)[:64], dev)
  g = torch.zeros(64, 8 + 16, dtype=BF, device=dev)
  lr = t.learning_rates()
  lr_arr = (C.c_float * len(lr))(*lr)
  stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

  def bwd(**over):
    good = dict(table=names.index("a8"), fids_dev=f.data_ptr(), n_fids=64, row_offsets_dev=None, n_rows=64,
                pooling=_lib.POOL_SUM, rows_dev=g.data_ptr(), stride=24, col=4, max_seq_len=0)
    good.update(over)
    ok = dict(good, col=0, rows_dev=g.data_ptr(), stride=24)
    arr = (PoolPartC * 2)(PoolPartC(**ok), PoolPartC(**good))
    return t._lib.mono_mtable_pool_backward_parts_bf16(t.handle, arr, 2, lr_arr, 200, 0, stream)

  before = {n: (t.size(n), _entries(t, n, _fids(700, s), dev)) for s, n in enumerate(names, start=1)}
  for what, over in {"col % 4": dict(col=2), "stride % 4": dict(stride=22), "base 4-byte aligned":
                     dict(rows_dev=g.data_ptr() + 4), "base 2-byte aligned": dict(rows_dev=g.data_ptr() + 2),
                     "bad table index": dict(table=-1)}.items():
    assert bwd(**over) == -1, what
  torch.cuda.synchronize()
  for s, n in enumerate(names, start=1):
    assert t.size(n) == before[n][0], n
    np.testing.assert_array_equal(_entries(t, n, _fids(700, s), dev), before[n][1])
  assert bwd(rows_dev=g.data_ptr() + 8, col=0) == 0   # 8-byte aligned is enough for bf16 rows


def test_python_rejects_mixed_and_other_dtypes(dev):
  from monolith_b200 import MultiHashTable, PoolPart
  t = MultiHashTable(_cfg(), device=dev)
  f = T(_fids(16, 1), dev)
  for rows in ([torch.zeros(16, 8, device=dev), torch.zeros(16, 8, dtype=BF, device=dev)],
               [torch.zeros(16, 8, dtype=torch.float16, device=dev)] * 2,
               [torch.zeros(16, 8, dtype=torch.float64, device=dev)] * 2):
    with pytest.raises(ValueError):
      t.pool_backward_parts([PoolPart("a8", f, rows=r) for r in rows], req_time=1)
    with pytest.raises(ValueError):
      t.lookup_pool_parts([PoolPart("a8", f, rows=r) for r in rows])
  with pytest.raises(ValueError):
    t.lookup_pool_parts([PoolPart("a8", f, rows=torch.zeros(16, 8, device=dev))], dtype=BF)


def test_every_bf16_forward_instantiation_ran():
  """Runs last in this file: the forward grid launched every bf16 forward instantiation."""
  assert SEEN == ({f"bf16_lookup_kernel<{g},{c}>" for g in GS for c in ("false", "true")} |
                  {f"bf16_seq_kernel<{g},{c}>" for g in GS for c in ("false", "true")} |
                  {f"bf16_pool_staged_kernel<{g}>" for g in GS} | {"bf16_pool_kernel<%d,%d,%d>" % v for v in POOL_VARIANTS})
