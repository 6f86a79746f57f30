"""Every dispatch path of the forward (lookup, fused lookup, lookup_pool, gather_pool, lookup_push, contains,
lookup_entry) against the CPU oracle, bit for bit.

Each case checks two things: (a) the result equals the oracle through uint32 views (-0.0 is not +0.0, a NaN's
payload is kept where the path only copies), and run twice it gives the same bits; (b) it ran exactly the kernel
instantiation it is aimed at, read from torch.profiler's CUDA kernel records.  The last test checks that the cases
together ran every forward instantiation of ops.cu / layout.cu and nothing else.  The dispatch rules the cases are
aimed with are pinned against the sources in tests/test_forward_paths_cpu.py.

Tables are SGD with a zeros initializer, filled with `assign`, so a row holds exactly the bits written to it.
"""
import contextlib
import re
import zlib

import numpy as np
import pytest
import torch

from tests import cuckoo_place as cp
from tests import orc
from tests.helpers import sgd_table

pytestmark = pytest.mark.gpu

I64 = np.iinfo(np.int64)
GS = (4, 8, 16, 32)
FAMILY = ("lookup_kernel", "lookup_tma_kernel", "lookup_pool_staged_kernel", "lookup_pool_kernel", "gather_rows_kernel",
          "gather_pool_kernel", "lookup_push_kernel", "contains_kernel", "lookup_entry_kernel")
POOL_VARIANTS = ((4, 1, 4), (8, 1, 4), (16, 1, 4), (32, 1, 4), (32, 2, 2), (32, 4, 1))
INVENTORY = frozenset(
    [f"lookup_kernel<{g},true,false,false>" for g in GS] +   # single table, same stream as the inserts
    [f"lookup_kernel<{g},true,false,true>" for g in GS] +    # single table, misses confirmed (inserts on another stream)
    [f"lookup_kernel<{g},true,true,true>" for g in GS] +     # knob lookup_dual
    [f"lookup_kernel<{g},false,false,true>" for g in GS] +   # several (shard, table) segments
    ["lookup_tma_kernel<128>", "lookup_tma_kernel<256>"] +
    [f"lookup_pool_staged_kernel<{g}>" for g in GS] +
    ["lookup_pool_kernel<%d,%d,%d>" % v for v in POOL_VARIANTS] +
    [f"gather_rows_kernel<{g}>" for g in GS] + [f"gather_pool_kernel<{g}>" for g in GS] +
    [f"lookup_push_kernel<{g}>" for g in GS] + ["contains_kernel", "lookup_entry_kernel"])
SEEN = set()
WIDTHS = [1, 2, 3, 4, 5, 7, 8, 12, 16, 17, 20, 31, 32, 33, 36, 64, 65, 100, 128, 129, 132, 200, 256, 257, 260, 384, 511,
          512]
NAN_SENTINEL = np.array([0x7FC0DEAD], np.uint32).view(np.float32)[0]


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


# ------------------------------------------------------------------------------------------------
# which instantiation a call selects (the rules pinned in test_forward_paths_cpu.py)
# ------------------------------------------------------------------------------------------------
def pick_group(d):
  v, g = (d + 3) // 4, 4
  while g < v and g < 32:
    g <<= 1
  return g


def k_lookup(d, confirm=False, dual=False, tma=True, packed=True):
  """Single-segment lookup / lookup_pool without row offsets."""
  if tma and packed and d % 4 == 0 and d * 4 in (128, 256):
    return f"lookup_tma_kernel<{d * 4}>"
  g = pick_group(d)
  if dual:
    return f"lookup_kernel<{g},true,true,true>"
  return f"lookup_kernel<{g},true,false,{'true' if confirm else 'false'}>"


def k_pool(d, staged_ok=True):
  """lookup_pool with row offsets; staged_ok: output stride, column and base pass the staged kernel's checks."""
  g = pick_group(d)
  if staged_ok and d % 4 == 0 and d <= 128:
    return f"lookup_pool_staged_kernel<{g}>"
  nv = -(-d // (4 * g))
  v = (g, 1, 4) if g < 32 else {1: (32, 1, 4), 2: (32, 2, 2)}.get(nv, (32, 4, 1))
  return "lookup_pool_kernel<%d,%d,%d>" % v


def k_gather(d, csr, rows_ok=True):
  g = pick_group(d)
  if not csr and rows_ok and d % 4 == 0 and d <= 4 * g:
    return f"gather_rows_kernel<{g}>"
  return f"gather_pool_kernel<{g}>"


# ------------------------------------------------------------------------------------------------
# running a case: profiled once (kernel names), then again (determinism)
# ------------------------------------------------------------------------------------------------
def _canon(name, family=FAMILY):
  m = re.search(r"(\w+)(<[^()]*?>)?\(", name)
  if not m or m.group(1) not in family:
    return None
  return m.group(1) + (m.group(2) or "").replace(" ", "")


def traced(fn, family=FAMILY):
  """-> (fn(), names of the kernels of `family` (default: the forward's) torch.profiler recorded while it ran)."""
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    out = fn()
    torch.cuda.synchronize()
  return out, {c for c in (_canon(e.name, family) for e in prof.events()) if c}


def _bytes(out):
  outs = out if isinstance(out, tuple) else (out,)
  return [np.ascontiguousarray(o).view(np.uint8) for o in outs]


def run(fn, expect, family=FAMILY, seen=SEEN):
  """fn() -> numpy array(s).  Asserts the kernels of `family` it launched are exactly `expect` and adds them to
  `seen`.  fn is called several times, so a case that changes state builds it from scratch inside fn.

  torch.profiler now and then loses a whole batch of device records (a few traces in a thousand, two or three in
  a row; the traces after them are complete).  A lost record can only make a kernel MISSING from a trace, never add
  one, so a trace that recorded a strict subset of `expect` is traced again; any kernel outside `expect` fails at
  once, and a case that really launches less than `expect` fails after ten traces."""
  expect = {expect} if isinstance(expect, str) else set(expect)
  for _ in range(10):
    out, names = traced(fn, family)
    if not names < expect:
      break
  seen.update(names)
  assert names == expect, f"ran {sorted(names)}, aimed at {sorted(expect)}"
  for a, b in zip(_bytes(out), _bytes(fn())):
    np.testing.assert_array_equal(a, b, err_msg="not bit-stable run to run")
  return out


def assert_bits(got, want):
  """All 32 bits (paths that only copy rows)."""
  np.testing.assert_array_equal(np.ascontiguousarray(got, np.float32).view(np.uint32),
                                np.ascontiguousarray(want, np.float32).view(np.uint32))


def assert_pooled(got, want):
  """Bit for bit except NaN payloads (the GPU's arithmetic returns its canonical NaN, x86 propagates an operand's)."""
  g, w = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
  gn, wn = np.isnan(g), np.isnan(w)
  np.testing.assert_array_equal(gn, wn)
  np.testing.assert_array_equal(np.where(gn, 0, g.view(np.uint32)), np.where(wn, 0, w.view(np.uint32)))


@contextlib.contextmanager
def options(**kv):
  from monolith_b200 import _lib
  lib = _lib.load()
  old = {k: lib.mono_get_option(k.encode()) for k in kv}
  try:
    for k, v in kv.items():
      assert lib.mono_set_option(k.encode(), int(v)) == 0
    yield
  finally:
    for k, v in old.items():
      lib.mono_set_option(k.encode(), v)


def sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def sweep_items(threads_per_item):
  """Upper bound on the items one grid-stride sweep covers: at most 2048 resident threads per SM."""
  return sms() * 2048 // threads_per_item


# ------------------------------------------------------------------------------------------------
# tables
# ------------------------------------------------------------------------------------------------
class Pair:
  """One GPU table set and its oracle, filled by one assign call."""

  def __init__(self, dev, dims, keys, vals, capacity=None, req_time=1000, **kw):
    from monolith_b200 import MultiHashTable
    self.dev = dev
    self.names = sorted(dims)
    cfg = {n: sgd_table(dims[n], capacity=capacity or max(keys[n].size, 1), **kw) for n in self.names}
    self.gpu = MultiHashTable(cfg, device=dev)
    self.cpu = orc.OracleMultiHashTable(cfg)
    self.assign(keys, vals, req_time)

  def assign(self, keys, vals, req_time):
    self.gpu.assign({n: (T(keys[n], self.dev), T(vals[n], self.dev)) for n in keys}, req_time=req_time, ids_unique=True)
    self.cpu.assign({n: (keys[n], vals[n]) for n in keys}, req_time=req_time)


def table1(dev, dim, keys, vals, **kw):
  return Pair(dev, {"t": dim}, {"t": keys}, {"t": vals}, **kw)


def rand_keys(rng, n, exclude=None):
  k = np.unique(rng.integers(I64.min, I64.max, n + 64, dtype=np.int64))
  if exclude is not None:
    k = k[~np.isin(k, exclude)]
  return rng.permutation(k)[:n]


def basic(dev, dim, n_keys=3000, seed=0, **kw):
  rng = np.random.default_rng(seed * 1000 + dim)
  keys = rand_keys(rng, n_keys)
  vals = rng.standard_normal((keys.size, dim)).astype(np.float32)
  absent = rand_keys(rng, 200, exclude=keys)
  return table1(dev, dim, keys, vals, **kw), keys, absent, rng


def queries(rng, keys, absent, n):
  pool = np.concatenate([keys, absent])
  return pool[rng.integers(0, pool.size, n)]


def csr(rng, n_rows, max_len, min_len=0):
  lens = rng.integers(min_len, max_len + 1, n_rows)
  return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


# ---- calls returning numpy ----
def g_lookup(p, ids_by_table):
  return lambda: tuple(v.cpu().numpy() for v in
                       p.gpu.lookup({k: T(v, p.dev) for k, v in ids_by_table.items()}).values())


def g_pool(p, fids, offs, pooling, slot="t", out=None, out_col=0):
  def f():
    o = None if out is None else out.clone()
    r = p.gpu.lookup_pool(slot, T(fids, p.dev), None if offs is None else T(offs, p.dev), pooling, out=o,
                          out_col=out_col)
    return (o if o is not None else r).cpu().numpy()
  return f


def g_gather(dev, fused, eo, dim, offs, pooling, out=None, out_col=0):
  from monolith_b200 import distribution_ops as dops
  def f():
    o = None if out is None else out.clone()
    r = dops.gather_pool(T(fused, dev), T(eo, dev), dim, None if offs is None else T(offs, dev), pooling, out=o,
                         out_col=out_col)
    return (o if o is not None else r).cpu().numpy()
  return f


# ------------------------------------------------------------------------------------------------
# widths
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", WIDTHS + [1000])
def test_lookup_every_width(dim, dev):
  p, keys, absent, rng = basic(dev, dim, seed=1)
  ids = queries(rng, keys, absent, 5000)
  got = run(g_lookup(p, {"t": ids}), k_lookup(dim))[0]
  assert_bits(got, p.cpu.lookup({"t": ids})["t"])


@pytest.mark.parametrize("dim", WIDTHS)
def test_lookup_pool_every_width(dim, dev):
  p, keys, absent, rng = basic(dev, dim, seed=2)
  offs = csr(rng, 1500, 9)
  offs[1:4] = offs[4]  # three empty rows up front
  fids = queries(rng, keys, absent, int(offs[-1]))
  fids[5:9] = fids[4]  # duplicates inside a row
  for pooling in ("sum", "mean"):
    got = run(g_pool(p, fids, offs, pooling), k_pool(dim))
    assert_bits(got, p.cpu.lookup_pool("t", fids, offs, pooling))
    got = run(g_pool(p, fids, None, pooling), k_lookup(dim))
    assert_bits(got, p.cpu.lookup_pool("t", fids, None, pooling))


@pytest.mark.parametrize("dim", WIDTHS)
def test_gather_pool_every_width(dim, dev):
  rng = np.random.default_rng(dim + 3)
  U = 700
  fused = rng.standard_normal(U * dim).astype(np.float32)
  offs = csr(rng, 900, 7)
  eo = (rng.integers(0, U, int(offs[-1])) * dim).astype(np.int32)
  for pooling in ("sum", "mean"):
    got = run(g_gather(dev, fused, eo, dim, offs, pooling), k_gather(dim, True))
    assert_bits(got, orc.gather_pool(fused, eo, dim, offs, pooling))
    got = run(g_gather(dev, fused, eo, dim, None, pooling), k_gather(dim, False))
    assert_bits(got, orc.gather_pool(fused, eo, dim, None, pooling))
  # rows at float offsets that are not 16-byte aligned (a fused buffer behind an odd-width table)
  eo1 = eo + 1 + 2 * (rng.integers(0, 2, eo.size)).astype(np.int32)
  fused1 = np.concatenate([fused, np.zeros(3, np.float32)])
  for c in (True, False):
    got = run(g_gather(dev, fused1, eo1, dim, offs if c else None, "sum"), k_gather(dim, c))
    assert_bits(got, orc.gather_pool(fused1, eo1, dim, offs if c else None, "sum"))


def test_lookup_pool_refuses_dim_513(dev):
  from monolith_b200._lib import MonoError
  p, keys, absent, rng = basic(dev, 513, n_keys=100, seed=4)
  fids = keys[:10]
  for offs in (np.array([0, 3, 10], np.int32), None):
    out = torch.full((10 if offs is None else 2, 513), float(NAN_SENTINEL), device=dev)
    before = out.cpu().numpy().copy()
    with pytest.raises(MonoError, match="InvalidArgument"):
      p.gpu.lookup_pool("t", T(fids, dev), None if offs is None else T(offs, dev), "sum", out=out)
    torch.cuda.synchronize()
    assert_bits(out.cpu().numpy(), before)


# ------------------------------------------------------------------------------------------------
# CSR shapes
# ------------------------------------------------------------------------------------------------
def _offs(lens, start=0):
  return (start + np.concatenate([[0], np.cumsum(lens)])).astype(np.int32)


def _every_offset_mod16():
  lens, cur = [], 0
  for L in range(1, 41):
    for o in range(16):
      pad = (o - cur) % 16
      if pad:
        lens.append(pad)
        cur += pad
      lens.append(L)
      cur += L
  return lens


def _shape(name, rng):
  """-> (row lengths, offset of row 0 into the FID array)"""
  if name.startswith("rows"):
    n = int(name[4:])
    return rng.integers(0, 6, n), 0
  if name == "large":
    return rng.integers(0, 6, 40000), 0
  if name == "empty_ends":
    return np.concatenate([[0] * 37, rng.integers(1, 5, 100), [0] * 41]), 0
  if name == "all_empty":
    return np.zeros(70, np.int64), 0
  if name == "len1_40_every_mod16":
    return np.asarray(_every_offset_mod16()), 0
  if name == "long_rows":
    return np.array([1000, 3, 100000, 0, 1, 999]), 0
  if name == "ragged_warp":
    return np.tile([1, 300, 0, 2, 57, 1, 16, 17, 33, 0, 5, 129], 40), 0
  if name == "sub_batch_view":
    return rng.integers(0, 9, 500), 37
  raise ValueError(name)


SHAPES = ["rows1", "rows2", "rows3", "rows4", "rows5", "rows31", "rows32", "rows33", "large", "empty_ends", "all_empty",
          "len1_40_every_mod16", "long_rows", "ragged_warp", "sub_batch_view"]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dim", [8, 17, 64, 200, 512])
def test_csr_shapes(dim, shape, dev):
  p, keys, absent, rng = basic(dev, dim, seed=5)
  lens, start = _shape(shape, rng)
  offs = _offs(lens, start)
  fids = queries(rng, keys, absent, int(offs[-1]))
  fids[:start] = -7
  if shape == "ragged_warp":  # absent FIDs first, last and on both sides of a 16-entry chunk boundary
    for b, n in zip(offs[:-1], lens):
      if n:
        fids[b] = absent[0]
        fids[b + n - 1] = absent[1]
      if n > 17:
        fids[b + 15:b + 17] = absent[2]
  if shape == "len1_40_every_mod16":
    fids[1::5] = fids[0::5][:fids[1::5].size]   # duplicates in a row
  n_rows = lens.size
  for pooling in ("sum", "mean"):
    out = torch.full((n_rows, dim), float(NAN_SENTINEL), device=dev)
    got = run(g_pool(p, fids, offs, pooling, out=out), k_pool(dim))
    want = p.cpu.lookup_pool("t", fids, offs, pooling)
    assert_bits(got, want)
    if shape == "all_empty":
      assert not got.view(np.uint32).any()   # +0.0 over the NaN sentinel
  # the same row structure through gather_pool (rows of a fused buffer instead of a table)
  U = 500
  fused = rng.standard_normal(U * dim).astype(np.float32)
  eo = (rng.integers(0, U, fids.size) * dim).astype(np.int32)
  got = run(g_gather(dev, fused, eo, dim, offs, "mean"), k_gather(dim, True))
  assert_bits(got, orc.gather_pool(fused, eo, dim, offs, "mean"))


# ------------------------------------------------------------------------------------------------
# output placement
# ------------------------------------------------------------------------------------------------
PLACEMENTS = [  # (out_col, stride - dim, base offset in floats)
    (0, 0, 0), (1, 1, 0), (2, 3, 0), (4, 4, 0), (5, 8, 0), (0, 1, 0), (0, 3, 0), (0, 4, 0), (0, 8, 0), (4, 8, 0),
    (0, 0, 1), (0, 4, 1), (3, 4, 1), (2, 8, 1)]


@pytest.mark.parametrize("dim", [4, 8, 17, 32, 64, 128, 200])
def test_output_placement(dim, dev):
  p, keys, absent, rng = basic(dev, dim, seed=6)
  offs = csr(rng, 700, 6)
  fids = queries(rng, keys, absent, int(offs[-1]))
  U = 300
  fused = rng.standard_normal(U * dim).astype(np.float32)
  eo = (rng.integers(0, U, fids.size) * dim).astype(np.int32)
  for col, extra, shift in PLACEMENTS:
    for with_csr in (True, False):
      n = offs.size - 1 if with_csr else fids.size
      W = dim + extra + shift   # row stride of the buffer; the output view starts `shift` floats into it
      buf = torch.full((n, W), float(NAN_SENTINEL), device=dev)
      aligned = shift == 0      # torch allocations are 256-byte aligned
      o = offs if with_csr else None
      ok16 = W % 4 == 0 and col % 4 == 0 and aligned
      expect = k_pool(dim, staged_ok=ok16) if with_csr else k_lookup(dim, packed=col == 0 and W == dim and aligned)
      got = run(_placed_pool(p, fids, o, buf, shift, col), expect)
      want = np.tile(NAN_SENTINEL, (n, W))
      want[:, shift + col:shift + col + dim] = p.cpu.lookup_pool("t", fids, o, "sum")
      assert_bits(got, want)   # the sentinel columns around the output are untouched
      # gather_pool into the same placement
      got = run(_placed_gather(dev, fused, eo, dim, o, buf, shift, col), k_gather(dim, with_csr, rows_ok=ok16))
      want[:, shift + col:shift + col + dim] = orc.gather_pool(fused, eo, dim, o, "sum")
      assert_bits(got, want)


def _placed_pool(p, fids, offs, buf, shift, col):
  def f():
    b = buf.clone()
    p.gpu.lookup_pool("t", T(fids, p.dev), None if offs is None else T(offs, p.dev), "sum", out=b[:, shift:],
                      out_col=col)
    return b.cpu().numpy()
  return f


def _placed_gather(dev, fused, eo, dim, offs, buf, shift, col):
  from monolith_b200 import distribution_ops as dops
  def f():
    b = buf.clone()
    dops.gather_pool(T(fused, dev), T(eo, dev), dim, None if offs is None else T(offs, dev), "sum", out=b[:, shift:],
                     out_col=col)
    return b.cpu().numpy()
  return f


# ------------------------------------------------------------------------------------------------
# grid-stride turnover: every instantiation with enough work that each warp loops at least twice (TMA: five
# times, so the mbarrier parity wraps), at the narrowest width that selects it
# ------------------------------------------------------------------------------------------------
NARROW = {4: 1, 8: 17, 16: 33, 32: 65}        # narrowest dim per lane group
NARROW16 = {4: 4, 8: 20, 16: 36, 32: 68}      # narrowest multiple of 4 per lane group
TURNOVER = ([("lookup", g, v) for g in GS for v in ("plain", "confirm", "dual", "multi")] +
            [("tma", 128, None), ("tma", 256, None)] + [("staged", g, None) for g in GS] +
            [("pool", v, None) for v in POOL_VARIANTS] + [("gather_rows", g, None) for g in GS] +
            [("gather_pool", g, None) for g in GS] + [("push", g, None) for g in GS] +
            [("contains", 4, None), ("entry", 8, None)])


@pytest.mark.parametrize("kind,arg,variant", TURNOVER, ids=lambda x: str(x))
def test_grid_stride_turnover(kind, arg, variant, dev):
  rng = np.random.default_rng(zlib.crc32(repr((kind, arg, variant)).encode()))
  if kind == "lookup":
    dim = NARROW[arg]
    n = 2 * sweep_items(1) + 7
    if variant == "multi":  # two tables: several segments
      keys = {"a": rand_keys(rng, 3000), "b": rand_keys(rng, 3000)}
      vals = {"a": rng.standard_normal((3000, dim)).astype(np.float32),
              "b": rng.standard_normal((3000, 1)).astype(np.float32)}
      p = Pair(dev, {"a": dim, "b": 1}, keys, vals)
      ids = {"a": queries(rng, keys["a"], keys["b"][:50], n // 2), "b": queries(rng, keys["b"], keys["a"][:50], n // 2)}
      got = run(g_lookup(p, ids), f"lookup_kernel<{arg},false,false,true>")
      want = p.cpu.lookup(ids)
      assert_bits(got[0], want["a"])
      assert_bits(got[1], want["b"])
      return
    p, keys, absent, rng = basic(dev, dim, seed=7)
    ids = queries(rng, keys, absent, n)
    if variant == "confirm":
      side = torch.cuda.Stream(dev)
      def f():
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
          r = p.gpu.lookup({"t": T(ids, dev)})["t"]
        torch.cuda.current_stream(dev).wait_stream(side)
        return r.cpu().numpy()
      got = run(f, k_lookup(dim, confirm=True))
    elif variant == "dual":
      with options(lookup_dual=1):
        got = run(lambda: g_lookup(p, {"t": ids})()[0], k_lookup(dim, dual=True))
    else:
      got = run(lambda: g_lookup(p, {"t": ids})()[0], k_lookup(dim))
    assert_bits(got, p.cpu.lookup({"t": ids})["t"])
  elif kind == "tma":
    dim = arg // 4
    p, keys, absent, rng = basic(dev, dim, seed=8)
    ids = queries(rng, keys, absent, 5 * sweep_items(1) + 33)
    got = run(lambda: g_lookup(p, {"t": ids})()[0], f"lookup_tma_kernel<{arg}>")
    assert_bits(got, p.cpu.lookup({"t": ids})["t"])
  elif kind in ("staged", "pool"):
    g, u = (arg, 4) if kind == "staged" else (arg[0], arg[2])
    dim = NARROW16[g] if kind == "staged" else {(32, 2, 2): 129, (32, 4, 1): 257}.get(arg, NARROW[g])
    p, keys, absent, rng = basic(dev, dim, seed=9)
    offs = csr(rng, 2 * sweep_items(max(g // u, 1)) + 7, 3)
    fids = queries(rng, keys, absent, int(offs[-1]))
    expect = f"lookup_pool_staged_kernel<{g}>" if kind == "staged" else "lookup_pool_kernel<%d,%d,%d>" % arg
    assert k_pool(dim) == expect
    got = run(g_pool(p, fids, offs, "mean"), expect)
    assert_bits(got, p.cpu.lookup_pool("t", fids, offs, "mean"))
  elif kind in ("gather_rows", "gather_pool"):
    dim = NARROW16[arg] if kind == "gather_rows" else NARROW[arg]
    U = 4000
    fused = rng.standard_normal(U * dim).astype(np.float32)
    if kind == "gather_rows":
      offs, n = None, 2 * sweep_items(1) + 7
    else:
      offs = csr(rng, 2 * sweep_items(arg) + 7, 3)
      n = int(offs[-1])
    eo = (rng.integers(0, U, n) * dim).astype(np.int32)
    got = run(g_gather(dev, fused, eo, dim, offs, "sum"), f"{kind}_kernel<{arg}>")
    assert_bits(got, orc.gather_pool(fused, eo, dim, offs, "sum"))
  elif kind == "push":
    dim = NARROW16[arg]
    p, keys, absent, rng = basic(dev, dim, seed=10)
    ids = queries(rng, keys, absent, 2 * sweep_items(1) + 7)
    got = run(_push(p, ids, dim), f"lookup_push_kernel<{arg}>")
    assert_bits(got, p.cpu.lookup({"t": ids})["t"])
  else:  # contains (4 lanes per id) / lookup_entry (8 lanes per id), grid of at most 8 blocks per SM
    dim = 3
    p, keys, absent, rng = basic(dev, dim, seed=11)
    ids = queries(rng, keys, absent, 2 * sweep_items(arg) + 7)
    if kind == "contains":
      got = run(lambda: p.gpu.contains("t", T(ids, dev)).cpu().numpy(), "contains_kernel")
      np.testing.assert_array_equal(got, p.cpu.contains("t", ids))
    else:
      got = run(lambda: p.gpu.lookup_entry("t", T(ids, dev))["raw"].cpu().numpy(), "lookup_entry_kernel")
      assert_bits(got, p.cpu.lookup_entry("t", ids))


def _push(p, ids, dim, slot="t"):
  from monolith_b200 import distribution_ops as dops
  def f():
    w = dops.PeerWindow(p.dev, 1, 0, ids.size * dim * 4 + 4096)
    try:
      w.view(0, ids.size * dim + 1024, torch.float32).fill_(float(NAN_SENTINEL))
      p.gpu.lookup_push(slot, T(ids, p.dev), [ids.size], w, 0, [4])
      w.barrier()
      torch.cuda.synchronize()
      got = w.view(0, ids.size * dim + 1024, torch.float32).cpu().numpy()
    finally:
      w.close()
    assert not (got[:4 * dim].view(np.uint32) != NAN_SENTINEL.view(np.uint32)).any()   # rows before the offset
    return got[4 * dim:(4 + ids.size) * dim].reshape(ids.size, dim)
  return f


# ------------------------------------------------------------------------------------------------
# knobs, the confirm path, several segments
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [8, 16, 32, 64, 100, 200, 512])
def test_lookup_knobs_give_identical_bits(dim, dev):
  p, keys, absent, rng = basic(dev, dim, n_keys=20000, seed=12)
  ids = queries(rng, keys, absent, 30000)
  want = p.cpu.lookup({"t": ids})["t"]
  for tma in (0, 1):
    for pf in (0, 1):
      for dual in (0, 1):
        with options(lookup_tma=tma, lookup_pf=pf, lookup_dual=dual):
          k = k_lookup(dim, dual=bool(dual), tma=bool(tma))
          assert_bits(run(lambda: g_lookup(p, {"t": ids})()[0], k), want)
          assert_bits(run(g_pool(p, ids, None, "mean"), k), want)


@pytest.mark.parametrize("dim", [1, 17, 33, 65, 32, 64])
def test_confirm_path_equals_same_stream(dim, dev):
  p, keys, absent, rng = basic(dev, dim, seed=13)   # fresh handle: inserts on the default stream
  ids = queries(rng, keys, absent, 20000)
  same = run(lambda: g_lookup(p, {"t": ids})()[0], k_lookup(dim))
  side = torch.cuda.Stream(dev)
  def f():
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
      r = p.gpu.lookup({"t": T(ids, dev)})["t"]
    torch.cuda.current_stream(dev).wait_stream(side)
    return r.cpu().numpy()
  other = run(f, k_lookup(dim, confirm=True))
  assert_bits(other, same)
  assert_bits(other, p.cpu.lookup({"t": ids})["t"])


def test_lookup_several_tables(dev):
  rng = np.random.default_rng(14)
  dims = {f"t{i}": d for i, d in enumerate([1, 3, 17, 32, 200, 512])}
  keys = {n: rand_keys(rng, 1500) for n in dims}
  vals = {n: rng.standard_normal((1500, d)).astype(np.float32) for n, d in dims.items()}
  p = Pair(dev, dims, keys, vals)
  names = sorted(dims)
  for empty in ([], ["t0"], ["t2", "t5"], ["t1", "t3", "t4"]):
    ids = {n: (np.zeros(0, np.int64) if n in empty else queries(rng, keys[n], keys[names[0]][:30], 700)) for n in names}
    g = pick_group(max(dims[n] for n in names if n not in empty))
    got = run(g_lookup(p, ids), f"lookup_kernel<{g},false,false,true>")
    want = p.cpu.lookup(ids)
    for i, n in enumerate(p.gpu.table_names):
      assert_bits(got[i], want[n])


@pytest.mark.parametrize("N", [1, 2, 8])
@pytest.mark.parametrize("dims", [(3, 17, 1), (5, 32, 7, 200)])
def test_fused_lookup_segments(dims, N, dev):
  rng = np.random.default_rng(sum(dims) * N)
  K = len(dims)
  d = {f"t{i}": x for i, x in enumerate(dims)}
  keys = {n: rand_keys(rng, 800) for n in d}
  vals = {n: rng.standard_normal((800, x)).astype(np.float32) for n, x in d.items()}
  p = Pair(dev, d, keys, vals)
  slot = rng.integers(0, 90, N * K).astype(np.int32)
  slot[rng.integers(0, N * K, max(1, N * K // 3))] = 0   # empty (shard, table) segments
  slot[-1] = max(slot[-1], 1)
  ids = np.concatenate([queries(rng, keys[f"t{j % K}"], keys[f"t{(j + 1) % K}"][:20], int(slot[j])) for j in range(N * K)])
  n_segs = int((slot > 0).sum())
  g = pick_group(max(dims[j % K] for j in range(N * K) if slot[j] > 0))
  expect = f"lookup_kernel<{g},false,false,true>" if n_segs > 1 else k_lookup(dims[int(np.flatnonzero(slot)[0]) % K])
  got = run(lambda: p.gpu.fused_lookup(T(ids, dev), slot.tolist(), N)[0].cpu().numpy(), expect)
  assert_bits(got, p.cpu.fused_lookup(ids, slot, N)[0])


@pytest.mark.parametrize("dim", [32, 64, 17])
def test_fused_lookup_one_table_across_shards_merges(dim, dev):
  """K = 1: the N shard segments are contiguous and merge into one; 128- and 256-byte rows go through TMA."""
  p, keys, absent, rng = basic(dev, dim, seed=15)
  N = 4
  slot = np.array([300, 0, 517, 41], np.int32)
  ids = queries(rng, keys, absent, int(slot.sum()))
  got = run(lambda: p.gpu.fused_lookup(T(ids, dev), slot.tolist(), N)[0].cpu().numpy(), k_lookup(dim))
  assert_bits(got, p.cpu.fused_lookup(ids, slot, N)[0])


# ------------------------------------------------------------------------------------------------
# key placement: second buckets, the stash, tombstones in stash chains
# ------------------------------------------------------------------------------------------------
def _placed_keys(rng, nb, short_slots):
  """Keys built (tests/cuckoo_place.py) to crowd chosen buckets.  -> (members, absent, short-expiry members)"""
  members, absent, short = [], [], []
  used = set()

  def fresh_bucket(lo=0):
    while True:
      b = int(rng.integers(lo, nb))
      if b not in used:
        used.add(b)
        return b
  # 8 keys per bucket pair: at most 4 fit in the first bucket, the rest sit in their second bucket (or the stash)
  for _ in range(24):
    k = cp.colliding_keys(nb, fresh_bucket(), fresh_bucket(), 11, rng)
    members += k[:8].tolist()
    absent += k[8:].tolist()
  # the last bucket, whose raw second choice wraps to bucket 0 in the fix-up
  used.update((nb - 1, 0))
  k = cp.colliding_keys(nb, nb - 1, nb - 1, 10, rng)
  members += k[:8].tolist()
  absent += k[8:].tolist()
  # 12 keys per bucket pair AND stash start: at least 4 share one stash probe chain; half of them expire early
  for _ in range(16):
    b1, b2 = fresh_bucket(), fresh_bucket()
    s = (int(rng.integers(*cp.word_range(b1, nb))) >> cp.STASH_SHIFT) & (cp.STASH_CAP - 1)
    ks = cp.colliding_keys(nb, b1, b2, 6, rng, stash_start=s, slots=short_slots)
    kl = cp.colliding_keys(nb, b1, b2, 16, rng, stash_start=s)
    kl = kl[~np.isin(cp.fid_slot(kl), list(short_slots)) & ~np.isin(kl, ks)]
    members += ks.tolist() + kl[:6].tolist()
    short += ks.tolist()
    absent += kl[6:10].tolist()
  # -1 has the bits of an empty entry's key: it and 7 keys of its bucket pair; the other extreme keys
  b1, b2 = (int(x) for x in cp.bucket_pair(-1, nb))
  k = cp.colliding_keys(nb, b1, b2, 11, rng)
  k = k[k != -1]
  members += [-1] + k[:7].tolist() + [0, int(I64.min), int(I64.max)]
  absent += k[7:10].tolist()
  members, absent = np.asarray(members, np.int64), np.asarray(absent, np.int64)
  assert np.unique(members).size == members.size and not np.isin(absent, members).any()
  return members, absent, np.asarray(short, np.int64)


def test_keys_in_second_buckets_stash_and_behind_tombstones(dev):
  rng = np.random.default_rng(16)
  CAP, T0, SHORT = 16384, 10 ** 6, {11, 12, 13, 14}
  nb = cp.buckets_for(CAP)
  members, absent, short = _placed_keys(rng, nb, SHORT)
  bg = rand_keys(rng, 4000, exclude=np.concatenate([members, absent]))
  bg = bg[~np.isin(cp.fid_slot(bg), list(SHORT))]
  keys = np.concatenate([bg, members])
  assert keys.size < 0.75 * nb * 4   # the fill does not rehash: the groups stay in the buckets they were built for
  dims = {"a": 8, "b": 17, "c": 64}   # staged + register lookup | probe_keys pooling | TMA + staged
  p = Pair(dev, dims, {n: keys for n in dims},
           {n: rng.standard_normal((keys.size, d)).astype(np.float32) for n, d in dims.items()},
           capacity=CAP, req_time=T0, default_expire_time=36500, slot_expire_times={s: 1 for s in SHORT})

  def check(extra=()):
    q = rng.permutation(np.concatenate([keys, absent, np.asarray(extra, np.int64)]))
    for n, d in dims.items():
      assert p.gpu.size(n) == p.cpu.size(n)
      want = p.cpu.lookup({n: q})[n]
      for dual in (0, 1):
        with options(lookup_dual=dual):
          assert_bits(run(lambda: g_lookup(p, {n: q})()[0], k_lookup(d, dual=bool(dual))), want)
      assert_bits(run(g_pool(p, q, None, "sum", slot=n), k_lookup(d)), want)
      offs = csr(rng, 3 * q.size // 10, 20)
      f = q[rng.integers(0, q.size, int(offs[-1]))]
      assert_bits(run(g_pool(p, f, offs, "mean", slot=n), k_pool(d)), p.cpu.lookup_pool(n, f, offs, "mean"))
      np.testing.assert_array_equal(run(lambda: p.gpu.contains(n, T(q, dev)).cpu().numpy(), "contains_kernel"),
                                    p.cpu.contains(n, q))
      assert_bits(run(lambda: p.gpu.lookup_entry(n, T(q, dev))["raw"].cpu().numpy(), "lookup_entry_kernel"),
                  p.cpu.lookup_entry(n, q))   # row, found flag and timestamp
      if d % 4 == 0:
        assert_bits(run(_push(p, q, d, slot=n), f"lookup_push_kernel<{pick_group(d)}>"), want)
    # all three tables in one call: several segments
    N = 2
    parts = [q[:500], q[500:1700], q[1700:2000], q[2000:2900], q[2900:3000], q[3000:]]
    slot = [x.size for x in parts]
    ids = np.concatenate(parts)
    got = run(lambda: p.gpu.fused_lookup(T(ids, dev), slot, N)[0].cpu().numpy(), "lookup_kernel<16,false,false,true>")
    assert_bits(got, p.cpu.fused_lookup(ids, slot, N)[0])

  check()
  # half of every stash group expires: tombstones inside the stash chains, the other half must still be found
  for n in dims:
    p.gpu.evict(n, T0 + 2 * 86400)
    p.cpu.evict(n, T0 + 2 * 86400)
  assert p.cpu.size("a") == keys.size - short.size
  check()
  # the next insert rehashes (a stash that held anything forces it) and empties the stash
  new = rand_keys(rng, 300, exclude=np.concatenate([keys, absent]))
  p.assign({n: new for n in dims}, {n: rng.standard_normal((new.size, d)).astype(np.float32) for n, d in dims.items()},
           T0 + 3 * 86400)
  check(new)


# ------------------------------------------------------------------------------------------------
# values: signed zeros, infinities, denormals, NaN payloads, sums that overflow
# ------------------------------------------------------------------------------------------------
SPECIAL = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x00400000,
                    0x80012345, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F000000, 0x7FC00001, 0x7FC12345, 0xFFC00077, 0x7FFFFFFF],
                   np.uint32).view(np.float32)


@pytest.mark.parametrize("dim", [4, 17, 32, 64, 129, 260])
def test_special_values(dim, dev):
  rng = np.random.default_rng(17 + dim)
  keys = rand_keys(rng, 2000)
  vals = rng.standard_normal((keys.size, dim)).astype(np.float32)
  mask = rng.random(vals.shape) < 0.4
  vals[mask] = SPECIAL[rng.integers(0, SPECIAL.size, int(mask.sum()))]
  vals[:100] = -0.0                                                        # rows of negative zeros
  den = rng.integers(1, 1 << 23, (100, dim)).astype(np.uint32) | (rng.integers(0, 2, (100, dim)).astype(np.uint32) << 31)
  vals[100:200] = den.view(np.float32)                                     # denormals of both signs
  vals[200:300] = np.float32(3e38)                                         # any two of them overflow
  p = table1(dev, dim, keys, vals)
  absent = rand_keys(rng, 50, exclude=keys)
  ids = queries(rng, keys, absent, 3000)
  # gather-only paths keep all 32 bits
  assert_bits(run(lambda: g_lookup(p, {"t": ids})()[0], k_lookup(dim)), p.cpu.lookup({"t": ids})["t"])
  for pooling in ("sum", "mean"):
    assert_bits(run(g_pool(p, ids, None, pooling), k_lookup(dim)), p.cpu.lookup_pool("t", ids, None, pooling))
  # pooled rows: from the zero rows only, the denormal rows only, the big rows only, and anything
  lens = rng.integers(0, 7, 800)
  offs = _offs(lens)
  fids = queries(rng, keys, absent, int(offs[-1]))
  for r, (b, e) in enumerate(zip(offs[:-1], offs[1:])):
    src = (keys[:100], keys[100:200], keys[200:300], None)[r % 4]
    if src is not None:
      fids[b:e] = src[rng.integers(0, src.size, e - b)]
  fused = vals.reshape(-1)
  eo = (rng.integers(0, keys.size, int(offs[-1])) * dim).astype(np.int32)
  for pooling in ("sum", "mean"):
    assert_pooled(run(g_pool(p, fids, offs, pooling), k_pool(dim)), p.cpu.lookup_pool("t", fids, offs, pooling))
    assert_pooled(run(g_gather(dev, fused, eo, dim, offs, pooling), k_gather(dim, True)),
                  orc.gather_pool(fused, eo, dim, offs, pooling))
    assert_bits(run(g_gather(dev, fused, eo, dim, None, pooling), k_gather(dim, False)),
                orc.gather_pool(fused, eo, dim, None, pooling))


# ------------------------------------------------------------------------------------------------
# inventory: keep last
# ------------------------------------------------------------------------------------------------
def test_every_forward_instantiation_ran_and_no_other():
  """The union of what the cases above ran (run this file whole: the inventory is collected from them)."""
  assert SEEN, "no forward kernel was recorded: the inventory is the union of this file's other tests"
  missing, extra = sorted(INVENTORY - SEEN), sorted(SEEN - INVENTORY)
  assert not missing and not extra, f"never ran: {missing}; ran but not listed: {extra}"
