"""Every Python wrapper that picks a _bf16, _scaled or fp16-input twin of a C call, run once per twin it serves: it
reaches the symbols written out in SYMBOLS, launches as many kernels as those symbols called directly with arguments
built here, and writes the same bits."""
import ctypes as C

import pytest
import torch

from monolith_b200 import _lib
from tests.helpers import table

pytestmark = pytest.mark.gpu

BF, F16 = torch.bfloat16, torch.float16
D, B, U = 8, 24, 40


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


class _Proxy:
  """The loaded library with every call recorded by name and forwarded unchanged."""

  def __init__(self, lib):
    self.lib, self.names = lib, []

  def __getattr__(self, name):
    fn = getattr(self.lib, name)
    if name in ("mono_last_error", "mono_kernel_launch_count"):
      return fn

    def rec(*args):
      self.names.append(name)
      return fn(*args)
    return rec


def _p(t):
  return None if t is None else C.c_void_p(t.data_ptr())


def _s(dev):
  return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _bits(t):
  return t.detach().contiguous().view(-1).view(torch.uint8)


def check(monkeypatch, symbols, wrapper, direct):
  """wrapper() through the recording proxy, then direct(the real symbols, in order): the symbols, the launch count and
  the bits of the returned tensors must agree."""
  symbols = [symbols] if isinstance(symbols, str) else list(symbols)
  lib = _lib.load()
  proxy = _Proxy(lib)
  torch.cuda.synchronize()
  n0 = lib.mono_kernel_launch_count()
  with monkeypatch.context() as m:
    m.setattr(_lib, "_lib", proxy)
    got = wrapper()
  torch.cuda.synchronize()
  n1 = lib.mono_kernel_launch_count()
  assert proxy.names == symbols
  assert _lib.load() is lib
  want = direct(*[getattr(lib, n) for n in symbols])
  torch.cuda.synchronize()
  assert lib.mono_kernel_launch_count() - n1 == n1 - n0, symbols
  assert len(got) == len(want)
  for g, w in zip(got, want):
    assert g.dtype == w.dtype and g.shape == w.shape, symbols
    assert torch.equal(_bits(g), _bits(w)), symbols


ALL, BF16 = ["f32", "bf16", "f32_scaled", "bf16_scaled"], ["f32", "bf16"]
SCALED, HALF = ["f32", "f32_scaled"], ["f32", "f16"]
# wrapper -> {variant: the C symbols it must call, in order}
SYMBOLS = {
    "gather_pool": {"f32": "mono_gather_pool", "bf16": "mono_gather_pool_bf16"},
    "gather_pool_grad": {"f32": "mono_gather_pool_grad", "bf16": "mono_gather_pool_grad_bf16",
                         "f32_scaled": "mono_gather_pool_grad_scaled",
                         "bf16_scaled": "mono_gather_pool_grad_bf16_scaled"},
    "scatter_grad_rows": {"f32": "mono_scatter_grad_rows", "bf16": "mono_scatter_grad_rows_bf16",
                          "f32_scaled": "mono_scatter_grad_rows_scaled",
                          "bf16_scaled": "mono_scatter_grad_rows_bf16_scaled"},
    "reduce_and_split": {"f32": "mono_reduce_and_split", "bf16": "mono_reduce_and_split_bf16"},
    "reduce_and_split_grad": {"f32": "mono_reduce_and_split_grad", "bf16": "mono_reduce_and_split_grad_bf16",
                              "f32_scaled": "mono_reduce_and_split_grad_scaled",
                              "bf16_scaled": "mono_reduce_and_split_grad_bf16_scaled"},
    "embedding_to_layout": {"f32": "mono_embedding_to_layout", "bf16": "mono_embedding_to_layout_bf16",
                            "f16in": "mono_embedding_to_layout_f16in",
                            "f16in_bf16": "mono_embedding_to_layout_f16in_bf16"},
    "embedding_to_layout_grad": {"f32": "mono_embedding_to_layout_grad", "bf16": "mono_embedding_to_layout_grad_bf16",
                                 "f32_scaled": "mono_embedding_to_layout_grad_scaled",
                                 "bf16_scaled": "mono_embedding_to_layout_grad_bf16_scaled"},
    "fill_with_offset_map": {"f32": "mono_fill_with_offset_map", "f16": "mono_fill_with_offset_map_f16"},
    "fill_with_offset_map_gradient": {"f32": "mono_fill_with_offset_map_grad",
                                      "f16": "mono_fill_with_offset_map_grad_f16"},
    "Grouping.reduce": {"f32": "mono_grouping_reduce", "f32_scaled": "mono_grouping_reduce_scaled"},
    "Grouping.reduce_push": {"f32": "mono_grouping_reduce_push", "f32_scaled": "mono_grouping_reduce_push_scaled"},
    "Grouping.reduce_parts": {"f32": "mono_grouping_reduce_parts", "bf16": "mono_grouping_reduce_parts_bf16",
                              "f32_scaled": "mono_grouping_reduce_parts_scaled",
                              "bf16_scaled": "mono_grouping_reduce_parts_bf16_scaled"},
    "Grouping.reduce_push_parts": {"f32": "mono_grouping_reduce_push_parts",
                                   "bf16": "mono_grouping_reduce_push_parts_bf16",
                                   "f32_scaled": "mono_grouping_reduce_push_parts_scaled",
                                   "bf16_scaled": "mono_grouping_reduce_push_parts_bf16_scaled"},
    "gather_pool_parts": {"f32": "mono_gather_pool_parts", "bf16": "mono_gather_pool_parts_bf16"},
    "MultiHashTable.pool_backward": {"f32": "mono_mtable_pool_backward",
                                     "f32_scaled": "mono_mtable_pool_backward_scaled"},
    "MultiHashTable.lookup_pool_parts": {"f32": "mono_mtable_lookup_pool_parts",
                                         "bf16": "mono_mtable_lookup_pool_parts_bf16"},
    "MultiHashTable.pool_backward_parts": {"f32": "mono_mtable_pool_backward_parts",
                                           "bf16": "mono_mtable_pool_backward_parts_bf16",
                                           "f32_scaled": "mono_mtable_pool_backward_parts_scaled",
                                           "bf16_scaled": "mono_mtable_pool_backward_parts_bf16_scaled"},
    "MultiHashTable.raw_lookup": {"f32": "mono_mtable_lookup", "f16": "mono_mtable_lookup_f16"},
    "ShardedStep.step": {"f32": ["mono_xstep_forward", "mono_xstep_backward"],
                         "f32_scaled": ["mono_xstep_forward", "mono_xstep_backward_scaled"]},
    "ShardedStep.step_parts": {"f32": ["mono_xstep_forward_parts", "mono_xstep_backward_parts"],
                               "bf16": ["mono_xstep_forward_parts_bf16", "mono_xstep_backward_parts_bf16"],
                               "f32_scaled": ["mono_xstep_forward_parts", "mono_xstep_backward_parts_scaled"],
                               "bf16_scaled": ["mono_xstep_forward_parts_bf16",
                                               "mono_xstep_backward_parts_bf16_scaled"]},
}


def _flags(variant, dev):
  """-> (bf16, scaled, the scale tensor or None) of a variant name."""
  scaled = variant.endswith("_scaled")
  return "bf16" in variant, scaled, (torch.tensor([0.3], device=dev) if scaled else None)


def _problem(dev, dtype=torch.float32):
  """U fused rows of D floats, one occurrence per row in a shuffled order (so float atomics add one term per
  element), rows of the B samples given by CSR offsets."""
  g = torch.Generator().manual_seed(5)
  fused = torch.randn(U * D, generator=g).to(dev)
  offs = (torch.randperm(U, generator=g).to(torch.int32) * D).to(dev)
  cuts = torch.sort(torch.randint(0, U + 1, (B - 1,), generator=g)).values
  ro = torch.cat([torch.zeros(1, dtype=torch.int64), cuts, torch.full((1,), U)]).to(torch.int32).to(dev)
  pg = torch.randn(B, D, generator=g).to(dtype).to(dev)
  return fused, offs, ro, pg


@pytest.mark.parametrize("variant", BF16)
def test_gather_pool(dev, monkeypatch, variant):
  bf16 = variant == "bf16"
  from monolith_b200 import distribution_ops as dops
  fused, offs, ro, _ = _problem(dev)
  dt = BF if bf16 else torch.float32

  def direct(fn):
    out = torch.empty(B, D, dtype=dt, device=dev)
    assert fn(dev.index, _p(fused), _p(offs), _p(ro), B, D, _lib.POOL_MEAN, _p(out), D, 0, _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["gather_pool"][variant],
        lambda: [dops.gather_pool(fused, offs, D, ro, "mean", dtype=dt)], direct)


@pytest.mark.parametrize("variant", ALL)
def test_gather_pool_grad(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  from monolith_b200 import distribution_ops as dops
  _, offs, ro, pg = _problem(dev, BF if bf16 else torch.float32)

  def direct(fn):
    grad = torch.zeros(U * D, device=dev)
    extra = (_p(sc),) if scaled else ()
    assert fn(dev.index, _p(pg), D, 0, _p(offs), _p(ro), B, D, _lib.POOL_MEAN, _p(grad), *extra, _s(dev)) == 0
    return [grad]
  check(monkeypatch, SYMBOLS["gather_pool_grad"][variant],
        lambda: [dops.gather_pool_grad(pg, offs, D, U * D, ro, "mean", scale=sc)], direct)


@pytest.mark.parametrize("variant", ALL)
def test_gather_pool_grad_into_atomic_branch(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  """CudaBackend's float-atomic branch (a table dim that is not a multiple of 4)."""
  from monolith_b200 import MultiHashTable
  from monolith_b200.distributed_ps import CudaBackend
  be = CudaBackend(MultiHashTable({"t": table([(6, "sgd", {})], [0.1], capacity=64)}, device=dev))
  assert not be.vec_ok
  _, offs, ro, pg = _problem(dev, BF if bf16 else torch.float32)

  def wrapper():
    buf = torch.zeros(U * D, device=dev)
    be.gather_pool_grad_into(buf, pg, offs, D, ro, "sum", **({"scale": sc} if scaled else {}))
    return [buf]

  def direct(fn):
    grad = torch.zeros(U * D, device=dev)
    extra = (_p(sc),) if scaled else ()
    assert fn(dev.index, _p(pg), D, 0, _p(offs), _p(ro), B, D, _lib.POOL_SUM, _p(grad), *extra, _s(dev)) == 0
    return [grad]
  check(monkeypatch, SYMBOLS["gather_pool_grad"][variant], wrapper, direct)


@pytest.mark.parametrize("variant", ALL)
def test_scatter_grad_rows(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  from monolith_b200 import distribution_ops as dops
  _, offs, ro, pg = _problem(dev, BF if bf16 else torch.float32)

  def direct(fn):
    grad = torch.full((U * D,), 7.0, device=dev)
    extra = (_p(sc),) if scaled else ()
    assert fn(dev.index, _p(pg), D, 0, _p(offs), U, _p(ro), B, D, _lib.POOL_MEAN, _p(grad), U * D, *extra,
              _s(dev)) == 0
    return [grad]
  check(monkeypatch, SYMBOLS["scatter_grad_rows"][variant],
        lambda: [dops.scatter_grad_rows(pg, offs, D, torch.full((U * D,), 7.0, device=dev), ro, "mean", scale=sc)],
        direct)


def _reduce_recs(splits, rows, slices, pooling):
  rec = (_lib.ReduceFeature * 1)()
  sl = (_lib.ReduceSlice * len(slices))()
  for j, t in enumerate(slices):
    sl[j].dim, sl[j].out_dev, sl[j].stride = t.size(1), t.data_ptr(), t.stride(0)
  rec[0].splits_dev, rec[0].batch_size = splits.data_ptr(), splits.numel() - 1
  rec[0].rows_dev, rec[0].n_rows, rec[0].row_stride = rows.data_ptr(), rows.size(0), rows.stride(0)
  rec[0].dim, rec[0].pooling, rec[0].slices, rec[0].n_slices = rows.size(1), pooling, sl, len(slices)
  return rec, sl


@pytest.mark.parametrize("variant", BF16)
def test_reduce_and_split(dev, monkeypatch, variant):
  bf16 = variant == "bf16"
  from monolith_b200 import distribution_ops as dops
  fused, _, ro, _ = _problem(dev)
  rows = fused.view(U, D)
  dt = BF if bf16 else torch.float32

  def direct(fn):
    outs = [torch.empty(B, 3, dtype=dt, device=dev), torch.empty(B, D - 3, dtype=dt, device=dev)]
    rec, keep = _reduce_recs(ro, rows, outs, _lib.POOL_SUM)
    assert fn(dev.index, rec, 1, None, _s(dev)) == 0
    return outs
  check(monkeypatch, SYMBOLS["reduce_and_split"][variant],
        lambda: dops.fused_reduce_and_split_gpu([ro], [rows], [[3, D - 3]], dtype=dt), direct)


@pytest.mark.parametrize("variant", ALL)
def test_reduce_and_split_grad(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  from monolith_b200 import distribution_ops as dops
  fused, _, ro, pg = _problem(dev, BF if bf16 else torch.float32)
  rows = fused.view(U, D)
  grads = [pg[:, :3], pg[:, 3:]]

  def direct(fn):
    out = torch.empty(U, D, device=dev)
    rec, keep = _reduce_recs(ro, out, grads, _lib.POOL_MEAN)
    extra = (_p(sc),) if scaled else ()
    assert fn(dev.index, rec, 1, None, *extra, _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["reduce_and_split_grad"][variant],
        lambda: dops.fused_reduce_and_split_gpu_grad([ro], [rows], grads, [[3, D - 3]], pooling="mean",
                                                     grad_scale=sc), direct)


def _layout(dev):
  """One MEAN feature of B samples over one table, one server: the sharding's index tensors and the task.  The FIDs
  are distinct, so the gradient's float atomics add one term per element."""
  from monolith_b200 import distribution_ops as dops
  g = torch.Generator().manual_seed(8)
  fids = (torch.randperm(U, generator=g) + 1).to(dev)
  cuts = torch.sort(torch.randint(0, U + 1, (B - 1,), generator=g)).values
  splits = torch.cat([torch.zeros(1, dtype=torch.int64), cuts, torch.full((1,), U)]).to(dev)
  sh = dops.sharding_sparse_fids({"f": (fids, splits)}, {"f": "t"}, {"f": D}, 1)
  n = sh["fid_list"][0].numel() * D
  tasks = [dops.SliceTask(0, 0, D, _lib.POOL_MEAN, 0, 0, D, 0, 0)]
  return sh["fid_offset"], sh["feature_offset"], sh["nfl_offset"], n, tasks


def _layout_args(dev, fo, feo, nfo, ptrs, tasks):
  from monolith_b200 import distribution_ops as dops
  pt = torch.tensor([t.data_ptr() for t in ptrs], dtype=torch.int64, device=dev)
  st = torch.ones(len(ptrs), dtype=torch.int32, device=dev)
  return (pt, st), (dev.index, _p(pt), _p(st), len(ptrs), _p(fo), fo.numel(), _p(feo), feo.numel(), _p(nfo),
                    nfo.numel(), B, dops._tasks_arr(tasks), len(tasks))


@pytest.mark.parametrize("variant", ["f32", "bf16", "f16in", "f16in_bf16"])
def test_embedding_to_layout(dev, monkeypatch, variant):
  bf16, f16_in = "bf16" in variant, variant.startswith("f16in")
  from monolith_b200 import distribution_ops as dops
  fo, feo, nfo, n, tasks = _layout(dev)
  emb = torch.randn(n, generator=torch.Generator().manual_seed(3)).to(F16 if f16_in else torch.float32).to(dev)
  dt = BF if bf16 else torch.float32

  def direct(fn):
    out = torch.zeros(B, D, dtype=dt, device=dev)
    keep, args = _layout_args(dev, fo, feo, nfo, [emb], tasks)
    op = torch.tensor([out.data_ptr()], dtype=torch.int64, device=dev)
    assert fn(*args, _p(op), _s(dev)) == 0
    torch.cuda.synchronize()
    return [out]
  check(monkeypatch, SYMBOLS["embedding_to_layout"][variant],
        lambda: dops.fused_embedding_to_layout([emb], [1], fo, feo, nfo, B, tasks, [(B, D)], dtype=dt), direct)


@pytest.mark.parametrize("variant", ALL)
def test_embedding_to_layout_grad(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  from monolith_b200 import distribution_ops as dops
  fo, feo, nfo, n, tasks = _layout(dev)
  og = torch.randn(B, D, generator=torch.Generator().manual_seed(4)).to(BF if bf16 else torch.float32).to(dev)

  def direct(fn):
    grad = torch.zeros(n, device=dev)
    keep, args = _layout_args(dev, fo, feo, nfo, [grad], tasks)
    op = torch.tensor([og.data_ptr()], dtype=torch.int64, device=dev)
    extra = (_p(sc),) if scaled else ()
    assert fn(*args, _p(op), *extra, _s(dev)) == 0
    torch.cuda.synchronize()
    return [grad]
  check(monkeypatch, SYMBOLS["embedding_to_layout_grad"][variant],
        lambda: dops.fused_embedding_to_layout_grad([n], [1], fo, feo, nfo, B, tasks, [og],
                                                    layout_tensors_grad_scale=sc), direct)


def _offset_map(dev):
  from monolith_b200 import distribution_ops as dops
  ids = torch.randint(1, 12, (U,), generator=torch.Generator().manual_seed(6)).to(dev)
  res = dops.unique_key_with_value_and_offset(ids, [0, U], [D])
  nu = res.num_unique
  pos = torch.randperm(nu, generator=torch.Generator().manual_seed(7)).to(dev)
  return res, nu, pos


@pytest.mark.parametrize("variant", HALF)
def test_fill_with_offset_map(dev, monkeypatch, variant):
  f16 = variant == "f16"
  from monolith_b200 import distribution_ops as dops
  res, nu, pos = _offset_map(dev)
  value = torch.randn(nu * D, generator=torch.Generator().manual_seed(2)).to(F16 if f16 else torch.float32).to(dev)
  offs, offs_split = res.value_offset

  def direct(fn):
    buf = torch.full((res.value_len,), 5.0, device=dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    assert fn(dev.index, _p(pos), (C.c_int64 * 2)(0, nu), 1, (C.c_int32 * 1)(D), _p(value), value.numel(), _p(offs),
              _p(offs_split), nu, _p(buf), _p(bad), _s(dev)) == 0
    return [buf]
  check(monkeypatch, SYMBOLS["fill_with_offset_map"][variant],
        lambda: [dops.fill_with_offset_map(pos, [0, nu], value, res.value_offset,
                                           torch.full((res.value_len,), 5.0, device=dev), [D], sync=False)], direct)


@pytest.mark.parametrize("variant", HALF)
def test_fill_with_offset_map_gradient(dev, monkeypatch, variant):
  f16 = variant == "f16"
  from monolith_b200 import distribution_ops as dops
  res, nu, pos = _offset_map(dev)
  grad = torch.randn(res.value_len, generator=torch.Generator().manual_seed(2)).to(dev)
  offs, offs_split = res.value_offset

  def direct(fn):
    out = torch.empty(nu * D, dtype=F16 if f16 else torch.float32, device=dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    assert fn(dev.index, _p(pos), (C.c_int64 * 2)(0, nu), 1, (C.c_int32 * 1)(D), _p(grad), _p(offs), _p(offs_split),
              nu, _p(out), _p(bad), _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["fill_with_offset_map_gradient"][variant],
        lambda: [dops.fill_with_offset_map_gradient(pos, [0, nu], grad, res.value_offset, [D], sync=False,
                                                    dtype=F16 if f16 else torch.float32)], direct)


@pytest.mark.parametrize("variant", SCALED)
def test_grouping_reduce(dev, monkeypatch, variant):
  _, scaled, sc = _flags(variant, dev)
  from monolith_b200 import distribution_ops as dops
  fids = torch.randint(1, 12, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev)
  grp = dops.Grouping(dev)
  n_u = grp.build(fids, 1, D)[0].numel()

  def direct(fn):
    out = torch.empty(n_u * D, device=dev)
    extra = (_p(sc),) if scaled else ()
    assert fn(grp._h, _p(pg), D, 0, _p(ro), B, _lib.POOL_MEAN, _p(out), *extra, _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["Grouping.reduce"][variant],
        lambda: [grp.reduce(pg, torch.empty(n_u * D, device=dev), ro, "mean", grad_scale=sc)], direct)


def _tables(dev):
  """Two tables in the same state: one for the wrapper, one for the direct call."""
  from monolith_b200 import MultiHashTable
  ids = torch.arange(1, 31, dtype=torch.int64, device=dev)
  ts = []
  for _ in range(2):
    t = MultiHashTable({"t": table([(D, "adagrad", {})], [0.1], capacity=256)}, device=dev)
    t.assign({"t": (ids, torch.linspace(-1, 1, 30 * D, device=dev).view(30, D))})
    ts.append(t)
  return ts, ids


def _rows(t, ids):
  return [t.lookup_entry("t", ids)["raw"]]


@pytest.mark.parametrize("variant", SCALED)
def test_pool_backward(dev, monkeypatch, variant):
  _, scaled, sc = _flags(variant, dev)
  (a, b), ids = _tables(dev)
  fids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev)

  def wrapper():
    a.pool_backward("t", fids, pg, ro, "mean", req_time=9, global_step=2, grad_scale=sc)
    return _rows(a, fids)

  def direct(fn):
    extra = (_p(sc),) if scaled else ()
    assert fn(b.handle, 0, _p(fids), U, _p(ro), B, _lib.POOL_MEAN, _p(pg), D, 0, (C.c_float * 1)(0.1), 9, 2, *extra,
              _s(dev)) == 0
    return _rows(b, fids)
  check(monkeypatch, SYMBOLS["MultiHashTable.pool_backward"][variant], wrapper, direct)


def _part_arr(fids, ro, rows):
  arr = (_lib.PoolPartC * 1)()
  arr[0] = _lib.PoolPartC(0, fids.data_ptr(), fids.numel(), ro.data_ptr(), ro.numel() - 1, _lib.POOL_MEAN,
                          rows.data_ptr(), rows.stride(0), 0, 0)
  return arr


@pytest.mark.parametrize("variant", BF16)
def test_lookup_pool_parts(dev, monkeypatch, variant):
  bf16 = variant == "bf16"
  from monolith_b200 import PoolPart
  (a, _), _ = _tables(dev)
  fids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, _ = _problem(dev)
  dt = BF if bf16 else torch.float32

  def direct(fn):
    out = torch.empty(B, D, dtype=dt, device=dev)
    assert fn(a.handle, _part_arr(fids, ro, out), 1, _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["MultiHashTable.lookup_pool_parts"][variant],
        lambda: a.lookup_pool_parts([PoolPart("t", fids, ro, "mean")], dtype=dt), direct)


@pytest.mark.parametrize("variant", ALL)
def test_pool_backward_parts(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  from monolith_b200 import PoolPart
  (a, b), _ = _tables(dev)
  fids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev, BF if bf16 else torch.float32)

  def wrapper():
    a.pool_backward_parts([PoolPart("t", fids, ro, "mean", pg)], req_time=9, global_step=2, grad_scale=sc)
    return _rows(a, fids)

  def direct(fn):
    extra = (_p(sc),) if scaled else ()
    assert fn(b.handle, _part_arr(fids, ro, pg), 1, (C.c_float * 1)(0.1), 9, 2, *extra, _s(dev)) == 0
    return _rows(b, fids)
  check(monkeypatch, SYMBOLS["MultiHashTable.pool_backward_parts"][variant], wrapper, direct)


@pytest.mark.parametrize("variant", HALF)
def test_raw_lookup(dev, monkeypatch, variant):
  f16 = variant == "f16"
  (a, _), _ = _tables(dev)
  ids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)

  def direct(fn):
    out = torch.empty(U * D, dtype=F16 if f16 else torch.float32, device=dev)
    assert fn(a.handle, _p(ids), (C.c_int64 * 2)(0, U), _p(out), _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["MultiHashTable.raw_lookup"][variant],
        lambda: [a.raw_lookup(ids, [0, U], dtype=F16 if f16 else torch.float32)], direct)


def _window_case(dev, fn):
  """fn(window) with a world-1 peer window of U * D floats, closed afterwards."""
  from monolith_b200 import distribution_ops as dops
  win = dops.PeerWindow(dev, 1, 0, U * D * 4)
  try:
    fn(win)
  finally:
    torch.cuda.synchronize()
    win.close()


def _pushed(win, n):
  return [win.view(0, n, torch.float32).clone()]


@pytest.mark.parametrize("variant", SCALED)
def test_grouping_reduce_push(dev, monkeypatch, variant):
  from monolith_b200 import distribution_ops as dops
  _, scaled, sc = _flags(variant, dev)
  fids = torch.randint(1, 12, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev)
  grp = dops.Grouping(dev)
  _, _, sizes = grp.build(fids, 1, D)
  n = sum(sizes) * D

  def case(win):
    def wrapper():
      win.view(0, n, torch.float32).fill_(7.0)
      grp.reduce_push(pg, sizes, win, 0, [0], ro, "mean", grad_scale=sc)
      return _pushed(win, n)

    def direct(fn):
      win.view(0, n, torch.float32).fill_(7.0)
      extra = (_p(sc),) if scaled else ()
      assert fn(grp._h, _p(pg), D, 0, _p(ro), B, _lib.POOL_MEAN, (C.c_int64 * 1)(*sizes), win._h, 0,
                (C.c_int64 * 1)(0), *extra, _s(dev)) == 0
      return _pushed(win, n)
    check(monkeypatch, SYMBOLS["Grouping.reduce_push"][variant], wrapper, direct)
  _window_case(dev, case)


def _parts_grouping(dev, dtype):
  """A table, a parts grouping of one MEAN part over it, and that part's FIDs, row offsets and gradient rows."""
  from monolith_b200 import distribution_ops as dops
  (t, _), _ = _tables(dev)
  fids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev, dtype)
  grp = dops.Grouping(dev)
  uniq, occ, sizes = grp.build_parts(t, _part_arr(fids, ro, torch.empty(B, D, device=dev)), 1, U, 1, D)
  return t, grp, fids, ro, pg, uniq.numel(), occ, sizes


@pytest.mark.parametrize("variant", ALL)
def test_grouping_reduce_parts(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  t, grp, fids, ro, pg, n_u, _, _ = _parts_grouping(dev, BF if bf16 else torch.float32)
  arr = _part_arr(fids, ro, pg)

  def direct(fn):
    out = torch.empty(n_u * D, device=dev)
    extra = (_p(sc),) if scaled else ()
    assert fn(grp._h, t.handle, arr, 1, _p(out), *extra, _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["Grouping.reduce_parts"][variant],
        lambda: [grp.reduce_parts(t, arr, 1, bf16, torch.empty(n_u * D, device=dev), grad_scale=sc)], direct)


@pytest.mark.parametrize("variant", ALL)
def test_grouping_reduce_push_parts(dev, monkeypatch, variant):
  bf16, scaled, sc = _flags(variant, dev)
  t, grp, fids, ro, pg, n_u, _, sizes = _parts_grouping(dev, BF if bf16 else torch.float32)
  arr = _part_arr(fids, ro, pg)

  def case(win):
    def wrapper():
      win.view(0, n_u * D, torch.float32).fill_(7.0)
      grp.reduce_push_parts(t, arr, 1, bf16, sizes, win, 0, [0], grad_scale=sc)
      return _pushed(win, n_u * D)

    def direct(fn):
      win.view(0, n_u * D, torch.float32).fill_(7.0)
      extra = (_p(sc),) if scaled else ()
      assert fn(grp._h, t.handle, arr, 1, (C.c_int64 * 1)(*sizes), win._h, 0, (C.c_int64 * 1)(0), *extra,
                _s(dev)) == 0
      return _pushed(win, n_u * D)
    check(monkeypatch, SYMBOLS["Grouping.reduce_push_parts"][variant], wrapper, direct)
  _window_case(dev, case)


@pytest.mark.parametrize("variant", BF16)
def test_gather_pool_parts(dev, monkeypatch, variant):
  from monolith_b200 import distribution_ops as dops
  bf16 = variant == "bf16"
  dt = BF if bf16 else torch.float32
  t, _, fids, ro, _, n_u, occ, _ = _parts_grouping(dev, torch.float32)
  rows_in = torch.randn(n_u * D, generator=torch.Generator().manual_seed(3)).to(dev)

  def wrapper():
    out = torch.empty(B, D, dtype=dt, device=dev)
    dops.gather_pool_parts(t, rows_in, occ, _part_arr(fids, ro, out), 1, bf16)
    return [out]

  def direct(fn):
    out = torch.empty(B, D, dtype=dt, device=dev)
    assert fn(t.handle, _p(rows_in), _p(occ), _part_arr(fids, ro, out), 1, _s(dev)) == 0
    return [out]
  check(monkeypatch, SYMBOLS["gather_pool_parts"][variant], wrapper, direct)


def _steps(dev, warm):
  """Two direct-exchange steps at world 1 over tables in the same state, both after the same warm-up step (which
  makes their device-driven step objects), for the wrapper and for the direct calls."""
  from monolith_b200.distributed_ps import ShardedStep
  (a, b), _ = _tables(dev)
  sts = [ShardedStep(t, "t", D, 1, 0, dev, exchange="direct") for t in (a, b)]
  for st in sts:
    warm(st)
  return sts


def _close(sts):
  torch.cuda.synchronize()
  for st in sts:
    st.close_direct()


@pytest.mark.parametrize("variant", SCALED)
def test_sharded_step(dev, monkeypatch, variant):
  _, scaled, sc = _flags(variant, dev)
  fids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev)
  sa, sb = _steps(dev, lambda st: st.step(fids, pg, torch.empty(B, D, device=dev), 5, ro, "mean"))
  try:
    def wrapper():
      out = torch.empty(B, D, device=dev)
      sa.step(fids, pg, out, 9, ro, "mean", grad_scale=sc)
      return [out] + _rows(sa.table, fids)

    def direct(fwd, bwd):
      out = torch.empty(B, D, device=dev)
      assert fwd(sb.xstep, _p(fids), U, _p(ro), B, _lib.POOL_MEAN, _p(out), D, 0, _s(dev)) == 0
      extra = (_p(sc),) if scaled else ()
      assert bwd(sb.xstep, _p(pg), D, 0, _p(ro), _lib.POOL_MEAN, (C.c_float * 1)(0.1), 9, *extra, _s(dev)) == 0
      return [out] + _rows(sb.table, fids)
    check(monkeypatch, SYMBOLS["ShardedStep.step"][variant], wrapper, direct)
  finally:
    _close([sa, sb])


@pytest.mark.parametrize("variant", ALL)
def test_sharded_step_parts(dev, monkeypatch, variant):
  from monolith_b200 import PoolPart
  bf16, scaled, sc = _flags(variant, dev)
  dt = BF if bf16 else torch.float32
  fids = torch.randint(1, 40, (U,), generator=torch.Generator().manual_seed(1)).to(dev)
  _, _, ro, pg = _problem(dev, dt)
  sa, sb = _steps(dev, lambda st: st.step_parts([PoolPart("t", fids, ro, "mean")], [pg], 5))
  try:
    def wrapper():
      out = torch.empty(B, D, dtype=dt, device=dev)
      sa.step_parts([PoolPart("t", fids, ro, "mean", out)], [pg], 9, grad_scale=sc)
      return [out] + _rows(sa.table, fids)

    def direct(fwd, bwd):
      out = torch.empty(B, D, dtype=dt, device=dev)
      assert fwd(sb.xstep, _part_arr(fids, ro, out), 1, _s(dev)) == 0
      extra = (_p(sc),) if scaled else ()
      assert bwd(sb.xstep, _part_arr(fids, ro, pg), 1, (C.c_float * 1)(0.1), 9, *extra, _s(dev)) == 0
      return [out] + _rows(sb.table, fids)
    check(monkeypatch, SYMBOLS["ShardedStep.step_parts"][variant], wrapper, direct)
  finally:
    _close([sa, sb])
