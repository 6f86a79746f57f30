"""transfer_float16 of the async parameter-server table on the device.  The three fp16 calls are checked bit for bit
against their fp32 twins: the lookup and the fill gradient against the twin's result rounded once to fp16 (numpy's
astype(np.float16)), the fill against the twin on the rows widened exactly.  NaN is compared as NaN.
DistributedMultiTypeHashTable(transfer_float16=True) is checked against oracle tables (tests/orc.py) driven by the
reference's per-slot path with its fp16 casts (tests/fp16_transfer_model.py)."""
import numpy as np
import pytest
import torch

from monolith_b200 import MultiHashTable, _lib, distribution_ops as dops
from monolith_b200.distributed_ps import DistributedMultiTypeHashTable
from tests import fp16_transfer_model as fm
from tests import orc
from tests.helpers import sgd_table, table

pytestmark = pytest.mark.gpu
I64_MIN = np.iinfo(np.int64).min
# values whose fp16 rounding is an edge: the largest fp16, a value just below the midpoint that rounds down to it, the
# midpoint that rounds to inf, the smallest fp16 subnormal, half of it (a tie, to even 0), three quarters of it (up to
# 2^-24), signed zeros, fp32 subnormals, infinities and NaN
EDGES = np.array([65504, 65519.99, 65520, -65520, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, -3 * 2.0 ** -26, 0.0, -0.0,
                  1e-45, -1e-40, np.inf, -np.inf, np.nan], np.float32)


@pytest.fixture(scope="module")
def dev():
  if not torch.cuda.is_available():
    pytest.skip("needs a GPU")
  return torch.device("cuda", 0)


def same_f16(got, want32):
  """got (fp16, any container) is want32 (fp32) rounded once to fp16, bit for bit; NaN as NaN"""
  got = np.asarray(got.cpu().numpy() if torch.is_tensor(got) else got, np.float16).reshape(-1)
  with np.errstate(over="ignore", invalid="ignore"):
    want = np.asarray(want32, np.float32).reshape(-1).astype(np.float16)
  assert got.shape == want.shape
  gn, wn = np.isnan(got), np.isnan(want)
  assert np.array_equal(gn, wn), "NaN positions differ"
  diff = np.nonzero(got[~gn].view(np.uint16) != want[~wn].view(np.uint16))[0]
  assert diff.size == 0, f"{diff.size} elements differ, first at {diff[:5]}: {got[~gn][diff[:5]]} {want[~wn][diff[:5]]}"


def same_f32(got, want):
  got, want = np.asarray(got, np.float32).reshape(-1), np.asarray(want, np.float32).reshape(-1)
  assert got.shape == want.shape
  gn, wn = np.isnan(got), np.isnan(want)
  assert np.array_equal(gn, wn), "NaN positions differ"
  diff = np.nonzero(got[~gn].view(np.uint32) != want[~wn].view(np.uint32))[0]
  assert diff.size == 0, f"{diff.size} floats differ, first at {diff[:5]}"


def with_edges(rng, x, share=0.05):
  at = rng.random(x.shape) < share
  x[at] = EDGES[rng.integers(0, EDGES.size, int(at.sum()))]
  return x


# ---- mono_mtable_lookup_f16 -------------------------------------------------------------------------------------------
LOOKUP_DIMS = [1, 2, 3, 5, 16, 17, 32, 33, 64, 128, 257]  # every lane-group width; 32 and 64 take TMA in fp32


@pytest.fixture(scope="module")
def lookup_table(dev):
  """one table per dim (names sort in dim order), 400 keys each assigned values with the fp16 edges"""
  rng = np.random.default_rng(1)
  cfg = {f"d{d:03d}": table([(d, "sgd", {})], [0.1]) for d in LOOKUP_DIMS}
  mt = MultiHashTable(cfg, device=dev)
  keys = {}
  for d in LOOKUP_DIMS:
    k = np.unique(rng.integers(I64_MIN, np.iinfo(np.int64).max, 400, dtype=np.int64))
    v = (rng.standard_normal((k.size, d)) * rng.choice([1e-6, 1.0, 3e4, 1e5], (k.size, 1))).astype(np.float32)
    v = with_edges(rng, v)
    v[:EDGES.size, 0] = EDGES  # every edge in column 0 of the first keys, and in the last column
    v[:EDGES.size, -1] = EDGES[::-1]
    mt.assign({f"d{d:03d}": (torch.from_numpy(k).to(dev), torch.from_numpy(v).to(dev))})
    keys[d] = k
  return mt, keys


def lookup_ids(rng, keys, n):
  """n ids of the assigned keys, repeats included, about one in five a miss"""
  ids = keys[rng.integers(0, keys.size, n)]
  miss = rng.random(n) < 0.2
  ids[miss] = rng.integers(1, 1 << 40, int(miss.sum()))
  return ids


def check_lookup(dev, mt, ids_per_dim):
  flat = np.concatenate([ids_per_dim.get(d, np.zeros(0, np.int64)) for d in LOOKUP_DIMS])
  split = np.cumsum([0] + [ids_per_dim.get(d, np.zeros(0)).size for d in LOOKUP_DIMS]).tolist()
  t = torch.from_numpy(flat).to(dev)
  f32 = mt.raw_lookup(t, split)
  f16 = mt.raw_lookup(t, split, dtype=torch.float16)
  assert f16.dtype == torch.float16 and f16.shape == f32.shape
  same_f16(f16, f32.cpu().numpy())
  return f16


@pytest.mark.parametrize("dim", LOOKUP_DIMS)
def test_lookup_f16_one_table(dev, lookup_table, dim):
  mt, keys = lookup_table
  rng = np.random.default_rng(dim)
  for n in (1, 31, 32, 33, 5000):
    check_lookup(dev, mt, {dim: lookup_ids(rng, keys[dim], n)})


def test_lookup_f16_every_table_in_one_call(dev, lookup_table):
  mt, keys = lookup_table
  rng = np.random.default_rng(2)
  for _ in range(3):  # odd row counts put later tables at unaligned fp16 offsets
    ids = {d: lookup_ids(rng, keys[d], int(rng.integers(1, 900))) for d in LOOKUP_DIMS}
    check_lookup(dev, mt, ids)
  ids = {d: lookup_ids(rng, keys[d], 700) for d in LOOKUP_DIMS[::3]}  # some tables empty
  check_lookup(dev, mt, ids)


def test_lookup_f16_edges_and_misses(dev, lookup_table):
  mt, keys = lookup_table
  k = keys[17][:EDGES.size]
  miss = np.array([12345, -1, I64_MIN], np.int64)
  got = check_lookup(dev, mt, {17: np.concatenate([k, miss])}).cpu().numpy().reshape(-1, 17)
  col0 = got[:EDGES.size, 0]
  want = np.array([65504, 65504, np.inf, -np.inf, 2.0 ** -24, 0, 2.0 ** -24, -2.0 ** -24, 0, -0.0, 0, -0.0, np.inf,
                   -np.inf, np.nan], np.float16)
  assert np.array_equal(np.isnan(col0), np.isnan(want))
  assert col0[:-1].view(np.uint16).tolist() == want[:-1].view(np.uint16).tolist()
  assert got[EDGES.size:].view(np.uint16).tolist() == np.zeros((3, 17), np.uint16).tolist()  # misses are +0.0


def test_lookup_f16_rejects_a_split_that_does_not_cover_the_ids(dev, lookup_table):
  mt, _ = lookup_table
  with pytest.raises(ValueError, match="cover"):
    mt.raw_lookup(torch.zeros(3, dtype=torch.int64, device=dev), [0] * len(LOOKUP_DIMS) + [2], dtype=torch.float16)


# ---- mono_fill_with_offset_map_f16 and mono_fill_with_offset_map_grad_f16 ---------------------------------------------
def f16_rows(rng, n):
  x = (rng.standard_normal(n) * rng.choice([1e-5, 1.0, 1e4], n)).astype(np.float32)
  with np.errstate(over="ignore"):  # the edges beyond the fp16 range become +-inf
    return with_edges(rng, x).astype(np.float16)


def grad_values(rng, n):
  return with_edges(rng, (rng.standard_normal(n) * rng.choice([1e-6, 1.0, 3e4], n)).astype(np.float32), 0.01)


def check_fills(dev, keys, split, dims, S, rng, g_in=None):
  """unique -> split by floormod(key, S) -> per server the fp16 fill against the fp32 fill on the widened rows, and the
  fp16 fill gradient against the fp32 one rounded"""
  res = dops.unique_key_with_value_and_offset(torch.from_numpy(keys).to(dev), split.tolist(), dims)
  U = res.num_unique
  sp = dops.ragged_split_by_indices(torch.remainder(res.unique_key[0], S), res.unique_key[0], res.unique_key[1], S)
  buf16 = res.value_buffer.fill_(-12345.0)  # not an fp16 value: no row can write it
  buf32 = buf16.clone()
  g_in = grad_values(rng, res.value_len) if g_in is None else g_in
  g_dev = torch.from_numpy(g_in).to(dev)
  for s in range(S):
    p, rs = sp.pos[s], sp.row_splits_host[s]
    rows = sum((rs[k + 1] - rs[k]) * dims[k] for k in range(len(dims)))
    val = torch.from_numpy(f16_rows(rng, rows)).to(dev)
    dops.fill_with_offset_map(p, rs, val, res.value_offset, buf16, dims, num_unique=U)
    dops.fill_with_offset_map(p, rs, val.float(), res.value_offset, buf32, dims, num_unique=U)
    g32 = dops.fill_with_offset_map_gradient(p, rs, g_dev, res.value_offset, dims, num_unique=U)
    g16 = dops.fill_with_offset_map_gradient(p, rs, g_dev, res.value_offset, dims, num_unique=U, dtype=torch.float16)
    assert g16.dtype == torch.float16 and g16.shape == g32.shape
    same_f16(g16, g32.cpu().numpy())
  got = buf16.cpu().numpy()
  assert not (got == -12345.0).any(), "the S fills left floats of the buffer unwritten"
  same_f32(got, buf32.cpu().numpy())
  return res


def _keys(rng, M, vocab):
  return rng.integers(0, vocab, M).astype(np.int64)


@pytest.mark.parametrize("M", [1, 31, 32, 33, 2047, 2048, 2049, 8191, 8192, 8193, 100_000])
def test_fills_at_tile_and_warp_boundaries(dev, M):
  rng = np.random.default_rng(M)
  check_fills(dev, _keys(rng, M, max(2, M // 3)), np.array([0, M]), [3], 2, rng)


@pytest.mark.parametrize("dim", [1, 2, 3, 5, 16, 17, 33, 128, 257])
def test_fills_at_odd_and_wide_dims(dev, dim):
  rng = np.random.default_rng(100 + dim)
  keys = np.concatenate([_keys(rng, 3000, 700), _keys(rng, 1000, 300)])
  keys[rng.integers(0, keys.size, 20)] = np.array([-1, I64_MIN, -7, 5], np.int64)[rng.integers(0, 4, 20)]
  check_fills(dev, keys, np.array([0, 3000, 4000]), [dim, 4], 3, rng)


def test_fill_gradient_runs_up_to_2_17_and_overflow_to_inf(dev):
  """run lengths 1, 2, 3, ..., 1000 and one key of 2^17 + 5 occurrences; terms uniform in [0.5, 1.5) make the long
  run's sum pass 65520 (inf in fp16), and short runs of +-4e4 overflow to +-inf too"""
  rng = np.random.default_rng(17)
  lens = np.concatenate([np.arange(1, 1001), [(1 << 17) + 5]])
  keys = rng.permutation(np.repeat(np.arange(lens.size, dtype=np.int64) * 7919 - 5000, lens))
  dims = [2]
  g = (rng.random(keys.size * 2) + 0.5).astype(np.float32)
  big = np.nonzero(np.isin(keys, [7919 * 2 - 5000, 7919 * 3 - 5000]))[0]  # the runs of lengths 3 and 4
  g[2 * big] = 4e4
  g[2 * big + 1] = -4e4
  check_fills(dev, keys, np.array([0, keys.size]), dims, 1, rng, g)
  # the long run's sum really is beyond the fp16 range
  res = dops.unique_key_with_value_and_offset(torch.from_numpy(keys).to(dev), [0, keys.size], dims)
  hot = int(np.nonzero(res.unique_key[0].cpu().numpy() == lens.size * 7919 - 7919 - 5000)[0][0])
  out = dops.fill_with_offset_map_gradient(torch.tensor([hot], device=dev), [0, 1], torch.from_numpy(g).to(dev),
                                           res.value_offset, dims, num_unique=res.num_unique, dtype=torch.float16)
  assert np.isinf(out.cpu().numpy()).all()


def test_fill_f16_rejects_a_short_value(dev):
  res = dops.unique_key_with_value_and_offset(torch.arange(4, device=dev), [0, 4], [3])
  with pytest.raises(ValueError, match="expected: 12, actual: 10"):
    dops.fill_with_offset_map(torch.arange(4, device=dev), [0, 4], torch.zeros(10, dtype=torch.float16, device=dev),
                              res.value_offset, res.value_buffer, [3])


# ---- DistributedMultiTypeHashTable(transfer_float16=True) -------------------------------------------------------------
def _cfgs(opt):
  params = {"sgd": ("sgd", {}), "adagrad": ("adagrad", {}), "ftrl": ("ftrl", {})}[opt]
  return {"1": table([(3, params[0], params[1])], [0.05]), "2": table([(16, params[0], params[1])], [0.1]),
          "3": table([(1, params[0], params[1])], [0.2])}


def _train_and_compare(S, opt, devices):
  rng = np.random.default_rng(S * 11 + len(opt))
  cfg = _cfgs(opt)
  dmt = DistributedMultiTypeHashTable(S, cfg, lambda i, c: MultiHashTable(_cfgs(opt), device=devices[i % len(devices)]),
                                      transfer_float16=True)
  assert dmt.transfer_float16
  orcs = [orc.OracleMultiHashTable(_cfgs(opt)) for _ in range(S)]
  dims = {"1": 3, "2": 16, "3": 1}
  dev0 = devices[0]

  def server_lookup(s, slot, ids):
    return orcs[s].lookup({slot: np.asarray(ids, np.int64)})[slot].reshape(-1, dims[slot])

  for step in range(4):
    ids = {"1": rng.integers(-50, 50, 300), "2": rng.zipf(1.3, 500) % 200 - 20, "3": rng.integers(-5, 5, 40)}
    if step == 2:
      ids.pop("3")
    ids = {k: v.astype(np.int64) for k, v in ids.items()}
    ids["1"][:2] = [-1, I64_MIN]
    grads = {k: (rng.standard_normal((v.size, dims[k])) * rng.choice([1e-4, 1.0, 2e4], (v.size, 1))).astype(np.float32)
             for k, v in ids.items()}
    tids = {k: torch.from_numpy(v).to(dev0) for k, v in ids.items()}
    dmt.apply_gradients({k: (tids[k], torch.from_numpy(grads[k]).to(dev0)) for k in ids}, global_step=step,
                        req_time=100 + step)
    for s, per_slot in enumerate(fm.apply_gradients(S, {k: (ids[k], grads[k]) for k in ids})):
      orcs[s].apply_gradients(per_slot, global_step=step, req_time=100 + step)
    got = dmt.lookup(tids)
    want = fm.lookup(server_lookup, S, ids)
    assert sorted(got) == sorted(want)
    for k in ids:
      assert got[k].dtype == torch.float32
      same_f32(got[k].cpu().numpy(), want[k])


@pytest.mark.parametrize("S", [1, 2, 3, 5])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "ftrl"])
def test_training_steps_one_device(dev, S, opt):
  _train_and_compare(S, opt, [dev])


@pytest.mark.parametrize("opt", ["sgd", "ftrl"])
def test_training_steps_across_two_devices(opt):
  if torch.cuda.device_count() < 2:
    pytest.skip("needs two GPUs")
  _train_and_compare(3, opt, [torch.device("cuda", 0), torch.device("cuda", 1)])


def test_reference_apply_gradients_float16(dev):
  """ref: distributed_ps_test.py:376-413 (test_apply_gradients_float16, 2 servers, SGD lr 1 from zeros)"""
  cfg = lambda: {"1": sgd_table(1), "2": sgd_table(2)}
  dmt = DistributedMultiTypeHashTable(2, cfg(), lambda i, c: MultiHashTable(cfg(), device=dev), transfer_float16=True)
  t = lambda x, dt=torch.int64: torch.tensor(x, dtype=dt, device=dev)
  ids1, ids2 = t([1, 2]), t([3])
  dmt.apply_gradients({"1": (ids1, t([[2.0], [2.0]], torch.float32)), "2": (ids2, t([[3.0, 3.0]], torch.float32))},
                      global_step=1)
  got = dmt.lookup({"1": ids1, "2": ids2})
  assert got["1"].cpu().tolist() == [[-2.0], [-2.0]]
  assert got["2"].cpu().tolist() == [[-3.0, -3.0]]


def _kernel_names(fn):
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  return {e.name.split("<")[0].split("(")[0].replace("void ", "").replace("mono::", "") for e in prof.events()}


def test_transfer_float16_false_runs_the_fp32_kernels(dev):
  """transfer_float16=False launches none of the fp16 kernels; True launches them, in as many engine launches"""
  rng = np.random.default_rng(4)
  lib = _lib.load()
  runs = {}
  for f16 in (False, True):
    cfg = lambda: {"a": table([(32, "adagrad", {})], [0.1]), "b": table([(5, "sgd", {})], [0.1])}
    dmt = DistributedMultiTypeHashTable(2, cfg(), lambda i, c: MultiHashTable(cfg(), device=dev),
                                        transfer_float16=f16)
    ids = {"a": torch.from_numpy(rng.integers(0, 500, 3000)).to(dev), "b": torch.from_numpy(rng.integers(0, 50, 70)).to(dev)}
    grads = {"a": torch.randn(3000, 32, device=dev), "b": torch.randn(70, 5, device=dev)}

    def step():
      dmt.apply_gradients({k: (ids[k], grads[k]) for k in ids}, req_time=1)
      dmt.lookup(ids)

    step()  # the first step inserts; the traced one finds every key
    n0 = lib.mono_kernel_launch_count()
    step()
    torch.cuda.synchronize()
    launches = lib.mono_kernel_launch_count() - n0
    for _ in range(5):  # the profiler may lose records; a lost record only removes names
      names = _kernel_names(step)
      if not f16 or {"f16_lookup_kernel", "f16_fill_copy_kernel", "f16_fill_grad_kernel"} <= names:
        break
    runs[f16] = (launches, names)
  assert not any(n.startswith("f16_") for n in runs[False][1]), sorted(runs[False][1])
  assert {"f16_lookup_kernel", "f16_fill_copy_kernel", "f16_fill_grad_kernel"} <= runs[True][1], sorted(runs[True][1])
  assert runs[False][0] == runs[True][0]


def test_sync_false_f16_calls_do_not_wait(dev, lookup_table):
  mt, keys = lookup_table
  rng = np.random.default_rng(6)
  k = torch.from_numpy(_keys(rng, 20_000, 3000)).to(dev)
  res = dops.unique_key_with_value_and_offset(k, [0, 20_000], [4])
  sp = dops.ragged_split_by_indices(torch.remainder(res.unique_key[0], 2), res.unique_key[0], res.unique_key[1], 2)
  p, rs = sp.pos[0], sp.row_splits_host[0]
  val = torch.randn(rs[-1] * 4, device=dev).half()
  g = torch.randn(res.value_len, device=dev)
  ids = torch.from_numpy(lookup_ids(rng, keys[16], 4000)).to(dev)
  split = [0] * (LOOKUP_DIMS.index(16) + 1) + [4000] * (len(LOOKUP_DIMS) - LOOKUP_DIMS.index(16))
  torch.cuda.synchronize()
  torch.cuda._sleep(1_000_000_000)  # about half a second of a busy stream
  out = dops.fill_with_offset_map_gradient(p, rs, g, res.value_offset, [4], num_unique=res.num_unique, sync=False,
                                           dtype=torch.float16)
  dops.fill_with_offset_map(p, rs, val, res.value_offset, res.value_buffer, [4], num_unique=res.num_unique, sync=False)
  rows = mt.raw_lookup(ids, split, dtype=torch.float16)
  assert not torch.cuda.current_stream(dev).query(), "an fp16 call waited for the stream"
  torch.cuda.synchronize()
  same_f16(out, dops.fill_with_offset_map_gradient(p, rs, g, res.value_offset, [4]).cpu().numpy())
  same_f16(rows, mt.raw_lookup(ids, split).cpu().numpy())
