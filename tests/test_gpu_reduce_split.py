"""mono_reduce_and_split[_grad][_bf16] on the device (the default pooling path: ReduceSum / ReduceMean /
FusedReduceAndSplitGPU and their gradients), bit for bit against the numpy restatement in
tests/reduce_split_model.py (sequential fp32 adds per sample).  NaN outputs of
the arithmetic are compared by position only (the GPU returns its canonical NaN, x86 keeps an operand's payload);
the SUM gradient is a copy and keeps every bit."""
import numpy as np
import pytest
import torch

from monolith_b200 import MultiHashTable, _lib, distribution_ops as dops, entry
from tests import orc, reduce_split_model as rsm

pytestmark = pytest.mark.gpu

RAN = set()   # (direction, element, lane-group width) of every kernel instantiation launched here


def pick_group(d):
  v, g = (d + 3) // 4, 4
  while g < v and g < 32:
    g *= 2
  return g


def launches(f, *a, **k):
  lib = _lib.load()
  torch.cuda.synchronize()
  c0 = lib.mono_kernel_launch_count()
  out = f(*a, **k)
  torch.cuda.synchronize()
  return out, lib.mono_kernel_launch_count() - c0


def special(rng, shape):
  """Random values with -0.0, +-inf, NaN payloads, subnormals and pairs whose sum overflows sprinkled in."""
  x = rng.standard_normal(shape).astype(np.float32)
  pick = rng.random(shape)
  x[pick < 0.02] = -0.0
  x[(pick >= 0.02) & (pick < 0.03)] = np.inf
  x[(pick >= 0.03) & (pick < 0.04)] = -np.inf
  x[(pick >= 0.04) & (pick < 0.05)] = np.uint32(0x7FC01234).view(np.float32)
  x[(pick >= 0.05) & (pick < 0.07)] = np.float32(1e-40)
  x[(pick >= 0.07) & (pick < 0.09)] = np.float32(3e38)
  return x


def same_bits(got, want):
  got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
  assert got.shape == want.shape
  nan = np.isnan(want)
  np.testing.assert_array_equal(np.isnan(got), nan)
  np.testing.assert_array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan])


def bf16_round(x):
  return torch.from_numpy(np.asarray(x, np.float32)).to(torch.bfloat16)


def make_case(rng, B, feats, values=special):
  """feats: [(dim, slice_dims, row_lens or None, pooling)] -> numpy splits, rows and the descriptions."""
  sps, rows = [], []
  for dim, sd, lens, _ in feats:
    assert sum(sd) == dim
    lens = rng.integers(0, 5, B) if lens is None else np.asarray(lens)
    sps.append(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32))
    rows.append(values(rng, (int(sps[-1][-1]), dim)))
  return sps, rows


def check_case(dev, B, feats, seed=0, dtype=torch.float32, values=special):
  rng = np.random.default_rng(seed)
  sps, rows = make_case(rng, B, feats, values)
  sdims, pools = [f[1] for f in feats], [f[3] for f in feats]
  want = rsm.reduce_and_split(sps, rows, sdims, pools)
  tsp = [torch.from_numpy(s).to(dev) for s in sps]
  trows = [torch.from_numpy(r).to(dev) for r in rows]
  got, n = launches(dops.fused_reduce_and_split_gpu, tsp, trows, sdims, pooling=pools, dtype=dtype)
  widths = {pick_group(max(sd)) for sd in sdims} if B else set()
  assert n == len(widths)
  RAN.update(("fwd", dtype, g) for g in widths)
  flat_want = [w for ws in want for w in ws]
  for g, w in zip(got, flat_want):
    if dtype == torch.float32:
      same_bits(g.cpu().numpy(), w)
    else:
      r = bf16_round(w)
      np.testing.assert_array_equal(torch.isnan(g.cpu()).numpy(), torch.isnan(r).numpy())
      m = ~torch.isnan(r)
      assert torch.equal(g.cpu()[m].view(torch.int16), r[m].view(torch.int16))
  # gradient: slice gradients with the same kinds of values
  grads = [special(rng, (B, d)) for sd in sdims for d in sd]
  it = iter(grads)
  per = [[next(it) for _ in sd] for sd in sdims]
  if dtype == torch.bfloat16:   # the widened bf16 values are what the fp32 model sees
    per = [[bf16_round(g).float().numpy() for g in gs] for gs in per]
  gwant = rsm.reduce_and_split_grad(sps, [r.shape for r in rows], per, pools)
  tg = [torch.from_numpy(g).to(dtype).to(dev) for gs in per for g in gs]   # exact: per holds bf16 values
  ggot, n = launches(dops.fused_reduce_and_split_gpu_grad, tsp, trows, tg, sdims, pooling=pools)
  assert n == len(widths)
  RAN.update(("bwd", dtype, g) for g in widths)
  for g, w, p in zip(ggot, gwant, pools):
    g = g.cpu().numpy()
    if p == "sum":
      np.testing.assert_array_equal(g.view(np.uint32), w.view(np.uint32))   # a copy: NaN payloads kept
    else:
      same_bits(g, w)


@pytest.fixture(scope="module")
def dev():
  torch.cuda.set_device(0)
  return torch.device("cuda", 0)


@pytest.mark.parametrize("dim", list(range(1, 34)) + [47, 63, 64, 65, 96, 127, 128, 129, 200, 203, 255, 256, 257])
@pytest.mark.parametrize("pooling", ["sum", "mean"])
def test_every_dim_as_one_slice_and_as_odd_slices(dev, dim, pooling):
  odd = [1] * dim if dim < 4 else [dim // 4] * 3 + [dim // 4 + dim % 4]
  check_case(dev, 37, [(dim, [dim], None, pooling), (dim, odd, None, pooling)], seed=dim)


@pytest.mark.parametrize("lens", [[0], [1], [2], [31], [32], [33], [4000], [0, 1, 2, 31, 32, 33, 0, 5000, 7]])
@pytest.mark.parametrize("dim", [1, 16, 33, 64, 128])
def test_row_lengths(dev, lens, dim):
  B = len(lens)
  check_case(dev, B, [(dim, [dim], lens, "sum"), (dim, [dim], lens, "mean")], seed=B + dim)


@pytest.mark.parametrize("B", [1, 37, 65536])
def test_batch_sizes(dev, B):
  check_case(dev, B, [(16, [16], None, "sum"), (32, [8, 24], None, "mean"), (7, [3, 4], None, "sum")], seed=B)


@pytest.mark.parametrize("F", [1, 2, 26, 102, 1000])
def test_many_features_in_one_call(dev, F):
  rng = np.random.default_rng(F)
  feats = []
  for f in range(F):
    d = int(rng.choice([1, 3, 4, 8, 13, 16, 32, 61, 64, 100, 128, 257]))
    cut = sorted(rng.choice(np.arange(1, d), min(d - 1, int(rng.integers(0, 4))), replace=False)) if d > 1 else []
    sd = list(np.diff([0] + list(cut) + [d]).astype(int))
    feats.append((d, [int(x) for x in sd], None, "mean" if f % 3 == 2 else "sum"))
  check_case(dev, 64 if F >= 102 else 300, feats, seed=F)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bf16_slices_and_gradients(dev, dtype):
  feats = [(d, [d], None, p) for d in (1, 5, 16, 32, 64, 128, 129) for p in ("sum", "mean")]
  check_case(dev, 211, feats, seed=5, dtype=dtype)


def test_special_rows_exactly(dev):
  """-0.0-only rows give +0.0; an empty MEAN row is NaN; inf - inf is NaN; 3e38 + 3e38 overflows to inf."""
  sp = torch.tensor([0, 2, 2, 4, 6], dtype=torch.int32, device=dev)
  v = torch.tensor([[-0.0], [-0.0], [np.inf], [-np.inf], [3e38], [3e38]], dtype=torch.float32, device=dev)
  s = dops.fused_reduce_and_split_gpu([sp], [v], [[1]])[0].cpu().reshape(-1)
  m = dops.fused_reduce_and_split_gpu([sp], [v], [[1]], pooling="mean")[0].cpu().reshape(-1)
  assert s.view(torch.int32).tolist()[:2] == [0, 0] and torch.isnan(s[2]) and s[3] == np.inf
  assert m[0].item() == 0 and torch.isnan(m[1]) and torch.isnan(m[2]) and m[3] == np.inf


def test_mean_factor_on_the_device(dev):
  """Rows of ones: the MEAN gradient of each occurrence is the factor (float)(1.0 / (double)(float)n) itself."""
  ns = list(range(1, 300)) + [1000, 4095, 4096, 4097, 65535, 100003, 1 << 20]
  sp = torch.tensor(np.concatenate([[0], np.cumsum(ns)]), dtype=torch.int32, device=dev)
  g = torch.ones(len(ns), 1, device=dev)
  out = dops.fused_reduce_and_split_gpu_grad([sp], [torch.empty(int(sum(ns)), 1, device=dev)], [g], [[1]],
                                             pooling="mean")[0].cpu().numpy().reshape(-1)
  want = np.repeat((1.0 / np.asarray(ns, np.float32).astype(np.float64)).astype(np.float32), ns)
  np.testing.assert_array_equal(out.view(np.uint32), want.view(np.uint32))


def test_slices_land_at_column_offsets_of_one_concat_buffer(dev):
  """Slices written straight into a tower input: every bit outside them keeps its value."""
  rng = np.random.default_rng(9)
  B = 333
  sps, rows = make_case(rng, B, [(13, [5, 8], None, "sum"), (16, [16], None, "mean"), (3, [1, 1, 1], None, "sum")])
  width, cols = 50, [[1, 7], [20], [40, 42, 45]]
  sentinel = np.uint32(0x7FA5A5A5).view(np.float32)
  buf = torch.full((B, width), float(sentinel), device=dev)
  buf.view(torch.int32).fill_(0x7FA5A5A5)
  sdims = [[5, 8], [16], [1, 1, 1]]
  outs = [[buf[:, c:c + d] for c, d in zip(cs, ds)] for cs, ds in zip(cols, sdims)]
  dops._reduce_split_call(False, [torch.from_numpy(s).to(dev) for s in sps], [torch.from_numpy(r).to(dev) for r in rows],
                          outs, ["sum", "mean", "sum"], None)
  want = np.full((B, width), sentinel, np.float32)
  for cs, ds, w in zip(cols, sdims, rsm.reduce_and_split(sps, rows, sdims, ["sum", "mean", "sum"])):
    for c, d, x in zip(cs, ds, w):
      want[:, c:c + d] = x
  got = buf.cpu().numpy()
  covered = np.zeros(width, bool)
  for cs, ds in zip(cols, sdims):
    for c, d in zip(cs, ds):
      covered[c:c + d] = True
  np.testing.assert_array_equal(got[:, ~covered].view(np.uint32), want[:, ~covered].view(np.uint32))
  same_bits(got[:, covered], want[:, covered])


def test_malformed_splits_set_the_flag_and_stay_inside_the_buffers(dev):
  v = torch.arange(12, dtype=torch.float32, device=dev).reshape(6, 2)
  flag = torch.full((1,), 7, dtype=torch.int32, device=dev)
  good = torch.tensor([0, 2, 6], dtype=torch.int32, device=dev)
  dops.fused_reduce_and_split_gpu([good], [v], [[2]], bad_splits=flag)
  assert flag.item() == 0
  for bad in ([1, 2, 6], [0, 4, 2], [0, 2, 5], [0, 2, 1 << 30], [-5, 2, 6], [0, -1, 6]):
    flag.fill_(0)
    sp = torch.tensor(bad, dtype=torch.int32, device=dev)
    out = dops.fused_reduce_and_split_gpu([sp], [v], [[2]], bad_splits=flag)[0]
    g = torch.zeros(6, 2, device=dev)
    dops.fused_reduce_and_split_gpu_grad([sp], [v], [torch.ones(2, 2, device=dev)], [[2]], out=[g], bad_splits=flag)
    torch.cuda.synchronize()
    assert flag.item() == 1, bad
    assert torch.isfinite(out).all()


def test_id_indices_forms(dev):
  idx = torch.tensor([[0], [0], [2]], dtype=torch.int64, device=dev)
  val = torch.tensor([[1, 1, 1], [2, 2, 1], [4, 4, 2]], dtype=torch.float32, device=dev)
  o = dops.fused_reduce_sum_and_split(idx[:, 0], val, 4, [1, 2])
  assert o[0].cpu().tolist() == [[3], [0], [4], [0]] and o[1].cpu().tolist() == [[3, 2], [0, 0], [4, 2], [0, 0]]
  g = dops.fused_reduce_sum_and_split_gradient(idx[:, 0], [torch.ones(4, 1, device=dev), torch.ones(4, 2, device=dev)],
                                               [1, 2])
  assert g.cpu().tolist() == [[1, 1, 1]] * 3
  assert dops.reduce_sum(idx, val[:, :2], [3]).cpu().tolist() == [[3, 3], [0, 0], [4, 4]]
  mean = dops.reduce_mean(torch.tensor([[0], [0], [1]], device=dev), torch.tensor([[4., 4], [2, 2], [1, 1]], device=dev),
                          [2])
  assert mean.cpu().tolist() == [[3, 3], [1, 1]]
  assert dops.reduce_mean_gradient(torch.tensor([[0], [0]], device=dev),
                                   torch.tensor([[-2., -2]], device=dev)).cpu().tolist() == [[-1, -1], [-1, -1]]
  assert dops.reduce_sum_gradient(torch.tensor([[0], [0]], device=dev),
                                  torch.tensor([[-1., -1]], device=dev)).cpu().tolist() == [[-1, -1], [-1, -1]]
  b = dops.reduce_sum(idx, val, [3], dtype=torch.bfloat16)
  assert b.dtype == torch.bfloat16 and b.float().cpu().tolist() == [[3, 3, 2], [0, 0, 0], [4, 4, 2]]
  for bad in ([1, 0], [0, 3], [-1, 0]):
    with pytest.raises(ValueError):
      dops.reduce_sum(torch.tensor(bad, device=dev), torch.ones(2, 2, device=dev), 3)


def test_sync_false_makes_no_host_round_trip(dev):
  idx = torch.arange(4096, device=dev) // 3
  val = torch.ones(4096, 16, device=dev)
  dops.reduce_sum(idx, val, 1366, sync=False)   # warm up
  torch.cuda.synchronize()
  s = torch.cuda.current_stream(dev)
  torch.cuda._sleep(100_000_000)
  out = dops.reduce_sum(idx, val, 1366, sync=False)
  busy = not s.query()
  torch.cuda.synchronize()
  assert busy
  assert (out[:-1] == 3).all() and (out[-1] == 1).all()


def _cfg(dim):
  seg = entry.CombineAsSegment(dim, entry.RandomUniformInitializer(-0.5, 0.5),
                               entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
  return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=4096, init_seed=3), [0.05])


def test_chain_lookup_reduce_grad_apply(dev):
  """lookup -> reduce_and_split -> tower gradients -> grad into the flat buffer -> raw_apply_gradients with dedup:
  the table equals the oracle's.  The SUM forward equals lookup_pool_parts except on rows of -0.0 only."""
  cfg = {"a": _cfg(16), "b": _cfg(32)}
  gpu, cpu = MultiHashTable(cfg, device=dev), orc.OracleMultiHashTable(cfg)
  rng = np.random.default_rng(11)
  B = 512
  vocab = {"a": rng.integers(1, 1 << 40, 300), "b": rng.integers(1, 1 << 40, 200)}
  for n in ("a", "b"):
    g0 = rng.standard_normal((vocab[n].size, cpu.dims[cpu.names.index(n)])).astype(np.float32)
    gpu.apply_gradients({n: (torch.from_numpy(vocab[n]).to(dev), torch.from_numpy(g0).to(dev))}, req_time=1,
                        ids_unique=True)
    cpu.apply_gradients({n: (vocab[n], g0)}, req_time=1)
  # features: two on table a (SUM and MEAN), one on b (SUM, sliced)
  feats = [("a", "sum", [16]), ("a", "mean", [4, 12]), ("b", "sum", [8, 8, 16])]
  fids, sps = [], []
  for t, _, _ in feats:
    lens = rng.integers(0, 6, B)
    sps.append(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32))
    fids.append(rng.choice(np.concatenate([vocab[t], [777, 778]]), int(lens.sum())))
  ids = {"a": np.concatenate([fids[0], fids[1]]), "b": fids[2]}
  emb = gpu.lookup({k: torch.from_numpy(v).to(dev) for k, v in ids.items()})
  na = fids[0].size
  rows = [emb["a"][:na], emb["a"][na:], emb["b"]]
  tsp = [torch.from_numpy(s).to(dev) for s in sps]
  sdims = [f[2] for f in feats]
  pools = [f[1] for f in feats]
  outs = dops.fused_reduce_and_split_gpu(tsp, rows, sdims, pooling=pools)
  # SUM forward against lookup_pool_parts
  for fi, sl in ((0, slice(0, 1)), (2, slice(3, 6))):
    part = gpu.lookup_pool(feats[fi][0], torch.from_numpy(fids[fi]).to(dev), tsp[fi], "sum")
    mine = torch.cat(outs[sl], 1)
    neg0 = (part.view(torch.int32) == np.int32(-2 ** 31)).all(1)
    assert torch.equal(mine[~neg0].view(torch.int32), part[~neg0].view(torch.int32))
  # tower gradients, then the grad call into the flat value buffer raw_apply_gradients takes
  tgrads = [torch.from_numpy(rng.standard_normal((B, d)).astype(np.float32)).to(dev) for sd in sdims for d in sd]
  flat = torch.empty(fids[0].size * 16 + fids[1].size * 16 + fids[2].size * 32, device=dev)
  o0 = flat[:na * 16].view(na, 16)
  o1 = flat[na * 16:(na + fids[1].size) * 16].view(-1, 16)
  o2 = flat[(na + fids[1].size) * 16:].view(-1, 32)
  dops.fused_reduce_and_split_gpu_grad(tsp, rows, tgrads, sdims, pooling=pools, out=[o0, o1, o2])
  all_ids = np.concatenate([ids["a"], ids["b"]])
  split = np.array([0, ids["a"].size, all_ids.size], np.int64)
  gpu.raw_apply_gradients(torch.from_numpy(all_ids).to(dev), split, flat, req_time=2, enable_dedup=True)
  # oracle: the same chain on the host
  cemb = cpu.lookup(ids)
  crows = [cemb["a"][:na], cemb["a"][na:], cemb["b"]]
  couts = rsm.reduce_and_split(sps, crows, sdims, pools)
  for g, w in zip(outs, [w for ws in couts for w in ws]):
    same_bits(g.cpu().numpy(), w)
  it = iter([t.cpu().numpy() for t in tgrads])
  per = [[next(it) for _ in sd] for sd in sdims]
  cg = rsm.reduce_and_split_grad(sps, [r.shape for r in crows], per, pools)
  same_bits(flat.cpu().numpy(), np.concatenate([g.reshape(-1) for g in cg]))
  cpu.raw_apply_gradients(all_ids, split, np.concatenate([g.reshape(-1) for g in cg]), req_time=2, enable_dedup=True)
  for n in ("a", "b"):
    keys = np.unique(ids[n])
    same_bits(gpu.lookup_entry(n, torch.from_numpy(keys).to(dev))["raw"].cpu().numpy(), cpu.lookup_entry(n, keys))


def test_every_new_kernel_instantiation_ran():
  want = {(d, t, g) for d in ("fwd", "bwd") for t in (torch.float32, torch.bfloat16) for g in (4, 8, 16, 32)}
  assert want <= RAN, sorted(map(str, want - RAN))
