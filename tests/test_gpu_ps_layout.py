"""PartitionedHashTable's parameter-server mode on one H100: ShardingSparseFids version 5, NormalizeMergedSplit, the
fp16-input layout forward and PartitionedHashTablePS (fp32 and transfer_float16) against tests/ps_layout_model.py,
bit for bit."""
import numpy as np
import pytest
import torch

from tests import ps_layout_model as pm
from tests.helpers import table
from tests.test_gpu_forward_paths import T
from tests.test_gpu_layout_paths import exact_terms
from tests.test_gpu_sharding_paths import as_numpy, assert_same, make_features, run
from tests.test_sharding_paths_cpu import check_against_fixture, fixture_cases

pytestmark = pytest.mark.gpu

SUM, MEAN, FIRSTN = 0, 1, 2
V5_KEYS = ("fid_list_row_splits_size", "emb_size", "nfl_size", "feature_size", "fid_size", "batch_size")


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def bits(x):
  x = x.detach().cpu()
  return x.view(torch.int16 if x.element_size() == 2 else torch.int32).numpy()


def check_v5(feats, table_of, dims, N, dev, shared=(), batch_size=None):
  for unique in (True, False):
    want = pm.sharding_v5(feats, table_of, dims, N, shared, unique, batch_size)
    for sync in (True, False):
      r = run(feats, table_of, dims, N, dev, shared, unique=unique, sync=sync, version=5, batch_size=batch_size)
      assert_same(as_numpy(r), want)
      rs_size = torch.cat(r["fid_list_row_splits_size"])
      assert all(t.dtype == torch.int32 and t.is_cuda and t.numel() == 1 for t in r["fid_list_row_splits_size"])
      np.testing.assert_array_equal(rs_size.cpu().numpy(), want["fid_list_row_splits_size"])
      for key in V5_KEYS[1:]:
        assert r[key].dtype == torch.int32 and r[key].is_cuda, key
        np.testing.assert_array_equal(r[key].cpu().numpy(), want[key], err_msg=key)
      # the row splits of every list have fid_list_row_splits_size entries
      assert [t.numel() for t in r["fid_list_row_splits"]] == want["fid_list_row_splits_size"].tolist()


# ---- ShardingSparseFids version 5 --------------------------------------------------------------------------------------
def test_v5_on_the_reference_fixtures(dev):
  n = 0
  for z, p, feats, table_of, dims, N, shared, K in fixture_cases():
    for unique in (True, False):
      r = run(feats, table_of, dims, N, dev, shared, unique=unique, version=5, batch_size=7)
      check_against_fixture(z, p, as_numpy(r), unique, N, K)
    check_v5(feats, table_of, dims, N, dev, shared, batch_size=7)
    n += 1
  assert n == 5


@pytest.mark.parametrize("N", [1, 2, 3, 8, 31, 64])
def test_v5_one_to_64_shards(N, dev):
  rng = np.random.default_rng(N)
  feats, table_of, dims = make_features(rng, [300, 0, 17, 1000, 5], 3, vocab=400)
  check_v5(feats, table_of, dims, N, dev, batch_size=11)


def test_v5_shared_and_empty_features(dev):
  rng = np.random.default_rng(5)
  B = 6
  feats = {"a": (np.arange(5, dtype=np.int64), np.array([0, 1, 1, 3, 3, 5, 5], np.int64)),
           "b": (np.zeros(0, np.int64), np.zeros(B + 1, np.int64)),
           "s": (rng.integers(-9, 9, 4).astype(np.int64), np.array([0, 4], np.int64)),
           "t": (np.zeros(0, np.int64), np.array([0], np.int64))}
  table_of, dims = {"a": "x", "b": "y", "s": "x", "t": "y"}, {"a": 4, "b": 2, "s": 4, "t": 2}
  for N in (1, 3, 5):
    check_v5(feats, table_of, dims, N, dev, shared=("s", "t"))


def test_v5_sync_false_does_not_wait(dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(9)
  feats, table_of, dims = make_features(rng, [20000, 3000], 2)
  tf = {n: (T(f, dev), T(r, dev)) for n, (f, r) in feats.items()}
  dops.sharding_sparse_fids(tf, table_of, dims, 4, unique=True, sync=False, version=5, batch_size=5)   # warm
  torch.cuda.synchronize()
  torch.cuda._sleep(200_000_000)                      # keep the stream busy well past the call
  ev = torch.cuda.Event()
  r = dops.sharding_sparse_fids(tf, table_of, dims, 4, unique=True, sync=False, version=5, batch_size=5)
  ev.record()
  assert not ev.query(), "sync=False version 5 waited for the stream"
  torch.cuda.synchronize()
  assert r["fid_list"] is None
  want = pm.sharding_v5(feats, table_of, dims, 4, batch_size=5)
  np.testing.assert_array_equal(r["emb_size"].cpu().numpy(), want["emb_size"])


# ---- NormalizeMergedSplit ----------------------------------------------------------------------------------------------
def test_normalize_merged_split_reference_example_and_random(dev):
  from monolith_b200 import distribution_ops as dops
  rs, sz = [0, 2, 5, 5, 9, 0, 0, 3, 4], [5, 4]
  got = dops.normalize_merged_split(T(np.array(rs, np.int64), dev), T(np.array(sz, np.int32), dev))
  assert got.cpu().tolist() == [0, 2, 5, 5, 9, 9, 12, 13] == pm.normalize_merged_split(rs, sz).tolist()
  rng = np.random.default_rng(3)
  for m in (1, 2, 7, 1023, 1024, 1025, 5000):
    sizes = rng.integers(1, 6, m).astype(np.int32)
    parts = [np.concatenate([[0], np.cumsum(rng.integers(0, 9, s - 1))]) for s in sizes]
    row = np.concatenate(parts).astype(np.int64)
    for sync in (True, False):
      got = dops.normalize_merged_split(T(row, dev), T(sizes, dev), sync=sync)
      np.testing.assert_array_equal(got.cpu().numpy(), pm.normalize_merged_split(row, sizes), err_msg=str(m))


def test_normalize_merged_split_flags_bad_sizes(dev):
  from monolith_b200 import distribution_ops as dops
  rs = T(np.array([0, 2, 5, 0, 3], np.int64), dev)
  for sz in ([2, 2], [3, 0, 2], [5, 1], [-5, 3], [2, -1, 4], [-2, 7]):
    with pytest.raises(ValueError, match="row_split_size"):
      dops.normalize_merged_split(rs, T(np.array(sz, np.int32), dev))
  # a split that ends at or below 0 after a negative size reads nothing outside row_split (no fault, sync=False)
  out = dops.normalize_merged_split(rs, T(np.array([-5, 3], np.int32), dev), sync=False)
  torch.cuda.synchronize()
  assert out.numel() == 4


# ---- the fp16-input layout forward and the fp16 rounding ---------------------------------------------------------------
def _layout_problem(rng, B=64, N=3):
  feats, table_of, dims, tasks, shapes = problem(rng, B)
  sh = pm.sharding_v5(feats, table_of, dims, N, shared=("f_shared",))
  return sh, tasks, shapes


def test_f16in_layout_equals_fp32_layout_on_the_widened_lists(dev):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(11)
  sh, tasks, shapes = _layout_problem(rng)
  B = int(sh["batch_size"][0])
  lists = []
  for k, n_floats in enumerate(sh["emb_size"]):
    x = (rng.standard_normal(int(n_floats)) * rng.choice([1e-6, 1.0, 3e4], int(n_floats))).astype(np.float16)
    x[rng.integers(0, 50, x.size) == 0] = np.float16(np.inf)
    x[rng.integers(0, 50, x.size) == 0] = np.float16(6e-8)
    x[rng.integers(0, 50, x.size) == 0] = np.float16(-0.0)
    lists.append(torch.from_numpy(x).to(dev))
  args = (T(sh["fid_offset"].view(np.int64), dev), T(sh["feature_offset"], dev), T(sh["nfl_offset"].view(np.int32), dev),
          B, tasks, shapes)
  for dtype in (torch.float32, torch.bfloat16):
    got = dops.fused_embedding_to_layout(lists, [1] * len(lists), *args, dtype=dtype)
    want = dops.fused_embedding_to_layout([x.float() for x in lists], [1] * len(lists), *args, dtype=dtype)
    for g, w in zip(got, want):
      assert g.dtype == dtype
      np.testing.assert_array_equal(bits(g), bits(w))


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 65537])
def test_round_to_f16_is_one_nearest_even_rounding(dev, n):
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(n)
  x = (rng.standard_normal(n + 1) * rng.choice([1e-7, 1.0, 7e4], n + 1)).astype(np.float32)
  x[::97] = np.nan
  t = T(x, dev)
  for v in (t[:n], t[1:]):                 # 16-byte aligned and not
    got, want = dops.round_to_f16(v), v.half()
    nan = torch.isnan(v).cpu().numpy()
    np.testing.assert_array_equal(torch.isnan(got).cpu().numpy(), nan)
    np.testing.assert_array_equal(bits(got)[~nan], bits(want)[~nan])


# ---- PartitionedHashTablePS ---------------------------------------------------------------------------------------------
DIMS = {"ta": 3, "tb": 5, "tc": 7}
L = 3


def problem(rng, B, vocab=60):
  """features on three tables; out 0 CONCAT [B, 17] (tb MEAN | tc SUM | tb shared SUM), out 1 ADDN [B, 3] of two ta
  SUM features, out 2 STACK FIRSTN [B, L, 7]."""
  from monolith_b200.distribution_ops import SliceTask
  spec = {"f_add1": ("ta", "sum"), "f_add2": ("ta", "sum"), "f_cat": ("tb", "mean"), "f_cat2": ("tc", "sum"),
          "f_seq": ("tc", "firstn"), "f_shared": ("tb", "shared")}
  feats = {}
  for slot, (name, (t, kind)) in enumerate(sorted(spec.items())):
    n_rows = 1 if kind == "shared" else B
    if kind == "mean":
      lens = rng.choice([1, 2, 4, 8], n_rows)
    elif kind == "firstn":
      lens = rng.integers(0, 2 * L + 1, n_rows)
    else:
      lens = rng.integers(0, 5, n_rows)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = rng.integers(-vocab // 2, vocab, int(rs[-1])).astype(np.int64)
    feats[name] = (ids * 1000 + slot, rs)    # some ids negative: shard (uint64)fid % N
  names = sorted(feats)
  ix = names.index
  tasks = [SliceTask(ix("f_cat"), 0, 5, MEAN, 0, 0, 17, 0, 0), SliceTask(ix("f_cat2"), 0, 7, SUM, 0, 0, 17, 5, 0),
           SliceTask(ix("f_shared"), 0, 5, SUM, 0, 0, 17, 12, 0),
           SliceTask(ix("f_add1"), 0, 3, SUM, 0, 1, 3, 0, 1), SliceTask(ix("f_add2"), 0, 3, SUM, 0, 1, 3, 0, 1),
           SliceTask(ix("f_seq"), 0, 7, FIRSTN, L, 2, L * 7, 0, 0)]
  shapes = [(B, 17), (B, 3), (B, L, 7)]
  table_of = {n: spec[n][0] for n in names}
  dims = {n: DIMS[table_of[n]] for n in names}
  return feats, table_of, dims, tasks, shapes


def _cfgs(opt):
  params = {"sgd": ("sgd", {}), "adagrad": ("adagrad", {"initial_accumulator_value": 0.1})}[opt]
  return {t: table([(d, params[0], params[1])], [0.25]) for t, d in DIMS.items()}


def _pht(S, opt, dev, unique, f16, devices=None):
  from monolith_b200 import MultiHashTable
  from monolith_b200.distributed_ps import PartitionedHashTablePS
  rng = np.random.default_rng(0)
  feats, table_of, dims, tasks, shapes = problem(rng, 4)
  devices = devices or [dev]
  return PartitionedHashTablePS(S, _cfgs(opt), lambda i, c: MultiHashTable(_cfgs(opt), device=devices[i % len(devices)]),
                                table_of, dims, tasks, [s[1:] for s in shapes], ("f_shared",), unique=unique,
                                transfer_float16=f16)


def test_ps_mode_refuses_a_task_wider_than_its_tensor(dev):
  from monolith_b200 import MultiHashTable
  from monolith_b200.distributed_ps import PartitionedHashTablePS
  feats, table_of, dims, tasks, shapes = problem(np.random.default_rng(0), 4)
  narrow = [s[1:] for s in shapes]
  narrow[0] = (16,)
  with pytest.raises(ValueError, match="out_row_stride"):
    PartitionedHashTablePS(2, _cfgs("sgd"), lambda i, c: MultiHashTable(_cfgs("sgd"), device=dev), table_of, dims,
                           tasks, narrow, ("f_shared",))


def _train(S, opt, dev, unique, f16, dtype=torch.float32, devices=None, steps=4):
  pht = _pht(S, opt, dev, unique, f16, devices)
  servers = [pm.DictTable(DIMS, opt, 0.25) for _ in range(S)]
  rng = np.random.default_rng(S * 7 + (opt == "sgd") + 2 * unique + 4 * f16)
  touched = {t: set() for t in DIMS}
  for step in range(steps):
    B = int(rng.integers(1, 90))
    feats, table_of, dims, tasks, shapes = problem(rng, B, vocab=60 + 40 * step)   # fresh FIDs every step
    tf = {n: (T(f, dev), T(r, dev)) for n, (f, r) in feats.items()}
    got, ctx = pht.lookup(tf, dtype=dtype)
    og = [exact_terms(rng, s) for s in shapes]
    want, sh = pm.ps_step(servers, feats, table_of, dims, S, tasks, shapes, layout_grads=None, shared=("f_shared",),
                          unique=unique, transfer_float16=f16)
    for g, w in zip(got, want):
      assert g.dtype == dtype
      np.testing.assert_array_equal(bits(g), bits(torch.from_numpy(w).to(dtype)))
    pm.ps_step(servers, feats, table_of, dims, S, tasks, shapes, layout_grads=og, shared=("f_shared",),
               unique=unique, transfer_float16=f16)
    pht.apply_gradients(ctx, [T(g, dev).to(dtype) for g in og], global_step=step, req_time=10 + step)
    for n, (f, _) in feats.items():
      touched[table_of[n]].update(int(x) for x in f)
  # every touched row, on its server, bit for bit
  for t, ids in touched.items():
    ids = np.array(sorted(ids), np.int64)
    for i, tbl in enumerate(pht.tables):
      mine = ids[(ids.astype(np.uint64) % np.uint64(S)) == i]
      got = tbl.lookup({t: T(mine, tbl.device)})[t].cpu().numpy()
      np.testing.assert_array_equal(got.view(np.int32), servers[i].lookup(t, mine).view(np.int32), err_msg=(t, i))
  return pht


@pytest.mark.parametrize("S", [1, 2, 3, 5])
@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
@pytest.mark.parametrize("unique", [True, False])
def test_ps_mode_trains_like_the_model(dev, S, opt, unique):
  _train(S, opt, dev, unique, False)


@pytest.mark.parametrize("S", [1, 2, 3, 5])
@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
def test_ps_mode_transfer_float16_trains_like_the_model(dev, S, opt):
  _train(S, opt, dev, True, True)
  _train(S, opt, dev, False, True, steps=2)


@pytest.mark.parametrize("f16", [False, True])
def test_ps_mode_bf16_layout(dev, f16):
  _train(3, "sgd", dev, True, f16, dtype=torch.bfloat16)


def test_ps_mode_servers_on_two_devices():
  if torch.cuda.device_count() < 2:
    pytest.skip("one CUDA device")
  devs = [torch.device("cuda", 0), torch.device("cuda", 1)]
  _train(3, "adagrad", devs[0], True, True, devices=devs)


def test_ps_forward_equals_the_layout_over_one_global_table(dev):
  """the union of the servers' rows in one table, looked up list by list, through fused_embedding_to_layout"""
  from monolith_b200 import MultiHashTable
  from monolith_b200 import distribution_ops as dops
  S = 3
  pht = _train(S, "sgd", dev, True, False, steps=2)
  glob = MultiHashTable(_cfgs("sgd"), device=dev)
  rng = np.random.default_rng(21)
  feats, table_of, dims, tasks, shapes = problem(rng, 40, vocab=100)
  for t in DIMS:
    ids = np.unique(np.concatenate([f for n, (f, _) in feats.items() if table_of[n] == t]))
    for i, tbl in enumerate(pht.tables):
      mine = ids[(ids.astype(np.uint64) % np.uint64(S)) == i]
      if mine.size:
        rows = tbl.lookup({t: T(mine, dev)})[t]
        glob.assign({t: (T(mine, dev), rows)})
  tf = {n: (T(f, dev), T(r, dev)) for n, (f, r) in feats.items()}
  got, _ = pht.lookup(tf)
  sh = dops.sharding_sparse_fids(tf, table_of, dims, S, ("f_shared",))
  tables = sh["table_names"]
  embs = [glob.lookup({tables[k]: sh["fid_list"][k * S + n]})[tables[k]].reshape(-1) for k in range(len(tables))
          for n in range(S)]
  want = dops.fused_embedding_to_layout(embs, [1] * len(embs), sh["fid_offset"], sh["feature_offset"], sh["nfl_offset"],
                                        40, tasks, shapes)
  for g, w in zip(got, want):
    np.testing.assert_array_equal(bits(g), bits(w))
