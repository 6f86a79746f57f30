"""mono_sharding_sparse_fids (dedup.cu: ShardingSparseFids on the device) through distribution_ops.sharding_sparse_fids:
versions 3 and 4, unique and non-unique, bit for bit against the reference's Python model fixture, the numpy
restatement (tests/sharding_model.py) and the adapter over the oracle's reorder; at the reorder's tile edges and at
6.5 M FIDs; 1 to 1000 features with empty ones anywhere; 1 to 64 shards; special FIDs; the 32-bit offset limit; the
launches of every call; no host round trip with sync=False; and the fused lookup -> layout -> grad -> fused apply
chain over the version-4 list."""
import numpy as np
import pytest
import torch

from tests import orc
from tests import sharding_model as sm
from tests.helpers import table
from tests.test_gpu_forward_paths import T, assert_bits
from tests.test_gpu_layout_paths import CHAIN_FEATS, CHAIN_TABLES, _chain_features, _chain_tasks, exact_terms
from tests.test_sharding_paths_cpu import check_against_fixture, fixture_cases

pytestmark = pytest.mark.gpu

TILE = 2048
I32_MAX = 2 ** 31 - 1
I64 = np.iinfo(np.int64)


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def run(feats, table_of, dims, N, dev, shared=(), **kw):
  from monolith_b200 import distribution_ops as dops
  return dops.sharding_sparse_fids({n: (T(f, dev), T(r, dev)) for n, (f, r) in feats.items()}, table_of, dims, N,
                                   list(shared), **kw)


def as_numpy(r):
  """the device op's dict in sharding_model's form"""
  N = r["fid_list_shard_row_length"].numel()
  total = int(r["fid_list_shard_row_length"].sum())
  rs = r["fid_list_row_splits"]
  out = {"fid_offset": r["fid_offset"].cpu().numpy().view(np.uint64),
         "feature_offset": r["feature_offset"].cpu().numpy(),
         "nfl_offset": r["nfl_offset"].cpu().numpy().view(np.uint32),
         "fid_list_row_splits": [x.cpu().numpy() for x in rs],
         "fid_list_fused": r["fid_list_fused"][:total].cpu().numpy()}
  K = len(rs) // N
  out["fid_list_row_splits_fused"] = np.concatenate([out["fid_list_row_splits"][k * N + n] for n in range(N)
                                                     for k in range(K)])
  for key in ("table_row_length", "shard_row_length", "emb_row_length"):
    out["fid_list_" + key] = r["fid_list_" + key].cpu().numpy()
  if r["fid_list"] is not None:
    out["fid_list"] = [x.cpu().numpy() for x in r["fid_list"]]
  else:                              # the version-3 lists as slices of the version-4 list
    lens, starts = out["fid_list_table_row_length"], np.concatenate([[0], np.cumsum(out["fid_list_table_row_length"])])
    out["fid_list"] = [out["fid_list_fused"][starts[n * K + k]:starts[n * K + k] + lens[n * K + k]] for k in range(K)
                       for n in range(N)]
  return out


def assert_same(got, want):
  for key in ("fid_offset", "feature_offset", "nfl_offset", "fid_list_fused", "fid_list_row_splits_fused",
              "fid_list_table_row_length", "fid_list_shard_row_length", "fid_list_emb_row_length"):
    np.testing.assert_array_equal(got[key], want[key], err_msg=key)
    assert got[key].dtype == want[key].dtype or key == "fid_list_fused", key
  for key in ("fid_list", "fid_list_row_splits"):
    assert len(got[key]) == len(want[key]), key
    for i, (g, w) in enumerate(zip(got[key], want[key])):
      np.testing.assert_array_equal(g, w, err_msg=f"{key}[{i}]")


def launches(fn):
  from monolith_b200 import _lib
  lib = _lib.load()
  n0 = lib.mono_kernel_launch_count()
  r = fn()
  return r, lib.mono_kernel_launch_count() - n0


def check(feats, table_of, dims, N, dev, shared=(), twin=True):
  """every mode against the numpy model (and unique against the adapter over the oracle's reorder), launches pinned"""
  M = sum(f.size for f, _ in feats.values())
  for unique in (True, False):
    want = sm.sharding(feats, table_of, dims, N, shared, unique)
    for sync in (True, False):
      r, n = launches(lambda: run(feats, table_of, dims, N, dev, shared, unique=unique, sync=sync))
      assert n == ((9 if unique else 8) if M else 2), (unique, sync, n)
      assert (r["fid_list"] is None) == (not sync)
      assert r["fid_offset"].dtype == torch.int64 and r["nfl_offset"].dtype == torch.int32
      assert r["feature_offset"].dtype == torch.int32 and r["fid_list_fused"].dtype == torch.int64
      assert r["fid_offset"].is_cuda and r["fid_list_fused"].is_cuda
      assert_same(as_numpy(r), want)
  if twin:
    def reorder_fn(lists, n, d):
      out, ss, sl, _, offs = orc.reorder_by_indices([l.numpy() for l in lists], n, d)
      return torch.from_numpy(out), ss.tolist(), sl.tolist(), None, torch.from_numpy(offs)
    from monolith_b200 import distribution_ops as dops
    w = dops.sharding_sparse_fids({n: (torch.from_numpy(f), torch.from_numpy(r)) for n, (f, r) in feats.items()},
                                  table_of, dims, N, list(shared), reorder_fn=reorder_fn)
    g = run(feats, table_of, dims, N, dev, shared)
    for key in ("fid_offset", "feature_offset", "nfl_offset"):
      np.testing.assert_array_equal(g[key].cpu().numpy(), w[key].numpy(), err_msg=key)
    for i, (a, b) in enumerate(zip(g["fid_list"], w["fid_list"])):
      np.testing.assert_array_equal(a.cpu().numpy(), b.numpy(), err_msg=f"fid_list[{i}]")


def make_features(rng, sizes, n_tables, vocab=50, rows_per=None, specials=False):
  """features named so that sorted-name order differs from table-major order; sizes[i] FIDs for feature i"""
  feats, table_of, dims = {}, {}, {}
  for i, m in enumerate(sizes):
    name = f"f{(i * 7919) % 100003:06d}_{i}"
    if rows_per is None:
      rows = max(1, m // 3) if m else int(rng.integers(0, 3))
    else:
      rows = rows_per
    cuts = np.sort(rng.integers(0, m + 1, max(rows - 1, 0))) if rows else np.zeros(0, np.int64)
    rs = np.concatenate([[0], cuts, [m]]) if rows else np.zeros(1, np.int64)
    keys = rng.integers(I64.min, I64.max, vocab, dtype=np.int64) if specials else \
        (np.int64(i + 1) << 48) | rng.integers(0, 1 << 40, vocab)
    fids = keys[rng.integers(0, vocab, m)]
    feats[name] = (fids.astype(np.int64), rs.astype(np.int64))
    table_of[name] = f"t{(i * 5) % n_tables:03d}"
    dims[name] = int(rng.integers(1, 40))
  return feats, table_of, dims


# ------------------------------------------------------------------------------------------------
def test_equals_the_reference_model_fixture_in_every_case_and_mode(dev):
  n = 0
  for z, p, feats, table_of, dims, N, shared, K in fixture_cases():
    for unique in (True, False):
      for sync in (True, False):
        r = run(feats, table_of, dims, N, dev, shared, unique=unique, sync=sync)
        check_against_fixture(z, p, as_numpy(r), unique, N, K)
        n += 1
  assert n == 20


@pytest.mark.parametrize("M", [0, 1, TILE - 1, TILE, TILE + 1])
def test_at_the_tile_edges(M, dev):
  rng = np.random.default_rng(M)
  feats, table_of, dims = make_features(rng, [M // 3, 0, M - M // 3], 2, vocab=max(M // 4, 1))
  check(feats, table_of, dims, 5, dev, shared=[sorted(feats)[1]])
  one = {"f": (rng.integers(0, 100, M).astype(np.int64), np.array([0, M], np.int64))}
  check(one, {"f": "t"}, {"f": 8}, 3, dev)


def test_six_and_a_half_million_fids(dev):
  rng = np.random.default_rng(65)
  sizes = rng.multinomial(6_500_000, np.ones(26) / 26)
  sizes[[0, 13, 25]] = 0
  sizes[1] += 6_500_000 - sizes.sum()
  feats, table_of, dims = make_features(rng, sizes.tolist(), 9, vocab=200_000)
  dims = {n: 1 + d % 8 for n, d in dims.items()}
  check(feats, table_of, dims, 64, dev, shared=[sorted(feats)[3]])


@pytest.mark.parametrize("F", [1, 26, 200, 1000])
def test_many_features_with_empty_ones_first_middle_and_last(F, dev):
  rng = np.random.default_rng(F)
  sizes = rng.integers(0, 60, F)
  sizes[[0, F // 2, F - 1]] = 0
  feats, table_of, dims = make_features(rng, sizes.tolist(), max(F // 7, 1), vocab=30)
  names = sorted(feats)
  empty = {names[0]: (np.zeros(0, np.int64), np.zeros(1, np.int64))}   # no rows at all
  feats.update(empty)
  check(feats, table_of, dims, 4, dev, shared=names[1:F:9], twin=F <= 200)


@pytest.mark.parametrize("N", [1, 2, 3, 7, 8, 31, 63, 64])
def test_one_to_64_shards(N, dev):
  rng = np.random.default_rng(N)
  feats, table_of, dims = make_features(rng, [300, 0, 1000, 77, 5], 3, vocab=400)
  check(feats, table_of, dims, N, dev, shared=[sorted(feats)[4]])


def test_negative_and_extreme_fids_use_the_unsigned_shard(dev):
  rng = np.random.default_rng(3)
  feats, table_of, dims = make_features(rng, [5000, 3000, 1], 2, vocab=700, specials=True)
  name = sorted(feats)[0]
  f, rs = feats[name]
  f[:8] = [-1, I64.min, I64.max, 0, -1, I64.min, I64.max, -2]
  for N in (3, 5, 64):
    check(feats, table_of, dims, N, dev)


def test_a_hot_fid_in_every_row(dev):
  rng = np.random.default_rng(4)
  B = 20000
  rs = np.arange(B + 1, dtype=np.int64) * 3
  fids = np.full(3 * B, 12345, np.int64)
  fids[1::3] = rng.integers(0, 1 << 40, B)
  check({"hot": (fids, rs), "other": (rng.integers(0, 9, 100), np.array([0, 40, 100]))}, {"hot": "t", "other": "t"},
        {"hot": 16, "other": 4}, 7, dev)


def test_the_32_bit_offset_limit(dev):
  """sum n_fids x dims_sum = 2^31 - 1 is served (the last FID's row starts at 2^31 - 1 - dims_sum); 2^31 is refused
  before anything launches"""
  from monolith_b200 import _lib
  ok = {"a": (np.array([7], np.int64), np.array([0, 1], np.int64)),
        "b": (np.array([9, 10], np.int64), np.array([0, 2], np.int64))}
  dims = {"a": 1, "b": 2 ** 30 - 1}
  for unique in (True, False):
    r = run(ok, {"a": "t", "b": "t"}, dims, 1, dev, unique=unique)
    assert r["fid_list_emb_row_length"].tolist() == [I32_MAX]
    assert (r["fid_offset"].cpu().numpy() & 0xFFFFFFFF).tolist() == [0, 1, 1 + 2 ** 30 - 1]
  lib = _lib.load()
  n0 = lib.mono_kernel_launch_count()
  with pytest.raises(_lib.MonoError, match="InvalidArgument"):
    run(ok, {"a": "t", "b": "t"}, {"a": 2, "b": 2 ** 30 - 1}, 1, dev)
  assert lib.mono_kernel_launch_count() == n0


def test_malformed_row_splits_are_reported(dev):
  from monolith_b200 import _lib
  f = np.arange(6, dtype=np.int64)
  for rs in ([1, 6], [0, 4, 3, 6], [0, 2, 5], [0, 7]):
    with pytest.raises(_lib.MonoError, match="row splits"):
      run({"a": (f, np.array(rs, np.int64))}, {"a": "t"}, {"a": 4}, 2, dev)
  with pytest.raises(_lib.MonoError, match="row splits"):
    run({"a": (f, np.array([0, 6], np.int64)), "b": (f[:2], np.zeros(1, np.int64))}, {"a": "t", "b": "t"},
        {"a": 4, "b": 4}, 2, dev)


def test_sync_false_makes_no_host_round_trip(dev):
  rng = np.random.default_rng(9)
  feats, table_of, dims = make_features(rng, [20000, 3000, 0, 9000], 2, vocab=5000)
  args = {n: (T(f, dev), T(r, dev)) for n, (f, r) in feats.items()}
  from monolith_b200 import distribution_ops as dops
  want = dops.sharding_sparse_fids(args, table_of, dims, 8)   # warm: the library is loaded, the pool has grown
  stream = torch.cuda.current_stream(dev)
  torch.cuda.synchronize()
  torch.cuda._sleep(100_000_000)                               # ~50 ms of device time queued ahead of the call
  r = dops.sharding_sparse_fids(args, table_of, dims, 8, sync=False)
  busy = not stream.query()
  torch.cuda.synchronize()
  assert busy, "the call waited for the stream"
  total = int(r["fid_list_shard_row_length"].sum())
  assert torch.equal(r["fid_list_fused"][:total], want["fid_list_fused"])
  assert torch.equal(r["fid_offset"], want["fid_offset"])


# ------------------------------------------------------------------------------------------------
# the chain: device sharding -> ONE fused lookup of the version-4 list -> layout -> grad -> ONE fused apply,
# against today's per-list chain
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2, 5])
def test_chain_fused_lookup_layout_grad_fused_apply(N, dev):
  from monolith_b200 import MultiHashTable
  from monolith_b200 import distribution_ops as dops
  rng = np.random.default_rng(200 + N)
  B = 37
  names_t = sorted(CHAIN_TABLES)
  cfg = lambda: {t: table([(d, "adagrad", {})], [0.25], capacity=4096) for t, d in CHAIN_TABLES.items()}
  fused_t, per_list_t = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
  assert list(fused_t.table_names) == names_t
  feats = _chain_features(rng, B)
  for t, d in CHAIN_TABLES.items():
    ids = np.unique(np.concatenate([f for n, (f, _) in feats.items() if CHAIN_FEATS[n][0] == t]))
    vals = rng.standard_normal((ids.size, d)).astype(np.float32)
    for tb in (fused_t, per_list_t):
      tb.assign({t: (T(ids, dev), T(vals, dev))}, req_time=10, ids_unique=True)
  feature_table = {n: v[0] for n, v in CHAIN_FEATS.items()}
  dims_sum = {n: CHAIN_TABLES[v[0]] for n, v in CHAIN_FEATS.items()}
  shared = [n for n, v in CHAIN_FEATS.items() if v[2]]
  r = run(feats, feature_table, dims_sum, N, dev, shared)
  tables, names = r["table_names"], r["feature_names"]
  K = len(tables)
  assert tables == names_t
  # today's path: one lookup per (table, shard) list
  embs_a = []
  for k, t in enumerate(tables):
    for n in range(N):
      ids = r["fid_list"][k * N + n]
      embs_a.append(per_list_t.lookup({t: ids})[t].reshape(-1) if ids.numel() else torch.zeros(1, device=dev))
  # the version-4 path: one fused lookup with the table row lengths as the slot sizes
  slot = r["fid_list_table_row_length"].tolist()
  out, _, id_off, emb_off, ids = fused_t.fused_lookup(r["fid_list_fused"], slot, N)
  embs_b = [out[emb_off[n * K + k]:emb_off[n * K + k + 1]] if slot[n * K + k] else torch.zeros(1, device=dev)
            for k in range(K) for n in range(N)]
  tasks, shapes, _ = _chain_tasks(names, B)
  lay = lambda embs: dops.fused_embedding_to_layout(embs, [1] * len(embs), r["fid_offset"], r["feature_offset"],
                                                    r["nfl_offset"], B, tasks, shapes)
  for a, b in zip(lay(embs_a), lay(embs_b)):
    assert_bits(b.cpu().numpy(), a.cpu().numpy())
  og = [T(exact_terms(rng, s), dev) for s in shapes]
  grads = dops.fused_embedding_to_layout_grad([e.numel() for e in embs_a], [1] * len(embs_a), r["fid_offset"],
                                              r["feature_offset"], r["nfl_offset"], B, tasks, og)
  lists = r["fid_list"]
  for k, t in enumerate(tables):
    d = CHAIN_TABLES[t]
    ids_k = torch.cat(list(lists[k * N:(k + 1) * N]))
    g_k = torch.cat([grads[k * N + n][:lists[k * N + n].numel() * d] for n in range(N)]).reshape(-1, d)
    per_list_t.apply_gradients({t: (ids_k, g_k)}, req_time=20, ids_unique=True)
  g_fused = torch.cat([grads[k * N + n][:slot[n * K + k] * CHAIN_TABLES[tables[k]]] for n in range(N)
                       for k in range(K)])
  fused_t.fused_apply_gradient(r["fid_list_fused"], ids, slot, g_fused, id_off, emb_off, global_step=1, req_time=20,
                               num_of_shards=N)
  for t in tables:
    keys = torch.unique(torch.cat([T(f, dev) for n, (f, _) in feats.items() if CHAIN_FEATS[n][0] == t]))
    assert_bits(fused_t.lookup_entry(t, keys)["raw"].cpu().numpy(), per_list_t.lookup_entry(t, keys)["raw"].cpu().numpy())
