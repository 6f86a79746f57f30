"""ShardingSparseFids versions 3 and 4, unique and non-unique, without a GPU: the numpy restatement
(tests/sharding_model.py) pinned bit for bit on the reference's own Python model (tests/golden/ref_sharding_v4.npz),
and mono_sharding_sparse_fids' argument checks, which reject before any device is touched."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import sharding_model as sm

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
I32_MAX = 2 ** 31 - 1


def fixture_cases():
  z = np.load(os.path.join(G, "ref_sharding_v4.npz"))
  for ci in range(int(z["n_cases"])):
    p = f"c{ci}_"
    names = [str(n) for n in z[p + "names"]]
    feats = {n: (z[p + "fids_" + n], z[p + "splits_" + n]) for n in names}
    table_of = {n: str(t) for n, t in zip(names, z[p + "tables"])}
    dims = {n: int(d) for n, d in zip(names, z[p + "dims_sum"])}
    shared = [n for n, s in zip(names, z[p + "shared"]) if s]
    yield z, p, feats, table_of, dims, int(z[p + "N"]), shared, int(z[p + "n_tables"])


def check_against_fixture(z, p, got, unique, N, K):
  """got: a dict of numpy arrays as sharding_model.sharding returns it"""
  q = p + ("unique_" if unique else "all_")
  assert got["nfl_offset"].view(np.uint32).tolist() == z[p + "nfl_offset"].tolist()
  assert got["feature_offset"].tolist() == z[p + "feature_offset"].tolist()
  assert got["fid_offset"].view(np.uint64).tolist() == z[q + "fid_offset"].tolist()
  for k in range(K):
    for n in range(N):
      assert got["fid_list"][k * N + n].tolist() == z[q + f"list_{k}_{n}"].tolist(), (q, k, n)
      assert got["fid_list_row_splits"][k * N + n].tolist() == z[q + f"row_splits_{k}_{n}"].tolist(), (q, k, n)
  assert got["fid_list_fused"].tolist() == z[q + "fused"].tolist()
  assert got["fid_list_row_splits_fused"].tolist() == z[q + "fused_row_splits"].tolist()
  for key in ("table_row_length", "shard_row_length", "emb_row_length"):
    assert got["fid_list_" + key].tolist() == z[q + key].tolist(), (q, key)


@pytest.mark.parametrize("unique", [True, False])
def test_numpy_model_equals_the_reference_model_fixture(unique):
  n_cases = 0
  for z, p, feats, table_of, dims, N, shared, K in fixture_cases():
    check_against_fixture(z, p, sm.sharding(feats, table_of, dims, N, shared, unique), unique, N, K)
    n_cases += 1
  assert n_cases == 5


def test_fixture_covers_its_cases():
  """shared features, features without rows or FIDs, a table with one feature, N = 1, 3 and 8"""
  Ns, shared, no_rows, no_fids, one = set(), 0, 0, 0, False
  for z, p, feats, table_of, dims, N, sh, K in fixture_cases():
    Ns.add(N)
    shared += len(sh)
    no_rows += sum(rs.size == 1 for _, rs in feats.values())
    no_fids += sum(f.size == 0 and rs.size > 1 for f, rs in feats.values())
    one |= min(list(table_of.values()).count(t) for t in set(table_of.values())) == 1
    assert (z[p + "unique_fused"].size < z[p + "all_fused"].size) or not any(f.size for f, _ in feats.values())
  assert Ns == {1, 3, 8} and shared >= 3 and no_rows >= 2 and no_fids >= 2 and one


def test_unique_model_equals_the_adapter_over_the_oracle_reorder():
  """The version-3 unique outputs of the numpy model == sharding_sparse_fids over the oracle's reorder, on negative
  FIDs and many shards."""
  from monolith_b200 import distribution_ops as dops
  from tests import orc
  rng = np.random.default_rng(8)
  feats = {}
  for i, n in enumerate(["b", "a", "d", "c", "e"]):
    lens = rng.integers(0, 6, 0 if n == "e" else 30)
    fids = rng.integers(-2 ** 63, 2 ** 63 - 1, 40)[rng.integers(0, 40, int(lens.sum()))]
    feats[n] = (fids, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
  table_of = {"a": "t1", "b": "t0", "c": "t1", "d": "t0", "e": "t2"}
  dims = {"a": 3, "b": 5, "c": 2, "d": 7, "e": 1}

  def reorder_fn(lists, n, d):
    out, ss, sl, _, offs = orc.reorder_by_indices([l.numpy() for l in lists], n, d)
    return torch.from_numpy(out), ss.tolist(), sl.tolist(), None, torch.from_numpy(offs)
  for N in (1, 3, 7):
    want = dops.sharding_sparse_fids({n: (torch.from_numpy(f), torch.from_numpy(r)) for n, (f, r) in feats.items()},
                                     table_of, dims, N, ["c"], reorder_fn=reorder_fn)
    got = sm.sharding(feats, table_of, dims, N, ["c"])
    assert got["fid_offset"].tolist() == want["fid_offset"].numpy().view(np.uint64).tolist()
    assert got["feature_offset"].tolist() == want["feature_offset"].numpy().tolist()
    assert got["nfl_offset"].tolist() == want["nfl_offset"].numpy().view(np.uint32).tolist()
    assert [x.tolist() for x in got["fid_list"]] == [x.numpy().tolist() for x in want["fid_list"]]


def test_reorder_fn_path_keeps_unique_and_synchronous_outputs_only():
  from monolith_b200 import distribution_ops as dops
  feats = {"a": (torch.tensor([1, 2, 1]), torch.tensor([0, 3]))}
  for kw in ({"unique": False}, {"sync": False}):
    with pytest.raises(ValueError):
      dops.sharding_sparse_fids(feats, {"a": "t"}, {"a": 4}, 2, reorder_fn=lambda *a: None, **kw)


def test_sharding_feature_struct_matches_the_header():
  from monolith_b200 import _lib
  assert C.sizeof(_lib.ShardingFeature) == 32
  assert [f for f, _ in _lib.ShardingFeature._fields_] == ["n_fids", "n_rows", "table", "dims_sum", "shared"]


# ------------------------------------------------------------------------------------------------
# argument checks: MONO_ERR_INVALID_ARGUMENT before the device is touched
# ------------------------------------------------------------------------------------------------
def call(recs, K, N, unique=1, null_out=False):
  from monolith_b200 import _lib
  lib = _lib.load()
  arr = (_lib.ShardingFeature * max(len(recs), 1))()
  for i, (n_fids, n_rows, table, dims, shared) in enumerate(recs):
    arr[i].n_fids, arr[i].n_rows, arr[i].table, arr[i].dims_sum, arr[i].shared = n_fids, n_rows, table, dims, shared
  fake = C.c_void_p(0x1000)   # never dereferenced: every check runs on the host first
  outs = [None if null_out else fake] + [fake] * 7
  return lib.mono_sharding_sparse_fids(0, fake, fake, arr, len(recs), K, N, unique, *outs, None, None, None)


@pytest.mark.parametrize("case", [
    dict(recs=[], K=1, N=1),                                            # no features
    dict(recs=[(1, 1, 0, 4, 0)], K=0, N=1),                             # no tables
    dict(recs=[(1, 1, 0, 4, 0)], K=1, N=0),                             # no shards
    dict(recs=[(1, 1, 0, 4, 0)], K=1, N=65),                            # more than 64 shards
    dict(recs=[(1, 1, 1, 4, 0)], K=1, N=2),                             # table index past the last table
    dict(recs=[(1, 1, -1, 4, 0)], K=1, N=2),                            # negative table index
    dict(recs=[(1, 1, 0, 0, 0)], K=1, N=2),                             # dims_sum 0
    dict(recs=[(1, 1, 0, -3, 0)], K=1, N=2),                            # negative dims_sum
    dict(recs=[(-1, 1, 0, 4, 0)], K=1, N=2),                            # negative n_fids
    dict(recs=[(1, -1, 0, 4, 0)], K=1, N=2),                            # negative n_rows
    dict(recs=[(2 ** 29, 1, 0, 1, 0), (2 ** 29 + 1, 1, 0, 1, 0)], K=1, N=2),   # more than 2^30 FIDs
    dict(recs=[(1, 2 ** 31 - 1, 0, 1, 0)], K=1, N=2),                   # 2^31 - 1 rows
    dict(recs=[(1, 1, 0, 2 ** 30, 0), (1, 1, 0, 2 ** 30, 0)], K=1, N=2),       # sum n_fids x dims_sum = 2^31
    dict(recs=[(3, 1, 0, 715827883, 0)], K=1, N=2, unique=0),           # 2^31 + 1, non-unique
    dict(recs=[(1, 1, 0, 4, 0)], K=1, N=2, null_out=True),              # a required output missing
], ids=lambda c: str(c))
def test_arguments_are_rejected_on_the_host(case):
  assert call(**case) == -1   # MONO_ERR_INVALID_ARGUMENT


def test_the_largest_sum_of_sizes_times_dims_passes_the_host_checks():
  """2^31 - 1 floats (a prime: one FID of dims_sum 2^31 - 1, or 1 + (2^31 - 2)) passes every check and goes on to the
  device, which a machine without a GPU reports as a CUDA error (not an argument error)."""
  if torch.cuda.is_available():
    pytest.skip("GPU present: tests/test_gpu_sharding_paths.py runs this call for real")
  assert call([(1, 1, 0, I32_MAX, 0)], 1, 2) == -3
  assert call([(1, 1, 0, 1, 0), (2, 1, 0, 2 ** 30 - 1, 0)], 1, 2) == -3
