"""What tests/test_gpu_ps_layout.py assumes, checked without a GPU: the PS-mode model (tests/ps_layout_model.py) on the
reference's fixtures and example, its dict tables against the oracle, the new C ABI's declarations and bindings, and
the wrappers' argument checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from monolith_b200 import _lib
from monolith_b200 import distribution_ops as dops
from tests import orc
from tests import ps_layout_model as pm
from tests.helpers import table
from tests.test_sharding_paths_cpu import check_against_fixture, fixture_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("mono_sharding_sparse_fids_v5", "mono_normalize_merged_split", "mono_round_to_f16",
       "mono_embedding_to_layout_f16in", "mono_embedding_to_layout_f16in_bf16")


@pytest.fixture(scope="module")
def lib():
  if not os.path.exists(_lib.LIB_PATH):
    import __graft_entry__
    __graft_entry__.build()
  return _lib.load()


def test_v5_model_is_v3_plus_sizes_on_the_reference_fixtures():
  n = 0
  for z, p, feats, table_of, dims, N, shared, K in fixture_cases():
    for unique in (True, False):
      got = pm.sharding_v5(feats, table_of, dims, N, shared, unique, batch_size=7)
      check_against_fixture(z, p, got, unique, N, K)
      q = p + ("unique_" if unique else "all_")
      np.testing.assert_array_equal(got["emb_size"], z[q + "emb_row_length"].reshape(N, K).T.reshape(-1))
      assert got["fid_list_row_splits_size"].tolist() == [z[q + f"row_splits_{k}_{n}"].size for k in range(K)
                                                           for n in range(N)]
      assert got["nfl_size"].tolist() == [z[p + "nfl_offset"].size]
      assert got["feature_size"].tolist() == [z[p + "feature_offset"].size]
      assert got["fid_size"].tolist() == [z[q + "fid_offset"].size]
      assert got["batch_size"].tolist() == [7]
    n += 1
  assert n == 5


def test_normalize_model_on_the_reference_example():
  assert pm.normalize_merged_split([0, 2, 5, 5, 9, 0, 0, 3, 4], [5, 4]).tolist() == [0, 2, 5, 5, 9, 9, 12, 13]
  assert pm.normalize_merged_split([0, 3], [2]).tolist() == [0, 3]
  assert pm.normalize_merged_split([0, 1, 0, 2, 0, 4], [2, 2, 2]).tolist() == [0, 1, 3, 7]


@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
def test_dict_tables_equal_the_oracle_tables(opt):
  """the model's per-server apply, duplicates in order, bit for bit against the oracle (dims below 8)"""
  params = {"sgd": ("sgd", {}), "adagrad": ("adagrad", {"initial_accumulator_value": 0.1})}[opt]
  cfg = {"a": table([(3, params[0], params[1])], [0.25]), "b": table([(7, params[0], params[1])], [0.25])}
  oracle, model = orc.OracleMultiHashTable(cfg), pm.DictTable({"a": 3, "b": 7}, opt, 0.25)
  rng = np.random.default_rng(4)
  for step in range(3):
    upd = {}
    for t, d in (("a", 3), ("b", 7)):
      ids = rng.integers(-20, 20, 60).astype(np.int64)
      g = (rng.standard_normal((60, d)) * rng.choice([1e-3, 1.0, 1e3], (60, 1))).astype(np.float32)
      upd[t] = (ids, g)
      model.apply(t, ids, g)
    oracle.apply_gradients(upd, global_step=step, req_time=1 + step)
    for t in ("a", "b"):
      ids = np.arange(-20, 20, dtype=np.int64)
      np.testing.assert_array_equal(oracle.lookup({t: ids})[t].reshape(ids.size, -1).view(np.int32),
                                    model.lookup(t, ids).view(np.int32))


def test_f16_round_trip_is_one_nearest_even_rounding():
  x = np.array([1.0, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 65520.0, 1e-8, -0.0], np.float32)
  assert pm.f16_round_trip(x).tolist() == [1.0, 1.0, 1 + 2 * 2.0 ** -10, np.inf, 0.0, -0.0]


def test_new_calls_are_declared_and_bound(lib):
  with open(os.path.join(ROOT, "include", "mono_emb.h")) as f:
    header = f.read()
  for name in NEW:
    assert re.search(r"\bint " + name + r"\(", header), name
    assert name in _lib.SIGNATURES and getattr(lib, name).argtypes is not None, name
  assert lib.mono_abi_version() == 1
  # each layout entry point takes its twin's arguments
  assert _lib.SIGNATURES["mono_embedding_to_layout_f16in"] == _lib.SIGNATURES["mono_embedding_to_layout"]
  assert _lib.SIGNATURES["mono_embedding_to_layout_f16in_bf16"] == _lib.SIGNATURES["mono_embedding_to_layout_bf16"]
  twin = _lib.SIGNATURES["mono_sharding_sparse_fids"][1]
  assert _lib.SIGNATURES["mono_sharding_sparse_fids_v5"][1][:len(twin) - 1] == twin[:-1]


def test_layout_f16in_kernels_are_in_the_library(lib):
  import subprocess
  syms = subprocess.run(["nm", "-C", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
  for k in ("f16in_layout_fwd_kernel", "f16in_bf16_layout_fwd_kernel"):
    assert {int(g) for g in re.findall(r"\bmono::" + k + r"<(\d+)>\(", syms)} == {4, 8, 16, 32}, k


def test_normalize_kernel_reads_stay_inside_row_split_for_any_sizes():
  """dedup.cu normalize_merged_split_kernel's index arithmetic restated: a group reads rs[start .. end - 1] only when
  sz >= 1, start >= 0 and end <= split_num, so negative, zero and oversized sizes never index outside [0, split_num)"""
  with open(os.path.join(ROOT, "monolith_b200", "csrc", "dedup.cu")) as f:
    assert "const bool ok = live && sz >= 1 && start >= 0 && end <= split_num;" in f.read()
  rng = np.random.default_rng(8)
  cases = [([-5, 3], 10), ([2, -1, 4], 5), ([-2, 7], 5)] + [
      (list(rng.integers(-6, 7, int(rng.integers(1, 9)))), int(rng.integers(1, 20))) for _ in range(2000)]
  unguarded_below = 0
  for sizes, split_num in cases:
    ends = np.cumsum(np.asarray(sizes, np.int64))
    for sz, end in zip(sizes, ends):
      start = end - sz
      if sz >= 1 and end <= split_num and start < 0:
        unguarded_below += 1            # without start >= 0 this group would read rs[end - 1] or rs[start] below 0
      if sz >= 1 and start >= 0 and end <= split_num:
        assert 0 <= start and end - 1 < split_num, (sizes, split_num)
  assert unguarded_below > 0


def test_normalize_merged_split_rejects_sizes_on_the_host(lib):
  i64 = (C.c_int64 * 4)()
  assert lib.mono_normalize_merged_split(0, i64, 2, i64, 3, i64, i64, None) == -1       # more splits than entries
  assert lib.mono_normalize_merged_split(0, i64, 2, i64, 0, i64, i64, None) == -1       # entries without a split
  assert lib.mono_normalize_merged_split(0, None, 0, None, 0, None, None, None) == 0     # nothing to do
  assert lib.mono_round_to_f16(0, None, -1, None, None) == -1
  assert lib.mono_round_to_f16(0, None, 0, None, None) == 0


def test_sharding_version_checks():
  feats = {"a": (torch.arange(4), torch.tensor([0, 2, 4])), "b": (torch.arange(3), torch.tensor([0, 3]))}
  with pytest.raises(ValueError, match="version"):
    dops.sharding_sparse_fids(feats, {"a": "x", "b": "x"}, {"a": 1, "b": 1}, 2, version=6)
  with pytest.raises(ValueError, match="version=5 needs CUDA"):
    dops.sharding_sparse_fids(feats, {"a": "x", "b": "x"}, {"a": 1, "b": 1}, 2, version=5)
  with pytest.raises(ValueError, match="batch_size"):
    dops._v5_batch_size(feats, ["a", "b"], set(), None)
  with pytest.raises(ValueError, match="every feature is shared"):
    dops._v5_batch_size(feats, ["a", "b"], {"a", "b"}, None)
  assert dops._v5_batch_size(feats, ["a", "b"], {"b"}, None) == 2
  assert dops._v5_batch_size(feats, ["a", "b"], set(), 9) == 9


def test_layout_grad_out_must_match_emb_sizes():
  fo, fe, nf = torch.zeros(1, dtype=torch.int64), torch.zeros(2, dtype=torch.int32), torch.zeros(2, dtype=torch.int32)
  with pytest.raises(ValueError):
    dops.fused_embedding_to_layout_grad([4], [1], fo, fe, nf, 1, [], [torch.zeros(1, 4)], out=[torch.zeros(3)])


def test_round_to_f16_refuses_other_tensors():
  with pytest.raises(ValueError, match="round_to_f16"):
    dops.round_to_f16(torch.zeros(4))
