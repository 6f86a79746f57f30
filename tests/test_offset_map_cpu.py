"""The async parameter-server worker ops without a GPU: the numpy restatement (tests/offset_map_model.py) pinned on
the reference's own test vectors (tests/golden/ref_offset_map.json), and the argument checks of the four C entry
points, which reject before any device is touched."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from monolith_b200 import _lib
from tests import offset_map_model as om

G = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_offset_map.json")))


def _ragged(rows):
  flat = [x for r in rows for x in r]
  return np.asarray(flat, np.int64), np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)


def test_ragged_split_model_matches_the_reference_vectors():
  g = G["ragged_split"]
  splits, pos = om.ragged_split_by_indices(g["indices"], g["values"], g["row_splits"], g["num_splits"])
  for (vals, rs), want in zip(splits, g["splits"]):
    wv, wrs = _ragged(want)
    assert vals.tolist() == wv.tolist() and rs.tolist() == wrs.tolist()
  for p, want in zip(pos, g["pos"]):
    assert p.tolist() == _ragged(want)[0].tolist()


def test_unique_fill_and_gradient_model_match_the_reference_vectors():
  g = G["unique_fill"]
  keys, split = _ragged(g["keys"])
  uk, uks, vo, vos, n = om.unique_key_with_value_and_offset(keys, split, g["dims"])
  want_uk, want_uks = _ragged(g["unique_key"])
  assert uk.tolist() == want_uk.tolist() and uks.tolist() == want_uks.tolist()
  per_key = [o for t in g["value_offset"] for o in t]
  assert vo.tolist() == [x for o in per_key for x in o]
  assert vos.tolist() == np.cumsum([0] + [len(o) for o in per_key]).tolist()
  assert n == len(g["buffer"])
  pos, pos_split = _ragged(g["fill_pos"])
  buf = np.full(n, np.nan, np.float32)
  om.fill_with_offset_map(pos, pos_split, np.asarray(g["fill_value"], np.float32), vo, vos, g["dims"], buf)
  assert buf.tolist() == g["buffer"]
  grad = om.fill_with_offset_map_gradient(pos, pos_split, np.asarray(g["grad_in"], np.float32), vo, vos, g["dims"])
  assert grad.tolist() == g["grad"]


def test_unique_model_empty_tables():
  g = G["unique_empty"]
  keys, split = _ragged(g["keys"])
  uk, uks, vo, vos, n = om.unique_key_with_value_and_offset(keys, split, g["dims"])
  assert uk.size == 0 and uks.tolist() == [0, 0, 0, 0] and vo.size == 0 and vos.tolist() == [0] and n == 0


def test_gradient_model_sums_in_occurrence_order_from_plus_zero():
  # one key, occurrences 1e8, 1, -1e8: (((+0 + 1e8) + 1) + -1e8) = 0 in float32, a reordered sum gives 1
  vo, vos = np.array([0, 1, 2], np.int64), np.array([0, 3], np.int64)
  g = om.fill_with_offset_map_gradient([0], [0, 1], np.array([1e8, 1, -1e8], np.float32), vo, vos, [1])
  assert g.tolist() == [0.0]
  g = om.fill_with_offset_map_gradient([0], [0, 1], np.array([-0.0], np.float32), vo[:1], np.array([0, 1]), [1])
  assert np.signbit(g).tolist() == [False]


# ---- the C entry points' argument checks: MONO_ERR_INVALID_ARGUMENT before the device is selected ----------------
_P = C.c_void_p(16)  # never dereferenced: every case below is rejected on the host


def _unique(split, dims):
  lib = _lib.load()
  K = len(dims)
  return lib.mono_unique_key_with_value_and_offset(0, _P, (C.c_int64 * len(split))(*split), K,
                                                   (C.c_int32 * max(K, 1))(*dims), _P, _P, _P, _P, None, None, None)


@pytest.mark.parametrize("split,dims,what", [
    ([0], [], "num_tables must be positive"),
    ([1, 2], [1], "start at 0"),
    ([0, 3, 2], [1, 1], "must not decrease"),
    ([0, 2], [0], "dims must be positive"),
    ([0, 1, 2], [1, -3], "dims must be positive"),
    ([0, (1 << 30) + 1], [1], "2^30"),
])
def test_unique_rejects(split, dims, what):
  assert _unique(split, dims) == -1
  assert what in _lib.load().mono_last_error().decode()


def test_unique_null_arguments():
  lib = _lib.load()
  assert lib.mono_unique_key_with_value_and_offset(0, _P, None, 1, (C.c_int32 * 1)(1), _P, _P, _P, _P, None, None,
                                                   None) == -1


@pytest.mark.parametrize("cap,K,S,what", [
    (4, 0, 2, "num_tables must be positive"),
    (4, 1, 0, "num_splits must be positive"),
    (4, 1, -1, "num_splits must be positive"),
    (-1, 1, 2, "capacity"),
    ((1 << 30) + 1, 1, 2, "capacity"),
    (4, 1 << 16, 1 << 16, "2^31"),
])
def test_ragged_split_rejects(cap, K, S, what):
  lib = _lib.load()
  assert lib.mono_ragged_split_by_indices(0, _P, _P, cap, _P, K, S, _P, _P, _P, _P, None, None, None) == -1
  assert what in lib.mono_last_error().decode()


def _fill(split, dims, value_len=100, num_unique=4, grad=False):
  lib = _lib.load()
  K = len(dims)
  cs, cd = (C.c_int64 * len(split))(*split), (C.c_int32 * max(K, 1))(*dims)
  if grad:
    return lib.mono_fill_with_offset_map_grad(0, _P, cs, K, cd, _P, _P, _P, num_unique, _P, None, None)
  return lib.mono_fill_with_offset_map(0, _P, cs, K, cd, _P, value_len, _P, _P, num_unique, _P, None, None)


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("kw,what", [
    (dict(split=[0], dims=[]), "num_tables must be positive"),
    (dict(split=[1, 2], dims=[1]), "start at 0"),
    (dict(split=[0, 2, 1], dims=[1, 1]), "must not decrease"),
    (dict(split=[0, 2], dims=[0]), "dims must be positive"),
    (dict(split=[0, (1 << 30) + 1], dims=[1], value_len=1 << 31), "2^30 rows"),
    (dict(split=[0, 2], dims=[1], num_unique=-1), "num_unique"),
])
def test_fill_rejects(kw, what, grad):
  assert _fill(grad=grad, **kw) == -1
  assert what in _lib.load().mono_last_error().decode()


def test_fill_rejects_a_short_value_and_accepts_a_longer_one_on_the_host():
  """ref: distribution_ops_test.py:110-120: 10 floats where 12 are needed"""
  g = G["unique_fill"]
  pos, pos_split = _ragged(g["fill_pos"])
  assert _fill(pos_split.tolist(), g["dims"], value_len=G["fill_error"]["value_len"]) == -1
  assert "expected: 12, actual: 10" in _lib.load().mono_last_error().decode()
  assert _fill(pos_split.tolist(), g["dims"], value_len=13, num_unique=-1) == -1  # a longer value passes this check
  assert "num_unique" in _lib.load().mono_last_error().decode()


def test_the_four_entry_points_are_bound():
  for name in ("mono_unique_key_with_value_and_offset", "mono_ragged_split_by_indices", "mono_fill_with_offset_map",
               "mono_fill_with_offset_map_grad"):
    assert name in _lib.SIGNATURES
