"""CPU checks of the parts backward (mono_mtable_pool_backward_parts): the ctypes record against the header, PoolPart
validation, and the concatenation rule the GPU file relies on, restated with tests/reduce_order.py."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from monolith_b200 import PoolPart, _lib
from tests import reduce_order as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "mono_emb.h")).read()


def test_pool_part_struct_matches_the_header():
  body = re.search(r"typedef struct mono_pool_part \{(.*?)\} mono_pool_part;", HEADER, re.S).group(1)
  body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
  fields = re.findall(r"([A-Za-z_][A-Za-z0-9_ ]*?[\s*]+)([a-z_]+);", body)
  names = [n for _, n in fields]
  assert names == [f[0] for f in _lib.PoolPartC._fields_]
  size = {"int32_t": 4, "int64_t": 8}
  for (ctype, name), (_, ct) in zip(fields, _lib.PoolPartC._fields_):
    want = 8 if "*" in ctype else size[ctype.strip().split()[-1]]
    assert C.sizeof(ct) == want, name
  assert C.sizeof(_lib.PoolPartC) == 72
  assert int(re.search(r"#define MONO_MAX_POOL_PARTS (\d+)", HEADER).group(1)) == _lib.MAX_POOL_PARTS


def test_binding_signature():
  res, args = _lib.SIGNATURES["mono_mtable_pool_backward_parts"]
  assert res is C.c_int
  assert args[1] == C.POINTER(_lib.PoolPartC) and len(args) == 7


def test_pool_part_validation():
  f = torch.zeros(4, dtype=torch.int64)
  PoolPart("t", f)
  PoolPart("t", f, pooling="mean", rows=torch.zeros(4, 8), col=4)
  with pytest.raises(ValueError):
    PoolPart("t", f, pooling="firstn")
  with pytest.raises(ValueError):
    PoolPart("t", f, col=-1)
  with pytest.raises(ValueError):
    PoolPart("t", f, rows=torch.zeros(8))


@pytest.mark.parametrize("G", [4, 8, 32])
def test_concatenation_rule_against_the_oracle_sequential_sums(G):
  """A table's terms are taken part by part, then in occurrence order, and the tree depth comes from the table's
  total: for runs of <= 64 terms reduce_order's sums equal the reference's sequential ScatterGrad (one add per
  occurrence into the FID's row) over the concatenation."""
  rng = np.random.default_rng(G)
  D = 4 * G
  parts = [rng.integers(0, 300, n) for n in (500, 200, 900)]
  keys = np.concatenate(parts)
  x = rng.standard_normal((keys.size, D)).astype(np.float32)
  u, sums, length = ro.call_sums(x, keys, G)
  assert length.max() <= 64
  want = np.zeros((u.size, D), np.float32)
  seen = np.zeros(u.size, bool)
  for m, k in enumerate(np.searchsorted(u, keys)):  # the reference's order: occurrence by occurrence
    want[k] = x[m] if not seen[k] else want[k] + x[m]
    seen[k] = True
  np.testing.assert_array_equal(sums.view(np.uint32), want.view(np.uint32))
  # the depth follows the table's own total, not the call's
  assert ro.tree_top(ro.n_pieces(16384))[0] == 0 and ro.tree_top(ro.n_pieces(16385))[0] == 1
