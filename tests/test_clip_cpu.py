"""Clip by global norm without a device: the numpy restatement of mono_global_norm's order
(tests/global_norm_model.py) against math.fsum, ClipByGlobalNorm's scale rule, the host-side argument checks of
mono_global_norm, and the new C symbols and struct."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from tests import global_norm_model as gm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["mono_global_norm", "mono_mtable_pool_backward_parts_scaled",
               "mono_mtable_pool_backward_parts_bf16_scaled", "mono_embedding_to_layout_grad_scaled",
               "mono_embedding_to_layout_grad_bf16_scaled", "mono_gather_pool_grad_scaled",
               "mono_gather_pool_grad_bf16_scaled", "mono_scatter_grad_rows_scaled", "mono_scatter_grad_rows_bf16_scaled"]


# ---- the restatement ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sizes", [[], [0], [1], [8191], [8192], [8193], [3, 0, 70000, 8192 * 3 + 5],
                                   [1] * 9000, [70000] * 5])
def test_restatement_within_the_fp64_bound_of_fsum(sizes):
  rng = np.random.default_rng(len(sizes) + sum(sizes))
  arrays = [(rng.standard_normal(n) * rng.choice([1e-20, 1.0, 1e18], n)).astype(np.float32) for n in sizes]
  got = gm.sum_of_squares(arrays)
  sq = [float(x) * float(x) for a in arrays for x in a]
  want = math.fsum(sq)
  # every add of a sum of non-negative terms errs by at most 2^-53 of its result; no result exceeds the total, and no
  # term passes through more than (32 + 8) adds per level
  levels = max(1, math.ceil(math.log(max(len(sq), 2), 8192)))
  assert abs(got - want) <= 40 * levels * 2.0 ** -53 * want
  if not sq:
    assert got == 0.0 and math.copysign(1.0, got) == 1.0


def test_restatement_is_sequential_per_lane():
  """Lane 0 of one chunk: 1 + 2^-53 + ... (31 terms of 2^-53) stays 1 when added in order from 1 (each add rounds
  back), whereas a pairwise sum would keep them; the chunk then adds nothing else."""
  a = np.zeros(8192, np.float64)
  a[0] = 1.0
  a[256::256] = 2.0 ** -53
  assert gm._level(a)[0] == 1.0


def test_norm_is_the_fp32_sqrt_of_the_rounded_sum():
  arrays = [np.array([3.0, 4.0], np.float32)]
  assert gm.norm(arrays) == np.float32(5.0)
  big = [np.full(4, np.sqrt(np.finfo(np.float32).max), np.float32)]
  assert np.isinf(gm.norm(big))               # the fp64 sum is finite, its fp32 rounding is not


# ---- ClipByGlobalNorm's scale (clip_by_global_norm.h:42-49) -------------------------------------------------------
@pytest.mark.parametrize("norm,clip,want", [(5.0, 1000.0, 1.0), (1000.0, 1000.0, 1.0), (2000.0, 1000.0, 0.5),
                                            (3.0, 1.0, np.float32(1.0) / np.float32(3.0)),
                                            (float("inf"), 1000.0, 0.0), (float("nan"), 1000.0, 1.0),
                                            (0.0, 1e-30, 1.0)])
def test_scale_rule(norm, clip, want):
  with np.errstate(all="ignore"):
    got = gm.scale(norm, clip)
  assert got.view(np.uint32) == np.float32(want).view(np.uint32)


# ---- host-side rejection ------------------------------------------------------------------------------------------
def _norm_call(tensors, clip=0.0, norm=64, scale=None, n=None):
  from monolith_b200 import _lib
  lib = _lib.load()
  arr = (_lib.NormTensor * max(len(tensors), 1))()
  for i, (p, m, d) in enumerate(tensors):
    arr[i] = _lib.NormTensor(p, m, d)
  return lib.mono_global_norm(0, arr, len(tensors) if n is None else n, clip, norm, scale, None)


OK = (64, 16, 0)
BAD = {
    "n_tensors negative": dict(tensors=[OK], n=-1),
    "n_tensors over the limit": dict(tensors=[OK] * 4097),
    "negative size": dict(tensors=[(64, -1, 0)]),
    "null data": dict(tensors=[(None, 1, 0)]),
    "unknown dtype": dict(tensors=[(64, 1, 2)]),
    "negative dtype": dict(tensors=[(64, 1, -1)]),
    "negative clip_norm": dict(tensors=[OK], clip=-1.0, scale=64),
    "NaN clip_norm": dict(tensors=[OK], clip=float("nan"), scale=64),
    "infinite clip_norm": dict(tensors=[OK], clip=float("inf"), scale=64),
    "clip_norm without scale": dict(tensors=[OK], clip=1.0),
    "null norm": dict(tensors=[OK], norm=None),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_bad_arguments_are_rejected_on_the_host(case):
  assert _norm_call(**BAD[case]) == -1   # MONO_ERR_INVALID_ARGUMENT, nothing launched


def test_python_rejects_bad_tensors():
  import torch
  from monolith_b200 import clip_ops
  with pytest.raises(ValueError):
    clip_ops.global_norm([torch.zeros(3)])                           # not CUDA
  with pytest.raises(ValueError):
    clip_ops.global_norm_scale([], 0.0)
  with pytest.raises(ValueError):
    clip_ops.scale_ptr(torch.ones(1), torch.device("cuda", 0))       # a CPU scale
  with pytest.raises(ValueError):
    clip_ops.global_norm([object()])


# ---- declarations, exports, structs ---------------------------------------------------------------------------------
def test_new_symbols_are_declared_bound_and_exported():
  from monolith_b200 import _lib
  header = open(os.path.join(ROOT, "include", "mono_emb.h")).read()
  lib = _lib.load()
  for name in NEW_SYMBOLS:
    assert re.search(r"\bint %s\(" % name, header), name
    assert name in _lib.SIGNATURES, name
    assert getattr(lib, name) is not None
  assert "#define MONO_MAX_NORM_TENSORS 4096" in header
  assert _lib.MAX_NORM_TENSORS == 4096
  assert "MONO_DTYPE_F32 = 0, MONO_DTYPE_BF16 = 1" in header


def test_scaled_signatures_are_the_unscaled_ones_plus_the_scale():
  from monolith_b200 import _lib
  for name in NEW_SYMBOLS[1:]:
    res, args = _lib.SIGNATURES[name]
    base_res, base = _lib.SIGNATURES[name[:-len("_scaled")]]
    assert res == base_res and args == base[:-1] + [C.c_void_p, base[-1]], name


def test_norm_tensor_struct_matches_the_header():
  from monolith_b200 import _lib
  assert C.sizeof(_lib.NormTensor) == 24
  assert [f for f, _ in _lib.NormTensor._fields_] == ["data_dev", "n", "dtype"]
  assert _lib.NormTensor.n.offset == 8 and _lib.NormTensor.dtype.offset == 16


def test_abi_version_stays_1():
  from monolith_b200 import _lib
  assert _lib.load().mono_abi_version() == 1
