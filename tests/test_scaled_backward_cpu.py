"""What tests/test_gpu_scaled_backward.py relies on, checked without a GPU: the six _scaled calls of the one-table
backward, the ReduceSum gradients and the sharded step are declared, bound and exported with their twin's arguments
plus the device scale before the stream, and every Python entry refuses a bad grad_scale before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from monolith_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWINS = {
    "mono_mtable_pool_backward_scaled": "mono_mtable_pool_backward",
    "mono_reduce_and_split_grad_scaled": "mono_reduce_and_split_grad",
    "mono_reduce_and_split_grad_bf16_scaled": "mono_reduce_and_split_grad_bf16",
    "mono_grouping_reduce_scaled": "mono_grouping_reduce",
    "mono_grouping_reduce_push_scaled": "mono_grouping_reduce_push",
    "mono_xstep_backward_scaled": "mono_xstep_backward",
}


@pytest.fixture(scope="module")
def lib():
  if not os.path.exists(_lib.LIB_PATH):
    import __graft_entry__
    __graft_entry__.build()
  return _lib.load()


def _header():
  with open(os.path.join(ROOT, "include", "mono_emb.h")) as f:
    return f.read()


def _params(src, name):
  """The parameter list of `name`'s declaration, whitespace squashed."""
  m = re.search(r"\bint " + name + r"\(([^;]*?)\);", src, flags=re.S)
  assert m, name
  return [re.sub(r"\s+", " ", p).strip() for p in m.group(1).split(",")]


def test_declared_bound_and_exported(lib):
  src = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
  for name in TWINS:
    assert re.search(r"\b" + name + r"\s*\(", src), name
    assert name in _lib.SIGNATURES, name
    assert hasattr(lib, name), name
  assert lib.mono_abi_version() == 1


def test_each_signature_is_its_twins_plus_the_scale():
  src = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
  for name, twin in TWINS.items():
    res, args = _lib.SIGNATURES[name]
    t_res, t_args = _lib.SIGNATURES[twin]
    assert res == t_res and args == t_args[:-1] + [C.c_void_p, t_args[-1]], name
    p, tp = _params(src, name), _params(src, twin)
    assert p == tp[:-1] + ["const float* grad_scale_dev", tp[-1]], name
    assert tp[-1] == "void* stream", twin


def test_header_semantics_cover_every_scaled_call():
  h = _header()
  assert "for all eight" not in h
  assert "for every _scaled call" in h


# ------------------------------------------------------------------------------------------------
# Python: a bad grad_scale is a ValueError before anything reaches the device
# ------------------------------------------------------------------------------------------------
BAD = [torch.ones(1, dtype=torch.float64), torch.ones(2), torch.ones(1), torch.ones(1, device="meta"),
       np.ones(1, np.float32), 0.5]
BAD_IDS = ["float64", "two elements", "cpu", "meta device", "numpy", "python float"]


@pytest.mark.parametrize("bad", BAD, ids=BAD_IDS)
def test_distribution_ops_refuse_bad_scales(bad):
  from monolith_b200 import distribution_ops as dops
  idx = torch.arange(6, dtype=torch.int64)[:, None]
  g = torch.zeros(6, 8)
  for call in (lambda: dops.reduce_sum_gradient(idx, g, grad_scale=bad),
               lambda: dops.reduce_mean_gradient(idx, g, grad_scale=bad),
               lambda: dops.fused_reduce_sum_and_split_gradient(idx, [g[:, :3], g[:, 3:]], [3, 5], grad_scale=bad),
               lambda: dops.fused_reduce_and_split_gpu_grad([torch.arange(7, dtype=torch.int32)], [g], [g], [[8]],
                                                            grad_scale=bad)):
    with pytest.raises(ValueError, match="grad_scale"):
      call()


def _bare(cls, **attrs):
  """An instance without its device state: a call that got past the argument check would fail on a missing
  attribute, not with ValueError."""
  obj = object.__new__(cls)
  for k, v in attrs.items():
    setattr(obj, k, v)
  return obj


@pytest.mark.parametrize("bad", BAD, ids=BAD_IDS)
def test_methods_refuse_bad_scales_first(bad):
  from monolith_b200 import MultiHashTable
  from monolith_b200.distributed_ps import ShardedStep
  from monolith_b200.distribution_ops import Grouping
  dev = torch.device("cuda", 0)
  g = torch.zeros(4, 8)
  ids = torch.arange(4, dtype=torch.int64)
  with pytest.raises(ValueError, match="grad_scale"):
    _bare(MultiHashTable, _device=dev).pool_backward("t", ids, g, grad_scale=bad)
  grp = _bare(Grouping, device=dev)
  with pytest.raises(ValueError, match="grad_scale"):
    grp.reduce(g, torch.empty(32), grad_scale=bad)
  with pytest.raises(ValueError, match="grad_scale"):
    grp.reduce_push(g, [4], None, 0, [0], grad_scale=bad)
  for exchange in ("direct", "peer", "nccl"):
    st = _bare(ShardedStep, device=dev, exchange=exchange)
    with pytest.raises(ValueError, match="grad_scale"):
      st.step(ids, g, torch.empty(4, 8), 1, grad_scale=bad)
