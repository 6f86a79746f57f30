"""bf16 tower-side tensors of the layout op, the gather calls and PartitionedHashTable, without a device: the
bindings, the wrappers' dtype rules (checked before the library is loaded) and the bf16 layout calls' task validation.
"""

import pytest
import torch

from monolith_b200 import _lib
from monolith_b200 import distribution_ops as dops
from monolith_b200.distribution_ops import SliceTask
from tests.test_layout_paths_cpu import BAD, GOOD, SUM, _args, lib  # noqa: F401  (lib: the module fixture)

TWINS = ("mono_embedding_to_layout", "mono_embedding_to_layout_grad", "mono_gather_pool", "mono_gather_pool_grad",
         "mono_scatter_grad_rows")


@pytest.mark.parametrize("name", TWINS)
def test_bf16_bindings_take_their_twins_arguments(name):
  assert _lib.SIGNATURES[name + "_bf16"] == _lib.SIGNATURES[name]


def test_bf16_symbols_are_declared_in_the_header():
  import os
  with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "mono_emb.h")) as f:
    hdr = f.read()
  for name in TWINS:
    assert f"int {name}_bf16(" in hdr


@pytest.fixture
def no_lib(monkeypatch):
  def boom():
    raise AssertionError("reached the library")
  monkeypatch.setattr(_lib, "load", boom)


TASK = [SliceTask(0, 0, 4, SUM, 0, 0, 4, 0, 0)]


@pytest.mark.parametrize("bad", [torch.float16, torch.float64, torch.int32])
def test_layout_wrappers_refuse_other_dtypes_before_loading(bad, no_lib):
  with pytest.raises(ValueError, match="dtype"):
    dops.fused_embedding_to_layout([torch.zeros(16)], [1], *_args(), 1, TASK, [(1, 4)], dtype=bad)
  with pytest.raises(ValueError, match="out_grads"):
    dops.fused_embedding_to_layout_grad([16], [1], *_args(), 1, TASK, [torch.zeros(1, 4, dtype=bad)])


def test_layout_grad_refuses_mixed_dtypes_before_loading(no_lib):
  mixed = [torch.zeros(1, 4, dtype=torch.bfloat16), torch.zeros(1, 4)]
  for og in (mixed, mixed[::-1]):
    with pytest.raises(ValueError, match="out_grads"):
      dops.fused_embedding_to_layout_grad([16], [1], *_args(), 1, TASK, og)


@pytest.mark.parametrize("bad", [torch.float16, torch.float64])
def test_gather_wrappers_refuse_other_dtypes_before_loading(bad, no_lib):
  fused, offs = torch.zeros(16), torch.zeros(4, dtype=torch.int32)
  with pytest.raises(ValueError, match="gather_pool's output"):
    dops.gather_pool(fused, offs, 4, out=torch.zeros(4, 4, dtype=bad))
  with pytest.raises(ValueError, match="gather_pool's output"):
    dops.gather_pool(fused, offs, 4, dtype=bad)
  with pytest.raises(ValueError, match="pooled_grad"):
    dops.gather_pool_grad(torch.zeros(4, 4, dtype=bad), offs, 4, 16)
  with pytest.raises(ValueError, match="pooled_grad"):
    dops.scatter_grad_rows(torch.zeros(4, 4, dtype=bad), offs, 4, torch.zeros(16))


@pytest.mark.parametrize("bad", [torch.bfloat16, torch.float16, torch.float64])
def test_scatter_refuses_a_non_float32_grad_fused_before_loading(bad, no_lib):
  offs = torch.zeros(4, dtype=torch.int32)
  for pg in (torch.zeros(4, 4), torch.zeros(4, 4, dtype=torch.bfloat16)):
    with pytest.raises(ValueError, match="grad_fused"):
      dops.scatter_grad_rows(pg, offs, 4, torch.zeros(16, dtype=bad))


def test_partitioned_lookup_refuses_other_dtypes():
  from monolith_b200.distributed_ps import PartitionedHashTable

  class _T:
    table_names = ("a",)
    device = torch.device("cpu")

    def get_table_dim_sizes(self):
      return [4]
  pht = PartitionedHashTable(_T(), 1, 0, backend=object())
  with pytest.raises(ValueError, match="dtype"):
    pht.lookup({"a": torch.zeros(3, dtype=torch.int64)}, dtype=torch.float16)


def _call_bf16(lib, grad, tasks, total_nfl=3):
  arr = dops._tasks_arr(tasks)
  fn = lib.mono_embedding_to_layout_grad_bf16 if grad else lib.mono_embedding_to_layout_bf16
  return fn(0, None, None, 1, None, 0, None, 0, None, total_nfl, 4, arr, len(tasks), None, None)


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("field,change", BAD, ids=[f"{f}-{i}" for i, (f, _) in enumerate(BAD)])
def test_bf16_layout_rejects_bad_tasks_before_the_device(field, change, grad, lib):
  good = SliceTask(**GOOD)
  bad = SliceTask(**{**GOOD, **change})
  assert _call_bf16(lib, grad, [good, bad]) == -1   # MONO_ERR_INVALID_ARGUMENT
  assert field.encode() in lib.mono_last_error()


def test_bf16_layout_accepts_edge_tasks_and_reaches_the_device(lib):
  if torch.cuda.is_available():
    pytest.skip("with a GPU the call would launch on null pointers")
  for grad in (False, True):
    assert _call_bf16(lib, grad, [SliceTask(**GOOD)]) == -3   # MONO_ERR_CUDA: validation passed, no device here


def test_abi_version_stays_1(lib):
  assert lib.mono_abi_version() == 1
