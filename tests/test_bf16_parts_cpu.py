"""bf16 rows of the parts calls, without a device: the bindings, the Python dtype rules, and the rounding the GPU
tests use as their reference.

The header promises each bf16 output element is the fp32 result rounded once to nearest even
(__float2bfloat16_rn).  tests/test_gpu_bf16_parts.py compares against torch's float32 -> bfloat16 conversion, so
that conversion is pinned here on the edge cases those tests rely on.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from monolith_b200 import PoolPart, _lib


def test_bindings_take_the_fp32_calls_arguments():
  sig = _lib.SIGNATURES
  assert sig["mono_mtable_lookup_pool_parts_bf16"] == sig["mono_mtable_lookup_pool_parts"]
  assert sig["mono_mtable_pool_backward_parts_bf16"] == sig["mono_mtable_pool_backward_parts"]
  assert sig["mono_mtable_lookup_pool_parts_bf16"] == (C.c_int, [C.c_void_p, C.POINTER(_lib.PoolPartC), C.c_int32,
                                                                 C.c_void_p])
  assert C.sizeof(_lib.PoolPartC) == 72


def rne_bf16(x):
  """Reference float32 -> bfloat16 bits, round to nearest even, written out on the integer bits."""
  u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
  nan = np.isnan(np.asarray(x, np.float32))
  r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
  return np.where(nan, 0x7FC0 | ((u >> 16) & 0x8000), r).astype(np.uint16)


def bits(f32):
  return np.uint32(f32).view(np.float32)


EDGES = {
    "tie to even (down)": bits(0x3F808000),     # 1 + 2^-8: halfway between 1 and 1 + 2^-7 -> 1
    "tie to even (up)": bits(0x3F818000),       # 1 + 3 * 2^-8: halfway -> 1 + 2^-6
    "above the tie": bits(0x3F808001),
    "below the tie": bits(0x3F807FFF),
    "largest finite float": np.finfo(np.float32).max,        # rounds up to inf
    "largest bf16": bits(0x7F7F0000),
    "just under the inf tie": bits(0x7F7F7FFF),                # stays the largest finite bf16
    "the inf tie": bits(0x7F7F8000),                           # odd mantissa: rounds up to inf
    "smallest subnormal": bits(0x00000001),                    # -> +0
    "bf16 subnormal": bits(0x00010000),
    "subnormal tie": bits(0x00018000),                         # -> 0x0002
    "-0.0": np.float32(-0.0),
    "inf": np.float32(np.inf),
    "-inf": np.float32(-np.inf),
    "negative tie": bits(0xBF808000),
}


@pytest.mark.parametrize("name", sorted(EDGES))
def test_torch_float_to_bfloat16_is_round_to_nearest_even(name):
  x = np.array([EDGES[name]], np.float32)
  got = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
  np.testing.assert_array_equal(got, rne_bf16(x), err_msg=name)


def test_the_edge_cases_land_where_the_gpu_tests_expect():
  r = {k: int(rne_bf16(np.array([v], np.float32))[0]) for k, v in EDGES.items()}
  assert r["tie to even (down)"] == 0x3F80 and r["tie to even (up)"] == 0x3F82
  assert r["largest finite float"] == 0x7F80 and r["the inf tie"] == 0x7F80 and r["just under the inf tie"] == 0x7F7F
  assert r["smallest subnormal"] == 0x0000 and r["subnormal tie"] == 0x0002 and r["-0.0"] == 0x8000
  assert r["inf"] == 0x7F80 and r["-inf"] == 0xFF80


def test_nan_stays_nan():
  x = np.array([np.nan, bits(0x7FC0DEAD), bits(0xFFFFFFFF)], np.float32)
  assert torch.isnan(torch.from_numpy(x).to(torch.bfloat16)).all()


def test_bf16_widening_is_exact():
  b = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
  f = b.float()
  ok = ~torch.isnan(f)
  assert torch.equal(f.view(torch.int32)[ok] >> 16, b.view(torch.int16)[ok].to(torch.int32))
  assert torch.equal(f.view(torch.int32)[ok] & 0xFFFF, torch.zeros_like(f.view(torch.int32)[ok]))


def _host_table():
  from monolith_b200.multi_hash_table_ops import MultiHashTable
  t = MultiHashTable.__new__(MultiHashTable)
  t._device = torch.device("cpu")
  t._table_names = ["t"]
  t._dims = [4]
  return t


def test_call_dtype_rules():
  t = _host_table()
  f = torch.arange(2, dtype=torch.int64)
  bf = torch.zeros(2, 4, dtype=torch.bfloat16)
  fp = torch.zeros(2, 4)
  assert t._parts_dtype([PoolPart("t", f)]) == torch.float32
  assert t._parts_dtype([PoolPart("t", f), PoolPart("t", f, rows=bf)]) == torch.bfloat16
  assert t._parts_dtype([PoolPart("t", f)], torch.bfloat16) == torch.bfloat16
  _, _, outs = t._parts_arr([PoolPart("t", f), PoolPart("t", f, rows=bf)], forward=True, dtype=torch.bfloat16)
  assert outs[0].dtype == torch.bfloat16 and outs[1] is bf
  with pytest.raises(ValueError):  # rows of another dtype than the call's
    t._parts_arr([PoolPart("t", f, rows=fp)], forward=True, dtype=torch.bfloat16)
  with pytest.raises(ValueError):  # mixed
    t._parts_dtype([PoolPart("t", f, rows=fp), PoolPart("t", f, rows=bf)])
  for bad in (torch.float16, torch.float64):
    with pytest.raises(ValueError):
      t._parts_dtype([PoolPart("t", f, rows=torch.zeros(2, 4, dtype=bad))])
    with pytest.raises(ValueError):
      t._parts_dtype([PoolPart("t", f)], bad)
