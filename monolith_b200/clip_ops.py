"""Clip gradients by global norm on the device (ref: monolith/native_training/clip_ops.py, GlobalL2Reduce in
runtime/ops/global_norm.cu.cc and ClipByGlobalNorm's scale rule, clip_by_global_norm.h:42-49).

The norm is one call of mono_global_norm: fp64 sums of exact squares in a fixed order that depends on the tensors'
sizes only (include/mono_emb.h states it), so its bits do not change from run to run.  The reference sums fp32
squares with float atomics.  Nothing here synchronises with the host: the norm and the scale stay on the device.

The sparse side takes the scale where the gradient rows are loaded; the dense side multiplies with torch:
- `grad_scale=` of MultiHashTable.pool_backward and pool_backward_parts, PartitionedHashTable.apply_gradients and
  ShardedStep.step (every exchange);
- `grad_scale=` of distribution_ops.reduce_sum_gradient, reduce_mean_gradient, fused_reduce_sum_and_split_gradient
  and fused_reduce_and_split_gpu_grad, and of Grouping.reduce / reduce_push;
- `layout_tensors_grad_scale=` of distribution_ops.fused_embedding_to_layout_grad, `scale=` of gather_pool_grad /
  scatter_grad_rows.
Each is bit for bit the call without the scale on the gradients multiplied by it in float32 first.
"""
import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib

_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.bfloat16: _lib.DTYPE_BF16}


def scale_ptr(scale: Optional[torch.Tensor], device: torch.device, what: str = "grad_scale"):
  """None -> None; otherwise the device pointer of a one-element float32 CUDA tensor on `device` (ValueError
  for anything else).  The value is read by the kernels, never by the host."""
  if scale is None:
    return None
  if not isinstance(scale, torch.Tensor) or scale.dtype != torch.float32 or scale.numel() != 1 or \
      scale.device.type != "cuda" or scale.device != torch.device(device):
    raise ValueError(f"{what} must be a one-element torch.float32 tensor on {device}")
  return C.c_void_p(scale.data_ptr())


def _device_of(t_list: Sequence[torch.Tensor]) -> torch.device:
  if len(t_list) > _lib.MAX_NORM_TENSORS:
    raise ValueError(f"at most {_lib.MAX_NORM_TENSORS} tensors per call, not {len(t_list)}")
  dev = None
  for t in t_list:
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
      raise ValueError("every tensor must be a CUDA tensor")
    if t.dtype not in _DTYPES:
      raise ValueError(f"tensors must be torch.float32 or torch.bfloat16, not {t.dtype}")
    if not t.is_contiguous():
      raise ValueError("tensors must be contiguous")
    if dev is None:
      dev = t.device
    elif t.device != dev:
      raise ValueError(f"all tensors must be on one device, not {dev} and {t.device}")
  return dev if dev is not None else torch.device("cuda", torch.cuda.current_device())


def _norm_call(t_list: Sequence[torch.Tensor], clip_norm: float) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
  t_list = list(t_list)
  dev = _device_of(t_list)
  clip_norm = float(clip_norm)
  lib = _lib.load()
  norm = torch.empty((), dtype=torch.float32, device=dev)
  scale = torch.empty((), dtype=torch.float32, device=dev) if clip_norm > 0 else None
  arr = (_lib.NormTensor * max(len(t_list), 1))()
  for i, t in enumerate(t_list):
    arr[i] = _lib.NormTensor(C.c_void_p(t.data_ptr()), t.numel(), _DTYPES[t.dtype])
  _lib.check(lib.mono_global_norm(dev.index, arr, len(t_list), clip_norm, _lib.ptr(norm), _lib.ptr(scale),
                                  _lib.stream(dev)))
  return scale, norm


def global_norm(t_list: Sequence[torch.Tensor]) -> torch.Tensor:
  """The L2 norm of all elements of all tensors (float32 and bfloat16 in any mix, contiguous, one CUDA device):
  a 0-d float32 tensor on that device.  ref: clip_ops._global_norm / GlobalL2Reduce."""
  return _norm_call(t_list, 0.0)[1]


def global_norm_scale(t_list: Sequence[torch.Tensor], clip_norm: float) -> Tuple[torch.Tensor, torch.Tensor]:
  """-> (scale, norm), both 0-d float32 on the device: scale = clip_norm / norm when norm > clip_norm, else 1
  (1 for a NaN norm, +0.0 for an infinite one).  This is the deferred path's scale: pass it as `grad_scale=`.
  clip_norm must be finite and > 0."""
  if not float(clip_norm) > 0 or float(clip_norm) == float("inf"):
    raise ValueError(f"clip_norm must be finite and > 0, not {clip_norm}")
  return _norm_call(t_list, clip_norm)


def clip_by_global_norm(t_list: Sequence[torch.Tensor], clip_norm: float) -> Tuple[List[torch.Tensor], torch.Tensor]:
  """-> (clipped tensors, global norm).  Each clipped tensor is torch's elementwise `t * scale` with the device
  scale of global_norm_scale (float32 arithmetic, the result in t's dtype): the reference's element_wise_mul.
  No host synchronisation decides whether to clip, so a tensor that needs no clipping comes back multiplied by
  1.0: a new tensor with t's values, never t itself."""
  t_list = list(t_list)
  scale, norm = global_norm_scale(t_list, clip_norm)
  return [t * scale for t in t_list], norm
