"""Times clip-by-global-norm on the bench_parts.py workload (4 tables of dims 16, 16, 32, 64; 26 one-FID features;
Zipf FIDs), all variants alternating in one process, CUDA events, median and [min, max] over the timed steps:

  1 norm: mono_global_norm over the 26 layout gradients against torch._foreach_norm + torch.linalg.vector_norm;
    bytes read over kernel time, as a share of the H100 SXM data sheet's 3.35 TB/s.
  2 backward: pool_backward_parts with grad_scale against the unscaled call on rows pre-multiplied outside the timing
    (the two tables must end bit-identical).
  3 the whole clip step: torch (foreach norm, stack, norm, where-scale, one mul per layout gradient, unscaled
    backward) against this engine (global_norm_scale + the scaled backward).

  python scripts/bench_clip.py [--batch 65536 16384] [--steps 30] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_parts import DIMS, N_FEATURES, batches, make_table  # noqa: E402
from monolith_b200 import PoolPart, clip_ops  # noqa: E402

CLIP = 1000.0


def timed(fn, reps=1):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(reps):
    out = fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps, out


def torch_norm(grads):
  return torch.linalg.vector_norm(torch.stack(torch._foreach_norm(grads)))


def torch_scale(grads):
  norm = torch_norm(grads)
  return torch.where(norm > CLIP, CLIP / norm, torch.ones((), device=norm.device))


def parts(feats, rows):
  return [PoolPart(s, f, rows=g) for (s, f, _), g in zip(feats, rows)]


def summary(xs):
  return {"median": float(np.median(xs)), "spread": [float(np.min(xs)), float(np.max(xs))]}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, nargs="+", default=[65536, 16384])
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_clip.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for B in args.batch:
    data = batches(B, 4, dev, seed=B)
    nbytes = sum(g.numel() * 4 for _, _, g in data[0])
    t_unscaled, t_scaled, t_torch, t_fused = (make_table(dev) for _ in range(4))
    times = {k: [] for k in ("norm_mono", "norm_torch", "bwd_unscaled", "bwd_scaled", "step_torch", "step_fused")}
    scale_rel = 0.0
    ts = 1
    for it in range(args.warmup + args.steps):
      feats = data[it % len(data)]
      grads = [g for _, _, g in feats]
      s_dev, _ = clip_ops.global_norm_scale(grads, CLIP)
      pre = [g * s_dev for g in grads]
      runs = [("norm_mono", lambda: clip_ops.global_norm(grads), 20),
              ("norm_torch", lambda: torch_norm(grads), 20),
              ("bwd_unscaled", lambda: t_unscaled.pool_backward_parts(parts(feats, pre), req_time=ts), 1),
              ("bwd_scaled", lambda: t_scaled.pool_backward_parts(parts(feats, grads), req_time=ts, grad_scale=s_dev), 1),
              ("step_torch", lambda: t_torch.pool_backward_parts(
                  parts(feats, [g * s for s in [torch_scale(grads)] for g in grads]), req_time=ts), 1),
              ("step_fused", lambda: t_fused.pool_backward_parts(
                  parts(feats, grads), req_time=ts, grad_scale=clip_ops.global_norm_scale(grads, CLIP)[0]), 1)]
      if it % 2:
        runs.reverse()
      for name, fn, reps in runs:
        ms, _ = timed(fn, reps)
        if it >= args.warmup:
          times[name].append(ms)
      scale_rel = max(scale_rel, abs(torch_scale(grads).item() / s_dev.item() - 1.0))
      ts += 1
    same = True
    for slot in DIMS:
      keys = torch.unique(torch.cat([f for d in data for s, f, _ in d if s == slot]))
      ea, eb = t_unscaled.lookup_entry(slot, keys)["raw"], t_scaled.lookup_entry(slot, keys)["raw"]
      same &= torch.equal(ea.view(torch.int32), eb.view(torch.int32))
    assert same, "scaled and pre-multiplied backward tables differ"
    norm_ms = float(np.median(times["norm_mono"]))
    res = {"batch": B, "features": N_FEATURES, "layout_grad_bytes": nbytes, "steps": args.steps,
           **{f"ms_{k}": summary(v) for k, v in times.items()},
           "norm_TBps": nbytes / (norm_ms * 1e-3) / 1e12, "norm_share_of_3.35TBps": nbytes / (norm_ms * 1e-3) / 3.35e12,
           "torch_vs_device_scale_max_rel_diff": scale_rel, "scaled_bwd_same_bits": same,
           "gpu": props.name, "power_limit": power}
    print(json.dumps(res))
    for t in (t_unscaled, t_scaled, t_torch, t_fused):
      t.close()


if __name__ == "__main__":
  main()
