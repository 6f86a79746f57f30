"""Times the fused sparse backward (`pool_backward`) of the C2 step alone and breaks it down per kernel.

Same table and batches as `bench.py` (one table, dim 32, 10 M resident keys, Adagrad; B = 1 048 576 samples x 2 slots,
M = 2 097 152 FID occurrences, Zipf(1.05) ranks, bench.make_batches with its seeds), four rotating batches.
  1. CUDA-event time of every `pool_backward` call over --steps calls after --warmup: median, min, max.
  2. A separate run of --profile-steps calls under torch.profiler: device time per call of every kernel, by name.
The card's name, SM clock limit and power limit are read in the same process.

  python scripts/bench_bwd.py [--steps 60] [--warmup 10] [--profile-steps 10]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the C2 workload's generator and constants)
from monolith_b200 import MultiHashTable, entry  # noqa: E402


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
  except OSError:
    out = ""
  return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": out}


def short_name(name):
  """Kernel name without namespace, argument list and return type: 'runs_apply_kernel<8, 1>'."""
  name = re.sub(r"\(.*$", "", name)
  name = re.sub(r"^void ", "", name)
  return name.replace("mono::", "")


def device_us(evt):
  for attr in ("self_device_time_total", "self_cuda_time_total"):
    v = getattr(evt, attr, None)
    if v is not None:
      return float(v)
  return 0.0


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=60)
  ap.add_argument("--warmup", type=int, default=10)
  ap.add_argument("--profile-steps", type=int, default=10)
  ap.add_argument("--batch", type=int, default=1 << 20)
  ap.add_argument("--keys", type=int, default=10_000_000)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_bwd.py measures on a GPU"
  assert args.steps >= 40, "at least 40 timed calls"
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)

  keys_per_slot = args.keys // bench.SLOTS
  seg = entry.CombineAsSegment(bench.DIM, entry.RandomUniformInitializer(-0.05, 0.05),
                               entry.AdagradOptimizer(bench.LR, bench.INIT_ACC))
  table = MultiHashTable({"item": entry.HashTableConfigInstance(
      entry.TableConfig([seg], initial_capacity=int(args.keys * 1.05), init_seed=1), [bench.LR])}, device=dev)
  for s in range(1, bench.SLOTS + 1):
    for lo in range(0, keys_per_slot, 1 << 22):
      hi = min(keys_per_slot, lo + (1 << 22))
      ids = torch.arange(lo, hi, device=dev, dtype=torch.int64) | (s << 48)
      table.assign_add({"item": (ids, torch.zeros(ids.numel(), bench.DIM, device=dev))}, req_time=1, ids_unique=True)
  M = args.batch * bench.SLOTS
  fids = [torch.from_numpy(b).to(dev) for b in bench.make_batches(4, args.batch, keys_per_slot, seed=2)]
  gen = torch.Generator(device=dev)
  gen.manual_seed(5)
  pgrad = torch.randn(M, bench.DIM, device=dev, generator=gen)
  n_unique = int(torch.unique(fids[0]).numel())
  step = [0]

  def bwd():
    table.pool_backward("item", fids[step[0] % len(fids)], pgrad, None, "sum", req_time=1000 + step[0])
    step[0] += 1

  # 1. CUDA-event time per call
  for _ in range(args.warmup):
    bwd()
  torch.cuda.synchronize()
  ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
  for e0, e1 in ev:
    e0.record()
    bwd()
    e1.record()
  torch.cuda.synchronize()
  ms = np.array([e0.elapsed_time(e1) for e0, e1 in ev])

  # 2. per-kernel device time, in a run of its own
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.profile_steps):
      bwd()
    torch.cuda.synchronize()
  per_kernel = {}
  for evt in prof.key_averages():
    us = device_us(evt)
    if us <= 0:
      continue
    k = short_name(evt.key)
    n, t = per_kernel.get(k, (0, 0.0))
    per_kernel[k] = (n + evt.count, t + us)
  rows = sorted(((k, n / args.profile_steps, t / args.profile_steps) for k, (n, t) in per_kernel.items()),
                key=lambda r: -r[2])
  total = sum(r[2] for r in rows)

  res = {"what": "pool_backward, C2 batch", "M": M, "unique_fids_batch0": n_unique, "dim": bench.DIM,
         "steps": args.steps, "ms_median": float(np.median(ms)), "ms_min": float(ms.min()), "ms_max": float(ms.max()),
         "profile_steps": args.profile_steps, "kernel_us_per_call_total": round(total, 2),
         "kernels_us_per_call": {k: round(t, 2) for k, _, t in rows},
         "card": card()}
  print(json.dumps(res))
  print(f"{'kernel':60s} {'launches/call':>13s} {'us/call':>9s} {'share':>6s}")
  for k, n, t in rows:
    print(f"{k[:60]:60s} {n:13.1f} {t:9.2f} {t / total:6.1%}")
  table.close()


if __name__ == "__main__":
  main()
