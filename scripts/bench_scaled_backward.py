"""Times the clip scale in the one-table fused backward and in the ReduceSum gradient, three variants each,
alternated in one process, device time (a sleep kernel queued first keeps the GPU busy while the host enqueues, so
the CUDA events bracket the device work), median and [min, max] over the timed calls:

  unscaled : the call without a scale, on rows pre-multiplied outside the timing (the lower bound);
  scaled   : the call with grad_scale= (the multiply where the kernels load the rows);
  torch    : `g * scale` in torch, then the unscaled call (what a user without grad_scale= writes).

  1 pool_backward: C2's backward (bench.py): one table, dim 32, Adagrad, batch B samples x 2 slots, one FID per
    pooled row, FID ranks Zipf(1.05) over 5 M ids per slot; the table holds what the warm-up batches inserted.
    The unscaled and scaled tables must end bit-identical.
  2 reduce_sum_gradient: the 26 features of scripts/bench_reduce_split.py (dims 16/16/32/64, every third multi-hot)
    in one fused_reduce_and_split_gpu_grad call, the kernel reduce_sum_gradient runs; scaled and pre-multiplied
    outputs must be bit-identical.

  python scripts/bench_scaled_backward.py [--c2-batch 1048576] [--rs-batch 65536 4096] [--steps 30] [--warmup 5]
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
from bench_reduce_split import DIMS as RS_DIMS, features  # noqa: E402
from monolith_b200 import MultiHashTable, distribution_ops as dops, entry  # noqa: E402

DIM, SLOTS, KEYS_PER_SLOT, ZIPF_S = 32, 2, 5_000_000, 1.05
SLEEP_CYCLES = 40_000_000   # ~20 ms at 1.98 GHz: longer than any host enqueue timed here
SCALE = 0.3


def timed(fn, times, key):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda._sleep(SLEEP_CYCLES)
  e0.record()
  out = fn()
  e1.record()
  torch.cuda.synchronize()
  if times is not None:
    times.setdefault(key, []).append(e0.elapsed_time(e1))
  return out


def summary(xs):
  return {"median": float(np.median(xs)), "spread": [float(np.min(xs)), float(np.max(xs))]}


def c2_table(dev):
  seg = entry.CombineAsSegment(DIM, entry.RandomUniformInitializer(-0.05, 0.05),
                               entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
  cfg = entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=1 << 22, init_seed=1), [0.05])
  return MultiHashTable({"t": cfg}, device=dev)


def c2_batches(B, n, dev):
  rng = np.random.default_rng(B)
  ranks = np.arange(1, KEYS_PER_SLOT + 1, dtype=np.float64)
  cdf = np.cumsum(ranks ** -ZIPF_S)
  cdf /= cdf[-1]
  out = []
  for _ in range(n):
    fids = np.empty(B * SLOTS, np.int64)
    for s in range(SLOTS):
      r = np.searchsorted(cdf, rng.random(B))
      fids[s::SLOTS] = (np.int64(s + 1) << 48) | r.astype(np.int64)
    g = torch.randn(B * SLOTS, DIM, device=dev)
    out.append((torch.from_numpy(fids).to(dev), g))
  return out


def bench_c2(B, steps, warmup, dev):
  data = c2_batches(B, 4, dev)
  sc = torch.tensor([SCALE], device=dev)
  tabs = {k: c2_table(dev) for k in ("unscaled", "scaled", "torch")}
  pre = [g * sc for _, g in data]
  times = {}
  for it in range(warmup + steps):
    fids, g = data[it % len(data)]
    p = pre[it % len(data)]
    ts = 1 + it
    runs = [("unscaled", lambda: tabs["unscaled"].pool_backward("t", fids, p, req_time=ts)),
            ("scaled", lambda: tabs["scaled"].pool_backward("t", fids, g, req_time=ts, grad_scale=sc)),
            ("torch", lambda: tabs["torch"].pool_backward("t", fids, g * sc, req_time=ts))]
    for key, fn in (runs if it % 2 == 0 else runs[::-1]):
      torch.cuda.synchronize()
      timed(fn, times if it >= warmup else None, key)
  keys = torch.unique(torch.cat([f for f, _ in data]))
  ea, eb = tabs["unscaled"].lookup_entry("t", keys)["raw"], tabs["scaled"].lookup_entry("t", keys)["raw"]
  same = torch.equal(ea.view(torch.int32), eb.view(torch.int32))
  res = {"leg": "pool_backward C2", "batch": B, "occurrences": B * SLOTS, "dim": DIM, "keys": tabs["scaled"].size("t"),
         "steps": steps, **{f"ms_{k}": summary(v) for k, v in times.items()},
         "grad_bytes": B * SLOTS * DIM * 4, "scaled_same_bits": bool(same)}
  for t in tabs.values():
    t.close()
  return res


def bench_rs(B, steps, warmup, dev):
  feats = features(B, dev, seed=B)
  dims = [RS_DIMS[s] for s, _, _ in feats]
  splits = [sp for _, _, sp in feats]
  embs = [torch.empty(f.numel(), d, device=dev) for (_, f, _), d in zip(feats, dims)]
  sdims = [[d] for d in dims]
  grads = [torch.randn(B, d, device=dev) for d in dims]
  sc = torch.tensor([SCALE], device=dev)
  pre = [g * sc for g in grads]
  outs = {}
  runs = [("unscaled", lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, pre, sdims)),
          ("scaled", lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, grads, sdims, grad_scale=sc)),
          ("torch", lambda: dops.fused_reduce_and_split_gpu_grad(splits, embs, [g * sc for g in grads], sdims))]
  times = {}
  for it in range(warmup + steps):
    for key, fn in (runs if it % 2 == 0 else runs[::-1]):
      torch.cuda.synchronize()
      outs[key] = timed(fn, times if it >= warmup else None, key)
  same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(outs["unscaled"], outs["scaled"]))
  n_occ = sum(f.numel() for _, f, _ in feats)
  return {"leg": "reduce_sum_gradient", "batch": B, "features": len(feats), "occurrences": int(n_occ), "steps": steps,
          **{f"ms_{k}": summary(v) for k, v in times.items()},
          "bytes": sum(4 * d * (f.numel() + B) for (_, f, _), d in zip(feats, dims)) + 4 * (B + 1),
          "scaled_same_bits": bool(same)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--c2-batch", type=int, nargs="+", default=[1 << 20])
  ap.add_argument("--rs-batch", type=int, nargs="+", default=[65536, 4096])
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_scaled_backward.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for B in args.c2_batch:
    print(json.dumps({**bench_c2(B, args.steps, args.warmup, dev), "gpu": props.name, "power_limit": power}))
  for B in args.rs_batch:
    print(json.dumps({**bench_rs(B, args.steps, args.warmup, dev), "gpu": props.name, "power_limit": power}))


if __name__ == "__main__":
  main()
