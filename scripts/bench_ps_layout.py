"""Times PartitionedHashTablePS (the parameter-server mode with the fused layout) with every server's table on one GPU,
per phase, with and without transfer_float16:

  shard        sharding_sparse_fids(version=5)             lookup   the servers' raw_lookup calls (fp16 rows with f16)
  layout       fused_embedding_to_layout (f16in kernels with f16)
  layout_grad  fused_embedding_to_layout_grad               round    the fp16 rounding of the layout gradient (f16)
  apply        the servers' raw_apply_gradients calls (Adagrad), each server's widening of fp16 gradients included

Device time per phase: CUDA events around each call of the phase, summed over the step; the median over --steps after
--warmup.  The events bracket the calls as the step issues them, so launch gaps inside a phase count.  The card's name
and power limit are read in the same run.

Workloads (one feature per table, one FID per sample, all pooled SUM into one CONCAT layout tensor [B, sum of dims]):
c3, Criteo-shaped: 26 tables of dim 16, per-table Zipf(1.1) FIDs; c2, MovieLens-shaped: 2 tables (uid, movie) of dim
32, Zipf(1.05) over 5 M ranks each.

  python scripts/bench_ps_layout.py [--workload c3 c2] [--num-ps 1 4] [--batch 65536] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from monolith_b200 import MultiHashTable, distribution_ops as dops, entry, multi_hash_table_ops  # noqa: E402
from monolith_b200 import distributed_ps  # noqa: E402
from monolith_b200.distribution_ops import SliceTask  # noqa: E402


def workload(name, B, rng):
  """feature -> (dim, fids)"""
  if name == "c3":
    return {f"slot_{i:02d}": (16, (rng.zipf(1.1, B) % (1 << 25)).astype(np.int64) + (i << 40)) for i in range(26)}
  return {s: (32, (rng.zipf(1.05, B) % 5_000_000).astype(np.int64) + (i << 40)) for i, s in enumerate(("movie", "uid"))}


def configs(shape):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=1 << 16, init_seed=1), [0.05])
  return {s: cfg(d) for s, (d, _) in shape.items()}


class PhaseTimer:
  """Wraps the calls of each phase with CUDA events; times[phase] = the step's sum of event intervals."""

  PHASES = (("shard", dops, "sharding_sparse_fids"), ("lookup", multi_hash_table_ops.MultiHashTable, "raw_lookup"),
            ("layout", dops, "fused_embedding_to_layout"), ("layout_grad", dops, "fused_embedding_to_layout_grad"),
            ("round", dops, "round_to_f16"), ("apply", multi_hash_table_ops.MultiHashTable, "raw_apply_gradients"))

  def __init__(self):
    self.marks = []
    self.saved = []
    for phase, owner, name in self.PHASES:
      fn = getattr(owner, name)
      self.saved.append((owner, name, fn))
      setattr(owner, name, self._wrap(phase, fn))

  def _wrap(self, phase, fn):
    def run(*a, **k):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      out = fn(*a, **k)
      e1.record()
      self.marks.append((phase, e0, e1))
      return out
    return run

  def step(self):
    torch.cuda.synchronize()
    t = {}
    for phase, e0, e1 in self.marks:
      t[phase] = t.get(phase, 0.0) + e0.elapsed_time(e1)
    self.marks = []
    return t

  def close(self):
    for owner, name, fn in self.saved:
      setattr(owner, name, fn)


def run(name, S, B, steps, warmup, f16, dev):
  rng = np.random.default_rng(0)
  shape = workload(name, B, rng)
  names = sorted(shape)
  dims = {n: shape[n][0] for n in names}
  width = sum(dims.values())
  tasks, col = [], 0
  for i, n in enumerate(names):
    tasks.append(SliceTask(i, 0, dims[n], 0, 0, 0, width, col, 0))
    col += dims[n]
  cfg = configs(shape)
  pht = distributed_ps.PartitionedHashTablePS(S, cfg, lambda i, c: MultiHashTable(configs(shape), device=dev),
                                              {n: n for n in names}, dims, tasks, [(width,)],
                                              transfer_float16=f16)
  splits = torch.arange(B + 1, dtype=torch.int64, device=dev)
  timer = PhaseTimer()
  times = {}
  try:
    for step in range(warmup + steps):
      fresh = workload(name, B, rng)
      feats = {n: (torch.from_numpy(fresh[n][1]).to(dev), splits) for n in names}
      torch.cuda.synchronize()
      timer.marks = []
      (out,), ctx = pht.lookup(feats)
      g = torch.randn_like(out) * 1e-3
      pht.apply_gradients(ctx, [g], global_step=step, req_time=step)
      t = timer.step()
      if step >= warmup:
        for k, v in t.items():
          times.setdefault(k, []).append(v)
  finally:
    timer.close()
  med = {k: round(float(np.median(v)), 4) for k, v in times.items()}
  med["total"] = round(sum(med.values()), 4)
  return med


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--workload", nargs="+", default=["c3", "c2"])
  ap.add_argument("--num-ps", nargs="+", type=int, default=[1, 4])
  ap.add_argument("--batch", type=int, default=65536)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=5)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_ps_layout needs a GPU")
  dev = torch.device("cuda", 0)
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip().splitlines()
  card = q[0] if q else torch.cuda.get_device_name(0)
  rows = []
  for name in a.workload:
    for S in a.num_ps:
      for f16 in (False, True):
        r = run(name, S, a.batch, a.steps, a.warmup, f16, dev)
        rows.append({"workload": name, "num_ps": S, "transfer_float16": f16, "ms": r})
        print(json.dumps(rows[-1]), flush=True)
  print(json.dumps({"card": card, "batch": a.batch, "steps": a.steps, "rows": rows}))


if __name__ == "__main__":
  main()
