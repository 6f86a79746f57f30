"""Times a C3-like multi-table step two ways in one process: the parts calls (lookup_pool_parts +
pool_backward_parts) against today's entry points (one lookup_pool per feature, then one pool_backward per table over
the table's features concatenated, the copy a caller needs to give shared FIDs one step).  T = 4 tables of dims 16,
16, 32 and 64, 26 one-FID features spread over them, Zipf-skewed FIDs.  The two ways run on two identical tables,
alternating, timed with CUDA events; afterwards the pooled outputs and every touched entry must be bit-identical.

  python scripts/bench_parts.py [--batch 65536 4096] [--steps 50] [--warmup 10]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monolith_b200 import MultiHashTable, PoolPart, entry  # noqa: E402

DIMS = {"t0": 16, "t1": 16, "t2": 32, "t3": 64}
N_FEATURES = 26
VOCAB = 1 << 20


def make_table(dev):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=VOCAB, init_seed=1), [0.05])
  return MultiHashTable({n: cfg(d) for n, d in DIMS.items()}, device=dev)


def batches(B, n, dev, seed):
  rng = np.random.default_rng(seed)
  names = list(DIMS)
  out = []
  for _ in range(n):
    feats = []
    for f in range(N_FEATURES):
      slot = names[f % len(names)]
      fids = (np.int64(f % len(names) + 1) << 48) | (rng.zipf(1.05, B) % VOCAB).astype(np.int64)
      grad = torch.from_numpy(rng.standard_normal((B, DIMS[slot])).astype(np.float32)).to(dev)
      feats.append((slot, torch.from_numpy(fids).to(dev), grad))
    out.append(feats)
  return out


def step_parts(t, feats, ts):
  outs = t.lookup_pool_parts([PoolPart(s, f) for s, f, _ in feats])
  t.pool_backward_parts([PoolPart(s, f, rows=g) for s, f, g in feats], req_time=ts)
  return outs


def step_loop(t, feats, ts):
  outs = [t.lookup_pool(s, f) for s, f, _ in feats]
  for slot in DIMS:
    mine = [(f, g) for s, f, g in feats if s == slot]
    t.pool_backward(slot, torch.cat([f for f, _ in mine]), torch.cat([g for _, g in mine]), req_time=ts)
  return outs


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, nargs="+", default=[65536, 4096])
  ap.add_argument("--steps", type=int, default=50)
  ap.add_argument("--warmup", type=int, default=10)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_parts.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    import subprocess
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for B in args.batch:
    ta, tb = make_table(dev), make_table(dev)
    data = batches(B, 4, dev, seed=B)
    lib = ta._lib
    times = {"parts": [], "loop": []}
    launches = {}
    ts = 1
    for it in range(args.warmup + args.steps):
      feats = data[it % len(data)]
      for name, t, fn in (("parts", ta, step_parts), ("loop", tb, step_loop)) if it % 2 == 0 else \
          (("loop", tb, step_loop), ("parts", ta, step_parts)):
        torch.cuda.synchronize()
        n0 = lib.mono_kernel_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        outs = fn(t, feats, ts)
        e1.record()
        torch.cuda.synchronize()
        launches[name] = lib.mono_kernel_launch_count() - n0
        if it >= args.warmup:
          times[name].append(e0.elapsed_time(e1))
        if name == "parts":
          out_parts = outs
        else:
          out_loop = outs
      ts += 1
      same_fwd = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(out_parts, out_loop))
      assert same_fwd, "forward outputs differ"
    same_tab = True
    for slot in DIMS:
      keys = torch.unique(torch.cat([f for s, f, _ in data[0] if s == slot]))
      ea, eb = ta.lookup_entry(slot, keys)["raw"], tb.lookup_entry(slot, keys)["raw"]
      same_tab &= torch.equal(ea.view(torch.int32), eb.view(torch.int32)) and ta.size(slot) == tb.size(slot)
    assert same_tab, "table entries differ"
    res = {"batch": B, "features": N_FEATURES, "tables": len(DIMS), "steps": args.steps,
           "ms_per_step_parts": float(np.median(times["parts"])), "ms_per_step_loop": float(np.median(times["loop"])),
           "ms_spread_parts": [float(np.min(times["parts"])), float(np.max(times["parts"]))],
           "ms_spread_loop": [float(np.min(times["loop"])), float(np.max(times["loop"]))],
           "launches_per_step_parts": launches["parts"], "launches_per_step_loop": launches["loop"],
           "same_bits": True, "gpu": props.name, "power_limit": power}
    print(json.dumps(res))
    ta.close()
    tb.close()


if __name__ == "__main__":
  main()
