"""Times a bf16 tower's embedding step two ways in one process, on twin tables, alternating, with CUDA events:

  (A) today: the fp32 parts calls, a .to(torch.bfloat16) of every pooled output, and the tower's bf16 gradients
      .float()-ed before pool_backward_parts;
  (B) the bf16 parts calls (lookup_pool_parts(..., dtype=torch.bfloat16), pool_backward_parts on bf16 rows).

Also timed: the forward alone and the backward alone, fp32 call against bf16 call with no casts (the backward's fp32
call gets gradients widened beforehand), which separates the byte saving from the removed torch passes.

Workload: scripts/bench_parts.py's 4 tables (dims 16, 16, 32, 64) and 26 features, every third one CSR SUM (1-7
FIDs per row) and the rest one FID per row, plus scripts/bench_seq.py's two FIRSTN features (L = 100, on the dim-32
and a dim-16 table).  Afterwards (A)'s cast outputs must equal (B)'s bit for bit, and so must every touched entry.

  python scripts/bench_bf16_parts.py [--batch 65536 4096] [--steps 40] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monolith_b200 import MultiHashTable, PoolPart, entry  # noqa: E402

DIMS = {"t0": 16, "t1": 16, "t2": 32, "t3": 64}
N_FEATURES = 26
SEQ = (("t2", 32), ("t0", 16))
L = 100
VOCAB = 1 << 20
BF = torch.bfloat16


def make_table(dev):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=VOCAB, init_seed=1), [0.05])
  return MultiHashTable({n: cfg(d) for n, d in DIMS.items()}, device=dev)


def batches(B, n, dev, seed):
  """Per batch: features (slot, fids, offs or None, pooling, max_seq_len, bf16 gradient rows)."""
  rng = np.random.default_rng(seed)
  names = list(DIMS)
  out = []
  for _ in range(n):
    feats = []
    for f in range(N_FEATURES):
      slot = names[f % len(names)]
      offs = None
      n_fids = B
      if f % 3 == 2:
        lens = rng.integers(1, 8, B)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        n_fids = int(offs[-1])
      fids = (np.int64(f % len(names) + 1) << 48) | (rng.zipf(1.05, n_fids) % VOCAB).astype(np.int64)
      g = torch.randn(B, DIMS[slot], device=dev).to(BF)
      feats.append((slot, torch.from_numpy(fids).to(dev), None if offs is None else torch.from_numpy(offs).to(dev),
                    "sum", 0, g))
    lens = np.minimum(rng.geometric(1 / 40, B), 160)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    for slot, D in SEQ:
      fids = (np.int64(names.index(slot) + 1) << 48) | (rng.zipf(1.05, int(offs[-1])) % VOCAB).astype(np.int64)
      g = torch.randn(B, L * D, device=dev).to(BF)
      feats.append((slot, torch.from_numpy(fids).to(dev), torch.from_numpy(offs).to(dev), "firstn", L, g))
    out.append(feats)
  return out


def fwd_parts(feats):
  return [PoolPart(s, f, o, p, max_seq_len=ln) for s, f, o, p, ln, _ in feats]


def bwd_parts(feats, rows):
  return [PoolPart(s, f, o, p, r, max_seq_len=ln) for (s, f, o, p, ln, _), r in zip(feats, rows)]


def step_a(t, feats, ts):
  outs = [o.to(BF) for o in t.lookup_pool_parts(fwd_parts(feats))]
  t.pool_backward_parts(bwd_parts(feats, [g.float() for *_, g in feats]), req_time=ts)
  return outs


def step_b(t, feats, ts):
  outs = t.lookup_pool_parts(fwd_parts(feats), dtype=BF)
  t.pool_backward_parts(bwd_parts(feats, [g for *_, g in feats]), req_time=ts)
  return outs


def alg_bytes(feats, row_bytes):
  """Bytes the step must move at least, from shapes: FIDs and offsets, one bucket (64 B) and one fp32 table row
  per occurrence looked up, the pooled rows written and the gradient rows read (row_bytes per element), and one
  table row + Adagrad state read and written per occurrence on the backward (an upper bound on distinct FIDs)."""
  n = 0
  for s, f, o, p, ln, g in feats:
    D, M = DIMS[s], f.numel()
    looked = min(M, g.shape[0] * ln) if p == "firstn" else M
    n += 8 * M + (0 if o is None else 4 * o.numel()) + (64 + 4 * D) * looked + 2 * row_bytes * g.numel()
    n += 4 * M * 4 * D
  return n


def timed(fn):
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  out = fn()
  e1.record()
  torch.cuda.synchronize()
  return out, e0.elapsed_time(e1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, nargs="+", default=[65536, 4096])
  ap.add_argument("--steps", type=int, default=40)
  ap.add_argument("--warmup", type=int, default=10)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_bf16_parts.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for B in args.batch:
    ta, tb = make_table(dev), make_table(dev)
    data = batches(B, 2, dev, seed=B)
    wide = [[g.float() for *_, g in feats] for feats in data]   # the fp32-only backward's pre-widened gradients
    lib = ta._lib
    keys = ("step_a", "step_b", "fwd_fp32", "fwd_bf16", "bwd_fp32", "bwd_bf16")
    times = {k: [] for k in keys}
    launches = {}
    ts = 1
    same_fwd = True
    for it in range(args.warmup + args.steps):
      feats = data[it % len(data)]
      w = wide[it % len(data)]
      work = {
          "step_a": lambda: step_a(ta, feats, ts),
          "step_b": lambda: step_b(tb, feats, ts),
          "fwd_fp32": lambda: ta.lookup_pool_parts(fwd_parts(feats)),
          "fwd_bf16": lambda: tb.lookup_pool_parts(fwd_parts(feats), dtype=BF),
          "bwd_fp32": lambda: ta.pool_backward_parts(bwd_parts(feats, w), req_time=ts + 1),
          "bwd_bf16": lambda: tb.pool_backward_parts(bwd_parts(feats, [g for *_, g in feats]), req_time=ts + 1),
      }
      order = keys if it % 2 == 0 else tuple(reversed(keys))
      outs = {}
      for k in order:
        n0 = lib.mono_kernel_launch_count()
        outs[k], ms = timed(work[k])
        launches[k] = lib.mono_kernel_launch_count() - n0
        if it >= args.warmup:
          times[k].append(ms)
      same_fwd &= all(torch.equal(a.view(torch.int16), b.view(torch.int16))
                      for a, b in zip(outs["step_a"], outs["step_b"]))
      ts += 2
      del outs
    same_tab = True
    for slot in DIMS:
      k = torch.unique(torch.cat([f for feats in data for s, f, *_ in feats if s == slot]))
      ea, eb = ta.lookup_entry(slot, k)["raw"], tb.lookup_entry(slot, k)["raw"]
      same_tab &= torch.equal(ea.view(torch.int32), eb.view(torch.int32)) and ta.size(slot) == tb.size(slot)
    res = {"batch": B, "features": N_FEATURES + len(SEQ), "tables": len(DIMS), "steps": args.steps,
           "same_bits": bool(same_fwd and same_tab), "gpu": props.name, "power_limit": power,
           "alg_bytes_per_step_fp32_rows": alg_bytes(data[0], 4), "alg_bytes_per_step_bf16_rows": alg_bytes(data[0], 2)}
    for k in keys:
      res[f"ms_{k}"] = float(np.median(times[k]))
      res[f"ms_spread_{k}"] = [float(np.min(times[k])), float(np.max(times[k]))]
      res[f"launches_{k}"] = launches[k]
    print(json.dumps(res), flush=True)
    ta.close()
    tb.close()
    del data, wide
    torch.cuda.empty_cache()


if __name__ == "__main__":
  main()
