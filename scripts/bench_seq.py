"""Times a DIN-shaped sparse step two ways in one process: FIRSTN parts in lookup_pool_parts + pool_backward_parts,
against the formulation available without them (every sequence occurrence as a one-FID SUM part, a torch scatter of
the looked-up rows into [B, L, dim], and a torch gather of the per-occurrence gradients with zero rows past L).

The step: two sequence features (clicked items on table "item", dim 32, and their categories on "cate", dim 16) with
lengths drawn so that some rows are longer than L = 100; the target item and category as one-FID features on the
same two tables; six other one-FID features on table "ctx" (dim 16).  FIDs are Zipf-skewed.  The two ways run on two
identical tables, alternating, timed with CUDA events; afterwards the outputs and every touched entry must be
bit-identical.

  python scripts/bench_seq.py [--batch 4096 1024] [--steps 40] [--warmup 10]
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

DIMS = {"cate": 16, "ctx": 16, "item": 32}
L = 100
N_CTX = 6
VOCAB = 1 << 20


def make_table(dev):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=VOCAB, init_seed=1), [0.05])
  return MultiHashTable({n: cfg(d) for n, d in DIMS.items()}, device=dev)


def zipf(rng, n, slot):
  return (np.int64(slot) << 48) | (rng.zipf(1.05, n) % VOCAB).astype(np.int64)


def batches(B, n, dev, seed):
  """Per batch: (sequence features, one-FID features).  A sequence feature is (slot, fids, offs, grad [B, L*dim]);
  a one-FID feature (slot, fids, grad [B, dim])."""
  rng = np.random.default_rng(seed)
  out = []
  for _ in range(n):
    lens = np.minimum(rng.geometric(1 / 40, B), 160)   # mean ~40, ~8% of the rows longer than L
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    M = int(offs[-1])
    seq = []
    for slot, s in (("item", 1), ("cate", 2)):
      f = zipf(rng, M, s)
      g = rng.standard_normal((B, L * DIMS[slot])).astype(np.float32)
      seq.append((slot, torch.from_numpy(f).to(dev), torch.from_numpy(offs).to(dev), torch.from_numpy(g).to(dev)))
    one = []
    for slot, s in [("item", 1), ("cate", 2)] + [("ctx", 3 + i) for i in range(N_CTX)]:
      g = rng.standard_normal((B, DIMS[slot])).astype(np.float32)
      one.append((slot, torch.from_numpy(zipf(rng, B, s)).to(dev), torch.from_numpy(g).to(dev)))
    out.append((seq, one))
  return out


def step_seq(t, batch, ts):
  seq, one = batch
  outs = t.lookup_pool_parts([PoolPart(s, f, o, "firstn", max_seq_len=L) for s, f, o, _ in seq] +
                             [PoolPart(s, f) for s, f, _ in one])
  t.pool_backward_parts([PoolPart(s, f, o, "firstn", g, max_seq_len=L) for s, f, o, g in seq] +
                        [PoolPart(s, f, rows=g) for s, f, g in one], req_time=ts)
  return outs


def _positions(offs, M):
  """-> (row, position) of every occurrence, as int64 device tensors."""
  lens = offs[1:] - offs[:-1]
  row = torch.repeat_interleave(torch.arange(lens.numel(), device=offs.device), lens.long())
  pos = torch.arange(M, device=offs.device) - offs[:-1].long()[row]
  return row, pos


def step_sum(t, batch, ts):
  """The same step through one-FID SUM parts and torch: occurrences looked up into [M, dim], scattered into
  [B, L, dim]; per-occurrence gradients gathered from [B, L, dim] with zero rows for positions >= L."""
  seq, one = batch
  occ = t.lookup_pool_parts([PoolPart(s, f) for s, f, _, _ in seq] + [PoolPart(s, f) for s, f, _ in one])
  outs = []
  terms = []
  for (slot, f, o, g), rows in zip(seq, occ):
    D = DIMS[slot]
    B = o.numel() - 1
    row, pos = _positions(o, f.numel())
    keep = pos < L
    out = torch.zeros(B, L, D, device=f.device)
    out[row[keep], pos[keep]] = rows[keep]
    outs.append(out.view(B, L * D))
    gv = g.view(B, L, D)
    term = torch.zeros(f.numel(), D, device=f.device)
    term[keep] = gv[row[keep], pos[keep]]
    terms.append(term)
  outs += occ[len(seq):]
  t.pool_backward_parts([PoolPart(s, f, rows=x) for (s, f, _, _), x in zip(seq, terms)] +
                        [PoolPart(s, f, rows=g) for s, f, g in one], req_time=ts)
  return outs


def alg_bytes(batch):
  """Bytes the step must move at least, from shapes: FIDs, offsets, one bucket (64 B) and one row read per
  occurrence looked up, the outputs written, the gradients read, and one row + state read and written per
  occurrence on the backward (an upper bound on distinct FIDs)."""
  seq, one = batch
  n = 0
  for slot, f, o, g in seq:
    D = DIMS[slot]
    M = f.numel()
    n += 8 * M + 4 * o.numel() + (64 + 4 * D) * M + 4 * g.numel() + 4 * g.numel() + 4 * M * 4 * D
  for slot, f, g in one:
    D = DIMS[slot]
    n += 8 * f.numel() + (64 + 4 * D) * f.numel() + 4 * g.numel() * 2 + 4 * f.numel() * 4 * D
  return n


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, nargs="+", default=[4096, 1024])
  ap.add_argument("--steps", type=int, default=40)
  ap.add_argument("--warmup", type=int, default=10)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_seq.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for B in args.batch:
    ta, tb = make_table(dev), make_table(dev)
    data = batches(B, 4, dev, seed=B)
    lib = ta._lib
    times = {"firstn": [], "sum": []}
    launches = {}
    ts = 1
    for it in range(args.warmup + args.steps):
      batch = data[it % len(data)]
      order = (("firstn", ta, step_seq), ("sum", tb, step_sum))
      for name, t, fn in order if it % 2 == 0 else order[::-1]:
        torch.cuda.synchronize()
        n0 = lib.mono_kernel_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        outs = fn(t, batch, ts)
        e1.record()
        torch.cuda.synchronize()
        launches[name] = lib.mono_kernel_launch_count() - n0
        if it >= args.warmup:
          times[name].append(e0.elapsed_time(e1))
        if name == "firstn":
          out_seq = outs
        else:
          out_sum = outs
      ts += 1
      assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(out_seq, out_sum)), \
          "forward outputs differ"
    same_tab = True
    for slot in DIMS:
      fs = [f for s, f, _, _ in data[0][0] if s == slot] + [f for s, f, _ in data[0][1] if s == slot]
      keys = torch.unique(torch.cat(fs))
      ea, eb = ta.lookup_entry(slot, keys)["raw"], tb.lookup_entry(slot, keys)["raw"]
      same_tab &= torch.equal(ea.view(torch.int32), eb.view(torch.int32)) and ta.size(slot) == tb.size(slot)
    assert same_tab, "table entries differ"
    M = data[0][0][0][1].numel()
    res = {"batch": B, "max_seq_len": L, "seq_occurrences": M,
           "rows_over_L": int((data[0][0][0][2].diff() > L).sum().item()), "steps": args.steps,
           "ms_per_step_firstn": float(np.median(times["firstn"])), "ms_per_step_sum": float(np.median(times["sum"])),
           "ms_spread_firstn": [float(np.min(times["firstn"])), float(np.max(times["firstn"]))],
           "ms_spread_sum": [float(np.min(times["sum"])), float(np.max(times["sum"]))],
           "mono_launches_per_step_firstn": launches["firstn"], "mono_launches_per_step_sum": launches["sum"],
           "alg_bytes_per_step": alg_bytes(data[0]), "same_bits": True, "gpu": props.name, "power_limit": power}
    print(json.dumps(res))
    ta.close()
    tb.close()


if __name__ == "__main__":
  main()
