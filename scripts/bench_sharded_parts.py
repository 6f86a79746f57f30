"""Times ShardedStep.step_parts (several features of one table in one sharded step) against what the same step costs
without it, world 1, direct exchange, in one process.  Each workload runs both sides on two identical tables, in
--rounds rounds that alternate the sides; in a round a side runs --warmup steps, then --steps steps back to back (no host
synchronisation between them, as a training loop enqueues them).  A step's device time is the interval between CUDA
events recorded before and after it on the current stream: launch gaps inside the step count, and so does any wait for
the host.  Reported per side: the median step time over all rounds and the host time to enqueue one step.  Afterwards
the forward outputs of the last step of both sides must be bit-identical.  The card's name and power limit are read in
the same run.

Workloads (table dim 16, Adagrad, Zipf(1.1) FIDs):
  c3     26 one-FID "sum" features, B = 65 536: step_parts into one [B, 416] tower tensor, against step() over the 26
         features' concatenated FIDs plus the torch copies of its [26 B, 16] output into the tower columns and of the
         tower gradient's columns back into [26 B, 16] rows.
  din    one "firstn" feature, L = 100, B = 4 096, rows of 1 .. L FIDs: step_parts into [B, L * 16], against step() with
         every occurrence as a one-FID "sum" row plus the torch scatter of the rows into [B, L, 16] and the gather of
         its gradient.
  c3bf16 c3 with a bfloat16 tower: the bf16 forms (bf16 outputs and gradients) against the fp32 forms plus the casts
         (the fp32 tower rounded to bf16, the bf16 gradient widened to fp32).

  python scripts/bench_sharded_parts.py [--workload c3 din c3bf16] [--steps 30] [--warmup 5] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monolith_b200 import MultiHashTable, PoolPart, entry  # noqa: E402
from monolith_b200.distributed_ps import ShardedStep  # noqa: E402

D = 16


def make_table(dev):
  seg = entry.CombineAsSegment(D, entry.RandomUniformInitializer(-0.05, 0.05),
                               entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
  cfg = entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=1 << 21, init_seed=1), [0.05])
  return MultiHashTable({"t": cfg}, device=dev)


def zipf(rng, n, feature):
  return (np.int64(feature) << 40) | (rng.zipf(1.1, n) % (1 << 25)).astype(np.int64)


def c3_batches(rng, B, n, dev):
  """[(fids of the 26 features [26, B], tower gradient [B, 416])]"""
  out = []
  for _ in range(n):
    f = np.stack([zipf(rng, B, i) for i in range(26)])
    g = torch.from_numpy((rng.standard_normal((B, 26 * D)) * 0.1).astype(np.float32)).to(dev)
    out.append((torch.from_numpy(f).to(dev), g))
  return out


def din_batches(rng, B, L, n, dev):
  """[(fids, offs [B + 1], gradient [B, L * 16])]"""
  out = []
  for _ in range(n):
    lens = rng.integers(1, L + 1, B)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    f = zipf(rng, int(offs[-1]), 0)
    g = torch.from_numpy((rng.standard_normal((B, L * D)) * 0.1).astype(np.float32)).to(dev)
    out.append((torch.from_numpy(f).to(dev), torch.from_numpy(offs).to(dev), g))
  return out


# ---- the two sides of each workload: step(i) runs batch i, returns the forward output ----
class C3Parts:
  def __init__(self, st, batches, bf16):
    self.st, self.batches, self.bf16 = st, batches, bf16

  def step(self, i):
    f, g = self.batches[i]
    B = f.shape[1]
    dt = torch.bfloat16 if self.bf16 else torch.float32
    tower = torch.empty(B, 26 * D, dtype=dt, device=f.device)
    gt = g.to(dt) if self.bf16 else g
    parts = [PoolPart("t", f[k], None, "sum", tower, k * D) for k in range(26)]
    self.st.step_parts(parts, [gt] * 26, 100 + i)
    return tower


class C3Flat:
  """step() over the concatenated FIDs; torch copies into and out of the tower columns."""

  def __init__(self, st, batches):
    self.st, self.batches = st, batches

  def step(self, i):
    f, g = self.batches[i]
    B = f.shape[1]
    out = torch.empty(26 * B, D, device=f.device)
    tower = torch.empty(B, 26 * D, device=f.device)

    def grad():
      tower.view(B, 26, D).copy_(out.view(26, B, D).transpose(0, 1))
      return g.view(B, 26, D).transpose(0, 1).reshape(26 * B, D)
    self.st.step(f.reshape(-1), grad, out, 100 + i)
    return tower


class C3Cast:
  """The fp32 forms plus the casts of a bf16 tower: the output rounded to bf16, the bf16 gradient widened."""

  def __init__(self, st, batches):
    self.st, self.batches = st, batches

  def step(self, i):
    f, g = self.batches[i]
    B = f.shape[1]
    tower = torch.empty(B, 26 * D, device=f.device)
    g16 = g.to(torch.bfloat16)
    parts = [PoolPart("t", f[k], None, "sum", tower, k * D) for k in range(26)]
    box = {}

    def grad():
      box["out"] = tower.to(torch.bfloat16)
      return [g16.float()] * 26
    self.st.step_parts(parts, grad, 100 + i)
    return box["out"]


class DinParts:
  def __init__(self, st, batches, L):
    self.st, self.batches, self.L = st, batches, L

  def step(self, i):
    f, offs, g = self.batches[i]
    B = offs.numel() - 1
    seq = torch.empty(B, self.L * D, device=f.device)
    self.st.step_parts([PoolPart("t", f, offs, "firstn", seq, 0, self.L)], [g], 100 + i)
    return seq


class DinFlat:
  """Every occurrence a one-FID SUM row; torch scatter into [B, L, 16] and gather of its gradient."""

  def __init__(self, st, batches, L):
    self.st, self.batches, self.L = st, batches, L
    self.idx = []
    for f, offs, _ in batches:   # row and position of every occurrence (rows have at most L FIDs)
      lens = offs[1:] - offs[:-1]
      row = torch.repeat_interleave(torch.arange(lens.numel(), device=f.device), lens)
      pos = torch.arange(f.numel(), device=f.device) - offs[:-1].long()[row]
      self.idx.append((row, pos))

  def step(self, i):
    f, offs, g = self.batches[i]
    B, L = offs.numel() - 1, self.L
    row, pos = self.idx[i]
    out = torch.empty(f.numel(), D, device=f.device)
    seq = torch.zeros(B, L, D, device=f.device)

    def grad():
      seq[row, pos] = out
      return g.view(B, L, D)[row, pos]
    self.st.step(f, grad, out, 100 + i)
    return seq.view(B, L * D)


def timed(a, b, n_batches, steps, warmup, rounds):
  """Rounds alternate the sides; in a round a side runs `warmup` steps, then `steps` steps back to back without a host
  synchronisation between them, with a CUDA event before and after each step.  -> (per side: the median per-step device
  time over all rounds, the median host time to enqueue one step), and the last outputs of both sides (the same batch
  on tables in the same state)."""
  res = {}
  out = {}
  for _ in range(rounds):
    for side in (a, b):
      for s in range(warmup):
        side.step(s % n_batches)
      torch.cuda.synchronize()
      ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
      t0 = time.perf_counter()
      for s in range(steps):
        ev[s][0].record()
        o = side.step((warmup + s) % n_batches)
        ev[s][1].record()
      host = (time.perf_counter() - t0) / steps
      torch.cuda.synchronize()
      dev_ms, host_ms = res.setdefault(id(side), ([], []))
      dev_ms += [e0.elapsed_time(e1) for e0, e1 in ev]
      host_ms.append(1e3 * host)
      out[id(side)] = o
  (da, ha), (db, hb) = res[id(a)], res[id(b)]
  return (float(np.median(da)), float(np.median(ha)), float(np.median(db)), float(np.median(hb)), out[id(a)],
          out[id(b)])


def same_bits(x, y):
  if x.dtype != y.dtype or x.shape != y.shape:
    return False
  v = torch.int16 if x.dtype == torch.bfloat16 else torch.int32
  return bool(torch.equal(x.contiguous().view(v), y.contiguous().view(v)))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--workload", nargs="+", default=["c3", "din", "c3bf16"])
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--rounds", type=int, default=3)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_sharded_parts needs a GPU")
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  rng = np.random.default_rng(0)
  for w in args.workload:
    ta, tb = make_table(dev), make_table(dev)
    sa, sb = ShardedStep(ta, "t", D, 1, 0, dev, exchange="direct"), ShardedStep(tb, "t", D, 1, 0, dev, exchange="direct")
    if w in ("c3", "c3bf16"):
      B = 65536
      data = c3_batches(rng, B, 4, dev)
      if w == "c3":
        a, b, what = C3Parts(sa, data, False), C3Flat(sb, data), ("step_parts", "step + torch copies")
      else:
        a, b, what = C3Parts(sa, data, True), C3Cast(sb, data), ("step_parts bf16", "step_parts fp32 + casts")
    elif w == "din":
      B, L = 4096, 100
      data = din_batches(rng, B, L, 4, dev)
      a, b, what = DinParts(sa, data, L), DinFlat(sb, data, L), ("step_parts firstn", "step + torch scatter/gather")
    else:
      raise SystemExit(f"unknown workload {w}")
    ms_a, host_a, ms_b, host_b, oa, ob = timed(a, b, len(data), args.steps, args.warmup, args.rounds)
    print(json.dumps({"workload": w, "batch": B, "a": what[0], "b": what[1], "a_ms": round(ms_a, 4),
                      "b_ms": round(ms_b, 4), "b_over_a": round(ms_b / ms_a, 3), "a_host_enqueue_ms": round(host_a, 4),
                      "b_host_enqueue_ms": round(host_b, 4), "same_output_bits": same_bits(oa, ob),
                      "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "gpu": props.name,
                      "power_limit": power}), flush=True)
    torch.cuda.synchronize()
    sa.close_direct()
    sb.close_direct()
    ta.close()
    tb.close()


if __name__ == "__main__":
  main()
