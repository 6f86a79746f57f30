"""Times a bf16 tower's step on the fused-layout path two ways in one process, on twin tables, alternating, with
CUDA events:

  (A) today: the fp32 layout, a .to(torch.bfloat16) of each output, the tower's bf16 gradients .float()-ed, and the
      fp32 layout grad;
  (B) the bf16 layout (fused_embedding_to_layout(..., dtype=torch.bfloat16)) and the bf16 layout grad.

Both look up every (table, shard) list first and apply the embedding gradients table by table afterwards.  Also
timed: the layout forward alone and the layout grad alone (fp32 call on pre-widened gradients against the bf16
call), and gather_pool / scatter_grad_rows at the C2 shape (M = 2 097 152 occurrences, dim 32), fp32 against bf16.

Workload: scripts/bench_bf16_parts.py's 4 tables (dims 16, 16, 32, 64) and 26 features, every third one CSR SUM (1-7
FIDs per row) and the rest one FID per row, through sharding_sparse_fids at one shard (outside the timed step: it
synchronises with the host), laid out as one CONCAT output.  The tower's gradients are exact-sum values, so the
float-atomic layout grad gives the same bits in any order.  Afterwards (A)'s cast outputs must equal (B)'s bit for
bit, and so must every touched entry.

  python scripts/bench_bf16_layout.py [--batch 65536 4096] [--steps 40] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monolith_b200 import MultiHashTable, _lib, distribution_ops as dops, entry  # noqa: E402
from monolith_b200.distribution_ops import SliceTask  # noqa: E402

DIMS = {"t0": 16, "t1": 16, "t2": 32, "t3": 64}
N_FEATURES = 26
VOCAB = 1 << 20
BF = torch.bfloat16
C2_M, C2_D = 2097152, 32


def make_table(dev):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=VOCAB, init_seed=1), [0.05])
  return MultiHashTable({n: cfg(d) for n, d in DIMS.items()}, device=dev)


def batch(B, dev, seed):
  """sharding_sparse_fids' outputs for 26 features, the CONCAT tasks and the tower's bf16 gradient."""
  rng = np.random.default_rng(seed)
  names = list(DIMS)
  feats, ftab, fdim = {}, {}, {}
  for f in range(N_FEATURES):
    slot = names[f % len(names)]
    lens = rng.integers(1, 8, B) if f % 3 == 2 else np.ones(B, np.int64)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    # a slot per feature: a table's list holds every FID once, as apply_gradients(ids_unique=True) requires
    fids = (np.int64(f + 1) << 48) | (rng.zipf(1.05, int(rs[-1])) % VOCAB).astype(np.int64)
    name = f"f{f:02d}"
    feats[name] = (torch.from_numpy(fids).to(dev), torch.from_numpy(rs).to(dev))
    ftab[name], fdim[name] = slot, DIMS[slot]
  r = dops.sharding_sparse_fids(feats, ftab, fdim, 1)
  tasks, col = [], 0
  for i, name in enumerate(r["feature_names"]):
    tasks.append(SliceTask(i, 0, fdim[name], _lib.POOL_SUM, 0, 0, -1, col, 0))
    col += fdim[name]
  for t in tasks:
    t.out_row_stride = col
  r["tasks"], r["shapes"] = tasks, [(B, col)]
  # k * 2^-6 with |k| <= 16: the float-atomic layout grad sums these exactly in any order (the hottest FID's element
  # stays below 2^15 at these sizes), so (A) and (B) can be compared bit for bit
  r["grad"] = [(torch.randint(-16, 17, (B, col), device=dev).float() * 2.0 ** -6).to(BF)]
  return r


def lookup(t, r):
  return [t.lookup({name: ids})[name].reshape(-1) if ids.numel() else torch.zeros(1, device=t.device)
          for name, ids in zip(r["table_names"], r["fid_list"])]


def layout(r, embs, dtype=torch.float32):
  return dops.fused_embedding_to_layout(embs, [1] * len(embs), r["fid_offset"], r["feature_offset"], r["nfl_offset"],
                                        r["shapes"][0][0], r["tasks"], r["shapes"], dtype=dtype)


def layout_grad(r, embs, og):
  return dops.fused_embedding_to_layout_grad([e.numel() for e in embs], [1] * len(embs), r["fid_offset"],
                                             r["feature_offset"], r["nfl_offset"], r["shapes"][0][0], r["tasks"], og)


def apply(t, r, grads, ts):
  for name, ids, g in zip(r["table_names"], r["fid_list"], grads):
    if ids.numel():
      t.apply_gradients({name: (ids, g[:ids.numel() * DIMS[name]].reshape(-1, DIMS[name]))}, req_time=ts,
                        ids_unique=True)


def step_a(t, r, ts):
  embs = lookup(t, r)
  outs = [o.to(BF) for o in layout(r, embs)]
  apply(t, r, layout_grad(r, embs, [g.float() for g in r["grad"]]), ts)
  return outs


def step_b(t, r, ts):
  embs = lookup(t, r)
  outs = layout(r, embs, BF)
  apply(t, r, layout_grad(r, embs, r["grad"]), ts)
  return outs


def timed(fn):
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  out = fn()
  e1.record()
  torch.cuda.synchronize()
  return out, e0.elapsed_time(e1)


def c2_work(dev):
  """gather_pool and scatter_grad_rows at M occurrences of dim-32 rows (Zipf offsets into the unique rows)."""
  rng = np.random.default_rng(2)
  u = rng.zipf(1.05, C2_M) % (C2_M // 4)
  offs = torch.from_numpy((u * C2_D).astype(np.int32)).to(dev)
  fused = torch.randn(C2_M // 4 * C2_D, device=dev)
  g_bf = torch.randn(C2_M, C2_D, device=dev).to(BF)
  g_32 = g_bf.float()
  out32, outbf = torch.empty(C2_M, C2_D, device=dev), torch.empty(C2_M, C2_D, device=dev, dtype=BF)
  buf = torch.zeros(fused.numel(), device=dev)
  return {
      "gather_fp32": lambda: dops.gather_pool(fused, offs, C2_D, out=out32),
      "gather_bf16": lambda: dops.gather_pool(fused, offs, C2_D, out=outbf),
      "scatter_fp32": lambda: dops.scatter_grad_rows(g_32, offs, C2_D, buf),
      "scatter_bf16": lambda: dops.scatter_grad_rows(g_bf, offs, C2_D, buf),
  }


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, nargs="+", default=[65536, 4096])
  ap.add_argument("--steps", type=int, default=40)
  ap.add_argument("--warmup", type=int, default=10)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_bf16_layout.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  lib = _lib.load()
  for B in args.batch:
    ta, tb = make_table(dev), make_table(dev)
    data = [batch(B, dev, seed=B + i) for i in range(2)]
    embs = [lookup(ta, r) for r in data]                       # fixed inputs of the layout-alone timings
    wide = [[g.float() for g in r["grad"]] for r in data]
    keys = ("step_a", "step_b", "fwd_fp32", "fwd_bf16", "grad_fp32", "grad_bf16")
    times = {k: [] for k in keys}
    launches = {}
    ts = 1
    same_fwd = True
    for it in range(args.warmup + args.steps):
      i = it % len(data)
      r, e, w = data[i], embs[i], wide[i]
      work = {
          "step_a": lambda: step_a(ta, r, ts),
          "step_b": lambda: step_b(tb, r, ts),
          "fwd_fp32": lambda: layout(r, e),
          "fwd_bf16": lambda: layout(r, e, BF),
          "grad_fp32": lambda: layout_grad(r, e, w),
          "grad_bf16": lambda: layout_grad(r, e, r["grad"]),
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
      ts += 1
      del outs
    same_tab = True
    for slot in DIMS:
      k = torch.unique(torch.cat([r["fid_list"][r["table_names"].index(slot)] for r in data]))
      ea, eb = ta.lookup_entry(slot, k)["raw"], tb.lookup_entry(slot, k)["raw"]
      same_tab &= torch.equal(ea.view(torch.int32), eb.view(torch.int32)) and ta.size(slot) == tb.size(slot)
    res = {"batch": B, "features": N_FEATURES, "tables": len(DIMS), "steps": args.steps,
           "same_bits": bool(same_fwd and same_tab), "gpu": props.name, "power_limit": power}
    for k in keys:
      res[f"ms_{k}"] = float(np.median(times[k]))
      res[f"ms_spread_{k}"] = [float(np.min(times[k])), float(np.max(times[k]))]
      res[f"launches_{k}"] = launches[k]
    print(json.dumps(res), flush=True)
    ta.close()
    tb.close()
    del data, embs, wide
    torch.cuda.empty_cache()
  # C2 shape: gather_pool and scatter_grad_rows alone
  work = c2_work(dev)
  times = {k: [] for k in work}
  for it in range(args.warmup + args.steps):
    for k in (work if it % 2 == 0 else reversed(list(work))):
      _, ms = timed(work[k])
      if it >= args.warmup:
        times[k].append(ms)
  res = {"shape": "C2", "occurrences": C2_M, "dim": C2_D, "steps": args.steps, "gpu": props.name,
         "power_limit": power}
  for k in work:
    res[f"ms_{k}"] = float(np.median(times[k]))
    res[f"ms_spread_{k}"] = [float(np.min(times[k])), float(np.max(times[k]))]
  print(json.dumps(res), flush=True)


if __name__ == "__main__":
  main()
