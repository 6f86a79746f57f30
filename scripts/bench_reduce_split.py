"""Times mono_reduce_and_split (the forward) and mono_reduce_and_split_grad (the backward) on the workload of
scripts/bench_parts.py: 4 tables of dims 16/16/32/64, 26 features, every third one multi-hot (0-8 FIDs per sample,
the others one FID), Zipf-skewed FIDs.  The per-occurrence rows come from MultiHashTable.lookup.  Per batch size:

  * device time (CUDA events, median of alternated calls after warm-up) of the forward and the backward, their
    algorithmic bytes sum_f 4 D_f (n_f + B) + 4 (B + 1) and the share of the H100 SXM data-sheet 3.35 TB/s;
  * what a PyTorch user writes instead: per feature segment_reduce (sum) or zeros().index_add_ (sum), then split,
    and repeat_interleave for the gradient; same_bits where the order of the adds is defined, else the max deviation;
  * for context, one op-by-op step (lookup -> reduce_and_split -> grad -> raw_apply_gradients with dedup) against
    lookup_pool_parts + pool_backward_parts on the same features (both SUM; two identical tables).

  python scripts/bench_reduce_split.py [--batch 65536 4096] [--steps 40] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monolith_b200 import MultiHashTable, PoolPart, distribution_ops as dops, entry  # noqa: E402

DIMS = {"t0": 16, "t1": 16, "t2": 32, "t3": 64}
N_FEATURES = 26
VOCAB = 1 << 20
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
SLEEP_CYCLES = 20_000_000   # ~10 ms at 1.98 GHz: longer than any host enqueue timed here


def make_table(dev):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=VOCAB, init_seed=1), [0.05])
  return MultiHashTable({n: cfg(d) for n, d in DIMS.items()}, device=dev)


def features(B, dev, seed):
  """[(slot, fids, row splits int32 [B + 1])]: feature f on table f % 4, multi-hot when f % 3 == 2."""
  rng = np.random.default_rng(seed)
  names = list(DIMS)
  out = []
  for f in range(N_FEATURES):
    slot = names[f % len(names)]
    lens = rng.integers(0, 9, B) if f % 3 == 2 else np.ones(B, np.int64)
    fids = (np.int64(f % len(names) + 1) << 48) | (rng.zipf(1.05, int(lens.sum())) % VOCAB).astype(np.int64)
    sp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    out.append((slot, torch.from_numpy(fids).to(dev), torch.from_numpy(sp).to(dev)))
  return out


def timed(fn, times, key):
  """Device time of fn's work: a sleep kernel queued first keeps the GPU busy while the host enqueues fn, so the
  events bracket the device work and not the host's Python and ctypes set-up."""
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda._sleep(SLEEP_CYCLES)
  e0.record()
  out = fn()
  e1.record()
  torch.cuda.synchronize()
  times.setdefault(key, []).append(e0.elapsed_time(e1))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, nargs="+", default=[65536, 4096])
  ap.add_argument("--steps", type=int, default=40)
  ap.add_argument("--warmup", type=int, default=10)
  ap.add_argument("--step-calls", type=int, default=4,
                  help="alternated op-by-op / parts steps (the op-by-op apply with dedup takes seconds at Zipf skew)")
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_reduce_split.py measures on a GPU"
  dev = torch.device("cuda", 0)
  props = torch.cuda.get_device_properties(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for B in args.batch:
    ta, tb = make_table(dev), make_table(dev)
    feats = features(B, dev, seed=B)
    dims = [DIMS[s] for s, _, _ in feats]
    # populate both tables identically, then take the per-occurrence rows from lookup
    for t in (ta, tb):
      t.pool_backward_parts([PoolPart(s, f, row_offsets=sp, rows=torch.zeros(B, DIMS[s], device=dev))
                             for s, f, sp in feats], req_time=1)
    per_slot = {s: [f for s2, f, _ in feats if s2 == s] for s in DIMS}
    ids = {s: torch.cat(v) for s, v in per_slot.items()}
    emb = ta.lookup(ids)
    rows, pos = [], {s: 0 for s in DIMS}
    for s, f, _ in feats:
      rows.append(emb[s][pos[s]:pos[s] + f.numel()])
      pos[s] += f.numel()
    splits = [sp for _, _, sp in feats]
    sdims = [[d] for d in dims]
    n_occ = [f.numel() for _, f, _ in feats]
    grads = [torch.randn(B, d, device=dev) for d in dims]
    lens = [sp[1:] - sp[:-1] for sp in splits]
    rowids = [torch.repeat_interleave(torch.arange(B, device=dev), ln) for ln in lens]

    def fwd():
      return dops.fused_reduce_and_split_gpu(splits, rows, sdims)

    def bwd():
      return dops.fused_reduce_and_split_gpu_grad(splits, rows, grads, sdims)

    def torch_segment():
      return [torch.segment_reduce(r, "sum", lengths=ln, unsafe=True).split([d], 1)[0] for r, ln, d in
              zip(rows, lens, dims)]

    def torch_index_add():
      return [torch.zeros(B, d, device=dev).index_add_(0, ri, r).split([d], 1)[0] for r, ri, d in
              zip(rows, rowids, dims)]

    def torch_bwd():
      return [torch.repeat_interleave(g, ln, dim=0) for g, ln in zip(grads, lens)]

    flat_ids = torch.cat([ids[s] for s in DIMS])
    id_split = np.cumsum([0] + [ids[s].numel() for s in DIMS]).tolist()
    order = [i for s in DIMS for i, (s2, _, _) in enumerate(feats) if s2 == s]

    def step_ops(ts):
      e = ta.lookup(ids)
      rr, p = [], {s: 0 for s in DIMS}
      for s, f, _ in feats:
        rr.append(e[s][p[s]:p[s] + f.numel()])
        p[s] += f.numel()
      outs = dops.fused_reduce_and_split_gpu(splits, rr, sdims)
      flat = torch.empty(sum(n * d for n, d in zip(n_occ, dims)), device=dev)
      views, off = [None] * N_FEATURES, 0
      for i in order:   # occurrence rows in the table-major order raw_apply_gradients takes
        views[i] = flat[off:off + n_occ[i] * dims[i]].view(n_occ[i], dims[i])
        off += n_occ[i] * dims[i]
      dops.fused_reduce_and_split_gpu_grad(splits, rr, grads, sdims, out=views)
      ta.raw_apply_gradients(flat_ids, id_split, flat, req_time=ts, enable_dedup=True)
      return outs

    def step_parts(ts):
      outs = tb.lookup_pool_parts([PoolPart(s, f, row_offsets=sp) for s, f, sp in feats])
      tb.pool_backward_parts([PoolPart(s, f, row_offsets=sp, rows=g) for (s, f, sp), g in zip(feats, grads)],
                             req_time=ts)
      return outs

    times = {}
    for it in range(args.warmup + args.steps):
      t = times if it >= args.warmup else {}
      pairs = [("fwd", fwd), ("torch_segment_reduce", torch_segment), ("torch_index_add", torch_index_add),
               ("bwd", bwd), ("torch_repeat_interleave", torch_bwd)]
      for key, fn in (pairs if it % 2 == 0 else pairs[::-1]):
        torch.cuda.synchronize()
        timed(fn, t, key)
    # outputs: ours against the torch forms
    mine, seg, iadd = fwd(), torch_segment(), torch_index_add()
    same_seg = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(mine, seg))
    dev_iadd = max(float((a - b).abs().max()) for a, b in zip(mine, iadd))
    same_iadd = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(mine, iadd))
    same_bwd = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(bwd(), torch_bwd()))
    # op-by-op step against the parts calls, alternated on two identical tables
    steps = {}
    lib = ta._lib
    launches = {}
    for it in range(1 + args.step_calls):
      t = steps if it >= 1 else {}
      pairs = [("step_ops", step_ops), ("step_parts", step_parts)]
      for key, fn in (pairs if it % 2 == 0 else pairs[::-1]):
        torch.cuda.synchronize()
        n0 = lib.mono_kernel_launch_count()
        timed(lambda: fn(2 + it), t, key)
        launches[key] = lib.mono_kernel_launch_count() - n0
    nbytes = sum(4 * d * (n + B) for d, n in zip(dims, n_occ)) + 4 * (B + 1)
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = {"batch": B, "features": N_FEATURES, "occurrences": int(sum(n_occ)), "calls": args.steps, "step_calls": args.step_calls,
           "fwd_ms": med["fwd"], "bwd_ms": med["bwd"],
           "fwd_spread_ms": [float(np.min(times["fwd"])), float(np.max(times["fwd"]))],
           "bwd_spread_ms": [float(np.min(times["bwd"])), float(np.max(times["bwd"]))],
           "bytes_each_way": nbytes,
           "fwd_share_of_3.35TBps": nbytes / (med["fwd"] * 1e-3) / HBM_BYTES_PER_S,
           "bwd_share_of_3.35TBps": nbytes / (med["bwd"] * 1e-3) / HBM_BYTES_PER_S,
           "torch_segment_reduce_ms": med["torch_segment_reduce"], "torch_segment_reduce_same_bits": same_seg,
           "torch_index_add_ms": med["torch_index_add"], "torch_index_add_same_bits": same_iadd,
           "torch_index_add_max_abs_dev": dev_iadd,
           "torch_repeat_interleave_ms": med["torch_repeat_interleave"], "torch_repeat_interleave_same_bits": same_bwd,
           "step_ops_ms": float(np.median(steps["step_ops"])), "step_parts_ms": float(np.median(steps["step_parts"])),
           "launches_step_ops": launches["step_ops"], "launches_step_parts": launches["step_parts"],
           "gpu": props.name, "power_limit": power}
    print(json.dumps(res))
    ta.close()
    tb.close()


if __name__ == "__main__":
  main()
