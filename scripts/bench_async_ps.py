"""Times the async parameter-server worker path (DistributedMultiTypeHashTable.lookup / apply_gradients on the raw
API, ref: NT/distributed_ps.py:266-337, 481-516) with every server's table on one GPU, per phase:

  unique     unique_key_with_value_and_offset    split   floormod + ragged_split_by_indices
  lookup     the servers' raw_lookup calls        fill    fill_with_offset_map, one call per server
  fill_grad  fill_with_offset_map_gradient        apply   the servers' raw_apply_gradients calls (Adagrad)

Device time per phase: CUDA events around the phase's calls, a sleep kernel queued first so that the events bracket
the device work and not the host's enqueue (median of --steps after --warmup).  Algorithmic bytes per phase (the
bytes each op must move at least, from the shapes; see phase_bytes) over that time, and the share of the H100 SXM
data sheet's 3.35 TB/s.  The longest run (occurrences of the most frequent key) and the device time of its row's
gradient alone, as a share of the whole fill gradient.  For comparison, the same worker step with the four ops on
the host (numpy restatement tests/offset_map_model.py; keys, rows and gradients copied between device and host), host
clock around a synchronised step.  The card's name and power limit are read in the same run.

Workloads: c3, Criteo-shaped: 26 tables of dim 16, B one key per sample per table, per-table Zipf(1.1) keys; c2,
MovieLens-shaped: 2 tables (uid, movie) of dim 32, Zipf(1.05) over 5 M ranks each.

--transfer-float16: the table's transfer_float16 path.  The servers' lookup writes fp16 rows, the fill reads them, the
fill gradient writes fp16 sums and the apply phase includes each server's widening of them to fp32.  Rows and
gradients between servers and worker then count 2 bytes per element in the algorithmic bytes.  --host-steps 0 skips
the host comparison step.

  python scripts/bench_async_ps.py [--workload c3 c2] [--num-ps 1 4] [--batch 65536] [--steps 20] [--warmup 5]
                                   [--host-steps 2] [--transfer-float16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from monolith_b200 import MultiHashTable, distribution_ops as dops, entry  # noqa: E402
from monolith_b200.distributed_ps import DistributedMultiTypeHashTable  # noqa: E402
from tests import offset_map_model as om  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
SLEEP_CYCLES = 20_000_000   # ~10 ms at 1.98 GHz: longer than any host enqueue timed here


def workload(name, B, rng):
  """slot -> (dim, keys)"""
  if name == "c3":
    return {f"slot_{i:02d}": (16, (rng.zipf(1.1, B) % (1 << 25)).astype(np.int64)) for i in range(26)}
  return {s: (32, (rng.zipf(1.05, B) % 5_000_000).astype(np.int64)) for s in ("movie", "uid")}


def configs(shape):
  def cfg(d):
    seg = entry.CombineAsSegment(d, entry.RandomUniformInitializer(-0.05, 0.05),
                                 entry.AdagradOptimizer(learning_rate=0.05, initial_accumulator_value=0.1))
    return entry.HashTableConfigInstance(entry.TableConfig([seg], initial_capacity=1 << 16, init_seed=1), [0.05])
  return {s: cfg(d) for s, (d, _) in shape.items()}


def timed(fn, times, key):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  torch.cuda._sleep(SLEEP_CYCLES)
  e0.record()
  out = fn()
  e1.record()
  torch.cuda.synchronize()
  if times is not None:
    times.setdefault(key, []).append(e0.elapsed_time(e1))
  return out


def phase_bytes(M, U, rows_floats, occ_floats, row_bytes=4):
  """M occurrences, U unique keys, rows_floats = sum over unique keys of their dim, occ_floats = the value buffer;
  row_bytes: bytes per element of the rows and row gradients between servers and worker (2 with transfer_float16)"""
  return {
      "unique": 8 * M + 8 * U + 8 * M + 8 * (U + 1),          # keys in; unique keys, offsets, offset splits out
      "split": 8 * U + 8 * U + 8 * U + 8 * U,                  # indices and keys in; keys and positions out
      "fill": 8 * U + 16 * U + 8 * M + row_bytes * rows_floats + 4 * occ_floats,   # pos, splits, offsets, rows in
      "fill_grad": 8 * U + 16 * U + 8 * M + 4 * occ_floats + row_bytes * rows_floats,
  }


def run(name, S, B, args, dev, power):
  rng = np.random.default_rng(1)
  shape = workload(name, B, rng)
  names = sorted(shape)
  dims = [shape[s][0] for s in names]
  f16 = args.transfer_float16
  row_dtype = torch.float16 if f16 else torch.float32
  dmt = DistributedMultiTypeHashTable(S, configs(shape), lambda i, c: MultiHashTable(configs(shape), device=dev),
                                      transfer_float16=f16)
  ids = {s: torch.from_numpy(shape[s][1]).to(dev) for s in names}
  grads = {s: torch.randn(shape[s][1].size, shape[s][0], device=dev) for s in names}
  dmt.apply_gradients({s: (ids[s], grads[s]) for s in names}, req_time=1)   # populate the servers
  t0 = dmt.tables[0]
  flat_ids, splits = t0.get_ragged_id(ids)
  flat_grad = t0.get_flat_value(grads)
  # one synchronised pass for the sizes the timed phases reuse
  res = dops.unique_key_with_value_and_offset(flat_ids, splits, dims)
  U, M = res.num_unique, flat_ids.numel()
  sp = dops.ragged_split_by_indices(torch.remainder(res.unique_key[0], S), res.unique_key[0], res.unique_key[1], S)
  vos = res.value_offset[1]
  runs = (vos[1:] - vos[:-1]).cpu().numpy()
  hot = int(np.argmax(runs))
  uks = res.unique_key[1].cpu().numpy()
  rows_floats = int(sum((uks[k + 1] - uks[k]) * dims[k] for k in range(len(dims))))
  lrs = {}

  def ph_unique():
    return dops.unique_key_with_value_and_offset(flat_ids, splits, dims, sync=False)

  def ph_split():
    return dops.ragged_split_by_indices(torch.remainder(res.unique_key[0], S), res.unique_key[0], res.unique_key[1], S,
                                        sync=False)

  def ph_lookup():
    lrs["rows"] = [t.raw_lookup(sp.splits[i][0], sp.row_splits_host[i], dtype=row_dtype) for i, t in
                   enumerate(dmt.tables)]

  def ph_fill():
    for i in range(S):
      dops.fill_with_offset_map(sp.pos[i], sp.row_splits_host[i], lrs["rows"][i], res.value_offset, res.value_buffer,
                                dims, num_unique=U, sync=False)

  def ph_fill_grad():
    lrs["g"] = [dops.fill_with_offset_map_gradient(sp.pos[i], sp.row_splits_host[i], flat_grad, res.value_offset, dims,
                                                   num_unique=U, sync=False, dtype=row_dtype) for i in range(S)]

  def ph_apply():
    for i, t in enumerate(dmt.tables):
      t.raw_apply_gradients(sp.splits[i][0], sp.row_splits_host[i], lrs["g"][i].float(), req_time=2)

  # the hot key's row alone: its server, its table and its place in that server's rows
  hot_ps = int(np.mod(res.unique_key[0][hot].item(), S))
  hot_row = int(np.nonzero(sp.pos[hot_ps].cpu().numpy() == hot)[0][0])
  hot_rs = sp.row_splits_host[hot_ps]
  hot_k = int(np.searchsorted(hot_rs, hot_row, side="right") - 1)
  one_split = [0] * (hot_k + 1) + [1] * (len(dims) - hot_k)

  def ph_hot_grad():
    dops.fill_with_offset_map_gradient(sp.pos[hot_ps][hot_row:hot_row + 1], one_split, flat_grad, res.value_offset,
                                       dims, num_unique=U, sync=False, dtype=row_dtype)

  phases = [("unique", ph_unique), ("split", ph_split), ("lookup", ph_lookup), ("fill", ph_fill),
            ("fill_grad", ph_fill_grad), ("apply", ph_apply), ("hot_row_grad", ph_hot_grad)]
  times = {}
  for it in range(args.warmup + args.steps):
    for key, fn in phases:
      timed(fn, times if it >= args.warmup else None, key)
  med = {k: float(np.median(v)) for k, v in times.items()}

  # whole worker steps through the public class (host clock, synchronised)
  def step_device():
    dmt.lookup(ids)
    dmt.apply_gradients({s: (ids[s], grads[s]) for s in names}, req_time=3)
    torch.cuda.synchronize()

  keys_np = flat_ids.cpu().numpy()
  g_np = flat_grad.cpu().numpy()

  def step_host():
    """the same step with the four ops on the host (numpy), the servers' calls on the device"""
    k_host = flat_ids.cpu().numpy()
    uk, uks_h, vo, vos_h, n = om.unique_key_with_value_and_offset(k_host, splits, dims)
    msp, mpos = om.ragged_split_by_indices(np.mod(uk, S), uk, uks_h, S)
    buf = np.empty(n, np.float32)
    for i, t in enumerate(dmt.tables):
      rows = t.raw_lookup(torch.from_numpy(msp[i][0]).to(dev), msp[i][1].tolist()).cpu().numpy()
      om.fill_with_offset_map(mpos[i], msp[i][1], rows, vo, vos_h, dims, buf)
    torch.from_numpy(buf).to(dev)
    g_host = flat_grad.cpu().numpy()
    for i, t in enumerate(dmt.tables):
      g = om.fill_with_offset_map_gradient(mpos[i], msp[i][1], g_host, vo, vos_h, dims)
      t.raw_apply_gradients(torch.from_numpy(msp[i][0]).to(dev), msp[i][1].tolist(), torch.from_numpy(g).to(dev),
                            req_time=3)
    torch.cuda.synchronize()

  steps = {}
  for it in range(1 + max(args.host_steps, 2)):
    for key, fn in (("step_device", step_device), ("step_host", step_host)):
      if key == "step_host" and (not args.host_steps or it > args.host_steps):
        continue
      torch.cuda.synchronize()
      t1 = time.perf_counter()
      fn()
      if it:
        steps.setdefault(key, []).append((time.perf_counter() - t1) * 1e3)
  # the device's outputs against the host's on this workload
  uk, uks_h, vo, vos_h, n = om.unique_key_with_value_and_offset(keys_np, splits, dims)
  same = (res.unique_key[0].cpu().numpy().tolist() == uk.tolist() and
          res.value_offset[0].cpu().numpy().tolist() == vo.tolist())
  msp, mpos = om.ragged_split_by_indices(np.mod(uk, S), uk, uks_h, S)
  for i in range(S):
    want = om.fill_with_offset_map_gradient(mpos[i], msp[i][1], g_np, vo, vos_h, dims)
    got = lrs["g"][i].cpu().numpy()
    if f16:
      with np.errstate(over="ignore"):
        want = want.astype(np.float16)
      same = same and np.array_equal(got.view(np.uint16), want.view(np.uint16))
    else:
      same = same and np.array_equal(got.view(np.uint32), want.view(np.uint32))
  nbytes = phase_bytes(M, U, rows_floats, res.value_len, 2 if f16 else 4)
  out = {"workload": name, "num_ps": S, "transfer_float16": f16, "batch": B, "tables": len(dims),
         "dims": sorted(set(dims)),
         "occurrences": M, "unique": U, "longest_run": int(runs[hot]), "steps": args.steps,
         "device_ms": {k: round(v, 4) for k, v in med.items() if k != "hot_row_grad"},
         "spread_ms": {k: [round(float(np.min(v)), 4), round(float(np.max(v)), 4)] for k, v in times.items()},
         "bytes": nbytes,
         "GBps": {k: round(b / (med[k] * 1e-3) / 1e9, 1) for k, b in nbytes.items()},
         "share_of_3.35TBps": {k: round(b / (med[k] * 1e-3) / HBM_BYTES_PER_S, 4) for k, b in nbytes.items()},
         "longest_run_grad_ms": round(med["hot_row_grad"], 4),
         "longest_run_share_of_fill_grad": round(med["hot_row_grad"] / med["fill_grad"], 4),
         "step_device_ms": round(float(np.median(steps["step_device"])), 3),
         "step_host_ops_ms": round(float(np.median(steps["step_host"])), 3) if "step_host" in steps else None,
         "host_ops_label": "unique, split, fill and fill gradient in numpy on the host (tests/offset_map_model.py)",
         "device_equals_host_bits": bool(same),
         "gpu": torch.cuda.get_device_properties(dev).name, "power_limit": power}
  print(json.dumps(out), flush=True)
  for t in dmt.tables:
    t.close()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--workload", nargs="+", default=["c3", "c2"], choices=["c3", "c2"])
  ap.add_argument("--num-ps", type=int, nargs="+", default=[1, 4])
  ap.add_argument("--batch", type=int, default=65536)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--host-steps", type=int, default=2)
  ap.add_argument("--transfer-float16", action="store_true")
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_async_ps.py measures on a GPU"
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
  except OSError:
    power = "unknown"
  for name in args.workload:
    for S in args.num_ps:
      run(name, S, args.batch, args, dev, power)


if __name__ == "__main__":
  main()
