"""ShardingSparseFids on the device against the host-driven adapter it replaces.

  python scripts/bench_sharding.py [--steps 10] [--warmup 2] [--legacy-steps 3]

Times, per call (host wall clock around work that ends in a device synchronise), at the C3 shape (26 features,
B = 65 536) and the C4 shape (200 features, B = 16 384) for 1, 4 and 8 shards:
  legacy      sharding_sparse_fids over fused_reorder_by_indices and host index arithmetic (the reorder_fn path,
              which is the adapter as it was before mono_sharding_sparse_fids: row_splits.tolist() per feature, the
              feature offsets built on the host)
  device      sharding_sparse_fids on CUDA inputs: one mono_sharding_sparse_fids call, sync=True
  device_nosync  the same call with sync=False
and reports the library's kernel launches per call and whether every output of the three is the same bit for bit.
One JSON line per shape and shard count, then one summary line.
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

from monolith_b200 import _lib  # noqa: E402
from monolith_b200 import distribution_ops as dops  # noqa: E402

SHAPES = {"c3": (26, 65536), "c4": (200, 16384)}


def features(rng, F, B, dev):
  """F features over F // 3 + 1 tables: every fifth a sequence feature (0-15 FIDs per row), one shared, the rest one
  FID per row; Zipf-like FIDs carrying their slot in the top bits"""
  feats, table_of, dims = {}, {}, {}
  for i in range(F):
    name = f"f_{i:04d}"
    rows = 1 if i == 3 else B
    lens = rng.integers(0, 16, rows) if i % 5 == 0 else np.ones(rows, np.int64)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fids = (np.int64(i + 1) << 48) | ((rng.zipf(1.2, int(rs[-1])) - 1) % 1_000_000)
    feats[name] = (torch.from_numpy(fids).to(dev), torch.from_numpy(rs).to(dev))
    table_of[name] = f"t_{i % (F // 3 + 1):03d}"
    dims[name] = 8 + 8 * (i % 4)
  return feats, table_of, dims, ["f_0003"]


def timed(fn, steps, warmup):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  lib = _lib.load()
  n0 = lib.mono_kernel_launch_count()
  t0 = time.perf_counter()
  for _ in range(steps):
    r = fn()
  torch.cuda.synchronize()
  dt = (time.perf_counter() - t0) / steps
  return r, dt * 1e3, (lib.mono_kernel_launch_count() - n0) / steps


def same_bits(legacy, dev, nosync):
  eq = lambda a, b: a.shape == b.shape and a.dtype == b.dtype and a.device == b.device and torch.equal(a, b)
  ok = all(eq(legacy[k], dev[k]) and eq(dev[k], nosync[k]) for k in ("fid_offset", "feature_offset", "nfl_offset"))
  ok &= len(legacy["fid_list"]) == len(dev["fid_list"]) and all(eq(a, b) for a, b in zip(legacy["fid_list"],
                                                                                          dev["fid_list"]))
  total = int(nosync["fid_list_shard_row_length"].sum())
  ok &= eq(dev["fid_list_fused"], nosync["fid_list_fused"][:total])
  for k in ("fid_list_table_row_length", "fid_list_shard_row_length", "fid_list_emb_row_length"):
    ok &= eq(dev[k], nosync[k])
  ok &= all(eq(a, b) for a, b in zip(dev["fid_list_row_splits"], nosync["fid_list_row_splits"]))
  return bool(ok)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--legacy-steps", type=int, default=3)
  ap.add_argument("--shards", type=int, nargs="+", default=[1, 4, 8])
  a = ap.parse_args()
  assert torch.cuda.is_available(), "bench_sharding.py needs a GPU"
  dev = torch.device("cuda", 0)
  gpu = torch.cuda.get_device_name(dev)
  try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    power = "unknown"
  rng = np.random.default_rng(0)
  legacy_reorder = lambda lists, n, d: dops.fused_reorder_by_indices(lists, n, d, rank0_empty_shard=False)
  all_same = True
  for shape, (F, B) in SHAPES.items():
    feats, table_of, dims, shared = features(rng, F, B, dev)
    M = sum(f.numel() for f, _ in feats.values())
    for N in a.shards:
      call = lambda **kw: dops.sharding_sparse_fids(feats, table_of, dims, N, shared, **kw)
      legacy, t_legacy, _ = timed(lambda: call(reorder_fn=legacy_reorder), a.legacy_steps, 1)
      device, t_dev, l_dev = timed(lambda: call(), a.steps, a.warmup)
      nosync, t_nosync, l_nosync = timed(lambda: call(sync=False), a.steps, a.warmup)
      same = same_bits(legacy, device, nosync)
      all_same &= same
      print(json.dumps({"shape": shape, "features": F, "batch": B, "fids": M, "shards": N,
                        "legacy_ms": round(t_legacy, 3), "device_ms": round(t_dev, 3),
                        "device_nosync_ms": round(t_nosync, 3), "launches_device": l_dev,
                        "launches_device_nosync": l_nosync, "same_bits": same}), flush=True)
  print(json.dumps({"gpu": gpu, "power_limit": power, "same_bits": all_same}))


if __name__ == "__main__":
  main()
