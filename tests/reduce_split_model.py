"""numpy restatement of ReduceSum / ReduceMean / FusedReduceSumAndSplit / FusedReduceAndSplitGPU and their
gradients (ref: RT/ops/reduce_op.cc:29-89,124-180,232-330; reduce_op.cu.cc:308-316): the reference the device calls
mono_reduce_and_split[_grad] are checked against, bit for bit.

Forward: sample b of a feature owns the occurrence rows splits[b] .. splits[b + 1] - 1; every column is summed from
+0.0 with fp32 adds in occurrence order (the k-th add of every sample happens in step k below, so the order per sample is
the sequential one), and MEAN then multiplies by float(1.0 / double(float(n))) (reduce_op.cc:81): an empty MEAN row
is 0 * inf = NaN.  The feature's columns are cut, in order, into its slices.
Gradient: every occurrence row of sample b is b's slice gradients, copied (SUM: every bit kept) or times the same
factor (MEAN, counted per sample)."""
import numpy as np


def mean_factor(n):
  """ReduceMeanOp's `float multiply = 1.0 / static_cast<float>(counter)` for an array of counts."""
  with np.errstate(divide="ignore"):
    return (1.0 / np.asarray(n).astype(np.float32).astype(np.float64)).astype(np.float32)


def _counts(splits):
  sp = np.asarray(splits, np.int64).reshape(-1)
  return sp[:-1], sp[1:] - sp[:-1]


def reduce_and_split(splits, rows, slice_dims, poolings):
  """Feature f's rows [n_f, D_f] pooled by splits[f] and cut into slice_dims[f]: a list (per feature) of [B, s]."""
  out = []
  for sp, r, dims, pool in zip(splits, rows, slice_dims, poolings):
    r = np.asarray(r, np.float32)
    lo, n = _counts(sp)
    acc = np.zeros((lo.size, r.shape[1]), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):   # inf - inf and overflowing sums are part of the inputs
      for k in range(int(n.max()) if n.size else 0):
        m = n > k
        acc[m] += r[lo[m] + k]
      if pool == "mean":
        acc = acc * mean_factor(n)[:, None]
    out.append(np.split(acc, np.cumsum(dims)[:-1], axis=1))
  return out


def reduce_and_split_grad(splits, shapes, grads, poolings):
  """grads[f]: feature f's slice gradients ([B, s] each); returns the [n_f, D_f] occurrence-row gradients (rows no
  sample covers stay 0)."""
  out = []
  for sp, shape, gs, pool in zip(splits, shapes, grads, poolings):
    lo, n = _counts(sp)
    g = np.concatenate([np.asarray(x, np.float32) for x in gs], axis=1)
    if pool == "mean":
      with np.errstate(invalid="ignore", over="ignore"):
        g = g * mean_factor(n)[:, None]
    o = np.zeros(shape, np.float32)
    occ = np.concatenate([np.arange(a, a + c) for a, c in zip(lo, n)] or [np.zeros(0, np.int64)]).astype(np.int64)
    o[occ] = g[np.repeat(np.arange(lo.size), n)]
    out.append(o)
  return out
