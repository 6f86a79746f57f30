"""The sparse backward's summation order, restated in numpy (no torch, no GPU).

Every backward of the engine (mono_mtable_pool_backward, mono_scatter_grad_rows, mono_grouping_reduce and
reduce_push, the device-driven sharded step) sums the gradient rows of one run -- the occurrences of one FID or
one destination row, in position order -- with the reduction of csrc/bwd.cu.  Its association is a fixed function
of the run length L, the lane-group width G = pick_group(dim) and the call's piece count np = ceil(M / 32):

* L <= 64: one sequential sum starting from the first row (acc = x0; acc += x1; ...).
* L > 64: 32-row blocks aligned to the run start, each summed sequentially from its first row.  Then, with
  top = 1, while np > top * 512: top *= 128 and one tree level is added; the levels run with stride
  s = 1, 128, ...  At each level the block sum at index k is replaced when k % (128 s) == 0 and k + s < nblk,
  by the node sum over the members k + i s (i < 128, k + i s < nblk).  A node splits its members into
  NG = 32 / G contiguous groups of PER = 128 / NG members; each group is summed from 0.0f and the group sums
  are added in group order (a group whose first member is out of range is skipped).  Final pass:
  acc = b[0], then acc += b[k] for k = top, 2 top, ... < nblk.

All arithmetic is np.float32, which rounds to nearest like __fadd_rn / __fdiv_rn (the library is built with
-fmad=false and without fast-math).  For MEAN pooling a row enters divided by its row length (an fp32
division), which `occurrence_rows` reproduces.  The constants below are checked against the CUDA sources by
tests/test_reduce_order_cpu.py.
"""
import numpy as np

PIECE = 32          # kPiece: occurrences per piece and per long-run block
SHORT_RUN = 64      # kShortRun: longest run summed as one sequential unit
TREE_FAN = 128      # kTreeFan: members of one tree node
FINISH_MAX = 512    # kFinishMax: terms the final pass may add per run before another level is added


def pick_group(dim):
  """Lanes per group of the backward kernels (ops.cu pick_group): (dim + 3) / 4 rounded up to a power of two
  in [4, 32]."""
  v = (dim + 3) // 4
  g = 4
  while g < v and g < 32:
    g <<= 1
  return g


def n_pieces(M):
  return (M + PIECE - 1) // PIECE


def tree_top(np_):
  """(levels, top) of a call with np_ pieces (launch_reduce)."""
  levels, top = 0, 1
  while np_ > top * FINISH_MAX:
    top *= TREE_FAN
    levels += 1
  return levels, top


def occurrence_rows(pooled_grad, M, row_offsets=None, pooling="sum"):
  """Gradient row of every occurrence (float32[M, D]) as the reduce reads it: pooled_grad[row(m)], divided by
  the row length for CSR MEAN pooling."""
  g = np.asarray(pooled_grad, np.float32)
  if row_offsets is None:
    return g[:M]
  ro = np.asarray(row_offsets, np.int64)
  lens = np.diff(ro)
  row = np.repeat(np.arange(lens.size), lens)
  x = g[row]
  if pooling == "mean":
    x = x / lens[row].astype(np.float32)[:, None]
  return np.ascontiguousarray(x, np.float32)


def _seq_sums(x, start, length):
  """Sequential fp32 sums x[start[r]] + x[start[r] + 1] + ... (length[r] >= 1 terms), vectorised over r."""
  out = np.empty((start.size,) + x.shape[1:], np.float32)
  if start.size == 0:
    return out
  order = np.argsort(-length, kind="stable")        # longest first: the runs still adding are a prefix
  st, ln = start[order], length[order]
  acc = x[st].copy()
  for i in range(1, int(ln[0])):
    n = int(np.searchsorted(-ln, -i, side="left"))   # runs with length > i
    acc[:n] += x[st[:n] + i]
  out[order] = acc
  return out


def reduce_runs(x, start, length, G, np_):
  """fp32 sums of the runs x[start[r] : start[r] + length[r]] (rows in occurrence order) as the kernels of a
  call with np_ pieces and lane groups of G produce them."""
  x = np.asarray(x, np.float32)
  start = np.asarray(start, np.int64)
  length = np.asarray(length, np.int64)
  assert (length >= 1).all()
  out = np.empty((start.size,) + x.shape[1:], np.float32)
  short = length <= SHORT_RUN
  out[short] = _seq_sums(x, start[short], length[short])
  long_ = np.flatnonzero(~short)
  if long_.size == 0:
    return out
  # blocks of the long runs: run-aligned, 32 rows, summed sequentially
  nblk = (length[long_] + PIECE - 1) // PIECE
  first = np.concatenate([[0], np.cumsum(nblk)[:-1]])       # index of each run's block 0 in b
  run_of = np.repeat(np.arange(long_.size), nblk)
  k = np.arange(run_of.size) - first[run_of]                 # block index inside its run
  bstart = start[long_][run_of] + PIECE * k
  blen = np.minimum(PIECE, start[long_][run_of] + length[long_][run_of] - bstart)
  b = _seq_sums(x, bstart, blen)
  nb = nblk[run_of]
  # tree levels
  levels, top = tree_top(np_)
  NG = 32 // G
  PER = TREE_FAN // NG
  s = 1
  for _ in range(levels):
    heads = np.flatnonzero((k % (TREE_FAN * s) == 0) & (k + s < nb))
    if heads.size:
      i = np.arange(TREE_FAN)
      valid = k[heads][:, None] + i[None, :] * s < nb[heads][:, None]          # [node, member]
      idx = np.where(valid, heads[:, None] + i[None, :] * s, heads[:, None])
      tot = None
      for g in range(NG):
        acc = np.zeros((heads.size,) + x.shape[1:], np.float32)
        for m in range(g * PER, (g + 1) * PER):
          v = valid[:, m].reshape((-1,) + (1,) * (x.ndim - 1))
          acc = np.where(v, acc + b[idx[:, m]], acc)
        if tot is None:
          tot = acc
        else:
          v = valid[:, g * PER].reshape((-1,) + (1,) * (x.ndim - 1))
          tot = np.where(v, tot + acc, tot)
      b[heads] = tot
    s *= TREE_FAN
  # final pass over blocks 0, top, 2 top, ...
  nterm = (nblk + top - 1) // top
  out[long_] = _seq_sums(b, first, nterm) if top == 1 else _strided_sums(b, first, nterm, top)
  return out


def _strided_sums(b, first, nterm, top):
  acc = b[first].copy()
  for j in range(1, int(nterm.max())):
    sel = nterm > j
    acc[sel] += b[first[sel] + j * top]
  return acc


def run_sum(x, G, np_):
  """fp32 sum of one run's rows x (occurrence order) in a call with np_ pieces."""
  x = np.asarray(x, np.float32)
  return reduce_runs(x, [0], [x.shape[0]], G, np_)[0]


def call_sums(x, keys, G, M=None):
  """Every run's sum in one call: occurrence m (row x[m]) belongs to the run of keys[m]; a run's rows are taken
  in position order.  M (the call's occurrence count, default len(keys)) fixes the tree depth.
  Returns (the distinct keys ascending, float32[n_keys, ...] sums, run lengths)."""
  keys = np.asarray(keys)
  M = keys.size if M is None else M
  order = np.argsort(keys, kind="stable")
  sk = keys[order]
  head = np.flatnonzero(np.concatenate([[True], sk[1:] != sk[:-1]])) if sk.size else np.zeros(0, np.int64)
  length = np.diff(np.concatenate([head, [sk.size]]))
  xs = np.asarray(x, np.float32)[order]
  return sk[head], reduce_runs(xs, head, length, G, n_pieces(M)), length


def depth(L, np_, G):
  """Longest chain of fp32 additions in the sum of a run of L rows in a call with np_ pieces."""
  if L <= SHORT_RUN:
    return L - 1
  nblk = (L + PIECE - 1) // PIECE
  levels, top = tree_top(np_)
  NG = 32 // G
  PER = TREE_FAN // NG
  return (PIECE - 1) + levels * (PER + NG - 1) + ((nblk + top - 1) // top - 1)


def error_bound(L, np_, G, abs_sum):
  """|fp32 result - exact sum| <= gamma(depth) * sum |x| (gamma(n) = n u / (1 - n u), u = 2^-24)."""
  n = depth(L, np_, G)
  u = 2.0 ** -24
  return n * u / (1.0 - n * u) * np.asarray(abs_sum, np.float64)
