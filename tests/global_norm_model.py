"""numpy float64 restatement of mono_global_norm's summation order (include/mono_emb.h), with explicit sequential
adds (np.sum is pairwise, so it is not used on the sums).

Chunks of CHUNK elements that never cross a tensor boundary; thread t of THREADS adds the squares of the chunk's
elements t + THREADS * i in increasing i from +0.0; then s[t] += s[t + h] for h = THREADS / 2 ... 1.  The chunk
partials, in (tensor, chunk) order, are reduced by the same rule until one value is left.
"""
import numpy as np

CHUNK, THREADS = 8192, 256


def _level(vals):
  """Every chunk of CHUNK float64 values (squares, or partials) by the rule, vectorised across chunks and lanes; the
  adds of one lane stay sequential (increasing i, then the tree)."""
  per = CHUNK // THREADS
  n_chunks = -(-vals.size // CHUNK)
  padded = np.zeros(n_chunks * CHUNK, np.float64)   # +0.0 past the end leaves a sum of squares unchanged
  padded[:vals.size] = vals
  cols = padded.reshape(n_chunks, per, THREADS)      # [chunk, i, t]: element t + THREADS * i
  s = np.zeros((n_chunks, THREADS), np.float64)
  for i in range(per):
    s = s + cols[:, i, :]
  h = THREADS // 2
  while h >= 1:
    s[:, :h] = s[:, :h] + s[:, h:2 * h]
    h //= 2
  return s[:, 0].copy()


def partials(arrays):
  """(tensor, chunk)-ordered partials of float32 arrays (bf16 inputs passed as their exact float32 values)."""
  out = []
  for a in arrays:
    x = np.asarray(a, np.float32).ravel().astype(np.float64)
    sq = x * x                            # exact: a float32 square fits a float64 mantissa
    out.append(_level(sq))
  return np.concatenate(out) if out else np.zeros(0, np.float64)


def sum_of_squares(arrays):
  p = partials(arrays)
  while p.size > 1:
    p = _level(p)
  return float(p[0]) if p.size else 0.0


def norm(arrays):
  return np.sqrt(np.float32(sum_of_squares(arrays)), dtype=np.float32)


def scale(norm_value, clip_norm):
  """ClipByGlobalNorm's rule (clip_by_global_norm.h:42-49): a NaN norm gives 1, an infinite one +0.0."""
  n, c = np.float32(norm_value), np.float32(clip_norm)
  return np.float32(c / n) if n > c else np.float32(1.0)
