"""Where a key lands in the device table, and keys built to land where a test wants them.

The table's hash (common.cuh `mix64`, the splitmix64 finalizer) is a bijection of the 64-bit words, so a key
with a chosen hash h is simply unmix64(h).  A key's two candidate buckets are the high halves of
lo(h) * nb and hi(h) * nb (`bucket_pair`), its stash probe starts at bits 17..28 of h, and its FID slot is bits
48..62 of the key itself.  `colliding_keys` therefore builds groups of keys that share a bucket pair (and,
optionally, a stash probe chain) without any search over the hash: it draws h inside the wanted intervals and
inverts the hash; only the FID slot filter is a rejection loop.

Everything here is a restatement of the CUDA sources; tests/test_forward_paths_cpu.py pins the two together.
"""
import numpy as np

M64 = (1 << 64) - 1
C1 = 0xBF58476D1CE4E5B9
C2 = 0x94D049BB133111EB
C1_INV = pow(C1, -1, 1 << 64)
C2_INV = pow(C2, -1, 1 << 64)
STASH_CAP = 4096          # table.cu table_init: d.stash_cap
STASH_SHIFT = 17          # (mix64(key) >> 17) & (stash_cap - 1)
SLOT_SHIFT, SLOT_MASK = 48, 0x7FFF   # common.cuh slot_id_v2


def _u64(x):
  """Python int / numpy integer array (any signedness) -> numpy uint64 array of the same bits."""
  a = np.asarray(x)
  if a.dtype == np.uint64:
    return a.copy()
  if a.dtype.kind == "i":
    return a.astype(np.int64).view(np.uint64)
  if a.dtype == object or a.dtype.kind not in "iu":
    return np.asarray([int(v) & M64 for v in np.ravel(a)], np.uint64).reshape(a.shape)
  return a.astype(np.uint64)


def _unshift(y, s):
  """Inverse of x -> x ^ (x >> s) on uint64."""
  x = y.copy()
  for _ in range(64 // s + 1):
    x = y ^ (x >> np.uint64(s))
  return x


def mix64(x):
  """common.cuh mix64 on uint64 (element-wise; numpy uint64 arithmetic wraps mod 2^64)."""
  x = _u64(x)
  with np.errstate(over="ignore"):
    x ^= x >> np.uint64(30)
    x *= np.uint64(C1)
    x ^= x >> np.uint64(27)
    x *= np.uint64(C2)
    x ^= x >> np.uint64(31)
  return x


def unmix64(h):
  """The inverse bijection: mix64(unmix64(h)) == h."""
  x = _u64(h)
  with np.errstate(over="ignore"):
    x = _unshift(x, 31)
    x *= np.uint64(C2_INV)
    x = _unshift(x, 27)
    x *= np.uint64(C1_INV)
    x = _unshift(x, 30)
  return x


def _umulhi(a, nb):
  return ((a.astype(np.uint64) * np.uint64(nb)) >> np.uint64(32)).astype(np.int64)


def bucket_pair(key, nb):
  """common.cuh bucket_pair: (b1, b2) of int64 key(s), with the b2 == b1 -> b1 + 1 (mod nb) fix-up."""
  h = mix64(np.asarray(key, np.int64))
  b1 = _umulhi(h & np.uint64(0xFFFFFFFF), nb)
  b2 = _umulhi(h >> np.uint64(32), nb)
  b2 = np.where(b2 == b1, np.where(b1 + 1 == nb, 0, b1 + 1), b2)
  return b1, b2


def buckets_for(capacity):
  """Bucket count of a fresh table of `initial_capacity` (table.cu table_init + buckets_for)."""
  return max(64, (max(int(capacity), 1024) + 1) // 2 + 1)


def stash_start(key):
  """First stash slot a key's probe (and its insert) visits."""
  return ((mix64(np.asarray(key, np.int64)) >> np.uint64(STASH_SHIFT)) & np.uint64(STASH_CAP - 1)).astype(np.int64)


def fid_slot(key):
  return ((np.asarray(key, np.int64).view(np.uint64) >> np.uint64(SLOT_SHIFT)) & np.uint64(SLOT_MASK)).astype(np.int64)


def word_range(b, nb):
  """The 32-bit words w with umulhi(w, nb) == b: [lo, hi)."""
  return (b * (1 << 32) + nb - 1) // nb, ((b + 1) * (1 << 32) + nb - 1) // nb


def colliding_keys(nb, b1, b2, n, rng, stash_start=None, slots=None):
  """n distinct int64 keys whose hash halves map to buckets b1 and b2 before the fix-up, so that
  bucket_pair(key, nb) == (b1, b2) (or (b1, b1 + 1 mod nb) when b1 == b2).

  stash_start: also fix bits 17..28 of the hash, so every key of the group starts its stash probe at that slot
  (it must be reachable from b1: some word of b1's range has those bits).
  slots: draw until the key's FID slot (bits 48..62 of the key) is in this set.
  """
  lo0, lo1 = word_range(b1, nb)
  hi0, hi1 = word_range(b2, nb)
  keys = []
  seen = set()
  slot_arr = None if slots is None else np.asarray(sorted(slots), np.int64)
  batch = 1 << 12 if slots is None else 1 << 16
  tries = 0
  while len(keys) < n:
    tries += 1
    if tries > 2000:
      raise ValueError("no keys with the requested bucket pair / stash start / slots")
    if stash_start is None:
      lo = rng.integers(lo0, lo1, batch, dtype=np.uint64)
    else:
      s = np.uint64(stash_start)
      top = rng.integers(0, 8, batch, dtype=np.uint64) << np.uint64(29)
      low = rng.integers(0, 1 << STASH_SHIFT, batch, dtype=np.uint64)
      lo = top | (s << np.uint64(STASH_SHIFT)) | low
      lo = lo[(lo >= np.uint64(lo0)) & (lo < np.uint64(lo1))]
    hi = rng.integers(hi0, hi1, lo.size, dtype=np.uint64)
    k = unmix64((hi << np.uint64(32)) | lo).view(np.int64)
    if slot_arr is not None:
      k = k[np.isin(fid_slot(k), slot_arr)]
    for v in k.tolist():
      if v not in seen:
        seen.add(v)
        keys.append(v)
        if len(keys) == n:
          break
  return np.asarray(keys, np.int64)
