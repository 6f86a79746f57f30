"""The counting admission filter restated in numpy, and FIDs built to land where a test wants them in it.

The filter (common.cuh filter_add / should_be_filtered, the oracle's HashFilter, the reference's
HashFilter<uint16_t>) keeps total + 64 cells of 16 bits, total = (uint64)(capacity * 1.5), at least 1.  A cell is
signature << 4 | count: the signature is bits 17..28 of the FID, the count saturates at 15, 0 is an empty cell.  A
FID's probe starts at cell mix64(fid) % total and walks at most 64 cells (the 64 spill cells past total are where a
window that starts near the end runs on); it stops at an empty cell or one with its signature.  add returns the count
before the addition (0 for a new cell, 15 when all 64 cells belong to others).

mix64 is a bijection, so a FID with a chosen start cell is unmix64(cell + m * total) for any m; fixing the FID's own
bits as well (signature, slot = bits 48..62) is a rejection loop over the free bits.  tests/test_filter_paths_cpu.py
pins all of this against the sources and the oracle.
"""
import numpy as np

from tests import cuckoo_place as cp

MAX_STEP = 64       # kMaxStep: probe window and spill cells
MAX_COUNT = 15      # kMaxCount: 4-bit saturating count
SIG_SHIFT, SIG_MASK = 17, 0xFFF
SLOT_SHIFT, SLOT_MASK = cp.SLOT_SHIFT, cp.SLOT_MASK


def total_for(capacity):
  return max(int(int(capacity) * 1.5), 1)


def n_cells(capacity):
  return total_for(capacity) + MAX_STEP


def signature(fid):
  return ((cp._u64(fid) >> np.uint64(SIG_SHIFT)) & np.uint64(SIG_MASK)).astype(np.int64)


def start_cell(fid, total):
  return (cp.mix64(np.asarray(fid, np.int64)) % np.uint64(total)).astype(np.int64)


class Filter:
  """hash_filter.h find / add / ShouldBeFiltered over one numpy cell array."""

  def __init__(self, capacity):
    self.total = total_for(capacity)
    self.cells = np.zeros(self.total + MAX_STEP, np.uint16)

  def find(self, fid):
    """The cell index add would write, or None when the 64-cell window holds only other signatures."""
    sign = int(signature(fid))
    pos = int(start_cell(fid, self.total))
    for _ in range(MAX_STEP):
      v = int(self.cells[pos])
      if v == 0 or (v >> 4) == sign:
        return pos
      pos += 1
      if pos == self.cells.size:
        pos = 0
    return None

  def add(self, fid, count):
    pos = self.find(fid)
    if pos is None:
      return MAX_COUNT
    count = min(int(count), MAX_COUNT)
    v = int(self.cells[pos])
    if v == 0:
      self.cells[pos] = (int(signature(fid)) << 4) + count
      return 0
    c = v & MAX_COUNT
    self.cells[pos] = v | MAX_COUNT if c + count >= MAX_COUNT else v + count
    return c

  def get(self, fid):
    pos = self.find(fid)
    return MAX_COUNT if pos is None else int(self.cells[pos]) & MAX_COUNT

  def should_be_filtered(self, fid, count, threshold):
    if threshold == 0:
      return False
    return self.add(fid, count) < threshold


def keys(total, cell, n, rng, sig=None, slot=None):
  """n distinct FIDs whose probe starts at `cell` of a filter with `total` cells, optionally with signature `sig`
  and FID slot `slot`."""
  cell = int(cell)
  assert 0 <= cell < total
  if sig is None and slot is None:
    hi = ((1 << 64) - 1 - cell) // total
    out = set()
    while len(out) < n:
      m = rng.integers(0, hi, n, dtype=np.uint64, endpoint=True)
      h = np.uint64(cell) + m * np.uint64(total)
      out.update(cp.unmix64(h).view(np.int64).tolist())
    return np.asarray(sorted(out)[:n], np.int64)
  fixed, mask = 0, 0
  if sig is not None:
    fixed |= (int(sig) & SIG_MASK) << SIG_SHIFT
    mask |= SIG_MASK << SIG_SHIFT
  if slot is not None:
    fixed |= (int(slot) & SLOT_MASK) << SLOT_SHIFT
    mask |= SLOT_MASK << SLOT_SHIFT
  out, tries = [], 0
  while len(out) < n:
    tries += 1
    if tries > 4000:
      raise ValueError("no FIDs with the requested start cell / signature / slot")
    r = rng.integers(0, 1 << 64, 1 << 16, dtype=np.uint64, endpoint=False)
    f = ((r & np.uint64(~mask & ((1 << 64) - 1))) | np.uint64(fixed)).view(np.int64)
    for v in f[start_cell(f, total) == cell].tolist():
      if v not in out:
        out.append(v)
  return np.asarray(out[:n], np.int64)


def distinct_start_keys(total, cells, rng):
  """One FID per entry of `cells` (distinct cells), starting its probe there: FIDs whose probes never leave their
  start cell, so that the filter state after any call is independent of the order of its adds."""
  cells = np.asarray(cells, np.int64)
  assert np.unique(cells).size == cells.size and (cells < total).all()
  hi = ((1 << 64) - 1 - int(cells.max())) // total
  m = rng.integers(0, hi, cells.size, dtype=np.uint64, endpoint=True)
  return cp.unmix64(cells.astype(np.uint64) + m * np.uint64(total)).view(np.int64)
