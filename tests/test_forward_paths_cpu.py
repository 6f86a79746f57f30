"""tests/cuckoo_place.py against the oracle and against itself, and the dispatch rules of the forward kernels that
tests/test_gpu_forward_paths.py aims its cases at.  A change to the hash, the table sizing, the stash or a dispatch
rule fails here by name; the GPU matrix then has to be re-aimed."""
import os
import re

import numpy as np
import pytest

from tests import cuckoo_place as cp
from tests import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "monolith_b200", "csrc")
I64 = np.iinfo(np.int64)


def _src(name):
  with open(os.path.join(CSRC, name)) as f:
    return f.read()


def _squash(s):
  return re.sub(r"\s+", " ", s.replace("\\\n", " "))  # macro line continuations too


def test_mix64_restatement_matches_the_oracle_initializer():
  """uniform_init(seed, fid, col, 0, 1) = top 24 bits of mix64(mix64(mix64(seed ^ G) + fid) + col * C) / 2^24."""
  rng = np.random.default_rng(1)
  lib = orc.lib()
  seeds = rng.integers(0, 1 << 63, 40, dtype=np.uint64)
  fids = np.concatenate([rng.integers(I64.min, I64.max, 40, dtype=np.int64), [0, -1, I64.min, I64.max]])
  with np.errstate(over="ignore"):
    for seed in seeds.tolist() + [0, (1 << 64) - 1]:
      inner = cp.mix64(np.uint64(seed) ^ np.uint64(0x9E3779B97F4A7C15))
      for fid in fids.tolist():
        for col in (0, 1, 31):
          h = cp.mix64(cp.mix64(inner + np.asarray(fid, np.int64).view(np.uint64)) + np.uint64(col) *
                       np.uint64(0xD1B54A32D192ED03))
          want = int(h >> np.uint64(40))
          got = lib.orc_uniform_init(seed, fid, col, 0.0, 1.0) * float(1 << 24)
          assert got == want, (seed, fid, col)


def test_unmix64_inverts_mix64():
  rng = np.random.default_rng(2)
  x = np.concatenate([rng.integers(I64.min, I64.max, 100000, dtype=np.int64), [0, -1, I64.min, I64.max]])
  u = x.view(np.uint64)
  np.testing.assert_array_equal(cp.unmix64(cp.mix64(u)), u)
  np.testing.assert_array_equal(cp.mix64(cp.unmix64(u)), u)
  # the constants are what the CUDA source multiplies by
  assert (cp.C1 * cp.C1_INV) % (1 << 64) == 1 and (cp.C2 * cp.C2_INV) % (1 << 64) == 1


def test_bucket_pair_fixup_and_sizing():
  assert cp.buckets_for(1) == cp.buckets_for(1024) == 513
  assert cp.buckets_for(0) == 513 and cp.buckets_for(4096) == 2049 and cp.buckets_for(4097) == 2050
  nb = 97
  rng = np.random.default_rng(3)
  keys = rng.integers(I64.min, I64.max, 200000, dtype=np.int64)
  b1, b2 = cp.bucket_pair(keys, nb)
  assert ((b1 >= 0) & (b1 < nb) & (b2 >= 0) & (b2 < nb)).all()
  assert (b1 != b2).all()
  # literal restatement with Python ints
  for k in keys[:2000].tolist():
    h = int(cp.mix64(np.int64(k)))
    r1, r2 = ((h & 0xFFFFFFFF) * nb) >> 32, ((h >> 32) * nb) >> 32
    if r2 == r1:
      r2 = 0 if r1 + 1 == nb else r1 + 1
    assert (r1, r2) == (int(cp.bucket_pair(k, nb)[0]), int(cp.bucket_pair(k, nb)[1]))


@pytest.mark.parametrize("nb", [64, 513, 2049, 40961])
def test_colliding_keys_land_where_asked(nb):
  rng = np.random.default_rng(nb)
  cases = [(0, 1), (nb - 1, 0), (nb - 1, 5 % nb), (7 % nb, 3 % nb), (nb // 2, nb // 2), (nb - 1, nb - 1)]
  for b1, b2 in cases:
    want2 = b2 if b2 != b1 else (0 if b1 + 1 == nb else b1 + 1)
    k = cp.colliding_keys(nb, b1, b2, 12, rng)
    assert np.unique(k).size == 12
    g1, g2 = cp.bucket_pair(k, nb)
    assert (g1 == b1).all() and (g2 == want2).all(), (b1, b2)
    # a shared stash probe chain: any start some word of b1's range has
    lo0, lo1 = cp.word_range(b1, nb)
    s = (int(rng.integers(lo0, lo1)) >> cp.STASH_SHIFT) & (cp.STASH_CAP - 1)
    k = cp.colliding_keys(nb, b1, b2, 12, rng, stash_start=s)
    g1, g2 = cp.bucket_pair(k, nb)
    assert (g1 == b1).all() and (g2 == want2).all() and (cp.stash_start(k) == s).all()
    # chosen FID slots (per-slot expiry picks members later)
    k = cp.colliding_keys(nb, b1, b2, 6, rng, stash_start=s, slots={3, 900})
    assert np.isin(cp.fid_slot(k), [3, 900]).all() and (cp.stash_start(k) == s).all()
    g1, g2 = cp.bucket_pair(k, nb)
    assert (g1 == b1).all() and (g2 == want2).all()


def test_fid_slot_and_stash_start_restatements():
  k = np.array([(5 << 48) | 77, -1, I64.min, I64.max, 0], np.int64)
  np.testing.assert_array_equal(cp.fid_slot(k), [5, 0x7FFF, 0, 0x7FFF, 0])
  h = cp.mix64(k)
  np.testing.assert_array_equal(cp.stash_start(k), ((h >> np.uint64(17)) & np.uint64(4095)).astype(np.int64))


# ------------------------------------------------------------------------------------------------
# source pins: what tests/cuckoo_place.py and tests/test_gpu_forward_paths.py assume about the CUDA sources
# ------------------------------------------------------------------------------------------------
def test_hash_and_placement_constants_match_the_cuda_sources():
  common = _squash(_src("common.cuh"))
  assert ("x ^= x >> 30; x *= 0x%xULL; x ^= x >> 27; x *= 0x%xULL; x ^= x >> 31; return x;" % (cp.C1, cp.C2)) in common, \
      "common.cuh mix64 changed: update tests/cuckoo_place.py"
  assert ("uint64_t h = mix64((uint64_t)key); b1 = __umulhi((uint32_t)h, nb); b2 = __umulhi((uint32_t)(h >> 32), nb); "
          "if (b2 == b1) b2 = (b1 + 1 == nb) ? 0u : b1 + 1;") in common, "common.cuh bucket_pair changed"
  assert "constexpr int kBucketSlots = 4;" in common
  assert "return (uint32_t)(((uint64_t)fid >> 48) & 0x7FFFu);" in common, "slot_id_v2 changed"
  table = _squash(_src("table.cu"))
  assert "uint64_t nb = (keys + 1) / 2 + 1; if (nb < 64) nb = 64;" in table, "table.cu buckets_for changed"
  assert "uint64_t rows = std::max<uint64_t>(cfg.initial_capacity, 1024);" in table
  assert "d.num_buckets = buckets_for(rows); d.stash_cap = 4096;" in table
  assert cp.STASH_CAP == 4096
  # the rehash that empties the stash: any stash entry (live or tombstone) forces one at the next insert
  assert "|| t.snap_stash > 0;" in table
  # every stash probe (and the stash insert) starts at bits 17.. of the hash
  rowops = _src("rowops.cuh")
  start = re.compile(r"\(uint32_t\)\(mix64\(\(uint64_t\)(?:key|key\[q\]|e\.key)\) >> 17\) & mask")
  assert len(start.findall(common)) == 3 and len(start.findall(rowops)) == 3, "stash start expression changed"


def test_forward_dispatch_rules_match_the_cuda_sources():
  ops = _squash(_src("ops.cu"))
  rowops = _squash(_src("rowops.cuh"))
  layout = _squash(_src("layout.cu"))
  assert "constexpr int kStage = 16;" in rowops
  assert "lookup_pool_staged_kernel(" in ops and re.search(r"lookup_pool_staged_kernel\([^{]*\) \{ constexpr int U = 4;", ops)
  # staged CSR pooling: 16-byte-aligned, packed-enough output, dims 4..128 in steps of 4
  assert ("if ((D & 3) == 0 && D <= 128 && (out_stride & 3) == 0 && (out_col & 3) == 0 && "
          "(reinterpret_cast<uintptr_t>(out) & 15) == 0 && n_rows < ((int64_t)1 << 31))") in ops
  # register-path pooling table
  assert ("if (G == 4) LP(4, 1, 4); else if (G == 8) LP(8, 1, 4); else if (G == 16) LP(16, 1, 4); "
          "else if (nv == 1) LP(32, 1, 4); else if (nv == 2) LP(32, 2, 2); else LP(32, 4, 1);") in ops
  assert 'if (D > 512) throw ArgError("lookup_pool supports dim <= 512");' in ops
  # TMA lookup: 128- and 256-byte rows, packed output at column 0, 16-byte aligned, contiguous table rows
  assert "if ((D & 3) || (rowb != 128 && rowb != 256)) return false;" in ops
  assert ("if (out_col != 0 || (out_stride > 0 && out_stride != D) || (reinterpret_cast<uintptr_t>(out_dev) & 15)) "
          "return false;") in ops
  assert "if (nsegs == 1 && h_segs[0].id_begin == 0 && try_lookup_tma(" in ops
  # single-table kernel selection order: dual knob, then same-stream, then confirm; several segments otherwise
  assert re.search(r"if \(nsegs == 1 && knob\(KNOB_LOOKUP_DUAL\)\) lookup_kernel<GG, true, true>.*"
                   r"else if \(nsegs == 1 && !mt->lookup_must_confirm\(s\)\) lookup_kernel<GG, true, false, false>.*"
                   r"else if \(nsegs == 1\) lookup_kernel<GG, true>.*else lookup_kernel<GG, false>", ops)
  assert "int pick_group(int max_dim) { int v = (max_dim + 3) / 4; int g = 4; while (g < v && g < 32) g <<= 1; return g; }" in ops
  # gather_pool: the two-phase row copy only without CSR and for 16-byte rows that one lane group covers
  assert ("if (row_offsets == nullptr && (dim & 3) == 0 && dim <= 4 * G && (out_stride & 3) == 0 && (out_col & 3) == 0 && "
          "((reinterpret_cast<uintptr_t>(fused_emb) | reinterpret_cast<uintptr_t>(out)) & 15) == 0)") in layout
  assert "const int grid = grid_for(n_rows, kThreads / G); #define GP(GG)" in layout
  # grid caps the turnover cases are sized against: at most 2048 resident threads per SM
  engine = _squash(_src("engine.h"))
  assert "if (max_blocks <= 0) max_blocks = device_sms() * 8;" in engine
  assert "constexpr int kThreads = 256;" in _squash(_src("common.cuh"))
