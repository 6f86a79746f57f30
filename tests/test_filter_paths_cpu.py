"""The counting admission filter without a GPU: the numpy restatement of tests/filter_place.py against the oracle's
HashFilter cell for cell, the reference's hash_filter_test.cc known answers replayed through the oracle, the FID
builder, and the rules tests/test_gpu_filter_paths.py aims its cases with, pinned against the CUDA sources.  A change
to the cell layout, the clamp, the sizing, an op's filter mode or the set of kernels that consult the filter fails
here by name."""
import os
import re

import numpy as np
import pytest

from tests import filter_place as fp
from tests import orc
from tests.test_write_paths_cpu import _body, _cu_sources, _src

I64 = np.iinfo(np.int64)


def model_run(capacity, fids, counts, thresholds=None):
  f = fp.Filter(capacity)
  counts = np.broadcast_to(np.asarray(counts), np.shape(fids))
  if thresholds is None:
    out = [f.add(x, c) for x, c in zip(np.asarray(fids).tolist(), counts.tolist())]
  else:
    thresholds = np.broadcast_to(np.asarray(thresholds), np.shape(fids))
    out = [int(f.should_be_filtered(x, c, t)) for x, c, t in zip(np.asarray(fids).tolist(), counts.tolist(),
                                                                 thresholds.tolist())]
  return np.asarray(out, np.uint32), f.cells


def same_as_oracle(capacity, fids, counts, thresholds=None):
  want, cells = model_run(capacity, fids, counts, thresholds)
  got, ocells = orc.hash_filter_run(capacity, fids, counts, thresholds)
  np.testing.assert_array_equal(got, want)
  np.testing.assert_array_equal(ocells, cells)
  return want, cells


# ------------------------------------------------------------------------------------------------
# the restatement against the oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capacity", [1, 2, 3, 40, 1001])
def test_model_equals_oracle_on_random_streams(capacity):
  """More FIDs than cells, counts 1..20 (clamped), repeats: windows fill up, counters saturate, signatures collide."""
  rng = np.random.default_rng(capacity)
  vocab = rng.integers(I64.min, I64.max, max(8, 2 * capacity), dtype=np.int64, endpoint=True)
  fids = rng.choice(vocab, 6 * vocab.size)
  counts = rng.integers(1, 21, fids.size)
  out, cells = same_as_oracle(capacity, fids, counts)
  assert (out == fp.MAX_COUNT).any() and (cells & 15 == 15).any()
  same_as_oracle(capacity, fids, counts, rng.integers(0, 18, fids.size))


def test_model_equals_oracle_on_adversarial_streams():
  rng = np.random.default_rng(1)
  cap = 200
  total = fp.total_for(cap)
  # a full window: 64 signatures from one start cell, then a 65th; two FIDs of one signature sharing a counter
  crowd = np.concatenate([fp.keys(total, 17, 1, rng, sig=s) for s in range(1, 66)])
  twins = fp.keys(total, 17, 2, rng, sig=3)
  out, cells = same_as_oracle(cap, np.concatenate([crowd, twins]), 1)
  assert out[64] == fp.MAX_COUNT and out[65:].tolist() == [1, 2]    # crowd[64] finds no cell; the twins share sig 3's
  assert (cells[17:17 + 64] != 0).all() and cells[17 + 64] == 0
  # the last start cell: the probe runs on into the spill cells; signature 0 and the extreme FIDs
  tail = np.concatenate([fp.keys(total, total - 1, 1, rng, sig=s) for s in range(0, 70)])
  extremes = np.asarray([I64.min, I64.max, -1, 0, 1, -(1 << 17), 1 << 17], np.int64)
  fids = np.concatenate([tail, extremes, tail[:3]])
  out, cells = same_as_oracle(cap, fids, np.resize([1, 7, 15, 16, 40], fids.size))
  assert (cells[total:total + 63] != 0).all()                          # 64 cells from total - 1: one short of the end
  assert (cells[total - 1] >> 4) == 0                                 # signature 0 is a valid cell
  fids = np.concatenate([tail, extremes])
  same_as_oracle(cap, fids, 1, np.resize([0, 1, 2, 15, 16], fids.size))


# ------------------------------------------------------------------------------------------------
# the reference's hash_filter_test.cc known answers, through the oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capacity", [1, 3, 100])
def test_simple_bloom_known_answers(capacity):
  """test_simple_bloom<uint16_t>(capacity): add(1, 1) returns 0, 1, ..., 15 while get(1) = min(i + 1, 15); then 15."""
  out, cells = orc.hash_filter_run(capacity, np.ones(17, np.int64), 1)
  assert out.tolist() == list(range(16)) + [15]
  f = fp.Filter(capacity)
  for i in range(16):
    assert f.add(1, 1) == i and f.get(1) == min(i + 1, 15)
  assert f.add(1, 1) == 15 and f.get(1) == 15
  np.testing.assert_array_equal(cells, f.cells)
  assert np.count_nonzero(cells) == 1


def test_skip_zero_threshold_features():
  """TestSkipZeroThresholdFeatures: threshold 0 never filters and adds nothing; threshold 1 filters a new FID; 5 FIDs
  end in the filter.  (The reference builds that filter with fill rate 10, the engine's is 1.5: the answers hold.)"""
  fids, thr = [], []
  for i in range(5):
    fids += [i, 2 * i]
    thr += [0, 1]
  out, cells = orc.hash_filter_run(1000000, fids, 1, thr)
  assert out.tolist() == [0, 1] * 5
  assert np.count_nonzero(cells) == 5


def test_count_repeated_add():
  """test_count's filter2: one FID added with 1, 20 (clamped to 15) and 1 is one element; the adds return the count
  before them."""
  fid = np.uint64(10000002961562801052).view(np.int64)
  out, cells = orc.hash_filter_run(1000000, [fid] * 3, [1, 20, 1])
  assert out.tolist() == [0, 1, 15]
  assert np.count_nonzero(cells) == 1 and cells[cells != 0][0] == (int(fp.signature(fid)) << 4 | 15)


# ------------------------------------------------------------------------------------------------
# the builder
# ------------------------------------------------------------------------------------------------
def test_filter_keys_land_where_asked():
  rng = np.random.default_rng(3)
  for cap in (1, 3, 1000, 1000003):
    total = fp.total_for(cap)
    for cell in {0, total // 2, total - 1}:
      k = fp.keys(total, cell, 50, rng)
      assert np.unique(k).size == 50 and (fp.start_cell(k, total) == cell).all()
  total = fp.total_for(1000)
  k = fp.keys(total, 123, 5, rng, sig=0xABC, slot=77)
  assert (fp.start_cell(k, total) == 123).all() and (fp.signature(k) == 0xABC).all()
  assert (((k.view(np.uint64) >> np.uint64(48)) & np.uint64(0x7FFF)) == 77).all()
  k = fp.keys(total, 5, 3, rng, sig=0)
  assert (fp.signature(k) == 0).all() and (fp.start_cell(k, total) == 5).all()
  cells = rng.choice(total, 300, replace=False)
  k = fp.distinct_start_keys(total, cells, rng)
  np.testing.assert_array_equal(fp.start_cell(k, total), cells)
  # such FIDs never leave their start cell, whatever the order of their adds
  a = model_run(1000, k, 3)[1]
  b = model_run(1000, k[::-1], 3)[1]
  np.testing.assert_array_equal(a, b)
  assert (a[cells] != 0).all() and np.count_nonzero(a) == cells.size


# ------------------------------------------------------------------------------------------------
# source pins
# ------------------------------------------------------------------------------------------------
# every kernel that consults the filter, and the GPU cases that reach it
CALL_SITES = {
    ("ops.cu", "resolve_hit_kernel"): ["test_path_matrix[assign_add-unique]",
                                       "test_defect2_optimize_duplicates_count_every_occurrence"],
    ("ops.cu", "resolve_miss_kernel"): ["test_counts_thresholds_and_saturation", "test_path_matrix[fused-n3-unique]"],
    ("bwd.cu", "claim_miss_kernel"): ["test_path_matrix[pool_backward-sum]", "test_path_matrix[parts-fp32]"],
    ("xstep.cu", "xmiss_insert_kernel"): ["test_path_matrix[xstep-direct]"],
}


def _kernel_of(src, pos):
  """Name of the __global__ function whose body holds src[pos]."""
  heads = [m for m in re.finditer(r"__global__ void (?:__launch_bounds__\([^)]*\) )?(\w+)\(", src) if m.start() < pos]
  return heads[-1].group(1)


def test_filter_call_sites_inventory():
  """should_be_filtered is called in exactly these kernels, and each is reached by a case of the GPU file."""
  found = set()
  for f, s in _cu_sources().items():
    for m in re.finditer(r"should_be_filtered\(", s):
      found.add((f, _kernel_of(s, m.start())))
  assert found == set(CALL_SITES)
  gpu = open(os.path.join(os.path.dirname(__file__), "test_gpu_filter_paths.py")).read()
  ids = set(re.findall(r'"([\w-]+)"', gpu))
  for site, cases in CALL_SITES.items():
    for c in cases:
      name, _, param = c.partition("[")
      assert f"def {name}(" in gpu, (site, c)
      assert not param or param.rstrip("]") in ids, (site, c)


def test_filter_cell_rules():
  c = _src("common.cuh")
  add = _body(c, "__device__ __forceinline__ uint32_t filter_add(")
  assert "constexpr uint32_t kMaxCount = 15, kMaxStep = 64;" in add
  assert fp.MAX_COUNT == 15 and fp.MAX_STEP == 64
  assert "const uint32_t sign = (uint32_t)(((fid >> 17) | (fid << 15)) & 0x0FFFu);" in add
  assert fp.SIG_SHIFT == 17 and fp.SIG_MASK == 0xFFF
  assert "const uint32_t ncell = t->flt_total + kMaxStep;" in add
  assert "uint32_t pos = (uint32_t)(mix64(fid) % (uint64_t)t->flt_total);" in add
  assert "if (count > kMaxCount) count = kMaxCount;" in add
  assert "const uint32_t nv = v == 0 ? ((sign << 4) + count) : (c + count >= kMaxCount ? (v | kMaxCount) : v + count);" in add
  assert "if (v != 0 && (v >> 4) != sign) break;" in add
  assert "const uint32_t old = atomicCAS(wp, w, nw);" in add and "if (++pos == ncell) pos = 0;" in add
  assert add.endswith("return kMaxCount; }")
  sbf = _body(c, "__device__ __forceinline__ bool should_be_filtered(")
  assert "if (t->flt_cells == nullptr) return false;" in sbf and "if (thr == 0) return false;" in sbf
  assert "return filter_add(t, fid, count) < thr;" in sbf
  assert "if (t->slot_thr[2 * i] == slot) thr = t->slot_thr[2 * i + 1];" in sbf   # the last matching pair wins


def test_filter_sizing():
  t = _body(_src("table.cu"), "void table_set_filter(")
  assert "uint64_t total = (uint64_t)(capacity * 1.5);" in t and "if (total == 0) total = 1;" in t
  assert "const size_t words = (size_t)((total + 64 + 1) / 2);" in t
  assert "MONO_CUDA(cudaMemset(d.flt_cells, 0, words * sizeof(uint32_t)));" in t   # set_hash_filter resets
  assert [fp.total_for(c) for c in (1, 2, 3, 100, 1000003)] == [1, 3, 4, 150, 1500004]
  cells = _body(_src("capi.cu"), "int mono_mtable_hash_filter_cells(")
  assert "n == (int64_t)d.flt_total + 64" in cells


def test_filter_mode_per_op():
  """Optimize and assign consult the filter for ids absent from the table (mode 1), assign_add for every id (mode 2),
  reinitialize and restore never; the grouped optimize and the backward's claims count 1 per FID."""
  ops = _src("ops.cu")
  ru = _body(ops, "void run_upsert(")
  assert ("a.filter_mode = !any_filter ? 0 : (op == kOpOptimize || op == kOpAssign) ? 1 : (op == kOpAssignAdd ? 2 : 0);"
          in ru)
  assert "a.filter_mode = call.any_filter ? 1 : 0;" in _body(ops, "void run_upsert_groups(")
  hit = _body(ops, "resolve_hit_kernel(UpsertArgs a)")
  assert "} else if (a.filter_mode == 2 && should_be_filtered(t, a.ids[i], 1)) {" in hit
  assert "if (a.absent0 && a.absent0[i]) (void)should_be_filtered(t, a.ids[i], 1);" in hit
  miss = _body(ops, "resolve_miss_kernel(UpsertArgs a)")
  assert "if (a.filter_mode != 0 && should_be_filtered(t, a.ids[i], a.occ_extra ? 1u + a.occ_extra[i] : 1u)) {" in miss
  # the duplicate rounds of a filtered optimize / assign note which ids were absent at call start
  assert "} else if (a.filter_mode == 1) {" in ru and "absent_at_start_kernel<<<" in ru
  assert "if (should_be_filtered(t, key, 1u)) continue;" in _body(_src("bwd.cu"), "claim_miss_kernel(")
  assert "should_be_filtered(t, key, 1u) ? kEmptyRow" in _body(_src("xstep.cu"), "xmiss_insert_kernel(")


def test_filtered_fused_optimize_goes_shard_by_shard():
  """With a filter the fused optimize runs the reference's per-shard BatchOptimize loop (a FID still absent counts
  once per shard); without one, unique ids take the grouped pass; a filtered table at world > 1 refuses the sharded
  step's backward."""
  fo = _body(_src("capi.cu"), "int mono_mtable_fused_optimize(")
  assert "if (fused_slot_size_host[s * K + k] > 0 && t->tables[k].dev.flt_cells) any_filter = true;" in fo
  assert ("if ((flags & MONO_FLAG_IDS_UNIQUE) && !(flags & MONO_FLAG_DEDUP_SUM) && num_shards > 1 && !any_filter) {"
          in fo)
  xb = _body(_src("xstep.cu"), "void xstep_backward(")
  assert "if (x->N > 1 && x->mt->tables[x->k].dev.flt_cells)" in xb
  assert xb.index("flt_cells") < xb.index("grouping_reduce_push(")
