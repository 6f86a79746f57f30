"""What tests/test_gpu_layout_paths.py assumes, checked without a GPU: the lane-group rules of layout.cu, the exact-sum
gradient generator, the chain sharding_sparse_fids -> lookup -> layout on the oracle, the wrappers' input checks and
the C ABI's task validation."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from monolith_b200 import _lib
from monolith_b200 import distribution_ops as dops
from monolith_b200.distribution_ops import SliceTask
from tests import orc
from tests.helpers import table
from tests.test_gpu_layout_paths import (CHAIN_FEATS, CHAIN_L, CHAIN_TABLES, DIM_SETS, FIRSTN, MEAN, SUM,
                                         _chain_features, _chain_tasks, exact_terms, layout_g, scatter_g,
                                         standard_problem, terms_model)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _layout_src():
  with open(os.path.join(ROOT, "monolith_b200", "csrc", "layout.cu")) as f:
    return re.sub(r"\s+", " ", f.read().replace("\\\n", " "))


@pytest.fixture(scope="module")
def lib():
  if not os.path.exists(_lib.LIB_PATH):
    import __graft_entry__
    __graft_entry__.build()
  return _lib.load()


def _oracle_reorder(lists, n, dims):
  out, ss, sl, _, offs = orc.reorder_by_indices([l.numpy() for l in lists], n, dims)
  return torch.from_numpy(out), ss.tolist(), sl.tolist(), None, torch.from_numpy(offs)


# ------------------------------------------------------------------------------------------------
# lane-group rules the GPU cases are aimed with
# ------------------------------------------------------------------------------------------------
def test_lane_group_rules_match_layout_cu():
  src = _layout_src()
  assert "int max_dim = 1; for (auto& t : ordered) max_dim = std::max(max_dim, t.dim);" in src
  assert "int G = 4; while (G < max_dim && G < 32) G <<= 1; // one float per lane" in src
  assert "const int G = std::min(32, std::max(4, pick_group(dim * 4))); // one float per lane" in src
  assert "static int pick_group(int dim) { int v = (dim + 3) / 4, g = 4; while (g < v && g < 32) g <<= 1; return g; }" in src
  for k in ("layout_fwd_kernel", "layout_bwd_kernel"):
    assert len(re.findall(k + r"<(4|8|16|32)>", src)) == 4, k
  assert "switch (G) { case 4: GG_(4); break; case 8: GG_(8); break; case 16: GG_(16); break; default: GG_(32); }" in src
  # gather_pool_grad's G restated: pick_group(4 * dim) clamped to [4, 32]
  for dim in range(1, 301):
    v, g = dim, 4
    while g < v and g < 32:
      g <<= 1
    assert scatter_g(dim) == min(32, max(4, g)), dim
  assert [scatter_g(d) for d in (1, 4, 5, 8, 9, 16, 17, 32, 33, 300)] == [4, 4, 8, 8, 16, 16, 32, 32, 32, 32]
  # the forward dim sets meet every G; grid units are chains (forward) or tasks (backward) times B
  rng = np.random.default_rng(0)
  gs = {layout_g(standard_problem(rng, 4, dims, 2)[1]) for dims in DIM_SETS}
  assert gs == {4, 8, 16, 32}
  assert "const int64_t units = (int64_t)(backward ? (int)ordered.size() : n_chains) * batch_size;" in src
  assert "const int grid = grid_for(units, kThreads / G);" in src


# ------------------------------------------------------------------------------------------------
# exact-sum inputs
# ------------------------------------------------------------------------------------------------
def test_exact_terms_sum_to_the_same_bits_in_any_order():
  rng = np.random.default_rng(1)
  t = exact_terms(rng, 1 << 15)
  assert np.abs(t * 64).max() <= 64 and (t * 64 == np.round(t * 64)).all()
  t[: 1 << 14] = np.float32(1.0)     # all of one sign: the largest partial sums the bound allows
  for n in (1, 2, 4, 8):
    x = (t / np.float32(n)).astype(np.float32)
    exact = x.astype(np.float64).sum()
    for _ in range(4):
      y = rng.permutation(x)
      s = np.cumsum(y, dtype=np.float32)        # sequential fp32 sums: every partial sum is exact
      np.testing.assert_array_equal(s.astype(np.float64), np.cumsum(y.astype(np.float64)))
      assert float(s[-1]) == exact


def test_exact_backward_problem_stays_within_2_15_terms():
  rng = np.random.default_rng(2)
  prob, tasks, shapes = standard_problem(rng, 256, (1, 17, 32, 4), 3, exact=True, hot=True)
  og = [exact_terms(rng, s) for s in shapes]
  model = terms_model(prob, tasks, og)
  assert 4096 <= max(int(n.max()) for _, _, n in model) <= 1 << 15
  # MEAN rows hold 1, 2, 4 or 8 FIDs, so every term is a multiple of 2^-9
  for fi in {t.nfl_idx for t in tasks if t.pooling == MEAN}:
    assert {len(r) for r in prob.rows_of[fi]} <= {1, 2, 4, 8}
  want = orc.embedding_to_layout_grad(prob.sizes(), prob.strides, prob.fo, prob.fe, prob.nfl, prob.B, tasks, og)
  for w, (s, _, _) in zip(want, model):
    np.testing.assert_array_equal(w.astype(np.float64), s)


# ------------------------------------------------------------------------------------------------
# the chain on the oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2, 5])
def test_chain_model_on_the_oracle(N):
  """sharding_sparse_fids (oracle reorder) -> oracle lookup of every (table, shard) list -> orc.embedding_to_layout
  with the outputs as they are == per-feature orc lookup_pool; read the way the int64 nfl_offset was (word f of the
  int64 buffer) it is not."""
  rng = np.random.default_rng(100 + N)
  B = 37
  o = orc.OracleMultiHashTable({t: table([(d, "adagrad", {})], [0.25], capacity=4096) for t, d in CHAIN_TABLES.items()})
  feats = _chain_features(rng, B)
  for t, d in CHAIN_TABLES.items():
    ids = np.unique(np.concatenate([f for n, (f, _) in feats.items() if CHAIN_FEATS[n][0] == t]))
    o.assign({t: (ids, rng.standard_normal((ids.size, d)).astype(np.float32))}, req_time=10)
  r = dops.sharding_sparse_fids({n: (torch.from_numpy(f), torch.from_numpy(rs)) for n, (f, rs) in feats.items()},
                                {n: v[0] for n, v in CHAIN_FEATS.items()},
                                {n: CHAIN_TABLES[v[0]] for n, v in CHAIN_FEATS.items()}, N,
                                [n for n, v in CHAIN_FEATS.items() if v[2]], reorder_fn=_oracle_reorder)
  tables, names = r["table_names"], r["feature_names"]
  embs = []
  for k, t in enumerate(tables):
    for n in range(N):
      ids = r["fid_list"][k * N + n].numpy()
      embs.append(o.lookup({t: ids})[t].reshape(-1) if ids.size else np.zeros(1, np.float32))
  tasks, shapes, cols = _chain_tasks(names, B)
  fo, fe, nfl = r["fid_offset"].numpy(), r["feature_offset"].numpy(), r["nfl_offset"].numpy()
  concat, seq = orc.embedding_to_layout(embs, [1] * len(embs), fo, fe, nfl, B, tasks, shapes)
  for name in names:
    t, pooling, sh = CHAIN_FEATS[name]
    f, rs = feats[name]
    if pooling == "firstn":
      d = CHAIN_TABLES[t]
      rows = o.lookup({t: f})[t]
      want = np.zeros((B, CHAIN_L, d), np.float32)
      for b in range(B):
        m = min(int(rs[b + 1] - rs[b]), CHAIN_L)
        want[b, :m] = rows[rs[b]:rs[b] + m]
      np.testing.assert_array_equal(seq.view(np.uint32), want.reshape(B, -1).view(np.uint32))
      continue
    want = o.lookup_pool(t, f, rs.astype(np.int32), pooling)
    if sh:
      want = np.repeat(want, B, axis=0)
    np.testing.assert_array_equal(concat[:, cols[name]:cols[name] + CHAIN_TABLES[t]].view(np.uint32),
                                  want.view(np.uint32))
  # the earlier int64 nfl_offset, read as the C ABI's uint32 words: features shift, feature 0 looks empty
  words = nfl.view(np.uint32).astype(np.int64).view(np.uint32)[:nfl.size]
  bad, _ = orc.embedding_to_layout(embs, [1] * len(embs), fo, fe, words, B, tasks, shapes)
  assert not np.array_equal(bad, concat)


def test_sharding_sparse_fids_nfl_offset_is_int32_with_the_uint32_bits():
  feats = {"a": (torch.tensor([1, 2, 3]), torch.tensor([0, 1, 3])), "b": (torch.tensor([7, 8]), torch.tensor([0, 2]))}
  r = dops.sharding_sparse_fids(feats, {"a": "t", "b": "t"}, {"a": 4, "b": 4}, 2, shared_features=["b"],
                                reorder_fn=_oracle_reorder)
  nfl = r["nfl_offset"]
  assert nfl.dtype == torch.int32
  assert nfl.numpy().astype(np.uint32).tolist() == [0, 2 | (1 << 31), 4]
  assert int(nfl[1]) < 0                                   # the shared bit is the sign bit
  assert r["feature_offset"].dtype == torch.int32 and r["fid_offset"].dtype == torch.int64


# ------------------------------------------------------------------------------------------------
# the wrappers refuse what the C ABI would reinterpret
# ------------------------------------------------------------------------------------------------
def _args(fo=torch.int64, fe=torch.int32, nf=torch.int32):
  return torch.zeros(3, dtype=fo), torch.zeros(2, dtype=fe), torch.zeros(2, dtype=nf)


@pytest.mark.parametrize("grad", [False, True])
def test_layout_wrappers_refuse_other_dtypes_and_cpu_tensors(grad):
  task = [SliceTask(0, 0, 4, SUM, 0, 0, 4, 0, 0)]

  def call(fo, fe, nf, rows=None):
    if grad:
      return dops.fused_embedding_to_layout_grad([16], [1], fo, fe, nf, 1, task, rows or [torch.zeros(1, 4)])
    return dops.fused_embedding_to_layout(rows or [torch.zeros(16)], [1], fo, fe, nf, 1, task, [(1, 4)])
  for kw, name in (({"nf": torch.int64}, "nfl_offset"), ({"nf": torch.uint8}, "nfl_offset"),
                   ({"fe": torch.int64}, "feature_offset"), ({"fo": torch.int32}, "fid_offset"),
                   ({"fo": torch.float64}, "fid_offset")):
    with pytest.raises(ValueError, match=name + " must be a torch.int"):
      call(*_args(**kw))
  with pytest.raises(ValueError, match="fid_offset must be a CUDA tensor"):
    call(*_args())
  with pytest.raises(ValueError, match="nfl_offset must be a torch.int32 tensor, not"):
    call(*_args()[:2], [0, 1])


def test_layout_wrappers_check_before_loading_anything(monkeypatch):
  def boom():
    raise AssertionError("reached the library")
  monkeypatch.setattr(_lib, "load", boom)
  with pytest.raises(ValueError, match="nfl_offset"):
    dops.fused_embedding_to_layout([torch.zeros(4)], [1], *_args(nf=torch.int64), 1,
                                   [SliceTask(0, 0, 4, SUM, 0, 0, 4, 0, 0)], [(1, 4)])


# ------------------------------------------------------------------------------------------------
# the C ABI's task validation (runs before the device is selected)
# ------------------------------------------------------------------------------------------------
def _call(lib, grad, tasks, total_nfl=3):
  arr = dops._tasks_arr(tasks)
  fn = lib.mono_embedding_to_layout_grad if grad else lib.mono_embedding_to_layout
  return fn(0, None, None, 1, None, 0, None, 0, None, total_nfl, 4, arr, len(tasks), None, None)


GOOD = dict(nfl_idx=1, slice_start=2, dim=4, pooling=SUM, max_seq_len=0, out_tensor=0, out_row_stride=8, out_col=4,
            accumulate=0)
BAD = [
    ("nfl_idx", dict(nfl_idx=3)), ("nfl_idx", dict(nfl_idx=-1)), ("dim", dict(dim=0)), ("dim", dict(dim=-4)),
    ("slice_start", dict(slice_start=-1)), ("out_col", dict(out_col=-1)), ("out_tensor", dict(out_tensor=-1)),
    ("pooling", dict(pooling=3)), ("pooling", dict(pooling=-1)),
    ("max_seq_len", dict(pooling=FIRSTN, max_seq_len=0, out_row_stride=100)),
    ("accumulate", dict(pooling=FIRSTN, max_seq_len=2, accumulate=1, out_row_stride=100)),
    ("out_row_stride", dict(out_row_stride=7)),
    ("out_row_stride", dict(pooling=FIRSTN, max_seq_len=2, out_row_stride=11)),
    ("out_row_stride", dict(out_col=2 ** 31 - 2, out_row_stride=2 ** 31 - 1)),
]


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("field,change", BAD, ids=[f"{f}-{i}" for i, (f, _) in enumerate(BAD)])
def test_cabi_rejects_bad_tasks_before_the_device(field, change, grad, lib):
  good = SliceTask(**GOOD)
  bad = SliceTask(**{**GOOD, **change})
  assert _call(lib, grad, [good, bad]) == -1   # MONO_ERR_INVALID_ARGUMENT
  assert field.encode() in lib.mono_last_error()


def test_cabi_accepts_edge_tasks_and_reaches_the_device(lib):
  if torch.cuda.is_available():
    pytest.skip("with a GPU the call would launch on null pointers")
  edge = [SliceTask(**GOOD), SliceTask(**{**GOOD, "nfl_idx": 2, "slice_start": 0, "out_col": 0, "out_row_stride": 4}),
          SliceTask(**{**GOOD, "pooling": FIRSTN, "max_seq_len": 2, "out_row_stride": 12}),
          SliceTask(**{**GOOD, "pooling": MEAN, "accumulate": 1, "nfl_idx": 0})]
  for grad in (False, True):
    assert _call(lib, grad, edge) == -3        # MONO_ERR_CUDA: validation passed, no device here
    assert _call(lib, grad, []) == -3
