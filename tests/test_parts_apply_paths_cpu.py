"""CPU checks for tests/test_gpu_parts_apply_paths.py: the numpy restatement of a parts call's per-occurrence gradient
terms, which the oracle is fed, and the dispatch rules the GPU cases are aimed with, pinned against the sources.

The fused backward over parts (csrc/bwd.cu run_pool_backward_parts) checks every part's rows (check_grad_rows), orders
the call's tables by table index (the sorted table names), reduces and applies each table over its sorted range with
the lane-group width of its dim, and picks the reduce and apply instantiations below.  If a rule here changes, the
GPU file's expected kernel names, launch counts and boundary offsets change with it.
"""
import re

import numpy as np

from tests import reduce_order as ro
from tests.test_apply_paths_cpu import _read, _squash
from tests.test_seq_parts_cpu import firstn_terms

BWD = ("monolith_b200", "csrc", "bwd.cu")

GS = (4, 8, 16, 32)
OPTS = (0, 1, 2, 3, -1)
OPT_CODE = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 3}   # MONO_OPT_*: the four with a register-resident apply
# the optimizer x width matrix: each row dtype meets every lane-group width; together they meet every pool dim
FP32_DIMS = [4, 12, 20, 64, 100]
BF16_DIMS = [8, 32, 36, 128]
# table A's one run of L_A occurrences, then table B's range starts at L_A: offsets 1, 31, 0, 1, 31, 1, 1, 1 mod 32
BOUNDARY_LENS = [65, 95, 96, 97, 127, 129, 4097, 16385]
SEQ_L = 5


# ------------------------------------------------------------------------------------------------
# the per-occurrence gradient terms of one part
# ------------------------------------------------------------------------------------------------
class Part:
  """One feature of a parts call in host form: FIDs of table `slot`, CSR offsets (None: one FID per row), pooling,
  FIRSTN length L, and the column `col` its rows start at in the call's shared [B, W] gradient array."""

  def __init__(self, slot, fids, offs=None, pooling="sum", L=0):
    self.slot, self.fids, self.pooling, self.L = slot, np.asarray(fids, np.int64), pooling, L
    self.offs = None if offs is None else np.asarray(offs, np.int32)
    self.col = 0

  def n_rows(self):
    return self.fids.size if self.offs is None else self.offs.size - 1

  def width(self, D):
    return D * (self.L if self.pooling == "firstn" else 1)

  def where(self):
    """(row, position in the row) of every occurrence."""
    M = self.fids.size
    if self.offs is None:
      return np.arange(M), np.zeros(M, np.int64)
    n = np.diff(self.offs).astype(np.int64)
    row = np.repeat(np.arange(n.size), n)
    return row, np.arange(M) - self.offs[:-1].astype(np.int64)[row]

  def cell(self, m, D):
    """(row, first column) of occurrence m's term in the shared array; None past a FIRSTN row's L."""
    row, pos = self.where()
    if self.pooling == "firstn":
      return None if pos[m] >= self.L else (int(row[m]), self.col + int(pos[m]) * D)
    return int(row[m]), self.col

  def terms(self, grad, D):
    """float32[M, D]: SUM the row, CSR MEAN the row / n (one fp32 division), FIRSTN position j's slice for j < L
    and +0.0 beyond (ScatterGrad leaves such a FID's gradient at its zero fill)."""
    grad = np.asarray(grad, np.float32)
    row, pos = self.where()
    if self.pooling == "firstn":
      t = np.zeros((row.size, D), np.float32)
      inl = pos < self.L
      t[inl] = grad[row[inl, None], self.col + pos[inl, None] * D + np.arange(D)]
      return t
    t = grad[row, self.col:self.col + D]
    if self.pooling == "mean" and self.offs is not None:
      t = t / np.diff(self.offs).astype(np.float32)[row][:, None]
    return np.ascontiguousarray(t, np.float32)


def table_sums(grad, parts, slot, D):
  """(keys ascending, sums, run lengths) of table `slot` in one call: its parts' terms in part order, then occurrence
  order, summed as the reduce of a call with that table's occurrence count does."""
  ps = [p for p in parts if p.slot == slot]
  x = np.concatenate([p.terms(grad, D) for p in ps])
  keys = np.concatenate([p.fids for p in ps])
  with np.errstate(all="ignore"):
    return ro.call_sums(x, keys, ro.pick_group(D), M=keys.size)


def bf16_widen(x):
  """float32 -> the nearest bfloat16 (ties to even, NaN kept NaN), widened back exactly (bits << 16)."""
  import torch
  return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).float().numpy()


# ------------------------------------------------------------------------------------------------
# what a call launches
# ------------------------------------------------------------------------------------------------
def seg_kernel(G, bf16, seg_vpl=1, seg_ahead=1):
  """The reduce instantiation launch_reduce picks for one table of a parts call (never the PLAIN form: the gradient
  rows come through the occurrence map)."""
  g, v = (G // 2, 2) if seg_vpl == 2 and G >= 8 else (G, 1)
  a = "true" if seg_ahead else "false"
  return f"bf16_seg_reduce_kernel<{g},{v},{a}>" if bf16 else f"seg_reduce_kernel<{g},{v},false,{a}>"


def opt_sel(segs):
  """apply_opt_sel: the register-resident apply for a single SGD / Adagrad / FTRL / Adam segment, else -1."""
  return OPT_CODE.get(segs[0][1], -1) if len(segs) == 1 else -1


def apply_kernel(G, opt, bf16):
  return f"{'bf16_' if bf16 else ''}runs_apply_kernel<{G},{opt}>"


def claim_set_slots(n):
  cap = 1024
  while cap < 2 * n:
    cap <<= 1
  return cap


def call_launches(per_table):
  """Kernel launches of one parts call whose tables get per_table occurrences: occurrence map, claim, miss,
  finalize, 3 per radix pass, 3 for the run list; per table the reduce, one per tree level, the finish, the apply."""
  cap = sum(claim_set_slots(m) for m in per_table)
  bits = int(cap - 1).bit_length()
  passes = max(1, -(-bits // 11))
  return 4 + 3 * passes + 3 + sum(3 + ro.tree_top(ro.n_pieces(m))[0] for m in per_table)


# ------------------------------------------------------------------------------------------------
# the term builder against the restatements
# ------------------------------------------------------------------------------------------------
def test_terms_match_scatter_grad_and_occurrence_rows():
  """A small call: a one-FID SUM part, a CSR MEAN part and a FIRSTN part in column slices of one array; the terms
  equal reduce_order.occurrence_rows (SUM, MEAN) and test_seq_parts_cpu.firstn_terms (ScatterGrad's FIRSTN branch)."""
  rng = np.random.default_rng(5)
  D, L = 8, 3
  lens = rng.integers(0, 7, 20)
  lens[:3] = [0, L, L + 3]
  fo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
  mo = np.concatenate([[0], np.cumsum(rng.integers(1, 5, 15))]).astype(np.int32)
  s = Part("t", rng.integers(0, 9, 12))
  m = Part("t", rng.integers(0, 9, int(mo[-1])), mo, "mean")
  f = Part("t", rng.integers(0, 9, int(fo[-1])), fo, "firstn", L)
  s.col, m.col, f.col = 4, 16, 28
  grad = rng.standard_normal((20, 28 + L * D + 4)).astype(np.float32)
  np.testing.assert_array_equal(s.terms(grad, D).view(np.uint32), grad[:12, 4:12].view(np.uint32))
  want_m = ro.occurrence_rows(grad[:15, 16:24], int(mo[-1]), mo, "mean")
  np.testing.assert_array_equal(m.terms(grad, D).view(np.uint32), want_m.view(np.uint32))
  want_f = firstn_terms(grad[:, 28:28 + L * D].reshape(20, L, D), fo, L, int(fo[-1]))
  np.testing.assert_array_equal(f.terms(grad, D).view(np.uint32), want_f.view(np.uint32))
  assert (f.terms(grad, D)[f.where()[1] >= L].view(np.uint32) == 0).all()   # +0.0, not -0.0
  for p in (s, m, f):
    t = p.terms(grad, D)
    for k in range(p.fids.size):
      c = p.cell(k, D)
      if c is None:
        continue
      r, col = c
      x = grad[r, col:col + D]
      if p.pooling == "mean":
        x = x / np.float32(np.diff(p.offs)[r])
      np.testing.assert_array_equal(t[k].view(np.uint32), x.view(np.uint32))


def test_bf16_widen_is_exact_and_rounds_to_nearest_even():
  x = np.array([0x3F808000, 0x3F818000, 0x3F808001, 0x80000001, 0x7F7FFFFF, 0xFF800000], np.uint32).view(np.float32)
  got = bf16_widen(x).view(np.uint32)
  assert got.tolist() == [0x3F800000, 0x3F820000, 0x3F810000, 0x80000000, 0x7F800000, 0xFF800000]
  assert (got & 0xFFFF == 0).all()


def test_table_sums_take_the_tables_own_occurrence_count():
  """The tree depth of a table's reduce follows its own range (launch_reduce: np from b.n - b.lo), not the call's."""
  src = _squash(_read(*BWD))
  assert "const int64_t np = (sa.b.n - sa.b.lo + kPiece - 1) / kPiece;" in src
  assert "sa.piece0 = range->lo / kPiece;" in src
  assert "sa.n_pieces = (range->hi + kPiece - 1) / kPiece - sa.piece0;" in src


# ------------------------------------------------------------------------------------------------
# rules pinned against the sources
# ------------------------------------------------------------------------------------------------
def test_check_grad_rows_rule():
  """dim % 4 == 0 and dim <= 128; stride and column multiples of 4 elements; the base 16-byte aligned for fp32 rows,
  8-byte for bf16 rows."""
  src = _squash(_read(*BWD))
  body = src[src.index("static void check_grad_rows("):]
  body = body[:body.index("// One table's share")]
  assert "if ((D & 3) || D > 128)" in body
  assert "const uintptr_t amask = 4 * (uintptr_t)elem_bytes - 1;" in body
  assert "(grad_stride & 3) || (grad_col & 3) || (reinterpret_cast<uintptr_t>(pooled_grad) & amask)" in body
  assert re.search(r'check_grad_rows\("pool_backward_parts", mt->tables\[p\.table\]\.dim, p\.rows_dev, p\.stride, '
                   r'p\.col, nullptr, bf16 \? 2 : 4\);', src)
  assert set(FP32_DIMS + BF16_DIMS) <= {d for d in range(4, 129, 4)}


def test_launch_reduce_halves_the_group_for_two_vectors_per_lane():
  src = _squash(_read(*BWD))
  assert "const bool two = knob(KNOB_SEG_VPL) == 2;" in src
  assert "if (two && GG >= 8) {" in src
  assert ("if (bf16) launch_seg<(GG >= 8 ? GG / 2 : GG), (GG >= 8 ? 2 : 1), false, true>(sa, po, defer_short, s);"
          in src)
  assert "if (bf16) launch_seg<GG, 1, false, true>(sa, po, defer_short, s);" in src
  assert "if (knob(KNOB_SEG_AHEAD)) launch_seg2<GL, VPL, PLAIN, true, BF16>" in src
  assert "BF16 ? bf16_seg_reduce_kernel<GL, VPL, AHEAD> : seg_reduce_kernel<GL, VPL, PLAIN, AHEAD>" in src
  # a parts call never takes the PLAIN form: its rows come through the occurrence map
  assert ("const bool plain = sa.b.occ_row == nullptr && sa.b.occ_src == nullptr &&" in src and
          "a.occ_src = w.occ_src;" in src)
  knobs = _squash(_read("monolith_b200", "csrc", "table.cu"))
  assert '{"seg_vpl", 1}' in knobs and '{"seg_ahead", 1}' in knobs   # the defaults


def test_every_reachable_bf16_reduce_instantiation_is_aimed_at():
  """The census target: <4|8|16|32, 1, true|false> and <4|8|16, 2, true|false>, 14 in all, reached by the default
  knobs, seg_vpl = 2 and seg_ahead = 0 at the four widths."""
  from tests.test_gpu_reduce_order import KNOBS
  got = {seg_kernel(G, True, **{k: v for k, v in s.items() if k in ("seg_vpl", "seg_ahead")})
         for G in GS for s in [{}] + KNOBS}
  want = ({f"bf16_seg_reduce_kernel<{g},1,{a}>" for g in GS for a in ("true", "false")} |
          {f"bf16_seg_reduce_kernel<{g},2,{a}>" for g in (4, 8, 16) for a in ("true", "false")})
  assert got == want and len(want) == 14


def test_apply_opt_sel_rule():
  src = _squash(_read(*BWD))
  assert ("const int opt_sel = (ht.segs.size() == 1 && ht.segs[0].opt_type <= MONO_OPT_ADAM) ? ht.segs[0].opt_type "
          ": -1;" in src)
  assert "bf16 ? bf16_runs_apply_kernel<GG, OO> : runs_apply_kernel<GG, OO>" in src
  assert "launch_apply(a, G, apply_opt_sel(ht), Mk, s, bf16);" in src
  hdr = _squash(_read("include", "mono_emb.h"))
  for name, code in OPT_CODE.items():
    assert f"MONO_OPT_{name.upper()} = {code}," in hdr


def test_tables_are_ranged_in_table_order():
  """run_pool_backward_parts gives table k's occurrences the range after those of tables < k (parts table-major, part
  order inside a table), and the Python tables are indexed in sorted-name order: so the boundary cases lay tables out
  by name."""
  src = _squash(_read(*BWD))
  body = src[src.index("void run_pool_backward_parts("):]
  body = body[:body.index("// Deterministic replacement")]
  assert "for (int k = 0; k < K; ++k) { const int lr_off = n_lr;" in body
  assert "c.occ_begin = occ; c.occ_end = occ + per_table[k];" in body
  assert "for (int k = 0; k < K; ++k) for (int i = 0; i < n_parts; ++i) { const mono_pool_part& p = parts[i]; " \
         "if (p.table != k || p.n_fids == 0) continue;" in body
  assert "const SortedRange rg = {ct[q].occ_begin, ct[q].occ_end, mean[k] != 0};" in body
  py = _squash(_read("monolith_b200", "multi_hash_table_ops.py"))
  assert "self._table_names: Tuple[str, ...] = tuple(sorted(configs.keys()))" in py
  assert [L % 32 for L in BOUNDARY_LENS] == [1, 31, 0, 1, 31, 1, 1, 1]
  assert {ro.tree_top(ro.n_pieces(L))[0] for L in BOUNDARY_LENS} == {0, 1}


def test_short_runs_are_summed_in_the_apply():
  src = _squash(_read(*BWD))
  assert "constexpr int kApplyRun = 8;" in src
  assert "if (re - rs > (uint32_t)kApplyRun) {" in src


def test_zero_row_holds_a_whole_gradient_row():
  """A FIRSTN occurrence past L reads D elements of the zero row: D <= 128 floats (fp32), 128 bf16 (256 bytes)."""
  capi = _squash(_read("monolith_b200", "csrc", "capi.cu"))
  assert "MONO_CUDA(cudaMalloc((void**)&mt->zero_row, sizeof(float) * 128));" in capi
  assert "MONO_CUDA(cudaMemset(mt->zero_row, 0, sizeof(float) * 128));" in capi
  src = _squash(_read(*BWD))
  assert "src_out[p.occ_begin + m] = !p.seq_len ? src : j < p.seq_len ? src + j * p.dim : zero_row;" in src


def test_launch_count_rule():
  src = _squash(_read(*BWD))
  assert "constexpr int kRadixBits = 11;" in src
  assert "static int sort_passes(int bits) { return std::max(1, (bits + kRadixBits - 1) / kRadixBits); }" in src
  eng = _squash(_read("monolith_b200", "csrc", "engine.h"))
  assert "uint32_t cap = 1024; while ((uint64_t)cap < 2 * (uint64_t)n) cap <<= 1;" in eng
  assert call_launches([100]) == 4 + 3 + 3 + 3
  assert call_launches([16385, 10]) == 4 + 3 * 2 + 3 + 4 + 3   # 2^16 + 2^10 slots: 17 bits, two passes; depth 1


def test_matrix_dims_meet_every_width_in_both_dtypes():
  from tests.test_gpu_apply_paths import POOL_DIMS
  assert sorted(FP32_DIMS + BF16_DIMS) == sorted(POOL_DIMS)
  for dims in (FP32_DIMS, BF16_DIMS):
    assert {ro.pick_group(d) for d in dims} == set(GS)
