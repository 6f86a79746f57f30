"""The sparse optimizers restated in numpy from the reference sources, against the oracle bit for bit; and the
dispatch rules tests/test_gpu_apply_paths.py aims its cases at, pinned against the CUDA sources.

The restatement is written from runtime/hash_table/optimizer/*_optimizer.cc of the reference (line numbers below),
independently of oracle/oracle.cc, so a mistake the oracle and the kernels share shows here.  Adagrad is left out:
vectors computed with the reference header avx_utils.h pin it (tests/golden/ref_adagrad*.npz).  Every operation is one numpy
float32 operation (round to nearest, no FMA: the oracle is built with -ffp-contract=off); RMSProp computes in
float64 like the reference.  Adam and AMSGrad call an unqualified sqrt on floats (adam_optimizer.cc:64,74,76,
amsgrad_optimizer.cc:66,77,79); the oracle, the kernels and this file take the float overload (NOTES.md).
"""
import ast
import os
import re

import numpy as np
import pytest

from tests import orc
from tests.helpers import opt_from, table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "monolith_b200", "csrc")
F = np.float32


def _read(*path):
  with open(os.path.join(ROOT, *path)) as f:
    return f.read()


def _squash(s):
  return re.sub(r"\s+", " ", s.replace("\\\n", " "))


# ------------------------------------------------------------------------------------------------
# the restatement: one row block [n, dim] per call, state as a list of float32 arrays
# ------------------------------------------------------------------------------------------------
def init_state(name, o, n, D):
  z = lambda: np.zeros((n, D), F)
  if name == "sgd" or name == "moving_average":
    return []
  if name == "ftrl":                                   # ftrl_optimizer.cc:45-52
    return [np.full((n, D), F(o.initial_accumulator_value if o.initial_accumulator_value is not None else 0.1)), z()]
  if name in ("adam", "amsgrad"):                      # adam_optimizer.cc:44-55, amsgrad_optimizer.cc:44-56
    k = 2 if name == "adam" else 3
    return [z() for _ in range(k)] + [np.full((n, 1), F(o.beta1)), np.full((n, 1), F(o.beta2))]
  if name in ("momentum", "rmsprop", "rmspropv2"):     # momentum_optimizer.cc:43-49, rmsprop_optimizer.cc
    return [z()]
  if name == "adadelta":                               # adadelta_optimizer.cc:43-49
    return [z(), z()]
  if name == "group_adagrad":                          # group_adagrad_optimizer.cc:45-48
    return [np.full((n, 1), F(o.initial_accumulator_value))]
  raise ValueError(name)


def step(name, o, lr, w, st, g):
  """One Optimize call on every row of w [n, dim] (in place), gradient g, learning rate lr (float32)."""
  one = F(1)
  lr = F(lr)
  if name == "sgd":                                    # sgd_optimizer.cc:45-47
    w[:] = w - lr * g
  elif name == "ftrl":                                 # ftrl_optimizer.cc:61-75
    norm, zero = st
    l1, l2, beta = F(o.l1_regularization or 0), F(o.l2_regularization or 0), F(o.beta or 0)
    norm_new = norm + g * g
    sigma = (np.sqrt(norm_new) - np.sqrt(norm)) / lr
    zero[:] = zero + (g - sigma * w)
    norm[:] = norm_new
    num = lr * (np.where(np.signbit(zero), one, F(0)) * l1 - zero)
    w[:] = np.where(np.abs(zero) > l1, num / (np.sqrt(norm) + beta + l2 * lr), F(0))
  elif name in ("adam", "amsgrad"):                    # adam_optimizer.cc:64-83, amsgrad_optimizer.cc:66-87
    m, v = st[0], st[1]
    b1p, b2p = st[-2], st[-1]
    b1, b2, eps, wd = F(o.beta1), F(o.beta2), F(o.epsilon), F(o.weight_decay_factor)
    lrt = lr * np.sqrt(one - b2p) / (one - b1p)
    cur = g + wd * w
    new_m = m + (cur - m) * (one - b1)
    new_v = v + (cur * cur - v) * (one - b2)
    den_v = new_v
    if name == "amsgrad":
      vhat = st[2]
      new_vhat = np.where(vhat < new_v, new_v, vhat)   # std::max(vhat, new_v)
      vhat[:] = new_vhat
      den_v = new_vhat
    if o.use_nesterov:
      w[:] = w - ((cur * (one - b1) + b1 * new_m) * lrt) / (np.sqrt(den_v) + eps)
    else:
      w[:] = w - (new_m * lrt) / (np.sqrt(den_v) + eps)
    m[:], v[:] = new_m, new_v
    b1p[:], b2p[:] = b1p * b1, b2p * b2
  elif name == "momentum":                             # momentum_optimizer.cc:56-70
    (n,) = st
    mom, wd = F(o.momentum), F(o.weight_decay_factor)
    dx = lr * (g + wd * w)
    prev = n.copy()
    n[:] = mom * prev - dx
    if o.use_nesterov:
      w[:] = w + (-mom * prev + (one + mom) * n)
    else:
      w[:] = w + n
  elif name in ("rmsprop", "rmspropv2"):               # rmsprop_optimizer.cc:54-67 (v1), :131-144 (v2)
    (n,) = st
    mom, wd = np.float64(F(o.momentum)), np.float64(F(o.weight_decay_factor))
    dx = g.astype(np.float64) + wd * w.astype(np.float64)
    if name == "rmsprop":
      n[:] = (mom * n.astype(np.float64) + (1 - mom) * dx * dx).astype(F)
      eta = np.float64(F(o.learning_rate)) / (np.sqrt(n) + one).astype(np.float64)   # the config's rate
    else:
      n[:] = (mom * n.astype(np.float64) + dx * dx).astype(F)
      eta = np.float64(lr) / (np.sqrt(n) + one).astype(np.float64)
    w[:] = (w.astype(np.float64) - eta * dx).astype(F)
  elif name == "adadelta":                             # adadelta_optimizer.cc:56-70
    acc, upd = st
    rho, eps, wd = F(o.averaging_ratio), F(o.epsilon), F(o.weight_decay_factor)
    cur = g + wd * w
    new_acc = acc * rho + cur * cur * (one - rho)
    u = np.sqrt(upd + eps) / np.sqrt(new_acc + eps) * cur
    w[:] = w - u * lr
    upd[:] = upd * rho + u * u * (one - rho)
    acc[:] = new_acc
  elif name == "moving_average":                       # moving_average_optimizer.cc:45-49
    mom = F(o.momentum)
    w[:] = mom * w + (one - mom) * g
  elif name == "group_adagrad":                        # group_adagrad_optimizer.cc:54-88: the segment is one group
    (gss,) = st
    wd, beta, l2 = F(o.weight_decay_factor), F(o.beta), F(o.l2_regularization_strength)
    D = w.shape[1]
    gd = g + wd * w
    mx = np.zeros((w.shape[0], 1), F)
    for i in range(D):                                 # if (g * g > max) max = g * g, in column order
      sq = gd[:, i:i + 1] * gd[:, i:i + 1]
      mx = np.where(sq > mx, sq, mx)
    gss[:] = gss + mx
    elr = lr / (beta + np.sqrt(gss))
    w[:] = gd - w / elr
    zn = np.zeros((w.shape[0], 1), F)
    for i in range(D):
      zn = zn + w[:, i:i + 1] * w[:, i:i + 1]
    zn = np.sqrt(zn)
    coef = -elr * (zn - l2) / zn
    w[:] = np.where(zn < l2, F(0), coef * w)
  else:
    raise ValueError(name)


# (optimizer, params, lr): the branches no reference golden covers are all here
CASES = [
    ("sgd", {}, 0.05),
    ("ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01}, 0.05),
    ("ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.0, "l2": 0.01}, 0.05),
    ("adam", {}, 0.01), ("adam", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.01),
    ("adam", {"beta1": 0.5, "beta2": 0.25}, 0.01),
    ("momentum", {"weight_decay_factor": 0.01}, 0.02),
    ("momentum", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.02),
    ("rmsprop", {"learning_rate": 0.02, "weight_decay_factor": 0.01}, 0.05),
    ("rmspropv2", {"weight_decay_factor": 0.01}, 0.02),
    ("adadelta", {"weight_decay_factor": 0.01, "averaging_ratio": 0.8, "epsilon": 1e-6}, 0.5),
    ("amsgrad", {}, 0.01), ("amsgrad", {"use_nesterov": True, "weight_decay_factor": 0.01}, 0.01),
    ("amsgrad", {"beta1": 0.5, "beta2": 0.25, "weight_decay_factor": 0.01}, 0.01),
    ("moving_average", {"momentum": 0.8}, 0.0),
    ("group_adagrad", {"l2": 0.05, "beta": 1.0, "initial_accumulator_value": 0.1, "weight_decay_factor": 0.01}, 0.05),
    ("group_adagrad", {"l2": 0.0, "beta": 0.5, "initial_accumulator_value": 0.1}, 0.05),
    ("group_adagrad", {"l2": 1e3, "beta": 1.0}, 0.05),
    ("group_adagrad", {"l2": 5.0, "beta": 1.0}, 0.05),
]
SPECIAL = np.concatenate([np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x7F7FFFFF, 0x7F800000, 0xFF800000,
                                    0x7FC00000], np.uint32).view(F), F([3e38, -3e38])])


def same_bits(got, want, what):
  """uint32 equality, signed zeros included; a NaN only has to meet a NaN (payloads are not compared)."""
  gn, wn = np.isnan(got), np.isnan(want)
  bad = (gn != wn) | (~gn & (got.view(np.uint32) != want.view(np.uint32)))
  assert not bad.any(), f"{what}: {int(bad.sum())} values differ, first at {np.argwhere(bad)[0]}"


def _run(case, D, w0, grads, steps_keys):
  """Oracle and restatement over the same history.  steps_keys[s] = row indices updated in step s."""
  name, params, lr = case
  n = w0.shape[0]
  o = opt_from(name, params, lr)
  cfg = {"t": table([(D, name, params)], [lr])}
  cpu = orc.OracleMultiHashTable(cfg)
  keys = np.arange(1, n + 1, dtype=np.int64) * 7919
  cpu.assign({"t": (keys, w0)}, req_time=1)
  w = w0.copy()
  st = init_state(name, o, n, D)
  with np.errstate(all="ignore"):
    for s, rows in enumerate(steps_keys):
      cpu.apply_gradients({"t": (keys[rows], grads[s][rows])}, req_time=2 + s)
      sub_w, sub_st = w[rows], [x[rows] for x in st]
      step(name, o, lr, sub_w, sub_st, grads[s][rows])
      w[rows] = sub_w
      for x, y in zip(st, sub_st):
        x[rows] = y
  got = cpu.lookup_entry("t", keys)
  want = np.concatenate([w] + [x.reshape(n, -1) for x in st], axis=1)
  same_bits(got[:, :want.shape[1]], want, f"{name} {params}")
  return got


@pytest.mark.parametrize("D", [1, 7, 16])
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}{sorted(c[1].items())}")
def test_restatement_matches_the_oracle_on_random_rows(case, D):
  rng = np.random.default_rng(D * 31 + CASES.index(case))
  n = 64
  w0 = (rng.standard_normal((n, D)) * 0.1).astype(F)
  grads = [(rng.standard_normal((n, D)) * rng.choice([1.0, 1e-3, 30.0], (n, 1))).astype(F) for _ in range(6)]
  _run(case, D, w0, grads, [rng.permutation(n)[:n // 2 + 8 * s] for s in range(6)])


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}{sorted(c[1].items())}")
def test_restatement_matches_the_oracle_on_special_values(case):
  """Weights of -0.0 and subnormals; gradient columns of +-0, +-smallest subnormal, FLT_MAX, +-3e38 (g^2 overflows),
  +-inf and NaN; rows with an all-zero gradient (GroupAdaGrad l2 = 0: 0 / 0, FTRL l1 = 0: z = 0) and rows whose
  gradient (3, 4, 0, ...) on a zero row gives a GroupAdaGrad norm of exactly 5."""
  rng = np.random.default_rng(CASES.index(case))
  n, D = 96, 12
  w0 = rng.standard_normal((n, D)).astype(F)
  w0[:16] = -0.0
  w0[16:32] = (rng.integers(1, 1 << 23, (16, D)).astype(np.uint32) |
               (rng.integers(0, 2, (16, D)).astype(np.uint32) << 31)).view(F)
  w0[80:] = 0.0
  grads = []
  for s in range(3):
    g = rng.standard_normal((n, D)).astype(F)
    m = rng.random(g.shape) < 0.3
    g[m] = SPECIAL[rng.integers(0, SPECIAL.size, int(m.sum()))]
    g[80:88] = 0.0
    g[88:] = 0.0
    g[88:, :2] = (3.0, 4.0)
    grads.append(g)
  got = _run(case, D, w0, grads, [np.arange(n)] * 3)
  if case[1].get("l2") == 5.0:   # zn == l2 exactly: coefficient -0, so the weights are -0.0
    assert (got[88:, :D].view(np.uint32) == 0x80000000).all()


def test_every_uncovered_branch_is_in_the_cases():
  """AMSGrad Nesterov and wd, Adadelta wd, RMSProp v1 / v2 wd, plain Momentum with wd, the GroupAdaGrad l2 edge
  (l2 = 0 and zn == l2) and FTRL with l1 = 0."""
  have = {(c[0], tuple(sorted(c[1].items()))) for c in CASES}
  need = [("amsgrad", "use_nesterov"), ("amsgrad", "weight_decay_factor"), ("adadelta", "weight_decay_factor"),
          ("rmsprop", "weight_decay_factor"), ("rmspropv2", "weight_decay_factor")]
  for opt, key in need:
    assert any(o == opt and any(k == key and v for k, v in p) for o, p in have), (opt, key)
  assert any(c[0] == "momentum" and not c[1].get("use_nesterov") and c[1].get("weight_decay_factor") for c in CASES)
  assert {c[1].get("l2") for c in CASES if c[0] == "group_adagrad"} >= {0.0, 5.0}
  assert any(c[0] == "ftrl" and c[1]["l1"] == 0.0 for c in CASES)


# ------------------------------------------------------------------------------------------------
# the dispatch rules of the GPU file, pinned against the sources
# ------------------------------------------------------------------------------------------------
def test_opt_sel_rule():
  s = _squash(_read("monolith_b200", "csrc", "bwd.cu"))
  assert ("const int opt_sel = (ht.segs.size() == 1 && ht.segs[0].opt_type <= MONO_OPT_ADAM) ? "
          "ht.segs[0].opt_type : -1;") in s
  for o in ("SGD", "ADAGRAD", "FTRL", "ADAM"):
    assert f"case MONO_OPT_{o}: BWD2(GG, MONO_OPT_{o}); break;" in s
  assert "default: BWD2(GG, -1); break;" in s


def test_apply_row_fast_path_condition():
  s = _squash(_read("monolith_b200", "csrc", "rowops.cuh"))
  assert ("if (t->num_segs == 1 && s0.opt_type <= MONO_OPT_ADAM && (D & 3) == 0 && "
          "((reinterpret_cast<uintptr_t>(vals) & 15) == 0)) {") in s
  # the generic path: GroupAdaGrad one lane per segment, the further optimizers element by element
  assert "if (s.opt_type == MONO_OPT_GROUP_ADAGRAD) group_adagrad_segment(" in s
  assert "if (s.opt_type > MONO_OPT_ADAM) {" in s


def test_pick_group():
  from tests.reduce_order import pick_group
  s = _squash(_read("monolith_b200", "csrc", "ops.cu"))
  assert ("int pick_group(int max_dim) { int v = (max_dim + 3) / 4; int g = 4; while (g < v && g < 32) g <<= 1; "
          "return g; }") in s
  assert [pick_group(d) for d in (1, 16, 17, 32, 33, 64, 65, 128, 129, 260)] == [4, 4, 8, 8, 16, 16, 32, 32, 32, 32]


def _state_rule(src, fn):
  """opt name -> state floats as a function of dim, from the switch of `fn` in src."""
  body = src[src.index(fn):]
  body = body[:body.index("\n}")]
  rule, pending = {}, []
  for m in re.finditer(r"case MONO_OPT_(\w+):|return ([^;]+);", body):
    if m.group(1):
      pending.append(m.group(1))
      continue
    expr = m.group(2).replace("s.dim", "d").replace("//", "")
    for p in pending:
      rule[p] = expr
    pending = []
  return rule


def test_state_floats_agree():
  """table.cu (the row layout), rowops.cuh (the kernels) and the oracle size every optimizer's state alike."""
  opts = re.findall(r"MONO_OPT_(\w+) = \d+", _read("include", "mono_emb.h"))
  a = _state_rule(_read("monolith_b200", "csrc", "table.cu"), "static int state_floats(")
  b = _state_rule(_read("monolith_b200", "csrc", "rowops.cuh"), "int state_floats_dev(")
  c = _state_rule(_read("oracle", "oracle.cc"), "int StateFloats(")
  for o in opts:
    for d in (1, 7, 16):
      got = [eval(r.get(o, "0"), {"d": d}) for r in (a, b, c)]   # rowops.cuh: default 0 (SGD, MovingAverage)
      assert len(set(got)) == 1, (o, d, got)
  assert set(a) == set(opts) and set(c) == set(opts)


def test_every_optimizer_is_in_the_gpu_matrix():
  """A new MONO_OPT_* cannot land without a row in test_gpu_apply_paths.CONFIGS."""
  opts = {o.lower() for o in re.findall(r"MONO_OPT_(\w+) = \d+", _read("include", "mono_emb.h"))}
  tree = ast.parse(_read("tests", "test_gpu_apply_paths.py"))
  configs = next(n.value for n in tree.body if isinstance(n, ast.Assign) and n.targets[0].id == "CONFIGS")
  names = {ast.literal_eval(e)[1] for e in configs.elts}
  assert opts == names, f"missing: {sorted(opts - names)}"
