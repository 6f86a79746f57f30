"""ShardedStep.step_parts: several features of one table in one sharded step, on every exchange.

At world 1 (one rank owns every FID), for the "direct" (csrc/xstep.cu), "peer" (push and pull bulk) and "nccl"
exchanges:
1. one "sum" or "mean" part is bit for bit step() on the same inputs (outputs and every table entry);
2. the forward of mixed parts (sum and mean, CSR and one-FID rows, firstn rows shorter than, equal to and longer than
   L, absent FIDs, parts writing disjoint columns of one tensor) is bit for bit lookup_pool_parts on a twin table that
   holds the same state, and the backward with gradients whose sums are exact in any order leaves the table bit for bit
   as pool_backward_parts leaves the twin;
3. with random gradients, every table entry equals the CPU oracle fed the per-FID sums in the reduce's association
   (tests/reduce_order.py) over the concatenated occurrences, a FID shared by several parts and one whose occurrences
   all lie past L included;
4. bfloat16 outputs are the float32 outputs rounded once, and bfloat16 gradients give the table of the same gradients
   widened to float32;
5. grad_scale is the unscaled step on gradients pre-multiplied in float32;
6. the forward adds at most one launch per distinct pooling kernel over step()'s forward, the backward at most one;
7. every rejected input raises before any device work and leaves the table unchanged.
8. A world-2 case against one global oracle table runs where two GPUs are present.
Every comparison goes through uint32 views."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import orc
from tests import reduce_order as ro
from tests.helpers import table

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 16
EXCHANGES = ["direct", "peer-push", "peer-pull", "nccl"]
BF = torch.bfloat16
SLOT = np.int64(5) << 48


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


@pytest.fixture
def exchange(request, dev, monkeypatch):
  """The exchange name of ShardedStep; world-1 NCCL needs a process group."""
  import torch.distributed as dist
  ex = request.param
  if ex.startswith("peer-"):
    monkeypatch.setenv("MONO_PEER_BULK", ex.split("-")[1])
  ex = ex.split("-")[0]
  if ex == "nccl":
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1, device_id=dev)
  yield ex
  if ex == "nccl":
    dist.destroy_process_group()


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def cfg():
  return {"t": table([(D, "adagrad", {"initial_accumulator_value": 0.1})], [0.1], capacity=1 << 16)}


def assert_same(got, want, what):
  g = np.ascontiguousarray(got.float().cpu().numpy() if isinstance(got, torch.Tensor) else got, np.float32)
  w = np.ascontiguousarray(want.float().cpu().numpy() if isinstance(want, torch.Tensor) else want, np.float32)
  assert g.shape == w.shape, f"{what}: shape {g.shape} vs {w.shape}"
  gn, wn = np.isnan(g), np.isnan(w)
  bad = (gn != wn) | (~gn & (g.view(np.uint32) != w.view(np.uint32)))
  if bad.any():
    r = tuple(np.argwhere(bad)[0])
    raise AssertionError(f"{what}: {int(bad.sum())} values differ, first at {r}: {g[r]!r} vs {w[r]!r}")


def assert_bits(got, want, what):
  """bf16 tensors bit for bit (int16 views)."""
  assert got.dtype == want.dtype == BF and got.shape == want.shape, what
  assert torch.equal(got.view(torch.int16), want.view(torch.int16)), what


def export(tab):
  ks, rows = [], []
  for ids, raw in tab.export("t", chunk=1 << 14):
    ks.append(ids.cpu().numpy())
    rows.append(raw.cpu().numpy())
  ks, rows = np.concatenate(ks), np.concatenate(rows)
  o = np.argsort(ks)
  return ks[o], rows[o]


def assert_tables(a, b, what):
  (ka, ra), (kb, rb) = a, b
  np.testing.assert_array_equal(ka, kb, err_msg=what)
  assert_same(ra, rb, what)


# ------------------------------------------------------------------------------------------------
# batches: the parts of one step (numpy), then as PoolParts
# ------------------------------------------------------------------------------------------------
L = 5


def make_step(rng, B, step, exact=False):
  """The parts of one step as dicts: fids, offs (None: one FID per row), pooling, L, and the gradient rows.
  Three parts write disjoint columns of one tower tensor ([B, 3 D]); the FirstN part has its own [B, L D] tensor.
  exact: gradients k / 16 with small integers k and MEAN rows of 1, 2 or 4 FIDs, so every sum is exact in any order."""
  vocab = SLOT | rng.integers(0, 400, 4000).astype(np.int64)
  absent = SLOT | (np.int64(1) << 40) | np.arange(50, dtype=np.int64)   # never trained: absent in the forward
  past_l = SLOT | np.int64(777_000 + step)                               # occurs only at positions >= L

  def fids_of(n):
    f = rng.choice(vocab, n)
    m = rng.random(n) < 0.05
    f[m] = rng.choice(absent, int(m.sum()))
    f[rng.random(n) < 0.1] = SLOT | np.int64(3)                           # shared by every part
    return f

  def grad(rows, width):
    if exact:
      return (rng.integers(-8, 9, (rows, width)) / 16).astype(np.float32)
    return (rng.standard_normal((rows, width)) * 2).astype(np.float32)

  parts = []
  # one-FID SUM rows
  parts.append(dict(fids=fids_of(B), offs=None, pooling="sum", L=0, col=0))
  # CSR SUM rows, some empty
  n = rng.integers(0, 4, B)
  parts.append(dict(fids=fids_of(int(n.sum())), offs=np.concatenate([[0], np.cumsum(n)]).astype(np.int32),
                    pooling="sum", L=0, col=D))
  # CSR MEAN rows
  n = rng.choice([1, 2, 4], B) if exact else rng.integers(1, 6, B)
  parts.append(dict(fids=fids_of(int(n.sum())), offs=np.concatenate([[0], np.cumsum(n)]).astype(np.int32),
                    pooling="mean", L=0, col=2 * D))
  # FirstN: rows shorter than, equal to and longer than L; past_l only past L
  n = rng.integers(0, 2 * L + 1, B)
  n[:3] = [L - 2, L, L + 3]
  offs = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
  f = fids_of(int(n.sum()))
  for r in range(B):
    if n[r] > L:
      f[offs[r] + L] = past_l
  parts.append(dict(fids=f, offs=offs.astype(np.int32), pooling="firstn", L=L, col=0))
  for p in parts:
    rows = B
    width = D * (p["L"] or 1)
    p["g"] = grad(rows, width)
  return parts


def pool_parts(parts, dev, dtype=torch.float32, tower=None):
  """PoolParts with output rows: the first three write columns 0, D, 2D of one [B, 3D] tensor."""
  from monolith_b200.multi_hash_table_ops import PoolPart
  B = parts[0]["g"].shape[0]
  tower = torch.full((B, 3 * D), float("nan"), dtype=dtype, device=dev) if tower is None else tower
  seq = torch.full((B, L * D), float("nan"), dtype=dtype, device=dev)
  out = []
  for p in parts:
    rows = seq if p["pooling"] == "firstn" else tower
    out.append(PoolPart("t", T(p["fids"], dev), None if p["offs"] is None else T(p["offs"], dev), p["pooling"], rows,
                        p["col"], p["L"]))
  return out, tower, seq


def grad_tensors(parts, dev, dtype=torch.float32, scale=None):
  """The gradient of each part in the layout of its output rows: the tower gradient [B, 3D] for the three tower parts
  (each at its column), the FirstN gradient [B, L D] for the FirstN part."""
  tower = T(np.concatenate([p["g"] for p in parts[:3]], axis=1), dev)
  seq = T(parts[3]["g"], dev)
  if scale is not None:
    tower, seq = tower * scale, seq * scale
  tower, seq = tower.to(dtype), seq.to(dtype)
  return [tower, tower, tower, seq]


def grad_parts(parts, dev, gs):
  from monolith_b200.multi_hash_table_ops import PoolPart
  return [PoolPart("t", T(p["fids"], dev), None if p["offs"] is None else T(p["offs"], dev), p["pooling"], g,
                   p["col"], p["L"]) for p, g in zip(parts, gs)]


def new_step(tab, exchange, dev):
  from monolith_b200.distributed_ps import ShardedStep
  return ShardedStep(tab, "t", D, 1, 0, dev, exchange=exchange)


def close(st):
  torch.cuda.synchronize()
  if st.exchange == "direct":
    st.close_direct()
  elif st.window is not None:
    st.window.close()


def prefill(tab, dev, seed=1):
  """Train most of the vocabulary once, so the steps mix resident and new FIDs."""
  rng = np.random.default_rng(seed)
  ids = np.unique(SLOT | rng.integers(0, 300, 300).astype(np.int64))
  g = rng.standard_normal((ids.size, D)).astype(np.float32)
  tab.apply_gradients({"t": (T(ids, dev), T(g, dev))}, req_time=10, ids_unique=True)
  return ids, g


# ------------------------------------------------------------------------------------------------
# 1. one part == step()
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pooling", ["sum", "mean"])
@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_one_part_is_step(exchange, pooling, dev):
  from monolith_b200 import MultiHashTable
  from monolith_b200.multi_hash_table_ops import PoolPart
  rng = np.random.default_rng(11)
  a, b = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
  prefill(a, dev), prefill(b, dev)
  sa, sb = new_step(a, exchange, dev), new_step(b, exchange, dev)
  try:
    for step in range(3):
      B = 3000 + 500 * step
      offs, rows, M = None, 4 * B, 4 * B
      if pooling == "mean":
        offs = np.concatenate([[0], np.cumsum(rng.integers(0, 8, B))]).astype(np.int32)
        rows, M = B, int(offs[-1])
      fids = SLOT | rng.integers(0, 600, M).astype(np.int64)
      fids[rng.random(M) < 0.2] = SLOT | np.int64(3)             # a long run: several pieces of the reduce
      g = (rng.standard_normal((rows, D)) * 3).astype(np.float32)
      ro_t = None if offs is None else T(offs, dev)
      out_a = torch.empty(rows, D, device=dev)
      sa.step(T(fids, dev), T(g, dev), out_a, 20 + step, ro_t, pooling)
      out_b = torch.empty(rows, D, device=dev)
      sb.step_parts([PoolPart("t", T(fids, dev), ro_t, pooling, out_b)], [T(g, dev)], 20 + step)
      torch.cuda.synchronize()
      assert_same(out_b, out_a, f"forward, step {step}")
    assert_tables(export(b), export(a), "table")
  finally:
    close(sa), close(sb)


# ------------------------------------------------------------------------------------------------
# 2. mixed parts: forward == lookup_pool_parts on a twin, backward == pool_backward_parts (exact sums)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_mixed_parts_match_the_parts_calls(exchange, dev):
  from monolith_b200 import MultiHashTable
  rng = np.random.default_rng(21)
  a, twin = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
  prefill(a, dev), prefill(twin, dev)
  st = new_step(a, exchange, dev)
  try:
    for step in range(3):
      parts = make_step(rng, 700 + 100 * step, step, exact=True)
      pa, tower_a, seq_a = pool_parts(parts, dev)
      pt, tower_t, seq_t = pool_parts(parts, dev)
      twin.lookup_pool_parts(pt)
      outs = st.step_parts(pa, grad_tensors(parts, dev), 30 + step)
      assert outs[0] is tower_a and outs[3] is seq_a
      twin.pool_backward_parts(grad_parts(parts, dev, grad_tensors(parts, dev)), req_time=30 + step)
      torch.cuda.synchronize()
      assert_same(tower_a, tower_t, f"tower columns, step {step}")
      assert_same(seq_a, seq_t, f"firstn positions, step {step}")
      assert not torch.isnan(tower_a).any() and not torch.isnan(seq_a).any()
      assert_tables(export(a), export(twin), f"table after step {step}")
  finally:
    close(st)


# ------------------------------------------------------------------------------------------------
# 3. random gradients: the CPU oracle with the reduce's association
# ------------------------------------------------------------------------------------------------
def occurrence_rows(parts):
  """The gradient term of every occurrence of the concatenated parts (part order, then occurrence order)."""
  xs, keys = [], []
  for p in parts:
    g, f = p["g"], p["fids"]
    if p["offs"] is None:
      xs.append(g)
    elif p["pooling"] == "firstn":
      offs = p["offs"]
      x = np.zeros((f.size, D), np.float32)
      for r in range(offs.size - 1):
        for j in range(min(offs[r + 1] - offs[r], p["L"])):
          x[offs[r] + j] = g[r, j * D:(j + 1) * D]
      xs.append(x)
    else:
      xs.append(ro.occurrence_rows(g, f.size, p["offs"], p["pooling"]))
    keys.append(f)
  return np.concatenate(xs), np.concatenate(keys)


def oracle_forward(cpu, parts):
  outs = []
  for p in parts:
    if p["pooling"] != "firstn":
      outs.append(cpu.lookup_pool("t", p["fids"], p["offs"], p["pooling"]))
      continue
    rows = cpu.lookup({"t": p["fids"]})["t"]
    offs = p["offs"]
    o = np.zeros((offs.size - 1, L * D), np.float32)
    for r in range(offs.size - 1):
      for j in range(min(offs[r + 1] - offs[r], L)):
        o[r, j * D:(j + 1) * D] = rows[offs[r] + j]
    outs.append(o)
  return outs


def oracle_step(cpu, parts, ts):
  x, keys = occurrence_rows(parts)
  with np.errstate(all="ignore"):
    u, sums, _ = ro.call_sums(x, keys, ro.pick_group(D))
  cpu.apply_gradients({"t": (u, sums)}, req_time=ts)


@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_mixed_parts_match_the_oracle(exchange, dev):
  from monolith_b200 import MultiHashTable
  rng = np.random.default_rng(31)
  a, cpu = MultiHashTable(cfg(), device=dev), orc.OracleMultiHashTable(cfg())
  ids, g0 = prefill(a, dev)
  cpu.apply_gradients({"t": (ids, g0)}, req_time=10)
  st = new_step(a, exchange, dev)
  try:
    for step in range(3):
      parts = make_step(rng, 1500 + 200 * step, step)
      want = oracle_forward(cpu, parts)
      pa, tower, seq = pool_parts(parts, dev)
      st.step_parts(pa, lambda: grad_tensors(parts, dev), 40 + step)    # the gradients from a callable
      oracle_step(cpu, parts, 40 + step)
      torch.cuda.synchronize()
      for i in range(3):
        assert_same(tower[:, i * D:(i + 1) * D], want[i], f"part {i}, step {step}")
      assert_same(seq, want[3], f"firstn part, step {step}")
      k, e = export(a)
      np.testing.assert_array_equal(k, cpu.keys("t"))
      assert_same(e, cpu.lookup_entry("t", k), f"table after step {step}")
      past = SLOT | np.int64(777_000 + step)
      assert past in k, "a FID seen only past L is still inserted and stepped"
  finally:
    close(st)


# ------------------------------------------------------------------------------------------------
# 4. bf16 forms, 5. grad_scale
# ------------------------------------------------------------------------------------------------
def run_steps(exchange, dev, batches, fwd_dtype, grad_dtype, scale=None, premul=None):
  """-> forward outputs of every step and the final table."""
  from monolith_b200 import MultiHashTable
  a = MultiHashTable(cfg(), device=dev)
  prefill(a, dev)
  st = new_step(a, exchange, dev)
  outs = []
  try:
    for step, parts in enumerate(batches):
      pa, tower, seq = pool_parts(parts, dev, fwd_dtype)
      gs = grad_tensors(parts, dev, grad_dtype, scale=premul)
      st.step_parts(pa, gs, 50 + step,
                    grad_scale=None if scale is None else torch.full((1,), scale, dtype=torch.float32, device=dev))
      outs += [tower.clone(), seq.clone()]
    torch.cuda.synchronize()
  finally:
    close(st)
  return outs, export(a)


@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_bf16_forms(exchange, dev):
  rng = np.random.default_rng(41)
  batches = [make_step(rng, 900, s) for s in range(2)]
  for b in batches:   # bf16-representable gradients: the widened rows are the same values
    for p in b:
      p["g"] = torch.from_numpy(p["g"]).to(BF).float().numpy()
  o16, t16 = run_steps(exchange, dev, batches, BF, BF)
  o32, t32 = run_steps(exchange, dev, batches, torch.float32, torch.float32)
  for i, (x, y) in enumerate(zip(o16, o32)):
    assert_bits(x, y.to(BF), f"bf16 output {i}")
  assert_tables(t16, t32, "table after bf16 gradients")


@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_grad_scale(exchange, dev):
  """The scaled step is the unscaled step on gradients pre-multiplied in float32; with bfloat16 gradients it is the
  float32 scaled step on the widened gradients."""
  rng = np.random.default_rng(51)
  batches = [make_step(rng, 900, s) for s in range(2)]
  for b in batches:
    for p in b:
      p["g"] = torch.from_numpy(p["g"]).to(BF).float().numpy()
  s = np.float32(0.3)
  o1, t1 = run_steps(exchange, dev, batches, torch.float32, torch.float32, scale=float(s))
  o2, t2 = run_steps(exchange, dev, batches, torch.float32, torch.float32, premul=torch.tensor(float(s)))
  for i, (x, y) in enumerate(zip(o1, o2)):
    assert_same(x, y, f"output {i}")
  assert_tables(t1, t2, "table with grad_scale")
  o3, t3 = run_steps(exchange, dev, batches, BF, BF, scale=float(s))
  for i, (x, y) in enumerate(zip(o3, o1)):
    assert_bits(x, y.to(BF), f"bf16 output {i}")
  assert_tables(t3, t1, "table with grad_scale and bf16 gradients")


# ------------------------------------------------------------------------------------------------
# 6. launches
# ------------------------------------------------------------------------------------------------
def launches():
  from monolith_b200 import _lib
  torch.cuda.synchronize()
  return int(_lib.load().mono_kernel_launch_count())


@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_launch_counts(exchange, dev):
  from monolith_b200 import MultiHashTable
  rng = np.random.default_rng(61)
  parts = make_step(rng, 800, 0)
  flat = np.concatenate([p["fids"] for p in parts])
  a, b = MultiHashTable(cfg(), device=dev), MultiHashTable(cfg(), device=dev)
  sa, sb = new_step(a, exchange, dev), new_step(b, exchange, dev)
  try:
    counts = {}
    for rep in range(2):   # the second step: windows, scratch and table capacity are in place
      mark = {}
      out = torch.empty(flat.size, D, device=dev)
      g = torch.zeros(flat.size, D, device=dev)
      c0 = launches()

      def flat_grad():
        mark["f"] = launches()
        return g
      sa.step(T(flat, dev), flat_grad, out, 60 + rep)
      counts["step"] = (mark["f"] - c0, launches() - mark["f"])
      pa, _, _ = pool_parts(parts, dev)
      gs = grad_tensors(parts, dev)
      c0 = launches()

      def parts_grad():
        mark["p"] = launches()
        return gs
      sb.step_parts(pa, parts_grad, 60 + rep)
      counts["parts"] = (mark["p"] - c0, launches() - mark["p"])
    kinds = 3   # the row copy (one-FID part), the pooling kernel (CSR parts), the FirstN kernel
    assert counts["parts"][0] <= counts["step"][0] + kinds, counts
    assert counts["parts"][1] <= counts["step"][1] + 1, counts
  finally:
    close(sa), close(sb)


# ------------------------------------------------------------------------------------------------
# 7. rejected inputs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exchange", EXCHANGES, indirect=True)
def test_rejected_inputs(exchange, dev):
  from monolith_b200 import MultiHashTable, _lib
  from monolith_b200.multi_hash_table_ops import PoolPart
  import dataclasses
  rng = np.random.default_rng(71)
  two = {"t": cfg()["t"], "u": table([(D, "sgd", {})], [0.1])}
  a = MultiHashTable(two, device=dev)
  prefill(a, dev)
  st = new_step(a, exchange, dev)
  parts = make_step(rng, 300, 0)
  try:
    st.step_parts(pool_parts(parts, dev)[0], grad_tensors(parts, dev), 70)   # a good step first
    before = export(a)

    def refused(pa, gs, err=(ValueError, _lib.MonoError)):
      c0 = launches()
      with pytest.raises(err):
        st.step_parts(pa, gs, 71)
      assert launches() == c0, "device work before the refusal"
      assert_tables(export(a), before, "table after a refused step")

    pa, _, _ = pool_parts(parts, dev)
    gs = grad_tensors(parts, dev)
    refused([dataclasses.replace(pa[0], slot="u")] + pa[1:], gs)                      # another table
    refused(pa[:1] + [dataclasses.replace(p, rows=p.rows.to(BF)) for p in pa[1:]], gs)   # mixed output dtypes
    refused(pa, gs[:1] + [g.to(BF) for g in gs[1:]])                                  # mixed gradient dtypes
    refused(pa, gs[:-1])                                                              # too few gradients
    refused(pa, gs + gs[:1])                                                          # too many
    refused(pa, gs[:1] + [gs[1][:-1]] + gs[2:])                                       # a gradient with too few rows
    wide = torch.zeros(gs[0].shape[0], 3 * D + 2, device=dev)                         # stride % 4 != 0
    refused(pa, [wide] + gs[1:])
    refused(pa, gs[0])                                                                # not a list
    # FirstN with n_rows * max_seq_len over 2^31 (its rows are a zero-stride view: no memory behind them)
    n_rows, Lbig = 1 << 20, 1 << 12
    f = torch.full((n_rows,), int(SLOT | 3), dtype=torch.int64, device=dev)
    rows = torch.zeros(Lbig * D, device=dev).as_strided((n_rows, Lbig * D), (0, 1))
    big = PoolPart("t", f, None, "firstn", rows, 0, Lbig)
    refused([big], [rows])
    refused([], [])
  finally:
    close(st)


# ------------------------------------------------------------------------------------------------
# 8. world 2 against one global oracle table
# ------------------------------------------------------------------------------------------------
def _world2_worker(rank, world, port, q, exchange):
  try:
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    if exchange.startswith("peer-"):
      os.environ["MONO_PEER_BULK"] = exchange.split("-")[1]
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from monolith_b200 import MultiHashTable
    from monolith_b200.distributed_ps import ShardedStep
    tab = MultiHashTable(cfg(), device=dev)
    st = ShardedStep(tab, "t", D, world, rank, dev, exchange=exchange.split("-")[0])
    outs = []
    for step in range(3):
      parts = make_step(np.random.default_rng(1000 * step + rank), 600, step)
      pa, tower, seq = pool_parts(parts, dev)
      st.step_parts(pa, grad_tensors(parts, dev), 80 + step)
      outs.append((tower.cpu().numpy(), seq.cpu().numpy()))
    torch.cuda.synchronize()
    q.put((rank, outs, export(tab)))
    dist.barrier()
    close(st)
    dist.destroy_process_group()
  except Exception:
    import traceback
    q.put((rank, "ERROR", traceback.format_exc()))
    raise


@pytest.mark.parametrize("exchange", EXCHANGES)
def test_world_2(exchange):
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  import torch.multiprocessing as mp
  world = 2
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = 29500 + (os.getpid() % 90) + {"peer-pull": 0, "peer-push": 3, "nccl": 7, "direct": 11}[exchange]
  procs = [ctx.Process(target=_world2_worker, args=(r, world, port, q, exchange)) for r in range(world)]
  for p in procs:
    p.start()
  got = sorted([q.get(timeout=300) for _ in range(world)], key=lambda x: x[0])
  for g in got:
    assert g[1] != "ERROR", g[2]
  for p in procs:
    p.join(timeout=60)
  glob = orc.OracleMultiHashTable(cfg())
  for step in range(3):
    batches = [make_step(np.random.default_rng(1000 * step + r), 600, step) for r in range(world)]
    for r, parts in enumerate(batches):
      want = oracle_forward(glob, parts)
      tower, seq = got[r][1][step]
      for i in range(3):
        assert_same(tower[:, i * D:(i + 1) * D], want[i], f"rank {r}, part {i}, step {step}")
      assert_same(seq, want[3], f"rank {r}, firstn part, step {step}")
    for parts in batches:   # every owner applies requester 0's sums, then requester 1's
      oracle_step(glob, parts, 80 + step)
  keys = glob.keys("t")
  for r in range(world):
    mine = keys[(keys.view(np.uint64) % np.uint64(world)) == r]
    k_r, e_r = got[r][2]
    np.testing.assert_array_equal(k_r, mine)
    assert_same(e_r, glob.lookup_entry("t", mine), f"rank {r} table")
