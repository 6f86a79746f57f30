"""2-GPU NCCL test of the FID-hash sharded exchange with the CUDA engine on every rank, against ONE
global oracle table (same protocol as tests/test_distributed_cpu.py).  Needs >= 2 GPUs; skipped
otherwise."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
  try:
    _worker_body(rank, world, port, q)
  except Exception as e:  # report instead of letting the parent wait for the queue timeout
    import traceback
    q.put((rank, "ERROR", traceback.format_exc()))
    raise


def _worker_body(rank, world, port, q):
  sys.path.insert(0, ROOT)
  import torch.distributed as dist
  from tests.test_distributed_cpu import _batch, _configs
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  torch.cuda.set_device(rank)
  dev = torch.device("cuda", rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
  from monolith_b200 import MultiHashTable
  from monolith_b200.distributed_ps import PartitionedHashTable
  table = MultiHashTable(_configs(), device=dev)
  pht = PartitionedHashTable(table, world, rank)
  res = []
  for step in range(3):
    fa, fb, offs_b, ga, gb = _batch(rank, step)
    t = lambda x: torch.from_numpy(x).to(dev)
    pooled, ctx = pht.lookup({"a": t(fa), "b": t(fb)}, row_offsets={"b": t(offs_b)}, pooling={"b": "mean"})
    res.append((pooled["a"].cpu().numpy(), pooled["b"].cpu().numpy()))
    pht.apply_gradients(ctx, {"a": t(ga), "b": t(gb)}, req_time=10 + step)
  state = {}
  for n in table.table_names:
    ks, rows = [], []
    for ids, raw in table.export(n, chunk=1 << 14):
      ks.append(ids.cpu().numpy())
      rows.append(raw.cpu().numpy())
    ks = np.concatenate(ks) if ks else np.zeros(0, np.int64)
    rows = np.concatenate(rows) if rows else np.zeros((0, 1), np.float32)
    order = np.argsort(ks)
    state[n] = (ks[order], rows[order])
  q.put((rank, res, state))
  dist.barrier()
  dist.destroy_process_group()


def test_sharded_exchange_two_gpus():
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  import torch.multiprocessing as mp
  from tests import orc
  from tests.test_distributed_cpu import _batch, _configs
  world = 2
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = 29700 + (os.getpid() % 200)
  procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
  for p in procs:
    p.start()
  got = [q.get(timeout=240) for _ in range(world)]
  for g in got:
    assert g[1] != "ERROR", g[2]
  got = sorted(got, key=lambda x: x[0])
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  glob = orc.OracleMultiHashTable(_configs())
  for step in range(3):
    batches = [_batch(r, step) for r in range(world)]
    for r, (fa, fb, offs_b, ga, gb) in enumerate(batches):
      # table b has dim 5 => unaligned fused buffers => float-atomic grad scatter (like the reference GPU
      # kernel): states, and therefore later lookups, agree to 1e-5 instead of bit for bit
      np.testing.assert_allclose(got[r][1][step][0], glob.lookup_pool("a", fa, None, "sum"), rtol=1e-5, atol=1e-6)
      np.testing.assert_allclose(got[r][1][step][1], glob.lookup_pool("b", fb, offs_b, "mean"), rtol=1e-5, atol=1e-6)
    for r, (fa, fb, offs_b, ga, gb) in enumerate(batches):
      for name, f, g, ro, pool, D in (("a", fa, ga, None, "sum", 8), ("b", fb, gb, offs_b, "mean", 5)):
        u, inv = orc.dedup(f)
        ug = orc.gather_pool_grad(g, inv * D, D, u.size * D, ro, pool).reshape(-1, D)
        glob.apply_gradients({name: (u, ug)}, req_time=10 + step)
  for name in glob.names:
    keys = glob.keys(name)
    for r in range(world):
      mine = keys[(keys.view(np.uint64) % np.uint64(world)) == r]
      k_r, e_r = got[r][2][name]
      np.testing.assert_array_equal(k_r, mine)
      want = glob.lookup_entry(name, mine)
      # table b has dim 5, so the fused buffers are not 16-byte aligned and the backward uses the
      # float-atomic scatter (like the reference GPU kernel): tolerance instead of bit equality
      np.testing.assert_allclose(e_r[:, :-2], want[:, :-2], rtol=1e-5, atol=1e-6)
      np.testing.assert_array_equal(e_r[:, -2:].view(np.uint32), want[:, -2:].view(np.uint32))


# ---- fast path: one grouping shared by forward and backward (ShardedStep) ------------------------
def _fast_batch(rank, step, n=6000):
  rng = np.random.default_rng(1000 * step + rank)
  ids = rng.integers(0, 900, n)
  r = rng.random(n)
  ids[r < 0.25] = 3                       # hot FID shared by both ranks (long run)
  fids = (np.int64(5) << 48) | ids.astype(np.int64)
  g = rng.standard_normal((n, 16)).astype(np.float32)
  return fids, g


def _fast_cfg():
  from tests.helpers import table
  return {"t": table([(16, "adagrad", {})], [0.1])}


def _fast_worker(rank, world, port, q, exchange="peer", filtered=False):
  try:
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from monolith_b200 import MultiHashTable
    from monolith_b200.distributed_ps import ShardedStep
    table = MultiHashTable(_fast_cfg(), device=dev)
    if filtered:
      table.set_hash_filter("t", 2_000_000, 2)
    if exchange.startswith("peer-"):
      os.environ["MONO_PEER_BULK"] = exchange.split("-")[1]
      exchange = "peer"
    st = ShardedStep(table, "t", 16, world, rank, dev, exchange=exchange)
    pooled_all = []
    devb = [torch.from_numpy(_fast_batch(rank, step)[0]).to(dev) for step in range(3)]
    for step in range(3):
      fids, g = _fast_batch(rank, step)
      out = torch.empty(fids.size, 16, device=dev)
      if filtered and exchange == "direct":   # refused before anything is pushed, on both ranks
        try:
          st.step(devb[step], torch.from_numpy(g).to(dev), out, 20 + step)
        except RuntimeError as e:
          assert "hash filter needs world 1" in str(e), e
          torch.cuda.synchronize()
          q.put((rank, "REFUSED", None))
          dist.barrier()
          st.close_direct()
          dist.destroy_process_group()
          return
        raise AssertionError("a filtered table's direct step at world 2 was not refused")
      st.step(devb[step], torch.from_numpy(g).to(dev), out, 20 + step)
      if exchange == "direct" and step + 1 < 3:
        st.prepare(devb[step + 1])          # next batch's grouping on a side stream, under this step's exchange
      pooled_all.append(out.cpu().numpy())
    ks, rows = [], []
    for ids, raw in table.export("t", chunk=1 << 14):
      ks.append(ids.cpu().numpy()); rows.append(raw.cpu().numpy())
    ks, rows = np.concatenate(ks), np.concatenate(rows)
    o = np.argsort(ks)
    q.put((rank, pooled_all, (ks[o], rows[o])))
    dist.barrier()
    if exchange == "direct":
      st.close_direct()
    dist.destroy_process_group()
  except Exception:
    import traceback
    q.put((rank, "ERROR", traceback.format_exc()))
    raise


@pytest.mark.parametrize("exchange", ["direct", "peer-pull", "peer-push", "nccl"])
def test_sharded_fast_step_two_gpus(exchange):
  """ShardedStep on 2 GPUs == one global oracle table; exchange over NVLink peer windows (bulk data pulled
  by the consumer, or pushed by the fused lookup+send / reduce+send kernels; flag barriers) and over NCCL."""
  _fast_step_two_gpus(exchange, False)


@pytest.mark.parametrize("exchange", ["direct", "peer-pull", "nccl"])
def test_sharded_fast_step_two_gpus_filtered(exchange):
  """The same with an admission filter of threshold 2 on every rank: the owners apply each requester's rows as one
  optimize, so the filter counts a new FID once per requester, as the global table does; the direct exchange refuses
  the backward (its owner insert would count a new FID once per step)."""
  _fast_step_two_gpus(exchange, True)


def _fast_step_two_gpus(exchange, filtered):
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  import torch.multiprocessing as mp
  from tests import orc
  world = 2
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = 29900 + (os.getpid() % 90) + {"peer-pull": 0, "peer-push": 3, "nccl": 7, "direct": 11}[exchange] + 13 * filtered
  procs = [ctx.Process(target=_fast_worker, args=(r, world, port, q, exchange, filtered)) for r in range(world)]
  for p in procs:
    p.start()
  got = [q.get(timeout=240) for _ in range(world)]
  for g in got:
    assert g[1] != "ERROR", g[2]
  got = sorted(got, key=lambda x: x[0])
  for p in procs:
    p.join(timeout=60)
  if filtered and exchange == "direct":
    assert [g[1] for g in got] == ["REFUSED"] * world
    return
  glob = orc.OracleMultiHashTable(_fast_cfg())
  if filtered:
    glob.set_hash_filter("t", 2_000_000, 2)
  for step in range(3):
    batches = [_fast_batch(r, step) for r in range(world)]
    for r, (fids, g) in enumerate(batches):
      want = glob.lookup_pool("t", fids, None, "sum")
      cold = fids != ((np.int64(5) << 48) | np.int64(3))
      np.testing.assert_array_equal(got[r][1][step][cold], want[cold])
      # the hot FID's gradient is a 1500-term fp32 sum, reduced piecewise on the GPU
      np.testing.assert_allclose(got[r][1][step][~cold], want[~cold], rtol=2e-3, atol=2e-3)
    for r, (fids, g) in enumerate(batches):   # owners apply requester 0's rows, then requester 1's
      u, inv = orc.dedup(fids)
      ug = orc.gather_pool_grad(g, inv * 16, 16, u.size * 16).reshape(-1, 16)
      glob.apply_gradients({"t": (u, ug)}, req_time=20 + step)
  keys = glob.keys("t")
  hot = (np.int64(5) << 48) | np.int64(3)
  for r in range(world):
    mine = keys[(keys.view(np.uint64) % np.uint64(world)) == r]
    k_r, e_r = got[r][2]
    np.testing.assert_array_equal(k_r, mine)
    want = glob.lookup_entry("t", mine)
    cold = mine != hot
    np.testing.assert_array_equal(e_r[cold].view(np.uint32), want[cold].view(np.uint32))   # reference order: bit-exact
    np.testing.assert_allclose(e_r[~cold][:, :-2], want[~cold][:, :-2], rtol=2e-3, atol=2e-3)
