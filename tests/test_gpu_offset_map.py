"""The async parameter-server worker path on the device, bit for bit against tests/offset_map_model.py (the reference's
loops in numpy) and, for DistributedMultiTypeHashTable, against the oracle tables of tests/orc.py, one per server:
unique_key_with_value_and_offset, ragged_split_by_indices, fill_with_offset_map and its gradient at tile and warp
boundaries up to millions of occurrences, K in {1, 4, 26, 200} with empty tables, odd and wide dims, Zipf keys with a
run of 2^17 and more, negative and INT64_MIN keys, special values in the gradients, launch counts, and no host
round trip with sync=False."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from monolith_b200 import MultiHashTable, _lib, distribution_ops as dops
from monolith_b200.distributed_ps import DistributedMultiTypeHashTable
from tests import offset_map_model as om
from tests import orc
from tests.helpers import table

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_offset_map.json")))
I64_MIN = np.iinfo(np.int64).min


@pytest.fixture(scope="module")
def dev():
  if not torch.cuda.is_available():
    pytest.skip("needs a GPU")
  return torch.device("cuda", 0)


def _same_bits(got, want):
  """float32 arrays equal bit for bit, NaNs compared by position"""
  got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
  assert got.shape == want.shape
  gn, wn = np.isnan(got), np.isnan(want)
  assert np.array_equal(gn, wn), "NaN positions differ"
  diff = np.nonzero(got.view(np.uint32)[~gn] != want.view(np.uint32)[~wn])[0]
  assert diff.size == 0, f"{diff.size} floats differ, first at {diff[:5]}"


def _keys(rng, split, vocab, zipf=None, specials=False):
  M = split[-1]
  if zipf:
    k = rng.zipf(zipf, M).astype(np.int64) % vocab
  else:
    k = rng.integers(0, vocab, M).astype(np.int64)
  if specials and M:
    sp = np.array([-1, -2, I64_MIN, I64_MIN + 1, np.iinfo(np.int64).max, -7], np.int64)
    at = rng.integers(0, M, min(M, 64))
    k[at] = sp[rng.integers(0, sp.size, at.size)]
  return k


def _splits(rng, counts):
  return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


def _grad_specials(rng, n):
  g = rng.standard_normal(n).astype(np.float32)
  if n:
    at = rng.integers(0, n, max(1, n // 97))
    g[at] = np.array([-0.0, 0.0, np.inf, -np.inf, np.nan, 3e38, -3e38, 1e-45], np.float32)[rng.integers(0, 8, at.size)]
  return g


def check_pipeline(dev, keys, split, dims, S, rng, sync=True):
  """unique -> split by floormod(key, S) -> S fills into a NaN buffer and S gradients, each against the model"""
  K = len(dims)
  t = torch.from_numpy(keys).to(dev)
  res = dops.unique_key_with_value_and_offset(t, split.tolist(), dims, sync=sync)
  uk, uks, vo, vos, n = om.unique_key_with_value_and_offset(keys, split, dims)
  U = uk.size
  assert res.value_len == n
  assert res.unique_key[1].cpu().tolist() == uks.tolist()
  assert res.unique_key[0].cpu().numpy()[:U].tolist() == uk.tolist()
  assert res.value_offset[0].cpu().numpy().tolist() == vo.tolist()
  assert res.value_offset[1].cpu().numpy()[:U + 1].tolist() == vos.tolist()
  if sync:
    assert res.num_unique == U and res.unique_key[0].numel() == U
  # floormod, not (uint64) % S
  index = torch.remainder(res.unique_key[0], S)
  sp = dops.ragged_split_by_indices(index, res.unique_key[0], res.unique_key[1], S)
  msplits, mpos = om.ragged_split_by_indices(np.mod(uk, S), uk, uks, S)
  buf = res.value_buffer.fill_(float("nan"))
  want_buf = np.full(n, np.nan, np.float32)
  g_in = _grad_specials(rng, n)
  g_dev = torch.from_numpy(g_in).to(dev)
  for s in range(S):
    (v, rs), p = sp.splits[s], sp.pos[s]
    assert v.cpu().tolist() == msplits[s][0].tolist() and rs.cpu().tolist() == msplits[s][1].tolist()
    assert sp.row_splits_host[s] == msplits[s][1].tolist()
    assert p.cpu().tolist() == mpos[s].tolist()
    rows = sum((msplits[s][1][k + 1] - msplits[s][1][k]) * dims[k] for k in range(K))
    val = rng.standard_normal(int(rows)).astype(np.float32)
    dops.fill_with_offset_map(p, sp.row_splits_host[s], torch.from_numpy(val).to(dev), res.value_offset, buf, dims,
                              num_unique=U)
    om.fill_with_offset_map(mpos[s], msplits[s][1], val, vo, vos, dims, want_buf)
    got_g = dops.fill_with_offset_map_gradient(p, sp.row_splits_host[s], g_dev, res.value_offset, dims, num_unique=U)
    _same_bits(got_g.cpu().numpy(), om.fill_with_offset_map_gradient(mpos[s], msplits[s][1], g_in, vo, vos, dims))
  got_buf = buf.cpu().numpy()
  assert not np.isnan(got_buf).any(), "the S fills left floats of the buffer unwritten"
  _same_bits(got_buf, want_buf)
  return U


def test_golden_vectors(dev):
  g = G["unique_fill"]
  keys = np.array([x for r in g["keys"] for x in r], np.int64)
  split = np.cumsum([0] + [len(r) for r in g["keys"]]).tolist()
  res = dops.unique_key_with_value_and_offset(torch.from_numpy(keys).to(dev), split, g["dims"])
  assert res.unique_key[0].cpu().tolist() == [x for r in g["unique_key"] for x in r]
  per_key = [o for tb in g["value_offset"] for o in tb]
  assert res.value_offset[0].cpu().tolist() == [x for o in per_key for x in o]
  pos = torch.tensor([x for r in g["fill_pos"] for x in r], dtype=torch.int64, device=dev)
  ps = np.cumsum([0] + [len(r) for r in g["fill_pos"]]).tolist()
  value = torch.arange(12, dtype=torch.float32, device=dev)
  buf = dops.fill_with_offset_map(pos, ps, value, res.value_offset, res.value_buffer, g["dims"])
  assert buf.cpu().tolist() == g["buffer"]
  grad = dops.fill_with_offset_map_gradient(pos, ps, torch.arange(19, dtype=torch.float32, device=dev),
                                            res.value_offset, g["dims"])
  assert grad.cpu().tolist() == g["grad"]
  with pytest.raises(ValueError, match="expected: 12, actual: 10"):
    dops.fill_with_offset_map(pos, ps, value[:10], res.value_offset, res.value_buffer, g["dims"])
  e = G["unique_empty"]
  res = dops.unique_key_with_value_and_offset(torch.zeros(0, dtype=torch.int64, device=dev), [0, 0, 0, 0], e["dims"])
  assert res.unique_key[0].numel() == 0 and res.unique_key[1].cpu().tolist() == [0, 0, 0, 0]
  assert res.value_offset[1].cpu().tolist() == [0] and res.value_buffer.numel() == 0
  r = G["ragged_split"]
  sp = dops.ragged_split_by_indices(torch.tensor(r["indices"], device=dev), torch.tensor(r["values"], device=dev),
                                    torch.tensor(r["row_splits"], device=dev), r["num_splits"])
  for (v, rs), p, want, wpos in zip(sp.splits, sp.pos, r["splits"], r["pos"]):
    assert v.cpu().tolist() == [x for row in want for x in row]
    assert rs.cpu().tolist() == np.cumsum([0] + [len(row) for row in want]).tolist()
    assert p.cpu().tolist() == [x for row in wpos for x in row]


@pytest.mark.parametrize("M", [1, 31, 32, 33, 2047, 2048, 2049, 8191, 8192, 8193, 100_000])
def test_tile_and_warp_boundaries(dev, M):
  rng = np.random.default_rng(M)
  check_pipeline(dev, _keys(rng, [0, M], max(2, M // 3)), np.array([0, M]), [3], 2, rng)


def test_several_million_occurrences(dev):
  rng = np.random.default_rng(7)
  counts = [1_500_000, 0, 2_000_001]
  split = _splits(rng, counts)
  check_pipeline(dev, _keys(rng, split, 1 << 20), split, [2, 5, 1], 3, rng)


@pytest.mark.parametrize("K", [1, 4, 26, 200])
def test_tables_with_empty_ones(dev, K):
  rng = np.random.default_rng(K)
  counts = rng.integers(0, 400, K)
  counts[rng.integers(0, K, max(1, K // 4))] = 0
  dims = [int(d) for d in rng.choice([1, 2, 3, 5, 16, 17, 33], K)]
  split = _splits(rng, counts)
  check_pipeline(dev, _keys(rng, split, 300), split, dims, 3, rng)


@pytest.mark.parametrize("dim", [1, 2, 3, 5, 16, 17, 33, 128, 257])
def test_odd_and_wide_dims(dev, dim):
  rng = np.random.default_rng(dim)
  split = _splits(rng, [3000, 1000])
  check_pipeline(dev, _keys(rng, split, 700), split, [dim, 4], 4, rng)


def test_zipf_keys_with_a_run_of_2_17(dev):
  rng = np.random.default_rng(11)
  split = _splits(rng, [400_000, 300_000])
  keys = _keys(rng, split, 1 << 22, zipf=1.1)
  keys[:200_000:1] = np.where(np.arange(200_000) % 3 == 0, keys[:200_000], 12345)  # one key, > 2^17 occurrences
  assert np.count_nonzero(keys[:400_000] == 12345) >= (1 << 17)
  check_pipeline(dev, keys, split, [16, 3], 4, rng)


def test_negative_and_int64_min_keys_use_floormod(dev):
  rng = np.random.default_rng(3)
  split = _splits(rng, [5000, 2000])
  check_pipeline(dev, _keys(rng, split, 1000, specials=True), split, [4, 2], 3, rng)
  # key -1 with 3 servers goes to server 2 (tf.math.floormod), where (uint64)fid % 3 would give 0
  keys = torch.tensor([-1, 5, I64_MIN], dtype=torch.int64, device=dev)
  res = dops.unique_key_with_value_and_offset(keys, [0, 3], [1])
  sp = dops.ragged_split_by_indices(torch.remainder(res.unique_key[0], 3), res.unique_key[0], res.unique_key[1], 3)
  assert [v.cpu().tolist() for v, _ in sp.splits] == [[], [I64_MIN], [-1, 5]]


def test_sync_false_stays_on_the_stream(dev):
  rng = np.random.default_rng(5)
  split = _splits(rng, [20_000, 7_000])
  keys = _keys(rng, split, 5000)
  dims = [3, 8]
  t = torch.from_numpy(keys).to(dev)
  torch.cuda.synchronize()
  torch.cuda._sleep(1_000_000_000)  # about half a second of a busy stream
  res = dops.unique_key_with_value_and_offset(t, split.tolist(), dims, sync=False)
  uniq, uks = res.unique_key
  sp = dops.ragged_split_by_indices(torch.remainder(uniq, 2), uniq, uks, 2, sync=False)
  assert res.num_unique is None and sp.splits is None
  assert not torch.cuda.current_stream(dev).query(), "a sync=False call waited for the stream"
  torch.cuda.synchronize()
  uk, uks_m, vo, vos, n = om.unique_key_with_value_and_offset(keys, split, dims)
  U = uk.size
  assert uniq.cpu().numpy()[:U].tolist() == uk.tolist() and uks.cpu().tolist() == uks_m.tolist()
  msplits, mpos = om.ragged_split_by_indices(np.mod(uk, 2), uk, uks_m, 2)
  offs = sp.offsets.cpu().tolist()
  assert offs == [0, msplits[0][0].size, U]
  for s in range(2):
    assert sp.values[offs[s]:offs[s + 1]].cpu().tolist() == msplits[s][0].tolist()
    assert sp.positions[offs[s]:offs[s + 1]].cpu().tolist() == mpos[s].tolist()
    assert sp.row_splits[s].cpu().tolist() == msplits[s][1].tolist()
  assert int(sp.bad.item()) == 0
  # the fills with sync=False
  g = torch.from_numpy(_grad_specials(rng, n)).to(dev)
  torch.cuda._sleep(1_000_000_000)
  out = dops.fill_with_offset_map_gradient(sp.positions[:offs[1]], msplits[0][1].tolist(), g, res.value_offset, dims,
                                           num_unique=U, sync=False)
  assert not torch.cuda.current_stream(dev).query()
  _same_bits(out.cpu().numpy(), om.fill_with_offset_map_gradient(mpos[0], msplits[0][1], g.cpu().numpy(), vo, vos,
                                                                  dims))


def test_bad_index_and_bad_pos_are_reported(dev):
  vals = torch.arange(4, dtype=torch.int64, device=dev)
  rs = torch.tensor([0, 4], dtype=torch.int64, device=dev)
  with pytest.raises(ValueError, match="outside"):
    dops.ragged_split_by_indices(torch.tensor([0, 1, 3, 0], device=dev), vals, rs, 3)
  sp = dops.ragged_split_by_indices(torch.tensor([0, -1, 1, 0], device=dev), vals, rs, 3, sync=False)
  assert int(sp.bad.item()) == 1
  res = dops.unique_key_with_value_and_offset(vals, [0, 4], [2])
  with pytest.raises(ValueError, match="pos"):
    dops.fill_with_offset_map(torch.tensor([0, 4], device=dev), [0, 2], torch.zeros(4, device=dev), res.value_offset,
                              res.value_buffer, [2])


def test_launch_counts_do_not_grow_with_tables(dev):
  lib = _lib.load()
  rng = np.random.default_rng(9)
  counts = {}
  for K in (1, 200):
    split = _splits(rng, np.full(K, 20_000 // K))
    t = torch.from_numpy(_keys(rng, split, 3000)).to(dev)
    dims = [4] * K
    n0 = lib.mono_kernel_launch_count()
    res = dops.unique_key_with_value_and_offset(t, split.tolist(), dims, sync=False)
    n1 = lib.mono_kernel_launch_count()
    sp = dops.ragged_split_by_indices(torch.remainder(res.unique_key[0], 4), res.unique_key[0], res.unique_key[1], 4)
    n2 = lib.mono_kernel_launch_count()
    U = sp.offsets[-1].item()
    dops.fill_with_offset_map(sp.pos[0], sp.row_splits_host[0], torch.zeros(res.value_len, device=dev),
                              res.value_offset, res.value_buffer, dims, num_unique=U, sync=False)
    n3 = lib.mono_kernel_launch_count()
    dops.fill_with_offset_map_gradient(sp.pos[0], sp.row_splits_host[0], torch.zeros(res.value_len, device=dev),
                                       res.value_offset, dims, num_unique=U, sync=False)
    n4 = lib.mono_kernel_launch_count()
    counts[K] = (n1 - n0, n2 - n1, n3 - n2, n4 - n3)
  # unique: claim, 3 rank passes, ordinal, 2 radix passes x 3 + run list 3, emit; split: count, scan, 1 radix pass x 3,
  # scatter; fill: tile counts, tile scan, row starts, copy; gradient: one
  assert counts[1] == counts[200] == (15, 6, 4, 1), counts


# ---- DistributedMultiTypeHashTable ------------------------------------------------------------------------------------
def _cfgs(opt):
  params = {"sgd": ("sgd", {}), "adagrad": ("adagrad", {}), "ftrl": ("ftrl", {})}[opt]
  return {"1": table([(3, params[0], params[1])], [0.05]), "2": table([(16, params[0], params[1])], [0.1]),
          "3": table([(1, params[0], params[1])], [0.2])}


def _model_step(orcs, S, dims, names, slot_to_id, slot_to_grad=None, global_step=0, req_time=0):
  """the worker path on numpy + oracle tables (PS s = orcs[s]): lookup, or apply_gradients with slot_to_grad"""
  parts, split = [], [0]
  for n in names:
    v = np.asarray(slot_to_id.get(n, np.zeros(0, np.int64)), np.int64).reshape(-1)
    parts.append(v)
    split.append(split[-1] + v.size)
  keys = np.concatenate(parts)
  uk, uks, vo, vos, n = om.unique_key_with_value_and_offset(keys, split, dims)
  splits, pos = om.ragged_split_by_indices(np.mod(uk, S), uk, uks, S)
  if slot_to_grad is None:
    buf = np.full(n, np.nan, np.float32)
    for s in range(S):
      om.fill_with_offset_map(pos[s], splits[s][1], orcs[s].raw_lookup(splits[s][0], splits[s][1]), vo, vos, dims, buf)
    out, off = {}, 0
    for k, nm in enumerate(names):
      c = split[k + 1] - split[k]
      if nm in slot_to_id:
        out[nm] = buf[off:off + c * dims[k]].reshape(c, dims[k])
      off += c * dims[k]
    return out
  flat = np.concatenate([np.asarray(slot_to_grad[nm], np.float32).reshape(-1) for nm in names if nm in slot_to_grad])
  for s in range(S):
    g = om.fill_with_offset_map_gradient(pos[s], splits[s][1], flat, vo, vos, dims)
    orcs[s].raw_apply_gradients(splits[s][0], splits[s][1], g, global_step, req_time)


def _train_and_compare(S, opt, devices):
  rng = np.random.default_rng(S * 7 + len(opt))
  cfg = _cfgs(opt)
  dmt = DistributedMultiTypeHashTable(S, cfg, lambda i, c: MultiHashTable(_cfgs(opt), device=devices[i % len(devices)]))
  orcs = [orc.OracleMultiHashTable(_cfgs(opt)) for _ in range(S)]
  names, dims = sorted(cfg), [3, 16, 1]
  dev0 = devices[0]
  for step in range(4):
    ids = {"1": rng.integers(-50, 50, 300), "2": rng.zipf(1.3, 500) % 200 - 20, "3": rng.integers(-5, 5, 40)}
    if step == 2:
      ids.pop("3")
    ids = {k: v.astype(np.int64) for k, v in ids.items()}
    grads = {k: rng.standard_normal((v.size, dims[names.index(k)])).astype(np.float32) for k, v in ids.items()}
    tids = {k: torch.from_numpy(v).to(dev0) for k, v in ids.items()}
    dmt.apply_gradients({k: (tids[k], torch.from_numpy(grads[k]).to(dev0)) for k in ids}, global_step=step,
                        req_time=100 + step)
    _model_step(orcs, S, dims, names, ids, grads, step, 100 + step)
    got = dmt.lookup(tids)
    want = _model_step(orcs, S, dims, names, ids)
    assert sorted(got) == sorted(want)
    for k in ids:
      _same_bits(got[k].cpu().numpy(), want[k])


@pytest.mark.parametrize("S", [1, 2, 3, 5])
@pytest.mark.parametrize("opt", ["sgd", "adagrad", "ftrl"])
def test_distributed_training_steps_one_device(dev, S, opt):
  _train_and_compare(S, opt, [dev])


@pytest.mark.parametrize("opt", ["sgd", "ftrl"])
def test_distributed_training_steps_across_two_devices(opt):
  if torch.cuda.device_count() < 2:
    pytest.skip("needs two GPUs")
  _train_and_compare(3, opt, [torch.device("cuda", 0), torch.device("cuda", 1)])


def _ref_configs():
  from tests.helpers import sgd_table
  return {"1": sgd_table(1), "2": sgd_table(2)}


def test_reference_basic(dev):
  """ref: distributed_ps_test.py:221-263 (native table, 2 PS)"""
  g = G["distributed_basic"]
  dmt = DistributedMultiTypeHashTable(2, _ref_configs(), lambda i, c: MultiHashTable(_ref_configs(), device=dev))
  t = lambda x, dt=torch.int64: torch.tensor(x, dtype=dt, device=dev)
  ids = {k: t(v) for k, v in g["ids"].items()}
  dmt.assign_add({k: (ids[k], t(g["values"][k], torch.float32)) for k in ids})
  got = dmt.lookup(ids)
  for k in ids:
    assert got[k].cpu().tolist() == g["after_assign_add"][k]
  dmt.apply_gradients({k: (ids[k], t(g["grads"][k], torch.float32)) for k in ids}, global_step=0, req_time=0)
  got = dmt.as_op().lookup(ids)
  for k in ids:
    assert got[k].cpu().tolist() == g["after_apply"][k]
  assert dmt.get_table_dim_sizes() == (1, 2)


def test_reference_assign_and_reinitialize(dev):
  """ref: distributed_ps_test.py:265-314 (native table, 2 PS)"""
  g = G["distributed_assign_reinit"]
  dmt = DistributedMultiTypeHashTable(2, _ref_configs(), lambda i, c: MultiHashTable(_ref_configs(), device=dev))
  t = lambda x, dt=torch.int64: torch.tensor(x, dtype=dt, device=dev)
  ids = {k: t(v) for k, v in g["ids"].items()}
  dmt.assign({k: (ids[k], t(g["values"][k], torch.float32)) for k in ids})
  got = dmt.lookup(ids)
  for k in ids:
    assert got[k].cpu().tolist() == g["values"][k]
  dmt.assign({k: (ids[k], t(g["values2"][k], torch.float32)) for k in ids})
  got = dmt.lookup(ids)
  for k in ids:
    assert got[k].cpu().tolist() == g["values2"][k]
  _, st1 = dmt.reinitialize("1", t(g["reinit_ids"]))
  _, st3 = dmt.reinitialize("3", t(g["reinit_ids"]))
  assert st1.cpu().tolist() == g["status_1"] and st3.cpu().tolist() == g["status_3"]
  got = dmt.lookup({"1": t(g["reinit_ids"]), "2": ids["2"]})
  assert got["1"].cpu().tolist() == g["after_reinit"]["1"] and got["2"].cpu().tolist() == g["after_reinit"]["2"]


def test_split_by_indices(dev):
  ids = torch.tensor([5, -1, 4, 9, -6, 2], dtype=torch.int64, device=dev)
  vals = torch.arange(12, dtype=torch.float32, device=dev).view(6, 2)
  index = torch.remainder(ids, 3)
  got = dops.split_by_indices(index, vals, 3)
  for s in range(3):
    sel = np.nonzero(np.mod(ids.cpu().numpy(), 3) == s)[0]
    assert got[s].cpu().tolist() == vals.cpu().numpy()[sel].tolist()
  assert [x.numel() for x in dops.split_by_indices(index[:0], vals[:0], 3)] == [0, 0, 0]
