"""The table's write side against the CPU oracle, with the table's structure checked after every call.

Every inserter (resolve_miss, claim_miss and xmiss_insert, which take their rows from common.cuh insert_new_row, and
rehash; all publish through common.cuh cuckoo_insert), growth, eviction, export and restore run on keys built
(tests/cuckoo_place.py) to land where a case wants them: a free slot of the first bucket, the second bucket, a
copy-first displacement that succeeds, closed bucket pairs of 9, 10 and 12 keys written in one call (threads carry
entries through the exchange chain and end in the stash), the keys -1, 0, INT64_MIN and INT64_MAX in full pairs, and
stash keys hit again.  After every call `World.check` compares:
  * lookup_entry of every key ever written, and of absent keys, with the oracle bit for bit (weights, state, found
    flag, timestamp);
  * the exported keys with the oracle's keys (no key twice), and each exported entry with its lookup_entry bits;
  * the counters (MultiHashTable.counters): size with the oracle, inflight == 0, error == 0, bump - free == size (no
    row leaked or freed twice), the stash count where groups were built for one, the exact number of moves a call of
    copy-first displacements makes, moves > 0 where exchange chains were aimed at.
Each case ends with one assign of a distinct value to every live key, which every key must read back (no two keys
share a row).  Each case asserts, through torch.profiler, the write-side kernels it launched, and that rehash_kernel
ran exactly as often as the counters predict; the last test checks the file ran all of them.  The rules the cases are aimed with are pinned
against the sources in tests/test_write_paths_cpu.py.
"""
import collections
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from tests import cuckoo_place as cp
from tests import orc
from tests.helpers import table
from tests.test_gpu_apply_paths import assert_same
from tests.test_gpu_forward_paths import _canon, pick_group

pytestmark = pytest.mark.gpu

I64 = np.iinfo(np.int64)
GS = (4, 8, 16, 32)
FAMILY = ("resolve_hit_kernel", "resolve_miss_kernel", "upsert_finalize_kernel", "dup_claim_kernel", "dup_split_kernel",
          "miss_split_kernel", "miss_follow_kernel", "upsert_apply_kernel", "claim_miss_kernel", "xowner_resolve_kernel",
          "xmiss_claim_kernel", "xmiss_insert_kernel", "xmiss_follow_kernel", "rehash_kernel", "evict_kernel",
          "export_kernel")
INVENTORY = frozenset(
    ["resolve_hit_kernel<false>", "resolve_hit_kernel<true>", "resolve_miss_kernel<false>", "resolve_miss_kernel<true>",
     "upsert_finalize_kernel", "dup_claim_kernel", "dup_split_kernel", "miss_split_kernel", "miss_follow_kernel",
     "claim_miss_kernel", "xowner_resolve_kernel", "xmiss_claim_kernel", "xmiss_insert_kernel", "xmiss_follow_kernel",
     "rehash_kernel", "evict_kernel", "export_kernel"] +
    [f"upsert_apply_kernel<{g},{op}>" for g in GS for op in range(5)])
SEEN = set()
OP_OPTIMIZE, OP_ASSIGN, OP_ASSIGN_ADD, OP_REINIT, OP_RESTORE = range(5)
T0 = 10 ** 6
DAY = 86400


@pytest.fixture(scope="module")
def dev():
  assert torch.cuda.is_available()
  return torch.device("cuda", 0)


def T(x, dev):
  return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def rehash_buckets(keys):
  """table.cu buckets_for: the bucket count that holds `keys` keys at load 0.5."""
  return max(64, (int(keys) + 1) // 2 + 1)


def upsert_kernels(G, op, unique):
  k = {f"resolve_hit_kernel<{'true' if op == OP_RESTORE else 'false'}>",
       f"resolve_miss_kernel<{'true' if op == OP_RESTORE else 'false'}>", f"upsert_apply_kernel<{G},{op}>",
       "upsert_finalize_kernel"}
  return k if unique else k | {"dup_claim_kernel", "dup_split_kernel"}


def traced_counts(fn):
  """-> (fn(), {kernel of FAMILY: launches torch.profiler recorded while it ran})."""
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    out = fn()
    torch.cuda.synchronize()
  return out, collections.Counter(c for c in (_canon(e.name, FAMILY) for e in prof.events()) if c)


def run_case(fn):
  """fn() -> (numpy arrays, the write-side kernels it aimed at, the rehashes it predicted: a count, or None for
  "at least one").  The kernels of FAMILY it launched must be exactly those, and rehash_kernel must have run as many
  times as predicted (one launch per table rehash).  A trace that lost records (a strict subset of the kernels, or
  fewer rehash launches) is taken again; a second run gives the same bits.  fn builds its tables itself."""
  for _ in range(10):
    (out, expect, rehashes), counts = traced_counts(fn)
    names = set(counts)
    if not (names < expect or (rehashes is not None and counts["rehash_kernel"] < rehashes)):
      break
  SEEN.update(names)
  assert names == expect, f"ran {sorted(names)}, aimed at {sorted(expect)}"
  if rehashes is None:
    assert counts["rehash_kernel"] >= 1
  else:
    assert counts["rehash_kernel"] == rehashes, f"rehash_kernel ran {counts['rehash_kernel']} times, {rehashes} predicted"
  again, expect2, rehashes2 = fn()
  assert expect2 == expect and rehashes2 == rehashes
  for a, b in zip(out, again):
    np.testing.assert_array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8),
                                  err_msg="not bit-stable run to run")
  return out


# ------------------------------------------------------------------------------------------------
# one MultiHashTable, its oracle, and the checks made after every call
# ------------------------------------------------------------------------------------------------
class World:

  def __init__(self, dev, cfgs, capacity, chunk=1 << 20):
    from monolith_b200 import MultiHashTable
    self.dev, self.names, self.chunk = dev, sorted(cfgs), chunk
    self.gpu = MultiHashTable(cfgs, device=dev)
    self.cpu = orc.OracleMultiHashTable(cfgs)
    self.dims = dict(zip(self.names, self.gpu.get_table_dim_sizes()))
    self.nb = {n: cp.buckets_for(capacity[n] if isinstance(capacity, dict) else capacity) for n in self.names}
    self.written = {n: set() for n in self.names}
    self.over = {n: {} for n in self.names}   # restored entries the oracle cannot hold: key -> entry row
    self.expect, self.out, self.rehashes = set(), [], {n: 0 for n in self.names}
    self.rehashes_known = True                  # False: calls made without before(), the count is not predicted
    self.moves = {n: 0 for n in self.names}     # ctrs[kCtrMoves] at the last check

  # ---- calls --------------------------------------------------------------------------------
  def before(self, counts):
    """Predict the rehash ensure_capacity makes for a call bringing counts[name] ids (table.cu: load 0.75 of the
    bucket slots, or a non-empty stash; the host's counter snapshot is current because every check synchronises)."""
    for n, m in counts.items():
      if m <= 0:
        continue
      c = self.gpu.counters(n)
      if c["size"] + m > 0.75 * self.nb[n] * cp.BUCKET_SLOTS or c["stash"] > 0:
        self.nb[n] = max(2 * self.nb[n], rehash_buckets(c["size"] + m))
        self.expect.add("rehash_kernel")
        self.rehashes[n] += 1

  def note(self, d):
    for n, k in d.items():
      self.written[n].update(np.asarray(k, np.int64).reshape(-1).tolist())

  def G(self, names):
    return pick_group(max(self.dims[n] for n in names))

  def assign(self, d, ts, unique=True, add=False):
    """d: name -> (keys, values)"""
    self.before({n: len(k) for n, (k, _) in d.items()})
    self.note({n: k for n, (k, _) in d.items()})
    f = self.gpu.assign_add if add else self.gpu.assign
    f({n: (T(k, self.dev), T(v, self.dev)) for n, (k, v) in d.items()}, req_time=ts, ids_unique=unique)
    (self.cpu.assign_add if add else self.cpu.assign)(d, req_time=ts)
    self.expect |= upsert_kernels(self.G(d), OP_ASSIGN_ADD if add else OP_ASSIGN, unique)

  def optimize(self, d, ts, unique=True, dedup=False):
    self.before({n: len(k) for n, (k, _) in d.items()})
    self.note({n: k for n, (k, _) in d.items()})
    self.gpu.apply_gradients({n: (T(k, self.dev), T(v, self.dev)) for n, (k, v) in d.items()}, req_time=ts,
                             ids_unique=unique, enable_dedup=dedup)
    self.cpu.apply_gradients(d, req_time=ts, enable_dedup=dedup)
    self.expect |= upsert_kernels(self.G(d), OP_OPTIMIZE, unique and not dedup)

  def fused(self, shards, ts):
    """shards: [{name: (keys, grads)}] — keys unique inside a shard, a key may be in several shards."""
    N, names = len(shards), self.names
    ids, g, ss = [], [], []
    for sh in shards:
      for n in names:
        k, v = sh.get(n, (np.zeros(0, np.int64), np.zeros((0, self.dims[n]), np.float32)))
        ids.append(np.asarray(k, np.int64))
        g.append(np.asarray(v, np.float32).reshape(-1))
        ss.append(len(k))
    ids, g = np.concatenate(ids), np.concatenate(g)
    self.before({n: sum(len(sh[n][0]) for sh in shards if n in sh) for n in names})
    self.note({n: np.concatenate([sh[n][0] for sh in shards if n in sh]) for n in names})
    _, _, ko, eo = self.gpu.fused_offsets(ss, N)
    ti = T(ids, self.dev)
    self.gpu.fused_apply_gradient(ti, ti, ss, T(g, self.dev), ko, eo, 0, ts, N)
    self.cpu.fused_apply_gradient(ids, ss, g, N, req_time=ts)
    used = [n for n in names if any(n in sh for sh in shards)]
    self.expect |= {"resolve_hit_kernel<false>", "dup_claim_kernel", "miss_split_kernel", "resolve_miss_kernel<false>",
                    "miss_follow_kernel", "upsert_finalize_kernel", f"upsert_apply_kernel<{self.G(used)},0>"}

  def reinit(self, n, keys, ts):
    from monolith_b200 import _lib
    keys = np.asarray(keys, np.int64)
    self.before({n: keys.size})
    self.note({n: keys})
    st = torch.empty(keys.size, dtype=torch.int32, device=self.dev)
    tk = T(keys, self.dev)
    _lib.check(_lib.load().mono_mtable_reinitialize(self.gpu.handle, self.names.index(n), C.c_void_p(tk.data_ptr()),
                                                    keys.size, C.c_void_p(st.data_ptr()), ts,
                                                    C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)))
    want = self.cpu.reinitialize(n, keys, ts)
    np.testing.assert_array_equal(st.cpu().numpy(), want, err_msg="reinitialize status")
    self.expect |= upsert_kernels(self.G([n]), OP_REINIT, False)
    return want

  def restore(self, n, keys, rows):
    """Rows in export layout; the oracle cannot restore, so the restored entries are what must be read back."""
    keys = np.asarray(keys, np.int64)
    self.before({n: keys.size})
    self.note({n: keys})
    self.gpu.restore_rows(n, T(keys, self.dev), T(rows, self.dev))
    last = {}
    for i, k in enumerate(keys.tolist()):   # duplicates: the last occurrence wins (rounds run in position order)
      last[k] = rows[i]
    self.over[n].update(last)
    self.expect |= upsert_kernels(self.G([n]), OP_RESTORE, False)

  def pool_backward(self, n, fids, grads, ts):
    """One FID per pooled row (SUM): each FID's gradient is the sum of its rows.  The gradients are small integers,
    so the sum is exact in any order and the oracle gets the same one."""
    fids = np.asarray(fids, np.int64)
    self.before({n: fids.size})
    self.note({n: fids})
    self.gpu.pool_backward(n, T(fids, self.dev), T(grads, self.dev), None, "sum", req_time=ts)
    self._cpu_sums(n, fids, grads, ts)
    self.expect |= {"claim_miss_kernel", "upsert_finalize_kernel"}

  def pool_backward_parts(self, parts, ts):
    """parts: [(name, fids, grads)]; a table's parts are one batch."""
    from monolith_b200 import PoolPart
    cnt = {}
    for n, f, _ in parts:
      cnt[n] = cnt.get(n, 0) + len(f)
    self.before(cnt)
    self.note({n: np.concatenate([f for m, f, _ in parts if m == n]) for n in cnt})
    self.gpu.pool_backward_parts([PoolPart(n, T(f, self.dev), None, "sum", T(g, self.dev)) for n, f, g in parts],
                                 req_time=ts)
    d = {}
    for n in cnt:
      f = np.concatenate([f for m, f, _ in parts if m == n])
      g = np.concatenate([g for m, _, g in parts if m == n])
      d[n] = self._sums(f, g)
    self.cpu.apply_gradients(d, req_time=ts)
    self.expect |= {"claim_miss_kernel", "upsert_finalize_kernel"}

  @staticmethod
  def _sums(fids, grads):
    u, inv = np.unique(fids, return_inverse=True)
    s = np.zeros((u.size, grads.shape[1]), np.float64)
    np.add.at(s, inv, grads.astype(np.float64))
    return u, s.astype(np.float32)

  def _cpu_sums(self, n, fids, grads, ts):
    self.cpu.apply_gradients({n: self._sums(fids, grads)}, req_time=ts)

  def xstep(self, n, fids, grads, ts):
    """The world-1 ShardedStep in direct mode (xstep.cu): owner resolve, miss claim / insert / follow, finalize and
    the apply of the window."""
    from monolith_b200.distributed_ps import ShardedStep
    fids = np.asarray(fids, np.int64)
    # ensure_capacity(min(N * C, 2 * last_m)): nothing is asked on the first step, so only a stash rehashes
    self.before({n: 0})
    c = self.gpu.counters(n)
    if c["stash"] > 0:
      self.before({n: 1})
    self.note({n: fids})
    st = ShardedStep(self.gpu, n, self.dims[n], 1, 0, self.dev, exchange="direct")
    try:
      out = torch.empty(fids.size, self.dims[n], device=self.dev)
      st.step(T(fids, self.dev), T(grads, self.dev), out, ts, None, "sum")
      torch.cuda.synchronize()
    finally:
      st.close_direct()
    self._cpu_sums(n, fids, grads, ts)
    self.expect |= {"xowner_resolve_kernel", "xmiss_claim_kernel", "xmiss_insert_kernel", "xmiss_follow_kernel",
                    "upsert_finalize_kernel", f"upsert_apply_kernel<{pick_group(self.dims[n])},0>"}

  def evict(self, n, max_ts):
    self.gpu.evict(n, max_ts)
    self.cpu.evict(n, max_ts)
    self.expect.add("evict_kernel")

  # ---- checks -------------------------------------------------------------------------------
  def live_keys(self, n):
    k = set(self.cpu.keys(n).tolist()) | set(self.over[n])
    return np.asarray(sorted(k), np.int64)

  def want_entries(self, n, keys):
    w = self.cpu.lookup_entry(n, keys)
    for i, k in enumerate(keys.tolist()):
      if k in self.over[n]:
        w[i] = self.over[n][k]
    return w

  def export(self, n, chunk=None):
    ids, rows = [], []
    for i, r in self.gpu.export(n, chunk or self.chunk):
      ids.append(i.cpu().numpy())
      rows.append(r.cpu().numpy())
    W = self.gpu.entry_width(n)
    self.expect.add("export_kernel")
    if not ids:
      return np.zeros(0, np.int64), np.zeros((0, W), np.float32)
    return np.concatenate(ids), np.concatenate(rows)

  def check(self, absent=(), stash=None, moves=False, moves_added=None):
    """Every table: entries, export and counters (see the module docstring).  moves_added[name]: the displacements
    the calls since the last check must have made, exactly."""
    absent = np.asarray(absent, np.int64)
    for n in self.names:
      keys = np.asarray(sorted(self.written[n] | set(absent.tolist())), np.int64)
      got = self.gpu.lookup_entry(n, T(keys, self.dev))["raw"].cpu().numpy()
      assert_same(got, self.want_entries(n, keys), f"table {n}: lookup_entry")
      live = self.live_keys(n)
      ids, rows = self.export(n)
      assert np.unique(ids).size == ids.size, f"table {n}: a key exported twice"
      np.testing.assert_array_equal(np.sort(ids), live, err_msg=f"table {n}: exported keys")
      order = np.argsort(ids)
      ent = self.gpu.lookup_entry(n, T(ids[order], self.dev))["raw"].cpu().numpy()
      np.testing.assert_array_equal(rows[order].view(np.uint32), ent.view(np.uint32),
                                    err_msg=f"table {n}: exported entry vs lookup_entry")
      c = self.gpu.counters(n)
      assert c["size"] == live.size, (n, c, live.size)
      assert c["inflight"] == 0 and c["error"] == 0, (n, c)
      assert c["bump"] - c["free"] == c["size"], (n, c)
      if stash is not None and n in stash:
        assert c["stash"] == stash[n], (n, c["stash"], stash[n])
      if moves:
        assert c["moves"] > 0, (n, c)
      if moves_added is not None and n in moves_added:
        assert c["moves"] - self.moves[n] == moves_added[n], (n, c["moves"] - self.moves[n], moves_added[n])
      self.moves[n] = c["moves"]
      self.out += [got, rows[order], ids[order]]

  def no_aliasing(self, ts):
    """One assign gives every live key a distinct value; every key reads back its own (no two keys share a row)."""
    d = {}
    for n in self.names:
      live = self.live_keys(n)
      v = np.zeros((live.size, self.dims[n]), np.float32)
      v[:, 0] = np.arange(1, live.size + 1, dtype=np.float32)
      d[n] = (live, v)
    self.assign(d, ts)
    for n in self.names:   # the last call of a case: the entries are not compared with the oracle any more
      live, v = d[n]
      got = self.gpu.lookup_entry(n, T(live, self.dev))
      np.testing.assert_array_equal(got["num"].cpu().numpy()[:, 0], v[:, 0], err_msg=f"table {n}: rows alias")
      assert bool(got["found"].all())
      c = self.gpu.counters(n)
      assert c["size"] == live.size and c["bump"] - c["free"] == c["size"] and c["error"] == 0, (n, c)
    return self.out, set(self.expect), sum(self.rehashes.values()) if self.rehashes_known else None


def sgd(dim, capacity, init=None, **kw):
  from monolith_b200 import entry
  return table([(dim, "sgd", {})], [0.5], capacity=capacity,
               init=init or entry.RandomUniformInitializer(-0.25, 0.25), init_seed=11, **kw)


def rand_keys(rng, n, exclude=()):
  k = np.unique(rng.integers(I64.min, I64.max, n + 64, dtype=np.int64))
  k = k[~np.isin(k, np.asarray(list(exclude), np.int64))]
  return rng.permutation(k)[:n]


def ivals(rng, n, d):
  """Small integers: sums of them are exact in any order."""
  return rng.integers(-4, 5, (n, d)).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# placement x inserter
# ------------------------------------------------------------------------------------------------
EXTREMES = (-1, 0, int(I64.min), int(I64.max))
CLOSED = (9, 10, 12)


class Placed:
  """Keys of one table of nb buckets: `free1` (alone in their first bucket), `second` (6 keys of one pair: two end in
  their second bucket), copy-first `fill` + `newcomers`, closed pairs of 9, 10 and 12 keys that keep their pair at
  2·nb, and 8-key full pairs around each of -1, 0, INT64_MIN, INT64_MAX (also kept at 2·nb)."""

  def __init__(self, nb, rng):
    pk = cp.BucketPicker(nb, rng, levels=1)
    # the extremes' pairs first: their companions share the pair at nb and 2·nb
    self.extreme = []
    for x in EXTREMES:
      f1, f2 = (int(v) for v in cp.bucket_pair(x, 2 * nb))
      c1, c2 = (int(v) for v in cp.bucket_pair(x, nb))
      assert not ({f1, f2} & pk.used[0]) and not ({c1, c2} & pk.used[1])
      pk.used[0].update((f1, f2))
      pk.used[1].update((c1, c2))
      h = cp.mix64(np.asarray([x], np.int64))   # the raw halves (key 0 hashes to 0: its pair is the fixed-up (0, 1))
      r1, r2 = (int(cp._umulhi(v, 2 * nb)[0]) for v in (h & np.uint64(0xFFFFFFFF), h >> np.uint64(32)))
      comp = cp.colliding_keys(2 * nb, r1, r2, 8, rng)
      comp = comp[~np.isin(comp, EXTREMES)][:7]
      for n in (nb, 2 * nb):
        want = [int(v[0]) for v in cp.bucket_pair(np.asarray([x], np.int64), n)]
        q1, q2 = cp.bucket_pair(comp, n)
        assert (q1 == want[0]).all() and (q2 == want[1]).all(), (x, n)
      self.extreme.append(np.concatenate([[x], comp]).astype(np.int64))
    self.extreme = np.concatenate(self.extreme)
    self.free1 = np.concatenate([cp.stable_keys(nb, pk.take(), pk.take(), 1, rng, levels=1) for _ in range(8)])
    self.second = cp.stable_keys(nb, pk.take(), pk.take(), 6, rng, levels=1)
    self.fill, self.new = [], []
    for _ in range(6):
      # copy-first groups built on the buckets of the 2·nb table: a bucket of the nb table is a pair of them halved,
      # and the picker keeps the halved images distinct too, so each group is a copy-first group at nb as well
      f, w = cp.copy_first_group(2 * nb, pk, rng)
      self.fill.append(f)
      self.new.append(w)
    self.fill, self.new = np.concatenate(self.fill), np.concatenate(self.new)
    self.closed = [cp.stable_keys(nb, pk.take(), pk.take(), m, rng, levels=1) for m in CLOSED]
    self.used = {nb: set(pk.used[1]), 2 * nb: set(pk.used[0])}
    self.stash = cp.predicted_stash(CLOSED)
    allk = np.concatenate([self.extreme, self.free1, self.second, self.fill, self.new] + self.closed)
    assert np.unique(allk).size == allk.size
    self.all = allk

  def background(self, rng, n, nb):
    k = cp.avoiding(rand_keys(rng, 4 * n, exclude=self.all), self.used, (nb, 2 * nb))
    assert k.size >= n
    return k[:n]


INSERTERS = ("assign", "assign_dup", "assign_add", "assign_add_dup", "optimize", "optimize_dup", "optimize_dedup",
             "fused", "reinit", "restore", "pool_backward", "pool_backward_parts", "xstep")
PLACE_CAP = 16384


def _write(w, how, d, ts, rng, dup=False):
  """Write d[name] = keys through inserter `how` (values the oracle can follow)."""
  dims = w.dims
  if how.startswith("assign"):
    add = how.startswith("assign_add")
    dd = {}
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      if dup:
        k = rng.permutation(np.repeat(k, rng.integers(1, 4, k.size)))
      dd[n] = (k, ivals(rng, k.size, dims[n]) * np.float32(0.125))
    w.assign(dd, ts, unique=not dup, add=add)
  elif how.startswith("optimize"):
    dd = {}
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      if dup:
        k = rng.permutation(np.repeat(k, rng.integers(1, 4, k.size)))
      dd[n] = (k, ivals(rng, k.size, dims[n]))
    w.optimize(dd, ts, unique=not dup, dedup=how == "optimize_dedup" and dup)
  elif how == "fused":
    # two shards; every second key is in both (a FID fresh in two shards: miss_split / miss_follow)
    sh = [{}, {}]
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      both = k[::2]
      a, b = np.concatenate([k[1::4], both]), np.concatenate([k[3::4], both])
      sh[0][n] = (rng.permutation(a), ivals(rng, a.size, dims[n]))
      sh[1][n] = (rng.permutation(b), ivals(rng, b.size, dims[n]))
    w.fused(sh, ts)
  elif how == "reinit":
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      w.reinit(n, rng.permutation(np.concatenate([k, k[::3]])), ts)   # duplicates within the call
  elif how == "restore":
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      W = w.gpu.entry_width(n)
      rows = rng.standard_normal((k.size, W)).astype(np.float32)
      rows[:, -2] = np.array([1], np.uint32).view(np.float32)[0]        # the found flag lookup_entry writes
      rows[:, -1] = np.asarray(ts - rng.integers(0, 5 * DAY, k.size), np.uint32).view(np.float32)   # ts backwards too
      w.restore(n, k, rows)
  elif how == "pool_backward":
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      f = rng.permutation(np.repeat(k, rng.integers(1, 4, k.size)))
      w.pool_backward(n, f, ivals(rng, f.size, dims[n]), ts)
  elif how == "pool_backward_parts":
    parts = []
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      for half in (k[::2], k[1::2], k[::5]):   # a table's parts share FIDs
        f = rng.permutation(np.repeat(half, rng.integers(1, 3, half.size)))
        parts.append((n, f, ivals(rng, f.size, dims[n])))
    w.pool_backward_parts(parts, ts)
  elif how == "xstep":
    for n, k in d.items():
      k = np.asarray(k, np.int64)
      f = rng.permutation(np.repeat(k, rng.integers(1, 3, k.size)))
      w.xstep(n, f, ivals(rng, f.size, dims[n]), ts)
  else:
    raise ValueError(how)


@pytest.mark.parametrize("how", INSERTERS)
def test_placement_by_inserter(how, dev):
  """Call 1 writes the singles, the second-bucket pair and the copy-first fillers; call 2 only the copy-first
  newcomers: each makes exactly one displacement (a copy-first move adds 1 to the move counter, an exchange that
  places its victim at once adds 2); call 3 (crafted groups in both tables at once where the inserter takes several
  tables) the closed pairs and the extreme keys' pairs: the predicted stash; call 4 hits every key again (the stash
  ones through resolve_hit's stash branch, after the rehash a non-empty stash forces, in which the closed pairs
  re-enter the stash)."""
  seed = zlib.crc32(how.encode())
  # the backward and the sharded step take dim % 4 == 0 up to 128; their per-table apply then runs at G = 8 and 32
  dims = {"a": 20, "b": 128} if how in ("pool_backward", "pool_backward_parts", "xstep") else {"a": 8, "b": 33}

  def fn():
    rng = np.random.default_rng(seed)
    w = World(dev, {n: sgd(d, PLACE_CAP) for n, d in dims.items()}, PLACE_CAP)
    nb = w.nb["a"]
    pl = {n: Placed(nb, rng) for n in dims}
    dup = how.endswith("_dup") or how == "optimize_dedup"
    absent = rand_keys(rng, 50, exclude=np.concatenate([p.all for p in pl.values()]))
    # call 1
    _write(w, how, {n: np.concatenate([p.free1, p.second, p.fill]) for n, p in pl.items()}, T0, rng, dup)
    w.check(absent, stash={n: 0 for n in dims})
    assert "rehash_kernel" not in w.expect
    # call 2: the copy-first newcomers alone
    _write(w, how, {n: rng.permutation(p.new) for n, p in pl.items()}, T0 + 5, rng, dup)
    w.check(absent, stash={n: 0 for n in dims}, moves_added={n: p.new.size for n, p in pl.items()})
    # call 3: the crafted groups, in one call (one per table for the single-table inserters)
    d2 = {n: rng.permutation(np.concatenate([p.extreme, p.background(rng, 200, nb)] + p.closed))
          for n, p in pl.items()}
    _write(w, how, d2, T0 + 10, rng, dup)
    w.check(absent, stash={n: pl[n].stash for n in dims}, moves=True)
    assert "rehash_kernel" not in w.expect
    # call 4: every key again plus new ones; the stash forces a rehash first, the closed pairs are closed at 2·nb too
    nb2 = max(2 * nb, rehash_buckets(0))
    d3 = {n: rng.permutation(np.concatenate([np.asarray(sorted(w.written[n]), np.int64),
                                              cp.avoiding(rand_keys(rng, 100, exclude=w.written[n]), pl[n].used,
                                                          (nb2,))]))
          for n in dims}
    _write(w, how, d3, T0 + 20, rng, dup)
    assert w.rehashes["a"] == 1 and w.rehashes["b"] == 1
    w.check(absent, stash={n: pl[n].stash for n in dims})
    return w.no_aliasing(T0 + 30)

  run_case(fn)


# ------------------------------------------------------------------------------------------------
# widths: assign_add, reinitialize and restore at every lane-group width
# ------------------------------------------------------------------------------------------------
WIDTH_DIMS = [1, 3, 4, 5, 8, 17, 32, 33, 64, 65, 128, 129, 257, 512]
SPECIAL = np.array([0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x7F7FFFFF, 0xFF7FFFFF], np.uint32).view(np.float32)


def width_tables(dim):
  """A single-segment table of `dim` and, of the same width, two multi-segment ones with eight optimizers' state
  layouts (with the single one's Adagrad, every optimizer with state) and all four initializers (seg_of_col /
  seg_of_state)."""
  from monolith_b200 import entry
  inits = [entry.RandomUniformInitializer(-0.25, 0.25), entry.ZerosInitializer(), entry.OnesInitializer(),
           entry.ConstantsInitializer(0.375)]
  out = {"s": table([(dim, "adagrad", {"initial_accumulator_value": 0.1})], [0.5], capacity=1, init=inits[0],
                    init_seed=5)}
  if dim >= 4:
    d = [dim - 3, 1, 1, 1]
    segs = [(d[0], "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0, "l1": 0.001, "l2": 0.01}),
            (d[1], "adam", {}), (d[2], "amsgrad", {}), (d[3], "group_adagrad", {"l2": 0.05, "beta": 1.0})]
    out["m"] = table(segs, [0.5] * 4, capacity=1, init=inits, init_seed=5)
    segs = [(d[0], "momentum", {"use_nesterov": True}), (d[1], "rmsprop", {"learning_rate": 0.02}),
            (d[2], "rmspropv2", {}), (d[3], "adadelta", {"averaging_ratio": 0.8, "epsilon": 1e-6})]
    out["z"] = table(segs, [0.5] * 4, capacity=1, init=inits[::-1], init_seed=6)
  return out


@pytest.mark.parametrize("dim", WIDTH_DIMS)
def test_widths_assign_add_reinit_restore(dim, dev):
  """upsert_apply_kernel<G, 2|3|4> at every G: assign_add onto fresh rows (init + value, uniform initializer) and
  resident ones with -0.0, subnormals and sums that overflow; reinitialize of resident and fresh keys; restore of
  rows exported from the table onto fresh and resident keys, with timestamps moving backwards."""
  seed = zlib.crc32(f"width/{dim}".encode())

  def fn():
    rng = np.random.default_rng(seed)
    w = World(dev, width_tables(dim), 1)
    names = w.names
    keys = {n: rand_keys(rng, 300) for n in names}
    sp = lambda n: SPECIAL[rng.integers(0, SPECIAL.size, (n, dim))]
    w.assign({n: (keys[n], rng.standard_normal((300, dim)).astype(np.float32)) for n in names}, T0, add=True)
    w.check()
    v = sp(300)
    v[:10] = np.float32(3e38)
    w.assign({n: (keys[n], v) for n in names}, T0 + 1, add=True)                  # resident: special sums
    w.assign({n: (keys[n][:10], np.full((10, dim), 3e38, np.float32)) for n in names}, T0 + 2, add=True)  # -> inf
    w.check()
    for n in names:   # reinitialize: resident and fresh keys, duplicates
      w.reinit(n, np.concatenate([keys[n][:100], rand_keys(rng, 50, exclude=keys[n]), keys[n][:7]]), T0 + 3)
    w.check()
    for n in names:   # restore the table's own rows shuffled onto other keys, fresh and resident, ts backwards
      ids, rows = w.export(n)
      rows = rows[np.argsort(ids)]
      rows[:, -1] = np.asarray(T0 - rng.integers(0, 10 * DAY, rows.shape[0]), np.uint32).view(np.float32)
      tgt = np.concatenate([keys[n][150:250], rand_keys(rng, 60, exclude=w.written[n])])
      w.restore(n, tgt, rows[rng.integers(0, rows.shape[0], tgt.size)])
    w.check()
    return w.no_aliasing(T0 + 4)

  run_case(fn)


def test_width_matrix_covers_every_lane_group():
  assert {pick_group(d) for d in WIDTH_DIMS} == set(GS)


# ------------------------------------------------------------------------------------------------
# growth
# ------------------------------------------------------------------------------------------------
def test_finalize_branches_and_row_growth_in_one_call(dev):
  """Three tables with 200 rows on the free list each; one assign call brings 150 (m < fc), 200 (m == fc) and 260
  (m > fc: the bump allocator continues) new keys.  The call asks for more rows than the 1024-row slab and the free
  list hold, so the slab grows in the same call; in the m > fc table the bump allocator then hands out rows past
  1024, which exist only because of that growth (without it error bit 2 is set and the row is not written)."""
  def fn():
    rng = np.random.default_rng(31)
    caps = {"lt": 1, "eq": 1, "gt": 1}
    w = World(dev, {n: sgd(4, 1, slot_expire_times={7: 1}, default_expire_time=36500) for n in caps}, 1)
    base = {n: rand_keys(rng, 1000) for n in caps}
    for n in caps:   # 200 of them in slot 7: they expire after a day
      base[n][:200] = (np.int64(7) << np.int64(48)) | (base[n][:200] & np.int64((1 << 48) - 1))
    w.assign({n: (base[n], ivals(rng, 1000, 4)) for n in caps}, T0)
    w.check()
    for n in caps:
      w.evict(n, T0 + DAY)
    w.check()
    for n in caps:
      c = w.gpu.counters(n)
      assert c["free"] == 200 and c["bump"] == 1000, c
    m = {"lt": 150, "eq": 200, "gt": 260}
    # with 400 resident keys besides: the call asks for more rows than the slab and the free list hold (224)
    new = {n: rand_keys(rng, m[n], exclude=w.written[n]) for n in caps}
    call = {n: np.concatenate([new[n], base[n][200:600]]) for n in caps}
    w.assign({n: (call[n], ivals(rng, call[n].size, 4)) for n in caps}, T0 + DAY)
    w.check()
    for n in caps:
      c = w.gpu.counters(n)
      assert c["free"] == max(0, 200 - m[n]) and c["bump"] == 1000 + max(0, m[n] - 200), (n, c)
    assert w.gpu.counters("gt")["bump"] > 1024
    return w.no_aliasing(T0 + DAY + 1)

  run_case(fn)


def test_stash_groups_survive_two_rehashes(dev):
  """Closed pairs of 9, 10 and 12 keys that share their pair at nb, 2·nb and 4·nb: each call after the first
  rehashes (the stash holds entries), rehash_kernel puts the same excess back into the stash."""
  def fn():
    rng = np.random.default_rng(32)
    w = World(dev, {"t": sgd(8, 1)}, 1)
    nb = w.nb["t"]
    pk = cp.BucketPicker(nb, rng, levels=2)
    groups = [cp.stable_keys(nb, pk.take(), pk.take(), m, rng, levels=2) for m in (9, 10, 12) * 3]
    used = {nb << j: pk.used[2 - j] for j in range(3)}
    want = cp.predicted_stash([g.size for g in groups])
    keys = np.concatenate(groups)
    w.assign({"t": (keys, ivals(rng, keys.size, 8))}, T0)
    w.check(stash={"t": want}, moves=True)
    for step in (1, 2):
      bg = cp.avoiding(rand_keys(rng, 400, exclude=w.written["t"]), used, (nb, 2 * nb, 4 * nb))[:60]
      k = np.concatenate([keys, bg])
      w.assign({"t": (k, ivals(rng, k.size, 8))}, T0 + step)
      assert w.rehashes["t"] == step and w.nb["t"] == nb << step
      w.check(stash={"t": want})
    return w.no_aliasing(T0 + 3)

  run_case(fn)


def test_back_to_back_duplicate_heavy_inserts_from_stale_snapshots(dev):
  """32 assign_add calls of 1200 ids (about 400 distinct, half of them new) on a table of capacity 1, with no host
  synchronisation between them: growth and rehash are decided from counter snapshots that lag the device."""
  def case():
    rng = np.random.default_rng(33)
    w = World(dev, {"t": sgd(16, 1)}, 1)
    live = np.zeros(0, np.int64)
    for i in range(32):
      new = rand_keys(rng, 200, exclude=w.written["t"])
      u = np.concatenate([new, rng.permutation(live)[:200]]) if live.size else new
      ids = rng.permutation(np.repeat(u, rng.integers(1, 6, u.size)))
      v = ivals(rng, ids.size, 16)
      w.note({"t": ids})
      w.gpu.assign_add({"t": (T(ids, dev), T(v, dev))}, req_time=T0 + i)
      w.cpu.assign_add({"t": (ids, v)}, req_time=T0 + i)
      live = np.union1d(live, u)
    w.expect |= upsert_kernels(pick_group(16), OP_ASSIGN_ADD, False) | {"rehash_kernel"}
    w.rehashes_known = False
    w.check()
    return w.no_aliasing(T0 + 40)

  run_case(case)


# ------------------------------------------------------------------------------------------------
# eviction
# ------------------------------------------------------------------------------------------------
def test_eviction_buckets_stash_boundaries_and_reuse(dev):
  """Per-slot expiry pairs and the default; an entry exactly expire·86400 old goes, one second younger stays;
  entries in buckets and in the stash (tombstones); then the evicted keys and new ones take the freed rows, and a
  second eviction.  The second round's update times cross 2^32: both stores keep the low 32 bits of the timestamp,
  so an entry written at or after 2^32 holds a small ts, and an eviction at a time past 2^32 removes it whatever its
  expiry, on the device as in the oracle; the entries written just before 2^32 follow their expiry."""
  def fn():
    rng = np.random.default_rng(34)
    cfg = {"t": sgd(8, 4096, slot_expire_times={1: 1, 2: 3, 3: 7}, default_expire_time=2)}
    w = World(dev, cfg, 4096)
    nb = w.nb["t"]
    pk = cp.BucketPicker(nb, rng, levels=3)   # the groups stay closed through the rehashes of the first round

    def in_slot(keys, s):
      return (np.int64(s) << np.int64(48)) | (keys & np.int64((1 << 48) - 1))

    groups = [cp.colliding_keys(nb << 3, pk.take(), pk.take(), 12, rng, slots={1, 2, 3, 4}) for _ in range(6)]
    crowd = np.concatenate(groups)
    bg = rand_keys(rng, 3000)
    bg = np.concatenate([in_slot(bg[i::4], s) for i, s in enumerate((1, 2, 3, 9))])
    levels = [nb << j for j in range(4)]
    bg = rng.permutation(cp.avoiding(bg, {nb << j: pk.used[3 - j] for j in range(4)}, levels))[:1200]
    keys = np.concatenate([crowd, bg])
    for base in (T0, (1 << 32) - 2 * DAY):     # the second round's update times cross 2^32
      ts = base + rng.integers(0, 3 * DAY, keys.size)
      wrapped = keys[(ts // DAY) * DAY + 17 >= 1 << 32]
      assert (wrapped.size > 0) == (base != T0)
      for t in np.unique(ts // DAY):   # one call per day of timestamps: every entry gets its own ts
        sel = keys[ts // DAY == t]
        w.assign({"t": (sel, ivals(rng, sel.size, 8))}, int(t * DAY + 17))
      w.check()
      if base == T0:
        assert w.gpu.counters("t")["stash"] > 0   # entries in the stash: evicting them leaves tombstones
      now = int(ts.max() // DAY * DAY + 17) + DAY
      w.evict("t", now - 1)            # one second short of the boundary for the youngest day
      w.check()
      w.evict("t", now)                # exactly on it
      w.check()
      assert w.cpu.size("t") < keys.size
      if wrapped.size:
        assert now >= 1 << 32 and not w.cpu.contains("t", wrapped).any()   # truncated ts: all of them expired
        kept = keys[((ts // DAY) * DAY + 17 < 1 << 32) & (ts // DAY == ts.max() // DAY - 1)]
        assert not kept.size or w.cpu.contains("t", kept).any()
      back = np.concatenate([keys[::3], rand_keys(rng, 100, exclude=w.written["t"])])
      w.assign({"t": (back, ivals(rng, back.size, 8))}, now)   # evicted keys and new ones into the freed rows
      w.check()
    return w.no_aliasing((1 << 32) + 10 * DAY)

  run_case(fn)


# ------------------------------------------------------------------------------------------------
# export and restore
# ------------------------------------------------------------------------------------------------
def test_export_chunks_and_restore_elsewhere(dev):
  """Export in chunks of 1, 3, 4096 and of exactly the bucket slots (the chunk ends at the stash); tombstones and
  empty tables export nothing; restore into a table of another capacity and into one that holds some of the keys
  with other values."""
  def fn():
    rng = np.random.default_rng(35)
    cfg = lambda cap: table([(5, "adam", {}), (3, "ftrl", {"initial_accumulator_value": 0.1, "beta": 1.0,
                                                           "l1": 0.0, "l2": 0.0})], [0.5, 0.5], capacity=cap,
                            init=None, init_seed=3, slot_expire_times={5: 1}, default_expire_time=100)
    w = World(dev, {"a": cfg(2048), "b": cfg(1), "c": cfg(8192), "e": cfg(1)}, {"a": 2048, "b": 1, "c": 8192,
                                                                                "e": 1})
    nb = w.nb["a"]
    ids, _ = w.export("e")
    assert ids.size == 0
    pk = cp.BucketPicker(nb, rng)
    grp = np.concatenate([cp.colliding_keys(nb, pk.take(), pk.take(), 11, rng, slots={5, 6}) for _ in range(4)])
    keys = np.concatenate([grp, cp.avoiding(rand_keys(rng, 1500), {nb: set(pk.used[0])}, (nb,))[:700]])
    w.optimize({"a": (keys, ivals(rng, keys.size, 8))}, T0)
    w.check(stash={"a": 12})
    w.evict("a", T0 + DAY)   # slot-5 keys go: tombstones in the stash
    w.check()
    full = w.export("a")
    for chunk in (1, 3, 4096, nb * cp.BUCKET_SLOTS):
      ids, rows = w.export("a", chunk)
      o, p = np.argsort(ids), np.argsort(full[0])
      np.testing.assert_array_equal(ids[o], full[0][p])
      np.testing.assert_array_equal(rows[o].view(np.uint32), full[1][p].view(np.uint32))
    o = np.argsort(full[0])   # export order is the device's: fix one before drawing from it
    ids, rows = full[0][o], full[1][o]
    # into a table of another capacity
    w.restore("b", ids, rows)
    w.check()
    # into one that already holds some keys with other values
    w.optimize({"c": (ids[::2], ivals(rng, ids[::2].size, 8))}, T0 + 5)
    w.check()
    w.restore("c", ids, rows)
    w.check()
    for n in ("b", "c"):
      np.testing.assert_array_equal(w.gpu.lookup_entry(n, T(ids, dev))["raw"].cpu().numpy().view(np.uint32),
                                    rows.view(np.uint32))
      assert w.gpu.size(n) == ids.size
    return w.no_aliasing(T0 + 6)

  run_case(fn)


# ------------------------------------------------------------------------------------------------
# stash overflow
# ------------------------------------------------------------------------------------------------
def test_stash_overflow_is_reported_and_other_tables_are_unaffected(dev):
  """4097 closed pairs of 9 keys in one call on a fresh table: 4097 entries for a 4096-entry stash.  The next size()
  raises "stash overflow"; the other table of the same MultiHashTable keeps working."""
  from monolith_b200 import _lib

  def fn():
    rng = np.random.default_rng(36)
    cap = 40000
    w = World(dev, {"full": sgd(4, cap), "ok": sgd(4, 1024)}, {"full": cap, "ok": 1024})
    nb = w.nb["full"]
    pk = cp.BucketPicker(nb, rng)
    keys = np.concatenate([cp.colliding_keys(nb, pk.take(), pk.take(), 9, rng) for _ in range(4097)])
    other = rand_keys(rng, 500)
    w.assign({"full": (keys, ivals(rng, keys.size, 4)), "ok": (other, ivals(rng, 500, 4))}, T0)
    with pytest.raises(_lib.MonoError, match="stash overflow"):
      w.gpu.size("full")
    c = w.gpu.counters("full")
    assert c["error"] & 1 and c["stash"] == 4097 and c["inflight"] == 0, c
    w.names = ["ok"]   # the other table: every check still holds, and it takes further calls
    w.check()
    more = rand_keys(rng, 300, exclude=w.written["ok"])
    w.assign({"ok": (more, ivals(rng, 300, 4))}, T0 + 1)
    w.check()
    return w.no_aliasing(T0 + 2)

  run_case(fn)


# ------------------------------------------------------------------------------------------------
# inventory: keep last
# ------------------------------------------------------------------------------------------------
def test_every_write_kernel_ran_and_no_other():
  """The union of what the cases above ran (run this file whole: the inventory is collected from them)."""
  assert SEEN, "no write-side kernel was recorded: the inventory is the union of this file's other tests"
  missing, extra = sorted(INVENTORY - SEEN), sorted(SEEN - INVENTORY)
  assert not missing and not extra, f"never ran: {missing}; ran but not listed: {extra}"
