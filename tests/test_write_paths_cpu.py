"""The rules tests/test_gpu_write_paths.py aims its cases at, pinned against the CUDA sources, and self-tests of the
write-side key builders of tests/cuckoo_place.py.  A change to a constant, a counter, an error bit, the growth or
eviction rule, the row allocation, the scratch-set claim or the upsert kernel sequence fails here by name; the GPU
cases then have to be re-aimed."""
import os
import re

import numpy as np

from tests import cuckoo_place as cp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "monolith_b200", "csrc")


def _src(name):
  with open(os.path.join(CSRC, name)) as f:
    return re.sub(r"\s+", " ", f.read())


def _body(src, head):
  """The brace-balanced body that follows the first occurrence of `head`."""
  i = src.index(head)
  i = src.index("{", i)
  depth = 0
  for j in range(i, len(src)):
    depth += {"{": 1, "}": -1}.get(src[j], 0)
    if depth == 0:
      return src[i:j + 1]
  raise AssertionError(f"unbalanced body after {head}")


def _cu_sources():
  return {f: _src(f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")}


# the three inserters of an upsert call, each of which takes its row from common.cuh insert_new_row
INSERTERS = (("ops.cu", "resolve_miss_kernel("), ("bwd.cu", "claim_miss_kernel("), ("xstep.cu", "xmiss_insert_kernel("))
# the two claims of the epoch-versioned scratch set (engine.h ClaimSet)
EPOCH_CLAIMS = (("bwd.cu", "fid_claim_kernel("), ("xstep.cu", "xmiss_claim_kernel("))


# counter words (common.cuh) as tests/test_gpu_write_paths.py and MultiHashTable.counters read them
COUNTERS = {"bump": 0, "free": 1, "size": 2, "stash": 3, "error": 4, "moves": 8, "inflight": 9}
ERROR_BITS = {1: "stash overflow", 2: "row slab overflow", 4: "lost a marked slot"}


def test_cuckoo_constants():
  c = _src("common.cuh")
  assert "constexpr int kBucketSlots = 4;" in c and cp.BUCKET_SLOTS == 4
  assert "constexpr int kMaxEvictions = 48;" in c
  assert "constexpr uint32_t kEmptyRow = 0xFFFFFFFFu;" in c and "constexpr uint32_t kTombRow = 0xFFFFFFFEu;" in c
  assert "d.stash_cap = 4096;" in _src("table.cu") and cp.STASH_CAP == 4096
  # the stash probe starts at bits 17.. of the hash, in the insert as in the probes
  assert "uint32_t s = (uint32_t)(mix64((uint64_t)e.key) >> 17) & mask;" in c and cp.STASH_SHIFT == 17


def test_counter_words_and_error_bits_with_one_row_allocator():
  """The counter words and where each error bit is set; bit 2 (row slab overflow) is set in insert_new_row alone,
  which every upsert inserter calls."""
  c = _src("common.cuh")
  for name, word in [("Bump", 0), ("Free", 1), ("Size", 2), ("Stash", 3), ("Error", 4), ("Moves", 8),
                     ("Inflight", 9)]:
    assert f"kCtr{name} = {word}," in c, name
  assert "kNumCtrs = 16" in c
  from monolith_b200.multi_hash_table_ops import MultiHashTable
  assert MultiHashTable.COUNTER_WORDS == COUNTERS
  # where each bit is set: 1 when the stash is full, 2 when the row slab is, 4 when a marked slot was lost
  ins = _body(c, "__device__ __forceinline__ void cuckoo_insert(")
  assert "atomicOr(t->ctrs + kCtrError, 1u);" in ins and "if (copied) atomicOr(t->ctrs + kCtrError, 4u);" in ins
  alloc = _body(c, "__device__ __forceinline__ uint32_t insert_new_row(")
  assert "if (row >= t->row_cap) { atomicOr(t->ctrs + kCtrError, 2u); return kEmptyRow; }" in alloc
  for f, head in INSERTERS:
    assert "insert_new_row(t, " in _body(_src(f), head), f
  # the stash count rises before the entry is visible, and only on the stash path
  assert ins.count("atomicAdd(t->ctrs + kCtrStash, 1u);") == 1


def test_read_counters_sync_raises_on_every_error_bit():
  """size(), ensure_capacity and every other reader of the counters raise on each error bit with its own message;
  mono_mtable_counters copies the words without checking them."""
  t = _src("table.cu")
  body = _body(t, "void read_counters_sync(")
  assert "copy_counters_sync(mt, k, s, out);" in body
  for bit, what in ERROR_BITS.items():
    m = re.search(r"if \(out\[kCtrError\] & %du\) throw CudaError\((.*?)\);" % bit, body)
    assert m and what in m.group(1), f"error bit {bit} ({what}) does not raise"
  copy = _body(t, "void copy_counters_sync(")
  assert "throw" not in copy
  capi = _body(_src("capi.cu"), "int mono_mtable_counters(")
  assert "copy_counters_sync(" in capi and "read_counters_sync" not in capi
  # a completed snapshot with any error bit set goes through the raising reader
  ens = _body(t, "void ensure_capacity(")
  assert ens.count("if (t.h_snap[kCtrError]) {") == 2 and ens.count("read_counters_sync(mt, k, s, tmp);") == 2


def test_ensure_capacity_rule():
  """Rehash when the keys may exceed 0.75 of the bucket slots, or when the stash holds anything (live or tombstone);
  grow the rows when the call may take more rows than the free list and the unused slab hold."""
  ens = _body(_src("table.cu"), "void ensure_capacity(")
  assert "uint64_t avail = (uint64_t)d.row_cap - t.snap_bump + t.snap_free;" in ens
  assert "rows = n_new + slack > avail;" in ens
  assert "buckets = (double)size_ub > 0.75 * (double)d.num_buckets * kBucketSlots || t.snap_stash > 0;" in ens
  assert "uint64_t size_ub = t.snap_size + slack + n_new;" in ens
  assert "if (nr) grow_rows(mt, k, t.snap_bump - t.snap_free + n_new, s);" in ens
  assert "if (nbk) rehash(mt, k, t.snap_size + n_new, s);" in ens


def test_rehash_and_grow_sizing():
  t = _src("table.cu")
  rh = _body(t, "static void rehash(")
  assert "uint32_t nnb = std::max<uint64_t>((uint64_t)d.num_buckets * 2, buckets_for(keys_target));" in rh
  assert "cudaMemsetAsync(d.ctrs + kCtrStash, 0, sizeof(uint32_t), s)" in rh   # the stash is rebuilt from scratch
  assert "rehash_kernel<<<" in rh
  gr = _body(t, "static void grow_rows(")
  assert "uint64_t ncap = std::max<uint64_t>((uint64_t)d.row_cap * 2, need_total + need_total / 8);" in gr
  bf = _body(t, "static uint32_t buckets_for(")
  assert "uint64_t nb = (keys + 1) / 2 + 1;" in bf and "if (nb < 64) nb = 64;" in bf
  assert "uint64_t rows = std::max<uint64_t>(cfg.initial_capacity, 1024);" in t
  # restated in cuckoo_place
  assert cp.buckets_for(1) == 513 and cp.buckets_for(40000) == 20001
  # the rehash re-inserts every live entry of the buckets and of the stash, tombstones dropped
  rk = _body(t, "rehash_kernel(")
  assert "if (e.row < kTombRow) {" in rk and "cuckoo_insert(nt, e);" in rk


def test_eviction_rule():
  """An entry expires when max_update_time - ts >= expire_days * 86400 (the boundary evicts); its slot becomes empty
  in a bucket and a tombstone in the stash (so that stash probe chains stay intact); the row goes to the free list."""
  ev = _body(_src("table.cu"), "evict_kernel(")
  assert "if (max_update_time - (int64_t)e.ts >= expire * 86400LL) {" in ev
  assert "int64_t expire = t->default_expire_days;" in ev
  assert "if (s_pairs[2 * j] == slot) { expire = s_pairs[2 * j + 1]; break; }" in ev
  assert "if (i >= slots) dead.row = kTombRow;" in ev and "Entry dead = empty;" in ev
  assert "t->free_list[idx] = e.row & kRowMask;" in ev and "atomicSub(t->ctrs + kCtrSize, 1u);" in ev
  assert "kCtrStash" not in ev           # a tombstone still counts as a stash entry until the next rehash
  # export skips empty slots and tombstones alike
  ex = _body(_src("table.cu"), "export_kernel(")
  assert "if (e.row >= kTombRow) continue;" in ex


def test_upsert_ops_kernel_sequence_and_row_allocator():
  """The UpsertOp values are the second template argument of upsert_apply_kernel in the kernel names; one upsert
  pass is resolve_hit, resolve_miss, upsert_apply (restore: the <true> resolves), then upsert_finalize; every
  inserter takes its row from insert_new_row, whose tickets upsert_finalize folds."""
  e = _src("engine.h")
  assert "enum UpsertOp { kOpOptimize = 0, kOpAssign = 1, kOpAssignAdd = 2, kOpReinit = 3, kOpRestore = 4 };" in e
  ops = _src("ops.cu")
  pair = _body(ops, "static void launch_upsert_pair(")
  seq = re.findall(r"(resolve_hit_kernel<R>|resolve_miss_kernel<R>|upsert_apply_kernel<G, OP>)\s*<<<", pair)
  assert seq == ["resolve_hit_kernel<R>", "resolve_miss_kernel<R>", "upsert_apply_kernel<G, OP>"]
  assert "constexpr bool R = OP == kOpRestore;" in pair
  ru = _body(ops, "void run_upsert(")
  assert ru.count("launch_upsert_finalize(") == 3      # unique, every duplicate round, the dedup-sum pass
  assert "dup_claim_kernel<<<" in ru and "dup_split_kernel<<<" in ru
  grp = _body(ops, "void run_upsert_groups(")
  seq = re.findall(r"(resolve_hit_kernel<false>|dup_claim_kernel|miss_split_kernel|resolve_miss_kernel<false>|"
                   r"miss_follow_kernel|launch_upsert_finalize|launch_optimize_apply)", grp)
  assert seq == ["resolve_hit_kernel<false>", "resolve_hit_kernel<false>", "dup_claim_kernel", "miss_split_kernel",
                 "resolve_miss_kernel<false>", "miss_follow_kernel", "launch_upsert_finalize", "launch_optimize_apply"]
  # finalize: both branches of the free-list fold
  fin = _body(ops, "__global__ void upsert_finalize_kernel(")
  assert "if (m <= fc) { t->ctrs[kCtrFree] = fc - m; } else { t->ctrs[kCtrFree] = 0; t->ctrs[kCtrBump] += m - fc; }" in fin
  # a fresh row is taken from the top of the free list first, then from the bump allocator, in one place that every
  # inserter calls; no other code takes a ticket that finalize folds
  alloc = _body(_src("common.cuh"), "__device__ __forceinline__ uint32_t insert_new_row(")
  assert "const uint32_t ticket = atomicAdd(t->ctrs + kCtrMiss, 1u);" in alloc
  assert "ticket < fc ? t->free_list[fc - 1 - ticket] : t->ctrs[kCtrBump] + (ticket - fc)" in alloc
  assert "cuckoo_insert(t, e);" in alloc
  for f, head in INSERTERS:
    assert "insert_new_row(t, " in _body(_src(f), head), f
  for f, s in _cu_sources().items():
    assert not re.search(r"atomicAdd\([^;]*kCtrMiss", s), f
  # the sharded step's insert pipeline
  xs = _src("xstep.cu")
  seq = re.findall(r"(xowner_resolve_kernel|xmiss_claim_kernel|xmiss_insert_kernel|xmiss_follow_kernel)<<<", xs)
  assert seq == ["xowner_resolve_kernel", "xmiss_claim_kernel", "xmiss_insert_kernel", "xmiss_follow_kernel"]


def test_epoch_set_claim():
  """Both claims of the epoch-versioned scratch set run common.cuh claim_epoch_slot from epoch_slot's start: a slot
  whose epoch is not the call's is empty and is claimed with a CAS against what was read."""
  c = _src("common.cuh")
  assert "return __umulhi((uint32_t)(mix64((uint64_t)key) >> 24), R);" in _body(c, "uint32_t epoch_slot(")
  claim = _body(c, "uint32_t claim_epoch_slot(")
  assert "for (uint32_t probes = 0; !BOUNDED || probes < R; ++probes) {" in claim
  assert "if (e.key == key) return base + idx;" in claim and claim.endswith("return kNoSlot; }")
  assert "while (e.ts != epoch) {" in claim and "const Entry old = cas_entry_old(p, e, ne);" in claim
  assert "if (same_entry(old, e)) { *won = true; e = ne; }" in claim
  # the backward's claim reads through L1 and gives up on a full region; the sharded step's set always has room
  for (f, head), targs in zip(EPOCH_CLAIMS, ("ld_entry, true", "ld_entry_cg, false")):
    assert re.search(r"claim_epoch_slot<%s>\([^;]*epoch_slot\(key, " % targs, _body(_src(f), head)), f
  # the claim kernel's prefetch aims at the same start slot
  assert "prefetch_l2(set + o_n * R + epoch_slot(key_next, R));" in _body(_src("bwd.cu"), "fid_claim_kernel(")
  for f, s in _cu_sources().items():
    assert "cas_entry_old" not in s, f


def test_pick_group():
  from tests.test_gpu_forward_paths import pick_group
  ops = _body(_src("ops.cu"), "int pick_group(int max_dim)")
  assert "int v = (max_dim + 3) / 4;" in ops and "while (g < v && g < 32) g <<= 1;" in ops
  assert [pick_group(d) for d in (1, 16, 17, 32, 33, 64, 65, 512)] == [4, 4, 8, 8, 16, 16, 32, 32]


# ------------------------------------------------------------------------------------------------
# the builders
# ------------------------------------------------------------------------------------------------
def test_stable_keys_keep_their_pair_through_two_doublings():
  rng = np.random.default_rng(5)
  nb = cp.buckets_for(1)
  pk = cp.BucketPicker(nb, rng, levels=2)
  for _ in range(20):
    b1, b2 = pk.take(), pk.take()
    k = cp.stable_keys(nb, b1, b2, 12, rng)
    assert np.unique(k).size == 12
    for j, n in enumerate((nb, 2 * nb, 4 * nb)):
      p1, p2 = cp.bucket_pair(k, n)
      assert (p1 == b1 >> (2 - j)).all() and (p2 == b2 >> (2 - j)).all(), n
  # images at every level are distinct across groups
  for u in pk.used:
    assert len(u) == 40


def test_copy_first_group_shape():
  rng = np.random.default_rng(6)
  nb = cp.buckets_for(4096)
  pk = cp.BucketPicker(nb, rng)
  fill, new = cp.copy_first_group(nb, pk, rng)
  b1, b2 = cp.bucket_pair(fill, nb)
  nb1, nb2 = (int(x[0]) for x in cp.bucket_pair(new, nb))
  assert list(b1[:4]) == [nb1] * 4 and list(b1[4:]) == [nb2] * 4
  # every filler's alternate bucket is its own and is neither of the newcomer's
  assert len(set(b2.tolist())) == 8 and not ({nb1, nb2} & set(b2.tolist()))


def test_predicted_stash():
  assert cp.predicted_stash([9, 10, 12]) == 1 + 2 + 4
  assert cp.predicted_stash([8, 3, 0]) == 0
  assert cp.predicted_stash([9] * 4097) == 4097 > cp.STASH_CAP


def test_avoiding():
  rng = np.random.default_rng(7)
  nb = 513
  keys = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, 5000, dtype=np.int64)
  used = {}
  for n in (nb, 2 * nb):
    b1, b2 = cp.bucket_pair(keys[:100], n)
    used[n] = set(b1.tolist()) | set(b2.tolist())
  kept = cp.avoiding(keys[100:], used, (nb, 2 * nb))
  assert 0 < kept.size < 4900
  for n in (nb, 2 * nb):
    b1, b2 = cp.bucket_pair(kept, n)
    assert not (set(b1.tolist()) | set(b2.tolist())) & used[n]
