"""What tests/test_gpu_reorder_paths.py assumes, checked without a GPU: dedup.cu's tile, grid and scan-chunk geometry,
the C ABI's argument checks (all before the device is selected), and the oracle on the shapes of the three sizes the
op used to get wrong."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from monolith_b200 import _lib
from tests import orc
from tests.test_gpu_reorder_paths import GRID_PER_SM, I32_MAX, MAX_IDS, SCAN_CHUNK, THREADS, TILE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(name):
  with open(os.path.join(ROOT, "monolith_b200", "csrc", name)) as f:
    return re.sub(r"\s+", " ", f.read())


@pytest.fixture(scope="module")
def lib():
  if not os.path.exists(_lib.LIB_PATH):
    import __graft_entry__
    __graft_entry__.build()
  return _lib.load()


# ------------------------------------------------------------------------------------------------
# the geometry the GPU sizes are aimed with
# ------------------------------------------------------------------------------------------------
def test_tile_grid_and_scan_chunk_match_dedup_cu():
  src = _src("dedup.cu")
  assert f"constexpr int kThreads = {THREADS};" in _src("common.cuh") + _src("engine.h")
  assert "constexpr int kTileItems = 8;" in src and "constexpr int kTile = kThreads * kTileItems;" in src
  assert TILE == THREADS * 8 == 2048
  assert "const int nblk = (int)std::max<int64_t>(1, (M + kTile - 1) / kTile);" in src
  # both rank passes run min(nblk, SMs * 8) blocks and walk the tiles grid-stride
  assert f"const int g = std::min(nblk, device_sms() * {GRID_PER_SM});" in src
  assert src.count("dd_rank_kernel<0><<<g, kThreads, 0, s>>>") == 1 and src.count("dd_rank_kernel<1><<<g, kThreads") == 1
  assert "for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {" in src
  # the scan: one block of SCAN_CHUNK threads walking the block counts chunk by chunk, with a carry
  assert f"dd_scan_kernel<<<1, {SCAN_CHUNK}, 0, s>>>" in src
  assert f"__launch_bounds__({SCAN_CHUNK}) dd_scan_kernel" in src
  assert "for (int base = 0; base < nblk; base += blockDim.x) {" in src
  assert "if (threadIdx.x == blockDim.x - 1) carry = carry + warp_tot[31];" in src
  # the limits the tests probe
  assert "constexpr int64_t kMaxIds = (int64_t)1 << 30;" in src and MAX_IDS == 1 << 30
  assert "constexpr int kMaxLists = 1 << 25;" in src
  assert "const int pair = cls >= 0 ? cls * K + m : -1;" in src


def test_geometry_sizes_of_the_gpu_matrix():
  """The named sizes hit the boundaries they are named after, on an H100 (132 SMs) and on any SM count."""
  for sms in (1, 78, 114, 132, 144):
    g = sms * GRID_PER_SM
    nblk = lambda M: max(1, -(-M // TILE))
    assert nblk(g * TILE) == g and nblk(g * TILE + 1) == g + 1
    assert nblk(3 * g * TILE + 1) == 3 * g + 1
  assert [max(1, -(-M // TILE)) for M in (2047, 2048, 2049)] == [1, 1, 2]
  assert [-(-M // TILE) for M in (SCAN_CHUNK * TILE - 1, SCAN_CHUNK * TILE, SCAN_CHUNK * TILE + 1)] == [1024, 1024, 1025]
  assert -(-(3 * 132 * 8 + 1) // SCAN_CHUNK) == 4                 # the 6.5 M-id case: four scan chunks on an H100
  assert (3 * 132 * 8 * TILE + 1) < 7_000_000


# ------------------------------------------------------------------------------------------------
# the C ABI's argument checks run before the device is selected
# ------------------------------------------------------------------------------------------------
def _reorder(lib, splits, K, N, dims, r0=0, host=True):
  sp = (C.c_int64 * len(splits))(*splits)
  dm = (C.c_int32 * len(dims))(*dims)
  fake = C.c_void_p(0x1000)                              # never dereferenced: the checks come first
  ss = (C.c_int32 * 64)()
  return lib.mono_reorder_by_indices(0, fake, sp, K, N, dm, r0, fake, None, fake, ss if host else None, None, None,
                                     None)


REJECT = [
    ("no lists", dict(splits=[0], K=0, N=1, dims=[1]), b"num_lists and num_shards must be positive"),
    ("no shards", dict(splits=[0, 4], K=1, N=0, dims=[1]), b"num_lists and num_shards must be positive"),
    ("65 shards", dict(splits=[0, 4], K=1, N=65, dims=[1]), b"num_shards > 64"),
    ("2^25+1 lists", dict(splits=[0, 4], K=(1 << 25) + 1, N=1, dims=[1]), b"num_lists > 2^25"),
    ("rank0_empty N1", dict(splits=[0, 4], K=1, N=1, dims=[1], r0=1), b"rank0_empty needs at least 2 shards"),
    ("split start", dict(splits=[1, 4], K=1, N=1, dims=[1]), b"id_split must start at 0"),
    ("split decreases", dict(splits=[0, 5, 4, 9], K=3, N=2, dims=[1, 1, 1]), b"id_split must not decrease"),
    ("2^30+1 ids", dict(splits=[0, MAX_IDS + 1], K=1, N=1, dims=[1]), b"more than 2^30 ids"),
    ("2^30+1 ids, K3", dict(splits=[0, 5, MAX_IDS, MAX_IDS + 1], K=3, N=4, dims=[1, 1, 1]), b"more than 2^30 ids"),
    ("dim 0", dict(splits=[0, 4], K=1, N=1, dims=[0]), b"dims must be positive"),
    ("dim -3 in the middle", dict(splits=[0, 1, 2, 3], K=3, N=2, dims=[4, -3, 4]), b"dims must be positive"),
    ("ids x dim, no host outputs", dict(splits=[0, 2048], K=1, N=1, dims=[1 << 20], host=False), b"ids x dim"),
    ("ids x dim, no host outputs, 2^30 ids", dict(splits=[0, MAX_IDS], K=1, N=4, dims=[2], host=False), b"ids x dim"),
]


@pytest.mark.parametrize("args,msg", [r[1:] for r in REJECT], ids=[r[0] for r in REJECT])
def test_cabi_rejects_bad_reorder_arguments_before_the_device(args, msg, lib):
  n0 = lib.mono_kernel_launch_count()
  assert _reorder(lib, **args) == -1                     # MONO_ERR_INVALID_ARGUMENT
  assert msg in lib.mono_last_error()
  assert lib.mono_kernel_launch_count() == n0


def test_cabi_dedup_rejects_more_than_2_30_ids(lib):
  fake = C.c_void_p(0x1000)
  assert lib.mono_dedup(0, fake, MAX_IDS + 1, fake, fake, None, None, None) == -1
  assert b"more than 2^30 ids" in lib.mono_last_error()


def test_cabi_accepts_edge_reorder_arguments_and_reaches_the_device(lib):
  if torch.cuda.is_available():
    pytest.skip("with a GPU the call would launch on fake pointers")
  edge = [dict(splits=[0, MAX_IDS], K=1, N=64, dims=[1]),                          # exactly 2^30 ids
          dict(splits=[0, 1], K=1, N=1, dims=[I32_MAX], host=False),               # 1 x (2^31 - 1) floats
          dict(splits=[0, 2048], K=1, N=1, dims=[(1 << 20) - 1], host=False),
          dict(splits=[0, 2048], K=1, N=1, dims=[1 << 20]),                        # host outputs: checked after
          dict(splits=[0, 0, 0, 3], K=3, N=2, dims=[1, 1, 1], r0=1),
          dict(splits=[0, 0], K=1, N=1, dims=[1])]
  for a in edge:
    assert _reorder(lib, **a) == -3, a                   # MONO_ERR_CUDA: the checks passed, no device here


# ------------------------------------------------------------------------------------------------
# the oracle on the three defect shapes
# ------------------------------------------------------------------------------------------------
def test_scratch_set_capacity_fits_uint32_up_to_2_30_ids():
  """run_reorder's sizing loop (uint32 cap = 1024; while (cap < 2 M) cap <<= 1) restated: 2^31 slots at 2^30 ids;
  past that the uint32 doubles to 0 and the loop would never end, so 2^30 is the limit."""
  def cap_u32(M, limit=40):
    cap = 1024
    for _ in range(limit):
      if cap >= 2 * max(M, 1):
        return cap
      cap = (cap << 1) & 0xFFFFFFFF
    return None                                          # did not terminate
  assert cap_u32(1) == 1024 and cap_u32(513) == 2048
  assert cap_u32(MAX_IDS) == 1 << 31
  assert cap_u32(MAX_IDS + 1) is None
  assert "uint32_t cap = 1024; while (cap < 2 * (uint64_t)std::max<int64_t>(M, 1)) cap <<= 1;" in _src("dedup.cu")
  # 16-byte set entries for 2^32 slots would be 64 GiB of an 80 GB card before the ids and per-id scratch
  assert 16 * 2 ** 32 + 16 * (MAX_IDS + 1) > 80e9


def test_oracle_keeps_shard_list_pairs_apart_past_65536_lists():
  """The shape the old (shard * 65536 + list) key merged: shard 1 of list 0 and shard 0 of list 65536, the lists
  between them empty.  The oracle keeps them apart; the new key cls * K + m is unique per pair."""
  K, N = 65537, 2
  lists = [np.zeros(0, np.int64) for _ in range(K)]
  lists[0] = np.array([3], np.int64)
  lists[K - 1] = np.array([4], np.int64)
  out, ss, sl, sz, offs = orc.reorder_by_indices(lists, N, [1] * K)
  assert out.tolist() == [4, 3] and ss.tolist() == [1, 1]
  assert sl[0 * K + 65536] == 1 and sl[1 * K + 0] == 1 and sl.sum() == 2
  assert offs.tolist() == [1, 0]
  assert 1 * 65536 + 0 == 0 * 65536 + 65536                 # the old key collides
  assert 1 * K + 0 != 0 * K + 65536                         # the new one does not
  cls, m = np.meshgrid(np.arange(64, dtype=np.int64), np.arange(K, dtype=np.int64))
  keys = cls * K + m
  assert np.unique(keys).size == keys.size and keys.max() < 2 ** 31
  assert 63 * (1 << 25) + (1 << 25) - 1 == 2 ** 31 - 1      # K = 2^25: the largest key is INT32_MAX


def _exact_offsets(lists, N, dims):
  """fused_emb_offset in int64: rank inside (shard, list) x dim + the (shard, list) segment's base."""
  shard = lambda v: (v % (1 << 64)) % N                  # (uint64)fid % N
  seen = [dict() for _ in lists]
  cnt = {}
  for m, l in enumerate(lists):
    for v in l.tolist():
      if v not in seen[m]:
        key = (shard(v), m)
        seen[m][v] = cnt.get(key, 0)
        cnt[key] = seen[m][v] + 1
  base, run = {}, 0
  for n in range(N):
    for m in range(len(lists)):
      base[(n, m)] = run
      run += cnt.get((n, m), 0) * dims[m]
  offs = [seen[m][v] * dims[m] + base[(shard(v), m)] for m, l in enumerate(lists) for v in l.tolist()]
  return np.array(offs, np.int64), run


def test_oracle_offsets_are_exact_up_to_2_31_minus_1_floats():
  """At exactly 2^31 - 1 floats the int32 offsets are the exact ones; one more float no longer fits an int32, which is
  why the op now refuses it.  Large dims keep the shapes small."""
  rng = np.random.default_rng(5)
  a = rng.integers(0, 1 << 40, 2047).astype(np.int64)
  cases = [([np.full(5, -9, np.int64)], 1, [I32_MAX]),
           ([np.concatenate([a, a[::2]]), np.array([9, 9], np.int64)], 3, [1 << 20, (1 << 20) - 1])]
  for lists, N, dims in cases:
    want, total = _exact_offsets(lists, N, dims)
    assert total == I32_MAX
    _, _, _, _, offs = orc.reorder_by_indices(lists, N, dims)
    np.testing.assert_array_equal(offs.astype(np.int64), want)
  # the 4096 x 2^20 shape: offsets up to 2^32 - 2^20, outside int32
  lists = [rng.integers(0, 1 << 40, 4096).astype(np.int64)]
  want, total = _exact_offsets(lists, 1, [1 << 20])
  assert total == 2 ** 32 and want.max() == 2 ** 32 - 2 ** 20 > I32_MAX
  # one list of 2048 ids of dim 2^20 is the smallest up-front rejection without host outputs: 2048 x 2^20 = 2^31
  assert 2048 * (1 << 20) == I32_MAX + 1 and 2048 * ((1 << 20) - 1) <= I32_MAX
