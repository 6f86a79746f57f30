// dedup.cu — requester-side FID dedup + shard partition on the GPU.
//
// Restates FusedReorderByIndicesOp (ref: RT/ops/fused_reorder_by_indices.cc:38-123) bit-exactly:
// per-list first-occurrence dedup, unique ids emitted shard-major / list-minor in first-occurrence
// order, and for every occurrence the float offset of its row in the post-all-to-all buffer.
// The reference walks the ids serially through an absl::flat_hash_map; here the order-defining
// quantity "rank of a first occurrence among earlier first occurrences of the same shard" is a
// stable multi-way partition computed with block histograms + a scan + warp match ballots
// (no atomics decide any output value, so the result is deterministic).
//
// passes (all coalesced streams over M ids; ~60 B/id of HBM traffic in total):
//   1 claim   : open-addressing scratch set keyed by (list, fid); 128-bit CAS claims a slot,
//               atomicMin keeps the lowest position = first occurrence
//   2 count   : per block, per shard: number of first occurrences  (+ per (shard,list) totals)
//   3 scan    : one block: exclusive scan of the block histograms per shard, and all the small
//               offset tables (shard_sizes, sharded_slot_sizes, output bases, emb offsets)
//   4 scatter : stable rank of every first occurrence -> output[] and rank[]
//   5 offsets : every occurrence -> fused_emb_offset[]
#include <algorithm>
#include <cstring>
#include <vector>

#include "engine.h"

namespace mono {

constexpr int kMaxShards = 64;
constexpr int kMaxLists = 1 << 25;                  // (shard, list) keys cls * K + m stay below 2^31
constexpr int64_t kMaxIds = (int64_t)1 << 30;       // the scratch set holds 2^31 16-byte slots at most
constexpr int kTileItems = 8;                       // ids per thread per tile
constexpr int kTile = kThreads * kTileItems;        // ids per block tile

struct DSet {  // 16-byte scratch-set entry, viewed as an Entry for the 128-bit CAS
  int64_t key;
  int32_t list;
  int32_t first_pos;
};

__device__ __forceinline__ int shard_of(int64_t fid, int n_eff, int rank0_empty) {
  // ref: shard_func, fused_reorder_by_indices.cc:121-123 (unsigned so that negative FIDs stay in range)
  return (int)((uint64_t)fid % (uint64_t)n_eff) + rank0_empty;
}

__device__ __forceinline__ int list_of(const int64_t* __restrict__ split, int K, int64_t i) {
  int lo = 0, hi = K - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (split[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads)
dd_claim_kernel(const int64_t* __restrict__ ids, int64_t M, const int64_t* __restrict__ split, int K,
                DSet* set, uint32_t mask, uint32_t* __restrict__ slot_of) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = ids[i];
    const int m = K > 1 ? list_of(split, K, i) : 0;
    uint32_t s = (uint32_t)(mix64((uint64_t)key * 0x9E3779B97F4A7C15ULL + (uint64_t)m) >> 20) & mask;
    while (true) {
      Entry e = ld_entry_cg(reinterpret_cast<Entry*>(set + s));
      if ((int32_t)e.row == -1) {  // list == -1: empty
        Entry v;
        v.key = key;
        v.row = (uint32_t)m;
        v.ts = (uint32_t)i;
        if (cas_entry(reinterpret_cast<Entry*>(set + s), empty_entry(), v)) break;
        continue;
      }
      if (e.key == key && (int32_t)e.row == m) {
        // first_pos only ever decreases: skip the atomic when the value just read is already
        // lower (this removes the same-address atomic storm of hot keys in Zipf batches)
        if ((int32_t)e.ts > (int32_t)i) atomicMin(&set[s].first_pos, (int32_t)i);
        break;
      }
      s = (s + 1) & mask;
    }
    slot_of[i] = s;
  }
}

// layout of the small device tables (int32), all inside one scratch block:
//   sizes      [N*K]    sharded_slot_sizes (shard-major)           -> also returned to the caller
//   shard_sz   [N]
//   out_base   [N*K]    first output index of segment (shard n, list m)
//   emb_base   [N*K]    float offset of segment (n, m) in the fused embedding buffer
//   list_rank0 [K*N]    number of first occurrences of shard n in lists < m   (index m*N+n)
//   n_unique   [1]
struct DDTables {
  int32_t* sizes;
  int32_t* shard_sz;
  int32_t* out_base;
  int32_t* emb_base;
  int32_t* list_rank0;
  int32_t* n_unique;
};

// Per tile: walk in position order; per warp keep running first-occurrence counts per shard.
// MODE 0: count only (writes blk_cnt[n * nblk + blk] and sizes via warp-aggregated atomics)
// MODE 1: scatter (needs blk_base from the scan)
template <int MODE>
__global__ void __launch_bounds__(kThreads)
dd_rank_kernel(const int64_t* __restrict__ ids, int64_t M, const int64_t* __restrict__ split, int K,
               int N, int n_eff, int rank0_empty, const DSet* __restrict__ set,
               const uint32_t* __restrict__ slot_of, int32_t* __restrict__ blk_cnt, int nblk,
               DDTables tb, int64_t* __restrict__ output, int32_t* __restrict__ rank) {
  __shared__ int32_t wcnt[kThreads / 32][kMaxShards];   // per-warp counts, then per-warp bases
  __shared__ int32_t bbase[kMaxShards];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  constexpr int NW = kThreads / 32;
  constexpr int kPerWarp = kTile / NW;  // consecutive ids handled by one warp
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    const int64_t wbeg = (int64_t)blk * kTile + (int64_t)w * kPerWarp;
    for (int n = lane; n < N; n += 32) wcnt[w][n] = 0;
    __syncwarp();
    // phase A: totals per warp
    for (int c = 0; c < kPerWarp; c += 32) {
      const int64_t i = wbeg + c + lane;
      int cls = -1, m = 0;
      if (i < M) {
        const bool first = set[slot_of[i]].first_pos == (int32_t)i;
        if (first) {
          cls = shard_of(ids[i], n_eff, rank0_empty);
          m = K > 1 ? list_of(split, K, i) : 0;
        }
      }
      const uint32_t same = __match_any_sync(0xffffffffu, cls);
      if (cls >= 0 && lane == (__ffs(same) - 1)) wcnt[w][cls] += __popc(same);
      if (MODE == 0) {
        // per (shard, list) totals: aggregate lanes that share both, one atomic per distinct pair
        // (cls * K + m < 64 * K <= 2^31 for K <= kMaxLists: the key is unique per pair)
        const int pair = cls >= 0 ? cls * K + m : -1;
        const uint32_t same2 = __match_any_sync(0xffffffffu, pair);
        if (cls >= 0 && lane == (__ffs(same2) - 1)) atomicAdd(tb.sizes + cls * K + m, __popc(same2));
      }
      __syncwarp();
    }
    __syncthreads();
    // phase B: exclusive scan over warps, per shard
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      int run = 0;
      for (int ww = 0; ww < NW; ++ww) {
        int v = wcnt[ww][n];
        wcnt[ww][n] = run;
        run += v;
      }
      if (MODE == 0) blk_cnt[(size_t)n * nblk + blk] = run;
      else bbase[n] = blk_cnt[(size_t)n * nblk + blk];
    }
    __syncthreads();
    if (MODE == 1) {
      // phase C: re-walk, assign stable ranks
      for (int c = 0; c < kPerWarp; c += 32) {
        const int64_t i = wbeg + c + lane;
        int cls = -1, m = 0;
        int64_t key = 0;
        if (i < M) {
          const bool first = set[slot_of[i]].first_pos == (int32_t)i;
          if (first) {
            key = ids[i];
            cls = shard_of(key, n_eff, rank0_empty);
            m = K > 1 ? list_of(split, K, i) : 0;
          }
        }
        const uint32_t same = __match_any_sync(0xffffffffu, cls);
        if (cls >= 0) {
          const int in_chunk = __popc(same & ((1u << lane) - 1u));
          const int r = bbase[cls] + wcnt[w][cls] + in_chunk;  // rank among first occs of this shard
          const int local = r - tb.list_rank0[m * N + cls];    // ordinal inside (shard, list)
          rank[i] = local;
          output[tb.out_base[cls * K + m] + local] = key;
        }
        __syncwarp();
        if (cls >= 0 && lane == (__ffs(same) - 1)) wcnt[w][cls] += __popc(same);
        __syncwarp();
      }
    }
    __syncthreads();
  }
}

// one block: scans + small tables.
// ref for the tables: fused_reorder_by_indices.cc:66-88 (sizes, shard_sizes, emb_offsets_cm)
__global__ void __launch_bounds__(1024)
dd_scan_kernel(int32_t* blk_cnt, int nblk, int N, int K, const int32_t* __restrict__ dims, int dim0,
               DDTables tb) {
  __shared__ int32_t carry;
  __shared__ int32_t warp_tot[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  // exclusive scan of blk_cnt[n][0..nblk) for every shard n (sequential over shards, parallel inside)
  for (int n = 0; n < N; ++n) {
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblk; base += blockDim.x) {
      const int idx = base + threadIdx.x;
      int v = idx < nblk ? blk_cnt[(size_t)n * nblk + idx] : 0;
      int x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) warp_tot[w] = x;
      __syncthreads();
      if (w == 0) {
        int t = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          int y = __shfl_up_sync(0xffffffffu, t, o);
          if (lane >= o) t += y;
        }
        warp_tot[lane] = t;  // inclusive scan of warp totals
      }
      __syncthreads();
      const int warp_off = w == 0 ? 0 : warp_tot[w - 1];
      const int excl = carry + warp_off + x - v;
      if (idx < nblk) blk_cnt[(size_t)n * nblk + idx] = excl;
      __syncthreads();
      if (threadIdx.x == blockDim.x - 1) carry = carry + warp_tot[31];
      __syncthreads();
    }
  }
  // small tables (serial; N*K is a few hundred at most)
  if (threadIdx.x == 0) {
    int uniq = 0, emb = 0;
    for (int n = 0; n < N; ++n) {
      int ss = 0;
      for (int m = 0; m < K; ++m) {
        const int sz = tb.sizes[n * K + m];
        tb.out_base[n * K + m] = uniq;
        tb.emb_base[n * K + m] = emb;
        uniq += sz;
        ss += sz;
        emb += sz * (K > 1 ? dims[m] : dim0);
      }
      tb.shard_sz[n] = ss;
    }
    for (int n = 0; n < N; ++n) {
      int run = 0;
      for (int m = 0; m < K; ++m) {
        tb.list_rank0[m * N + n] = run;
        run += tb.sizes[n * K + m];
      }
    }
    *tb.n_unique = uniq;
  }
}

// every occurrence: offset of its row in the fused buffer
// ref: fused_reorder_by_indices.cc:101-112: ids_sets[m][val] + emb_offsets_cm[shard + m*N]
__global__ void __launch_bounds__(kThreads)
dd_offsets_kernel(const int64_t* __restrict__ ids, int64_t M, const int64_t* __restrict__ split, int K,
                  int N, int n_eff, int rank0_empty, const DSet* __restrict__ set,
                  const uint32_t* __restrict__ slot_of, const int32_t* __restrict__ rank,
                  const int32_t* __restrict__ dims, int dim0, DDTables tb,
                  int32_t* __restrict__ fused_emb_offset) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t fp = set[slot_of[i]].first_pos;
    const int m = K > 1 ? list_of(split, K, i) : 0;
    const int n = shard_of(ids[i], n_eff, rank0_empty);
    fused_emb_offset[i] = rank[fp] * (K > 1 ? dims[m] : dim0) + tb.emb_base[n * K + m];
  }
}

void run_reorder(int device, const int64_t* ids_dev, const int64_t* id_split_host, int K, int N,
                 const int32_t* dims_host, int rank0_empty, int64_t* output_dev, int32_t* sizes_dev,
                 int32_t* fused_emb_offset_dev, int32_t* shard_sizes_host,
                 int32_t* sharded_slot_sizes_host, int64_t* n_unique_host, int32_t* n_unique_dev,
                 cudaStream_t s) {
  // every argument check runs before the device is touched
  if (K <= 0 || N <= 0) throw ArgError("num_lists and num_shards must be positive");
  if (K > kMaxLists) throw ArgError("num_lists > 2^25 is not supported");
  if (N > kMaxShards) throw ArgError("num_shards > 64 is not supported");
  if (rank0_empty && N < 2) throw ArgError("rank0_empty needs at least 2 shards");
  if (id_split_host[0] != 0) throw ArgError("id_split must start at 0");
  for (int m = 0; m < K; ++m)
    if (id_split_host[m + 1] < id_split_host[m]) throw ArgError("id_split must not decrease");
  const int64_t M = id_split_host[K];
  if (M > kMaxIds) throw ArgError("more than 2^30 ids in one call");
  for (int m = 0; m < (K > 1 ? K : 1); ++m)
    if (dims_host[m] <= 0) throw ArgError("dims must be positive");
  const int dim0 = dims_host[0];
  const bool want_host = shard_sizes_host || sharded_slot_sizes_host || n_unique_host;
  // The pageable H2D sources (id_split_host, dims_host; K > 1 only) and the host outputs must stay valid until the
  // copies have run: synchronise in those cases.  K == 1 without host outputs (mono_dedup in the fused train step)
  // stays fully asynchronous, so its float offsets (< M * dim0) are bounded up front instead of checked afterwards.
  const bool sync = K > 1 || want_host;
  if (!sync && M * (int64_t)dim0 > INT32_MAX) throw ArgError("ids x dim exceeds 2^31 - 1 float offsets");
  MONO_CUDA(cudaSetDevice(device));
  const int n_eff = N - (rank0_empty ? 1 : 0);
  const int nblk = (int)std::max<int64_t>(1, (M + kTile - 1) / kTile);

  // one scratch allocation (stream-ordered); M <= 2^30 keeps cap <= 2^31
  uint32_t cap = 1024;
  while (cap < 2 * (uint64_t)std::max<int64_t>(M, 1)) cap <<= 1;
  const size_t NK = (size_t)N * K;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_set = take(sizeof(DSet) * cap);
  const size_t o_slot = take(sizeof(uint32_t) * (size_t)std::max<int64_t>(M, 1));
  const size_t o_rank = take(sizeof(int32_t) * (size_t)std::max<int64_t>(M, 1));
  const size_t o_blk = take(sizeof(int32_t) * (size_t)N * nblk);
  const size_t o_split = take(sizeof(int64_t) * (K + 1));
  const size_t o_dims = take(sizeof(int32_t) * K);
  const size_t o_small = take(sizeof(int32_t) * (4 * NK + N + 8));
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, off, s));
  DSet* set = reinterpret_cast<DSet*>(ws + o_set);
  uint32_t* slot_of = reinterpret_cast<uint32_t*>(ws + o_slot);
  int32_t* rank = reinterpret_cast<int32_t*>(ws + o_rank);
  int32_t* blk_cnt = reinterpret_cast<int32_t*>(ws + o_blk);
  int64_t* split_dev = reinterpret_cast<int64_t*>(ws + o_split);
  int32_t* dims_dev = reinterpret_cast<int32_t*>(ws + o_dims);
  int32_t* small = reinterpret_cast<int32_t*>(ws + o_small);
  DDTables tb;
  tb.sizes = small;
  tb.shard_sz = small + NK;
  tb.out_base = tb.shard_sz + N;
  tb.emb_base = tb.out_base + NK;
  tb.list_rank0 = tb.emb_base + NK;
  tb.n_unique = tb.list_rank0 + NK;

  // the two tiny host arrays go through pageable H2D copies: copied to a staging vector that
  // outlives the async copy only if we sync; keep it simple and correct: synchronous small copies.
  if (K > 1) {  // K == 1 needs neither table on the device (dim passed by value): no pageable H2D
    MONO_CUDA(cudaMemcpyAsync(split_dev, id_split_host, sizeof(int64_t) * (K + 1), cudaMemcpyHostToDevice, s));
    MONO_CUDA(cudaMemcpyAsync(dims_dev, dims_host, sizeof(int32_t) * K, cudaMemcpyHostToDevice, s));
  }
  MONO_CUDA(cudaMemsetAsync(set, 0xFF, sizeof(DSet) * cap, s));
  MONO_CUDA(cudaMemsetAsync(small, 0, sizeof(int32_t) * (4 * NK + N + 8), s));

  if (M > 0) {
    dd_claim_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(ids_dev, M, split_dev, K, set, cap - 1, slot_of);
    MONO_CHECK_LAUNCH();
    const int g = std::min(nblk, device_sms() * 8);
    dd_rank_kernel<0><<<g, kThreads, 0, s>>>(ids_dev, M, split_dev, K, N, n_eff, rank0_empty ? 1 : 0, set,
                                            slot_of, blk_cnt, nblk, tb, output_dev, rank);
    MONO_CHECK_LAUNCH();
    dd_scan_kernel<<<1, 1024, 0, s>>>(blk_cnt, nblk, N, K, dims_dev, dim0, tb);
    MONO_CHECK_LAUNCH();
    dd_rank_kernel<1><<<g, kThreads, 0, s>>>(ids_dev, M, split_dev, K, N, n_eff, rank0_empty ? 1 : 0, set,
                                            slot_of, blk_cnt, nblk, tb, output_dev, rank);
    MONO_CHECK_LAUNCH();
    dd_offsets_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(ids_dev, M, split_dev, K, N, n_eff,
                                                                rank0_empty ? 1 : 0, set, slot_of, rank,
                                                                dims_dev, dim0, tb, fused_emb_offset_dev);
    MONO_CHECK_LAUNCH();
  }
  // results: sizes_dev = [shard_sizes (N) | sharded_slot_sizes (N*K)]
  if (sizes_dev) {
    MONO_CUDA(cudaMemcpyAsync(sizes_dev, tb.shard_sz, sizeof(int32_t) * N, cudaMemcpyDeviceToDevice, s));
    MONO_CUDA(cudaMemcpyAsync(sizes_dev + N, tb.sizes, sizeof(int32_t) * NK, cudaMemcpyDeviceToDevice, s));
  }
  if (n_unique_dev)
    MONO_CUDA(cudaMemcpyAsync(n_unique_dev, tb.n_unique, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  std::vector<int32_t> h(NK + N + 1);
  if (sync) {
    MONO_CUDA(cudaMemcpyAsync(h.data(), tb.shard_sz, sizeof(int32_t) * N, cudaMemcpyDeviceToHost, s));
    MONO_CUDA(cudaMemcpyAsync(h.data() + N, tb.sizes, sizeof(int32_t) * NK, cudaMemcpyDeviceToHost, s));
    MONO_CUDA(cudaMemcpyAsync(h.data() + N + NK, tb.n_unique, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  }
  MONO_CUDA(cudaFreeAsync(ws, s));
  if (sync) {
    MONO_CUDA(cudaStreamSynchronize(s));
    // the device accumulates the float offsets in int32: the exact sum of sizes x dims must fit
    int64_t floats = 0;
    for (size_t nm = 0; nm < NK; ++nm) floats += (int64_t)h[N + nm] * (K > 1 ? dims_host[nm % K] : dim0);
    if (floats > INT32_MAX) throw ArgError("float offsets exceed 2^31 - 1 (sum of unique ids x dims)");
  }
  if (want_host) {
    if (shard_sizes_host) std::memcpy(shard_sizes_host, h.data(), sizeof(int32_t) * N);
    if (sharded_slot_sizes_host) std::memcpy(sharded_slot_sizes_host, h.data() + N, sizeof(int32_t) * NK);
    if (n_unique_host) *n_unique_host = h[N + NK];
  }
}

}  // namespace mono
