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
#include <numeric>
#include <vector>

#include "engine.h"

namespace mono {

constexpr int kMaxShards = 64;
constexpr int kMaxLists = 1 << 25;                  // (shard, list) keys cls * K + m stay below 2^31
constexpr int64_t kMaxIds = (int64_t)1 << 30;       // the scratch set holds 2^31 16-byte slots at most
constexpr int kTileItems = 8;                       // ids per thread per tile
constexpr int kTile = kThreads * kTileItems;        // ids per block tile

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
                FirstOcc* set, uint32_t mask, uint32_t* __restrict__ slot_of) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = ids[i];
    const int m = K > 1 ? list_of(split, K, i) : 0;
    slot_of[i] = claim_first_occ(set, mask, first_occ_slot(key, m, mask), key, m, (int32_t)i);
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
               int N, int n_eff, int rank0_empty, const FirstOcc* __restrict__ set,
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
                  int N, int n_eff, int rank0_empty, const FirstOcc* __restrict__ set,
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

// passes 2-4 over M > 0 ids, once slot_of and the scratch set's first positions are written: the small tables, the
// unique ids in output[] and every first occurrence's ordinal inside its (shard, list) in rank[]
static void rank_scan_passes(const int64_t* ids_dev, int64_t M, const int64_t* split_dev, int K, int N, int n_eff,
                             int rank0_empty, const FirstOcc* set, const uint32_t* slot_of, int32_t* blk_cnt, int nblk,
                             const int32_t* dims_dev, int dim0, DDTables tb, int64_t* output_dev, int32_t* rank,
                             cudaStream_t s) {
  const int g = std::min(nblk, device_sms() * 8);
  dd_rank_kernel<0><<<g, kThreads, 0, s>>>(ids_dev, M, split_dev, K, N, n_eff, rank0_empty, set, slot_of, blk_cnt,
                                          nblk, tb, output_dev, rank);
  MONO_CHECK_LAUNCH();
  dd_scan_kernel<<<1, 1024, 0, s>>>(blk_cnt, nblk, N, K, dims_dev, dim0, tb);
  MONO_CHECK_LAUNCH();
  dd_rank_kernel<1><<<g, kThreads, 0, s>>>(ids_dev, M, split_dev, K, N, n_eff, rank0_empty, set, slot_of, blk_cnt,
                                          nblk, tb, output_dev, rank);
  MONO_CHECK_LAUNCH();
}

// passes 2-5: the above, then every occurrence's float offset
static void rank_passes(const int64_t* ids_dev, int64_t M, const int64_t* split_dev, int K, int N, int n_eff,
                        int rank0_empty, const FirstOcc* set, const uint32_t* slot_of, int32_t* blk_cnt, int nblk,
                        const int32_t* dims_dev, int dim0, DDTables tb, int64_t* output_dev, int32_t* rank,
                        int32_t* fused_emb_offset_dev, cudaStream_t s) {
  rank_scan_passes(ids_dev, M, split_dev, K, N, n_eff, rank0_empty, set, slot_of, blk_cnt, nblk, dims_dev, dim0, tb,
                   output_dev, rank, s);
  dd_offsets_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(ids_dev, M, split_dev, K, N, n_eff, rank0_empty, set,
                                                              slot_of, rank, dims_dev, dim0, tb, fused_emb_offset_dev);
  MONO_CHECK_LAUNCH();
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
  const size_t o_set = take(sizeof(FirstOcc) * cap);
  const size_t o_slot = take(sizeof(uint32_t) * (size_t)std::max<int64_t>(M, 1));
  const size_t o_rank = take(sizeof(int32_t) * (size_t)std::max<int64_t>(M, 1));
  const size_t o_blk = take(sizeof(int32_t) * (size_t)N * nblk);
  const size_t o_split = take(sizeof(int64_t) * (K + 1));
  const size_t o_dims = take(sizeof(int32_t) * K);
  const size_t o_small = take(sizeof(int32_t) * (4 * NK + N + 8));
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, off, s));
  FirstOcc* set = reinterpret_cast<FirstOcc*>(ws + o_set);
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
  MONO_CUDA(cudaMemsetAsync(set, 0xFF, sizeof(FirstOcc) * cap, s));
  MONO_CUDA(cudaMemsetAsync(small, 0, sizeof(int32_t) * (4 * NK + N + 8), s));

  if (M > 0) {
    dd_claim_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(ids_dev, M, split_dev, K, set, cap - 1, slot_of);
    MONO_CHECK_LAUNCH();
    rank_passes(ids_dev, M, split_dev, K, N, n_eff, rank0_empty ? 1 : 0, set, slot_of, blk_cnt, nblk, dims_dev, dim0, tb,
                output_dev, rank, fused_emb_offset_dev, s);
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

// ---- ShardingSparseFids (ref: parse_sparse_feature.cc:187-330, parse_sparse_feature.h:714-920) ----------------
//
// The features arrive in sorted-name order ("name order", index f); the reference's lists are table-major,
// feature-minor ("list order", index j).  The FIDs are gathered into list order and run through the reorder's
// claim / count / scan / scatter / offsets passes with one list per feature: its output buffer is then the
// version-4 fid_list (shard-major, table-minor, feature-minor), tb.sizes the per-(shard, feature) counts and
// tb.emb_base the float offset of every (shard, feature) block.  unique = false replaces the claim by an identity
// grouping (every occurrence its own first occurrence), so the same passes keep every occurrence, ranked in input
// order inside its (feature, shard).  Three small kernels then write the remaining outputs.

// Per-call tables staged from the host (one H2D copy), all indexed as named.
struct ShardStage {
  int64_t* split_lo;   // [F + 1] occurrence start of list j in the gathered (list-order) FIDs
  int64_t* split_in;   // [F + 1] occurrence start of feature f in the caller's (name-order) FIDs
  int64_t* row_start;  // [F + 1] first feature_offset entry of feature f; row_start[F] = R
  int32_t* list_of_f;  // [F]     list index of feature f
  int32_t* feat_of_j;  // [F]     feature index of list j
  int32_t* table_of_j; // [F]
  int32_t* dims_lo;    // [F]     dims_sum of list j
  int32_t* first_j;    // [K + 1] first list of table k
  uint32_t* nfl;       // [F + 1] nfl_offset (bit 31 = shared)
};

// list-order FIDs; unique = false also writes the identity grouping the rank passes read
__global__ void __launch_bounds__(kThreads)
sh_gather_kernel(const int64_t* __restrict__ fids, int64_t M, int F, ShardStage st, int identity,
                 int64_t* __restrict__ ids_lo, FirstOcc* __restrict__ set, uint32_t* __restrict__ slot_of) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < M; p += (int64_t)gridDim.x * blockDim.x) {
    const int j = F > 1 ? list_of(st.split_lo, F, p) : 0;
    ids_lo[p] = fids[st.split_in[st.feat_of_j[j]] + (p - st.split_lo[j])];
    if (identity) {
      slot_of[p] = (uint32_t)p;
      set[p].first_pos = (int32_t)p;
    }
  }
}

// one thread per (shard n, table k): version-4 row splits [n][k][0, c1, c1 + c2, ...], table and embedding row
// lengths ([n * K + k]); the k == 0 thread writes the shard row length
__global__ void __launch_bounds__(kThreads)
sh_tables_kernel(int N, int K, int F, ShardStage st, DDTables tb, int64_t* __restrict__ row_splits,
                 int32_t* __restrict__ table_len, int32_t* __restrict__ shard_len, int32_t* __restrict__ emb_len) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * K) return;
  const int n = idx / K, k = idx % K;
  const int j0 = st.first_j[k], j1 = st.first_j[k + 1];
  int64_t* rs = row_splits + (size_t)n * (F + K) + j0 + k;
  int32_t cnt = 0, emb = 0;
  rs[0] = 0;
  for (int j = j0; j < j1; ++j) {
    const int32_t c = tb.sizes[(size_t)n * F + j];
    cnt += c;
    emb += c * st.dims_lo[j];
    rs[j - j0 + 1] = cnt;
  }
  table_len[idx] = cnt;
  emb_len[idx] = emb;
  if (k == 0) shard_len[n] = tb.shard_sz[n];
}

// every occurrence, in name order: (table * N + shard) << 32 | float offset of its row inside its (table, shard)
// list (ref: parse_sparse_feature.cc:199-240)
__global__ void __launch_bounds__(kThreads)
sh_fid_offset_kernel(const int64_t* __restrict__ fids, int64_t M, int N, int F, ShardStage st, DDTables tb,
                     const int32_t* __restrict__ offs_lo, uint64_t* __restrict__ fid_offset) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
    const int f = F > 1 ? list_of(st.split_in, F, i) : 0;
    const int j = st.list_of_f[f];
    const int k = st.table_of_j[j];
    const int n = (int)((uint64_t)fids[i] % (uint64_t)N);
    const int32_t local = offs_lo[st.split_lo[j] + (i - st.split_in[f])] - tb.emb_base[(size_t)n * F + st.first_j[k]];
    fid_offset[i] = ((uint64_t)(k * N + n) << 32) | (uint32_t)local;
  }
}

// feature_offset[R + 1]: every feature's row splits shifted by the occurrences before it; nfl_offset[F + 1] from
// the staged table.  Checks every feature's row splits: 0 first, non-decreasing, n_fids last (bad = 1 otherwise).
__global__ void __launch_bounds__(kThreads)
sh_feature_offset_kernel(const int64_t* __restrict__ rs_in, int64_t R, int F, ShardStage st,
                         int32_t* __restrict__ feature_offset, uint32_t* __restrict__ nfl_offset,
                         int32_t* __restrict__ bad) {
  const int64_t items = (R > F ? R : F) + 1;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < items; r += (int64_t)gridDim.x * blockDim.x) {
    if (r <= F) {
      nfl_offset[r] = st.nfl[r];
      if (r < F && st.row_start[r + 1] == st.row_start[r]) {  // a feature without rows: its splits are [0]
        if (rs_in[st.row_start[r] + r] != 0 || st.split_in[r + 1] != st.split_in[r]) *bad = 1;
      }
    }
    if (r > R) continue;
    if (r == R) {
      feature_offset[r] = (int32_t)st.split_in[F];
      continue;
    }
    const int f = F > 1 ? list_of(st.row_start, F, r) : 0;
    const int64_t local = r - st.row_start[f];
    const int64_t at = st.row_start[f] + f + local;  // feature f's splits start after f earlier end entries
    const int64_t v = rs_in[at], next = rs_in[at + 1];
    if ((local == 0 && v != 0) || next < v ||
        (r + 1 == st.row_start[f + 1] && next != st.split_in[f + 1] - st.split_in[f]))
      *bad = 1;
    feature_offset[r] = (int32_t)(st.split_in[f] + v);
  }
}

// version 5 (ref: parse_sparse_feature.cc:287-301,329-336,390-404, parse_sparse_feature.h:837-893): one thread per
// list (table k, shard n) writes fid_list_row_splits_size (features of table k + 1) and emb_size (the list's floats:
// the version-4 emb_row_length of (n, k), transposed to table-major); thread 0 also writes nfl_size = F + 1,
// feature_size = R + 1, fid_size = M and batch_size
__global__ void __launch_bounds__(kThreads)
sh_v5_sizes_kernel(int N, int K, int F, int64_t R, int64_t M, ShardStage st, const int32_t* __restrict__ emb_len,
                   ShardingV5 v5) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx == 0) {
    v5.sizes[0] = F + 1;
    v5.sizes[1] = (int32_t)(R + 1);
    v5.sizes[2] = (int32_t)M;
    v5.sizes[3] = v5.batch_size;
  }
  if (idx >= N * K) return;
  const int k = idx / N, n = idx % N;
  v5.row_splits_size[idx] = st.first_j[k + 1] - st.first_j[k] + 1;
  v5.emb_size[idx] = emb_len[(size_t)n * K + k];
}

void run_sharding(int device, const int64_t* fids_dev, const int64_t* row_splits_dev,
                  const mono_sharding_feature* feats, int F, int K, int N, int unique, int64_t* fid_list_dev,
                  uint64_t* fid_offset_dev, int32_t* feature_offset_dev, uint32_t* nfl_offset_dev,
                  int64_t* row_splits_out_dev, int32_t* table_len_dev, int32_t* shard_len_dev, int32_t* emb_len_dev,
                  int32_t* bad_row_splits_dev, int32_t* table_len_host, cudaStream_t s, const ShardingV5* v5) {
  // every argument check runs before the device is touched
  if (F <= 0 || K <= 0 || N <= 0) throw ArgError("num_features, num_tables and num_shards must be positive");
  if (F > kMaxLists) throw ArgError("num_features > 2^25 is not supported");
  if (N > kMaxShards) throw ArgError("num_shards > 64 is not supported");
  int64_t M = 0, R = 0, floats = 0;
  for (int f = 0; f < F; ++f) {
    const mono_sharding_feature& a = feats[f];
    if (a.n_fids < 0 || a.n_rows < 0) throw ArgError("n_fids and n_rows must not be negative");
    if (a.table < 0 || a.table >= K) throw ArgError("table index out of range");
    if (a.dims_sum <= 0) throw ArgError("dims_sum must be positive");
    M += a.n_fids;
    R += a.n_rows;
    if (M > kMaxIds) throw ArgError("more than 2^30 ids in one call");
    if (R >= INT32_MAX) throw ArgError("more than 2^31 - 2 rows in one call");
    floats += a.n_fids * a.dims_sum;
    if (floats > INT32_MAX) throw ArgError("sum of n_fids x dims_sum exceeds 2^31 - 1 float offsets");
  }
  MONO_CUDA(cudaSetDevice(device));

  // staged tables: name order -> list order is a stable sort by table
  std::vector<int32_t> feat_of_j(F);
  std::iota(feat_of_j.begin(), feat_of_j.end(), 0);
  std::stable_sort(feat_of_j.begin(), feat_of_j.end(), [&](int a, int b) { return feats[a].table < feats[b].table; });
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 15) & ~(size_t)15; return o; };
  const size_t o_split_lo = take(sizeof(int64_t) * (F + 1)), o_split_in = take(sizeof(int64_t) * (F + 1)),
               o_row = take(sizeof(int64_t) * (F + 1)), o_list = take(sizeof(int32_t) * F),
               o_feat = take(sizeof(int32_t) * F), o_tab = take(sizeof(int32_t) * F), o_dims = take(sizeof(int32_t) * F),
               o_first = take(sizeof(int32_t) * (K + 1)), o_nfl = take(sizeof(uint32_t) * (F + 1));
  const size_t stage_bytes = off;
  std::vector<char> h(stage_bytes);
  auto H = [&](size_t o, auto* type) { return reinterpret_cast<decltype(type)>(h.data() + o); };
  int64_t* split_lo = H(o_split_lo, (int64_t*)nullptr);
  int64_t* split_in = H(o_split_in, (int64_t*)nullptr);
  int64_t* row_start = H(o_row, (int64_t*)nullptr);
  int32_t* list_of_f = H(o_list, (int32_t*)nullptr);
  int32_t* table_of_j = H(o_tab, (int32_t*)nullptr);
  int32_t* dims_lo = H(o_dims, (int32_t*)nullptr);
  int32_t* first_j = H(o_first, (int32_t*)nullptr);
  uint32_t* nfl = H(o_nfl, (uint32_t*)nullptr);
  std::memcpy(h.data() + o_feat, feat_of_j.data(), sizeof(int32_t) * F);
  split_lo[0] = split_in[0] = row_start[0] = 0;
  for (int f = 0; f < F; ++f) {
    split_in[f + 1] = split_in[f] + feats[f].n_fids;
    row_start[f + 1] = row_start[f] + feats[f].n_rows;
    nfl[f] = (uint32_t)row_start[f] | (feats[f].shared ? 0x80000000u : 0u);
  }
  nfl[F] = (uint32_t)(R + 1);
  for (int k = 0; k <= K; ++k) first_j[k] = F;
  for (int j = F - 1; j >= 0; --j) {
    const mono_sharding_feature& a = feats[feat_of_j[j]];
    list_of_f[feat_of_j[j]] = j;
    table_of_j[j] = a.table;
    dims_lo[j] = a.dims_sum;
    first_j[a.table] = j;
  }
  for (int k = K - 1; k >= 0; --k) first_j[k] = std::min(first_j[k], first_j[k + 1]);  // tables without features
  for (int j = 0; j < F; ++j) split_lo[j + 1] = split_lo[j] + feats[feat_of_j[j]].n_fids;

  // one stream-ordered scratch allocation: the reorder's scratch, the gathered FIDs and offsets, the staged tables
  const int nblk = (int)std::max<int64_t>(1, (M + kTile - 1) / kTile);
  const size_t M1 = (size_t)std::max<int64_t>(M, 1);
  const uint32_t cap = unique ? claim_set_slots(std::max<int64_t>(M, 1)) : (uint32_t)M1;
  const size_t NF = (size_t)N * F;
  off = 0;
  auto take256 = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_set = take256(sizeof(FirstOcc) * cap), o_slot = take256(sizeof(uint32_t) * M1),
               o_rank = take256(sizeof(int32_t) * M1), o_blk = take256(sizeof(int32_t) * (size_t)N * nblk),
               o_ids = take256(sizeof(int64_t) * M1), o_offs = take256(sizeof(int32_t) * M1),
               o_small = take256(sizeof(int32_t) * (4 * NF + N + 8)), o_stage = take256(stage_bytes);
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, off, s));
  FirstOcc* set = reinterpret_cast<FirstOcc*>(ws + o_set);
  uint32_t* slot_of = reinterpret_cast<uint32_t*>(ws + o_slot);
  int32_t* rank = reinterpret_cast<int32_t*>(ws + o_rank);
  int32_t* blk_cnt = reinterpret_cast<int32_t*>(ws + o_blk);
  int64_t* ids_lo = reinterpret_cast<int64_t*>(ws + o_ids);
  int32_t* offs_lo = reinterpret_cast<int32_t*>(ws + o_offs);
  int32_t* small = reinterpret_cast<int32_t*>(ws + o_small);
  char* stage = ws + o_stage;
  DDTables tb;
  tb.sizes = small;
  tb.shard_sz = small + NF;
  tb.out_base = tb.shard_sz + N;
  tb.emb_base = tb.out_base + NF;
  tb.list_rank0 = tb.emb_base + NF;
  tb.n_unique = tb.list_rank0 + NF;
  int32_t* bad = tb.n_unique + 1;
  ShardStage st;
  st.split_lo = reinterpret_cast<int64_t*>(stage + o_split_lo);
  st.split_in = reinterpret_cast<int64_t*>(stage + o_split_in);
  st.row_start = reinterpret_cast<int64_t*>(stage + o_row);
  st.list_of_f = reinterpret_cast<int32_t*>(stage + o_list);
  st.feat_of_j = reinterpret_cast<int32_t*>(stage + o_feat);
  st.table_of_j = reinterpret_cast<int32_t*>(stage + o_tab);
  st.dims_lo = reinterpret_cast<int32_t*>(stage + o_dims);
  st.first_j = reinterpret_cast<int32_t*>(stage + o_first);
  st.nfl = reinterpret_cast<uint32_t*>(stage + o_nfl);

  // a pageable H2D copy is staged by the driver before the call returns: h may go out of scope after it
  MONO_CUDA(cudaMemcpyAsync(stage, h.data(), stage_bytes, cudaMemcpyHostToDevice, s));
  if (unique) MONO_CUDA(cudaMemsetAsync(set, 0xFF, sizeof(FirstOcc) * cap, s));
  MONO_CUDA(cudaMemsetAsync(small, 0, sizeof(int32_t) * (4 * NF + N + 8), s));

  if (M > 0) {
    sh_gather_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(fids_dev, M, F, st, unique ? 0 : 1, ids_lo, set,
                                                               slot_of);
    MONO_CHECK_LAUNCH();
    if (unique) {
      dd_claim_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(ids_lo, M, st.split_lo, F, set, cap - 1, slot_of);
      MONO_CHECK_LAUNCH();
    }
    rank_passes(ids_lo, M, st.split_lo, F, N, N, 0, set, slot_of, blk_cnt, nblk, st.dims_lo, dims_lo[0], tb,
                fid_list_dev, rank, offs_lo, s);
  }
  sh_tables_kernel<<<(N * K + kThreads - 1) / kThreads, kThreads, 0, s>>>(N, K, F, st, tb, row_splits_out_dev,
                                                                         table_len_dev, shard_len_dev, emb_len_dev);
  MONO_CHECK_LAUNCH();
  if (v5) {
    sh_v5_sizes_kernel<<<(N * K + kThreads - 1) / kThreads, kThreads, 0, s>>>(N, K, F, R, M, st, emb_len_dev, *v5);
    MONO_CHECK_LAUNCH();
  }
  if (M > 0) {
    sh_fid_offset_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(fids_dev, M, N, F, st, tb, offs_lo,
                                                                   fid_offset_dev);
    MONO_CHECK_LAUNCH();
  }
  sh_feature_offset_kernel<<<grid_for(std::max<int64_t>(R, F) + 1, kThreads), kThreads, 0, s>>>(
      row_splits_dev, R, F, st, feature_offset_dev, nfl_offset_dev, bad);
  MONO_CHECK_LAUNCH();
  if (bad_row_splits_dev)
    MONO_CUDA(cudaMemcpyAsync(bad_row_splits_dev, bad, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  std::vector<int32_t> back((size_t)N * K + 1);
  if (table_len_host) {
    MONO_CUDA(cudaMemcpyAsync(back.data(), table_len_dev, sizeof(int32_t) * N * K, cudaMemcpyDeviceToHost, s));
    MONO_CUDA(cudaMemcpyAsync(back.data() + (size_t)N * K, bad, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  }
  MONO_CUDA(cudaFreeAsync(ws, s));
  if (table_len_host) {
    MONO_CUDA(cudaStreamSynchronize(s));
    if (back[(size_t)N * K]) throw ArgError("row splits must start at 0, not decrease and end at the feature's n_fids");
    std::memcpy(table_len_host, back.data(), sizeof(int32_t) * N * K);
  }
}

// ---- NormalizeMergedSplit (ref: RT/ops/normalize_merged_split_op.cc:33-90) ---------------------------------------
//
// row_split holds merge_num row splits end to end, split i being row_split_size[i] entries that start at 0.  The
// output joins them: split i's entries after its first, shifted by the sum of the last entries of splits 0 .. i - 1
// (split 0 keeps its first entry).  One block: the sizes and the last entries are scanned 1024 groups at a time,
// then each thread writes its group's entries.  bad = 1 for a size below 1 or sizes that do not add up to split_num.
constexpr int kNmsThreads = 1024;

__global__ void __launch_bounds__(kNmsThreads)
normalize_merged_split_kernel(const int64_t* __restrict__ rs, int64_t split_num, const int32_t* __restrict__ sizes,
                              int64_t merge_num, int64_t* __restrict__ out, int32_t* __restrict__ bad) {
  __shared__ int64_t sc[kNmsThreads];
  __shared__ int64_t carry_off, carry_pre;
  __shared__ int any_bad;
  if (threadIdx.x == 0) carry_off = carry_pre = 0, any_bad = 0;
  __syncthreads();
  for (int64_t base = 0; base < merge_num; base += kNmsThreads) {
    const int64_t i = base + threadIdx.x;
    const bool live = i < merge_num;
    const int64_t sz = live ? (int64_t)sizes[i] : 0;
    if (live && sz < 1) any_bad = 1;
    // inclusive scan of the sizes -> this group's first entry
    sc[threadIdx.x] = sz;
    __syncthreads();
    for (int d = 1; d < kNmsThreads; d <<= 1) {
      const int64_t v = threadIdx.x >= d ? sc[threadIdx.x - d] : 0;
      __syncthreads();
      sc[threadIdx.x] += v;
      __syncthreads();
    }
    const int64_t end = carry_off + sc[threadIdx.x], start = end - sz;
    const int64_t chunk_sizes = sc[kNmsThreads - 1];
    __syncthreads();
    // start >= 0: after a negative size a later split can end at or below 0; every read stays in [0, split_num)
    const bool ok = live && sz >= 1 && start >= 0 && end <= split_num;
    if (live && end > split_num) any_bad = 1;
    const int64_t last = ok ? rs[end - 1] : 0;
    // inclusive scan of the last entries -> the shift of this group (the exclusive prefix)
    sc[threadIdx.x] = last;
    __syncthreads();
    for (int d = 1; d < kNmsThreads; d <<= 1) {
      const int64_t v = threadIdx.x >= d ? sc[threadIdx.x - d] : 0;
      __syncthreads();
      sc[threadIdx.x] += v;
      __syncthreads();
    }
    const int64_t pre = carry_pre + sc[threadIdx.x] - last;
    const int64_t chunk_last = sc[kNmsThreads - 1];
    if (ok) {
      const int64_t n_out = split_num + 1 - merge_num;  // malformed sizes must not write outside the output
      for (int64_t j = (i == 0 ? start : start + 1); j < end; ++j)
        if (j - i >= 0 && j - i < n_out) out[j - i] = pre + rs[j];
    }
    __syncthreads();
    if (threadIdx.x == 0) carry_off += chunk_sizes, carry_pre += chunk_last;
    __syncthreads();
  }
  if (threadIdx.x == 0 && (any_bad || carry_off != split_num)) *bad = 1;
}

void run_normalize_merged_split(int device, const int64_t* row_split_dev, int64_t split_num,
                                const int32_t* row_split_size_dev, int64_t merge_num, int64_t* out_dev,
                                int32_t* bad_dev, cudaStream_t s) {
  if (split_num < 0 || merge_num < 0) throw ArgError("normalize_merged_split: negative size");
  if (merge_num > split_num) throw ArgError("normalize_merged_split: more merged splits than entries");
  if (merge_num == 0) {
    if (split_num != 0) throw ArgError("normalize_merged_split: entries without a merged split");
    return;
  }
  MONO_CUDA(cudaSetDevice(device));
  normalize_merged_split_kernel<<<1, kNmsThreads, 0, s>>>(row_split_dev, split_num, row_split_size_dev, merge_num,
                                                          out_dev, bad_dev);
  MONO_CHECK_LAUNCH();
}

// ---- UniqueKeyWithValueAndOffset (ref: unique_mapping_ops.cc:51-124) ---------------------------------------------
//
// The distinct keys of every table in first-occurrence order are the reorder's claim and rank passes with one shard
// and one list per table: the rank scatter writes them table after table, and out_base[k] + rank is every key's
// unique ordinal.  The occurrences are then grouped by ordinal with the backward's stable radix sort of (ordinal,
// position): sorted entry q is an occurrence of ordinal run(q), runs in ordinal order and occurrences in position
// order, which is the reference's value_offset order; the run starts are value_offset_split.

// Per-call tables staged from the host (one H2D copy)
struct UoStage {
  int64_t* split;  // [K + 1] key_split
  int64_t* base;   // [K]     float offset of table k's first occurrence in the value buffer
  int32_t* dims;   // [K]
  int32_t* ones;   // [K]     the rank passes' row widths: their float offsets are not used
};

// every occurrence: its unique ordinal (the sort key); the first K + 1 threads write unique_key_split
__global__ void __launch_bounds__(kThreads)
uo_ordinal_kernel(int64_t M, int K, UoStage st, const FirstOcc* __restrict__ set, const uint32_t* __restrict__ slot_of,
                  const int32_t* __restrict__ rank, DDTables tb, uint32_t* __restrict__ ord,
                  int64_t* __restrict__ unique_key_split) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M || i <= K;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (i <= K) unique_key_split[i] = i < K ? tb.out_base[i] : *tb.n_unique;
    if (i >= M) continue;
    const int m = K > 1 ? list_of(st.split, K, i) : 0;
    ord[i] = (uint32_t)(tb.out_base[m] + rank[set[slot_of[i]].first_pos]);
  }
}

// sorted entry q -> value_offset[q]; run j -> value_offset_split[j] (run_start[U] = M)
__global__ void __launch_bounds__(kThreads)
uo_emit_kernel(int64_t M, int K, UoStage st, const uint2* __restrict__ sorted, const uint32_t* __restrict__ run_start,
               const uint32_t* __restrict__ n_runs, int64_t* __restrict__ value_offset,
               int64_t* __restrict__ value_offset_split) {
  const int64_t U = *n_runs;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < M || q <= U;
       q += (int64_t)gridDim.x * blockDim.x) {
    if (q <= U) value_offset_split[q] = run_start[q];
    if (q >= M) continue;
    const int64_t i = sorted[q].y;
    const int m = K > 1 ? list_of(st.split, K, i) : 0;
    value_offset[q] = st.base[m] + (i - st.split[m]) * st.dims[m];
  }
}

static int key_bits(int64_t n) {  // bits of a key in [0, n)
  int bits = 1;
  while (((int64_t)1 << bits) < n) ++bits;
  return bits;
}

void run_unique_offset(int device, const int64_t* key_dev, const int64_t* key_split_host, int K,
                       const int32_t* dims_host, int64_t* unique_key_dev, int64_t* unique_key_split_dev,
                       int64_t* value_offset_dev, int64_t* value_offset_split_dev, int64_t* value_len_host,
                       int64_t* unique_key_split_host, cudaStream_t s) {
  // every argument check runs before the device is touched
  if (K <= 0) throw ArgError("unique_key_with_value_and_offset: num_tables must be positive");
  if (K > kMaxLists) throw ArgError("unique_key_with_value_and_offset: num_tables > 2^25 is not supported");
  if (key_split_host[0] != 0) throw ArgError("unique_key_with_value_and_offset: key_split must start at 0");
  for (int k = 0; k < K; ++k) {
    if (key_split_host[k + 1] < key_split_host[k])
      throw ArgError("unique_key_with_value_and_offset: key_split must not decrease");
    if (dims_host[k] <= 0) throw ArgError("unique_key_with_value_and_offset: dims must be positive");
  }
  const int64_t M = key_split_host[K];
  if (M > kMaxIds) throw ArgError("unique_key_with_value_and_offset: more than 2^30 keys in one call");
  MONO_CUDA(cudaSetDevice(device));

  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 15) & ~(size_t)15; return o; };
  const size_t o_split = take(sizeof(int64_t) * (K + 1)), o_base = take(sizeof(int64_t) * K),
               o_dims = take(sizeof(int32_t) * K), o_ones = take(sizeof(int32_t) * K);
  const size_t stage_bytes = off;
  std::vector<char> h(stage_bytes);
  int64_t* hbase = reinterpret_cast<int64_t*>(h.data() + o_base);
  int32_t* hones = reinterpret_cast<int32_t*>(h.data() + o_ones);
  std::memcpy(h.data() + o_split, key_split_host, sizeof(int64_t) * (K + 1));
  std::memcpy(h.data() + o_dims, dims_host, sizeof(int32_t) * K);
  int64_t floats = 0;
  for (int k = 0; k < K; ++k) {
    hbase[k] = floats;
    hones[k] = 1;
    floats += (key_split_host[k + 1] - key_split_host[k]) * dims_host[k];
  }
  if (value_len_host) *value_len_host = floats;

  const int nblk = (int)std::max<int64_t>(1, (M + kTile - 1) / kTile);
  const size_t M1 = (size_t)std::max<int64_t>(M, 1);
  const uint32_t cap = claim_set_slots((int64_t)M1);
  const int bits = key_bits((int64_t)M1);
  off = 0;
  auto take256 = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_set = take256(sizeof(FirstOcc) * cap), o_slot = take256(sizeof(uint32_t) * M1),
               o_rank = take256(sizeof(int32_t) * M1), o_ord = take256(sizeof(uint32_t) * M1),
               o_blk = take256(sizeof(int32_t) * nblk), o_small = take256(sizeof(int32_t) * (4 * (size_t)K + 9)),
               o_stage = take256(stage_bytes), o_sort = take256(key_sort_bytes((int64_t)M1, bits));
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, off, s));
  FirstOcc* set = reinterpret_cast<FirstOcc*>(ws + o_set);
  uint32_t* slot_of = reinterpret_cast<uint32_t*>(ws + o_slot);
  int32_t* rank = reinterpret_cast<int32_t*>(ws + o_rank);
  uint32_t* ord = reinterpret_cast<uint32_t*>(ws + o_ord);
  int32_t* blk_cnt = reinterpret_cast<int32_t*>(ws + o_blk);
  int32_t* small = reinterpret_cast<int32_t*>(ws + o_small);
  char* stage = ws + o_stage;
  DDTables tb;
  tb.sizes = small;
  tb.shard_sz = small + K;
  tb.out_base = tb.shard_sz + 1;
  tb.emb_base = tb.out_base + K;
  tb.list_rank0 = tb.emb_base + K;
  tb.n_unique = tb.list_rank0 + K;
  UoStage st;
  st.split = reinterpret_cast<int64_t*>(stage + o_split);
  st.base = reinterpret_cast<int64_t*>(stage + o_base);
  st.dims = reinterpret_cast<int32_t*>(stage + o_dims);
  st.ones = reinterpret_cast<int32_t*>(stage + o_ones);

  // a pageable H2D copy is staged by the driver before the call returns: h may go out of scope after it
  MONO_CUDA(cudaMemcpyAsync(stage, h.data(), stage_bytes, cudaMemcpyHostToDevice, s));
  MONO_CUDA(cudaMemsetAsync(small, 0, sizeof(int32_t) * (4 * (size_t)K + 9), s));
  if (M > 0) {
    MONO_CUDA(cudaMemsetAsync(set, 0xFF, sizeof(FirstOcc) * cap, s));
    dd_claim_kernel<<<grid_for(M, kThreads), kThreads, 0, s>>>(key_dev, M, st.split, K, set, cap - 1, slot_of);
    MONO_CHECK_LAUNCH();
    rank_scan_passes(key_dev, M, st.split, K, 1, 1, 0, set, slot_of, blk_cnt, nblk, st.ones, 1, tb, unique_key_dev,
                     rank, s);
  }
  uo_ordinal_kernel<<<grid_for(std::max<int64_t>(M, K + 1), kThreads), kThreads, 0, s>>>(
      M, K, st, set, slot_of, rank, tb, ord, unique_key_split_dev);
  MONO_CHECK_LAUNCH();
  if (M > 0) {
    const uint2* sorted = nullptr;
    const SortWs sw = key_sort(ws + o_sort, ord, M, bits, true, &sorted, s);
    uo_emit_kernel<<<grid_for(M + 1, kThreads), kThreads, 0, s>>>(M, K, st, sorted, sw.run_start, sw.n_runs,
                                                                  value_offset_dev, value_offset_split_dev);
    MONO_CHECK_LAUNCH();
  } else {
    MONO_CUDA(cudaMemsetAsync(value_offset_split_dev, 0, sizeof(int64_t), s));
  }
  if (unique_key_split_host)
    MONO_CUDA(cudaMemcpyAsync(unique_key_split_host, unique_key_split_dev, sizeof(int64_t) * (K + 1),
                              cudaMemcpyDeviceToHost, s));
  MONO_CUDA(cudaFreeAsync(ws, s));
  if (unique_key_split_host) MONO_CUDA(cudaStreamSynchronize(s));
}

// ---- RaggedSplitByIndices (ref: split_by_indices_op.cc:188-243) -------------------------------------------------
//
// A counting partition of the n (<= capacity) values by index, stable: (index, position) pairs through the backward's
// radix sort, the (split, table) counts by a count pass and one scan block.  The outputs are the S ragged tensors
// concatenated split after split: split s owns [split_offsets[s], split_offsets[s + 1]) of values_out and pos_out,
// and its own K + 1 row splits at row_splits_out[s * (K + 1)].  The value count n is num_split[K], read on the
// device; entries from n to the capacity sort behind every split (key S) and are not written.

// every entry: its sort key, and the (split, table) counts; bad = 1 for an index outside [0, S) (sorted and counted
// as split 0, as a defined stand-in) or a num_split that does not start at 0, decreases or exceeds the capacity
__global__ void __launch_bounds__(kThreads)
rsi_count_kernel(const int64_t* __restrict__ indices, int64_t cap, const int64_t* __restrict__ num_split, int K, int S,
                 uint32_t* __restrict__ keys, uint32_t* __restrict__ cnt, int32_t* __restrict__ bad) {
  const int64_t n = num_split[K];
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < cap || t < K;
       t += (int64_t)gridDim.x * blockDim.x) {
    if (t < K && (num_split[t + 1] < num_split[t] || (t == 0 && num_split[0] != 0) || (t == K - 1 && n > cap)))
      *bad = 1;
    int64_t cell = -1;  // the (split, table) counter of a counted entry
    if (t < cap) {
      int64_t sp = S;
      if (t < n && n <= cap) {
        sp = indices[t];
        if (sp < 0 || sp >= S) {
          *bad = 1;
          sp = 0;
        }
        cell = sp * K + (K > 1 ? list_of(num_split, K, t) : 0);
      }
      keys[t] = (uint32_t)sp;
    }
    // one atomic per distinct counter of the warp (few counters take all of a batch: S * K is small)
    const uint32_t peers = __match_any_sync(__activemask(), cell);
    if (cell >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(cnt + cell, (uint32_t)__popc(peers));
  }
}

// one block: every split's row splits from its table counts, then the split offsets (exclusive scan over splits)
__global__ void __launch_bounds__(1024)
rsi_scan_kernel(const uint32_t* __restrict__ cnt, int K, int S, int64_t* __restrict__ row_splits,
                int64_t* __restrict__ split_offsets) {
  __shared__ int64_t wsum[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int per = (S + 1023) / 1024;
  const int b = min(S, (int)threadIdx.x * per), e = min(S, b + per);
  int64_t sum = 0;
  for (int s = b; s < e; ++s) {
    int64_t run = 0;
    int64_t* rs = row_splits + (size_t)s * (K + 1);
    rs[0] = 0;
    for (int k = 0; k < K; ++k) {
      run += cnt[(size_t)s * K + k];
      rs[k + 1] = run;
    }
    sum += run;
  }
  int64_t x = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  if (w == 0) {
    int64_t t = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    wsum[lane] = t;
  }
  __syncthreads();
  int64_t run = (w ? wsum[w - 1] : 0) + x - sum;
  for (int s = b; s < e; ++s) {
    split_offsets[s] = run;
    run += row_splits[(size_t)s * (K + 1) + K];
  }
  if (threadIdx.x == 1023) split_offsets[S] = wsum[31];
}

__global__ void __launch_bounds__(kThreads)
rsi_scatter_kernel(const int64_t* __restrict__ values, const uint2* __restrict__ sorted, int64_t cap,
                   const int64_t* __restrict__ split_offsets, int S, int64_t* __restrict__ values_out,
                   int64_t* __restrict__ pos_out) {
  const int64_t n = split_offsets[S];
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n && q < cap;
       q += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t t = sorted[q].y;
    values_out[q] = values[t];
    pos_out[q] = t;
  }
}

void run_ragged_split(int device, const int64_t* indices_dev, const int64_t* values_dev, int64_t cap,
                      const int64_t* num_split_dev, int K, int S, int64_t* values_out_dev, int64_t* pos_out_dev,
                      int64_t* row_splits_out_dev, int64_t* split_offsets_dev, int32_t* bad_dev,
                      int64_t* row_splits_host, cudaStream_t s) {
  if (K <= 0) throw ArgError("ragged_split_by_indices: num_tables must be positive");
  if (S <= 0) throw ArgError("ragged_split_by_indices: num_splits must be positive");
  if (cap < 0 || cap > kMaxIds) throw ArgError("ragged_split_by_indices: capacity outside [0, 2^30]");
  if ((int64_t)S * K > ((int64_t)1 << 31)) throw ArgError("ragged_split_by_indices: num_splits x num_tables > 2^31");
  MONO_CUDA(cudaSetDevice(device));
  const size_t C1 = (size_t)std::max<int64_t>(cap, 1);
  const int bits = key_bits((int64_t)S + 1);  // keys 0 .. S
  size_t off = 0;
  auto take256 = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_keys = take256(sizeof(uint32_t) * C1), o_cnt = take256(sizeof(uint32_t) * (size_t)S * K),
               o_bad = take256(sizeof(int32_t)), o_sort = take256(key_sort_bytes((int64_t)C1, bits));
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, off, s));
  uint32_t* keys = reinterpret_cast<uint32_t*>(ws + o_keys);
  uint32_t* cnt = reinterpret_cast<uint32_t*>(ws + o_cnt);
  int32_t* bad = reinterpret_cast<int32_t*>(ws + o_bad);
  MONO_CUDA(cudaMemsetAsync(ws + o_cnt, 0, o_sort - o_cnt, s));  // the counters and the flag
  rsi_count_kernel<<<grid_for(std::max<int64_t>(cap, K), kThreads), kThreads, 0, s>>>(indices_dev, cap, num_split_dev,
                                                                                      K, S, keys, cnt, bad);
  MONO_CHECK_LAUNCH();
  rsi_scan_kernel<<<1, 1024, 0, s>>>(cnt, K, S, row_splits_out_dev, split_offsets_dev);
  MONO_CHECK_LAUNCH();
  if (cap > 0) {
    const uint2* sorted = nullptr;
    key_sort(ws + o_sort, keys, cap, bits, false, &sorted, s);
    rsi_scatter_kernel<<<grid_for(cap, kThreads), kThreads, 0, s>>>(values_dev, sorted, cap, split_offsets_dev, S,
                                                                    values_out_dev, pos_out_dev);
    MONO_CHECK_LAUNCH();
  }
  if (bad_dev) MONO_CUDA(cudaMemcpyAsync(bad_dev, bad, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  int32_t bad_host = 0;
  if (row_splits_host) {
    MONO_CUDA(cudaMemcpyAsync(row_splits_host, row_splits_out_dev, sizeof(int64_t) * (size_t)S * (K + 1),
                              cudaMemcpyDeviceToHost, s));
    MONO_CUDA(cudaMemcpyAsync(&bad_host, bad, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  }
  MONO_CUDA(cudaFreeAsync(ws, s));
  if (row_splits_host) {
    MONO_CUDA(cudaStreamSynchronize(s));
    if (bad_host)
      throw ArgError("ragged_split_by_indices: an index outside [0, num_splits), or num_split does not start at 0, "
                     "decreases or exceeds the capacity");
  }
}

}  // namespace mono
