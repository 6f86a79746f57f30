// bwd.cu — the fused sparse backward: pooled-gradient scatter + sparse optimizer + expiry bump, deterministic,
// without float atomics; and the owner grouping of the sharded step that shares its machinery.
//
// Replaces (for one table) the reference's ScatterGrad / BackwardBatchKernel (fused_embedding_to_layout.h:286-347,
// .cu.cc:337-381: float atomicAdd per occurrence into a per-unique-FID gradient buffer) followed by
// MultiHashTableOptimize (multi_hash_table_update_op.cc:47-89; embedding_hash_table_tf_bridge.cc:258-341).
// Pipeline, all on the caller's stream, nothing returns to the host:
//   1 claim   : every occurrence finds / claims the scratch-set slot of its FID (same slot <=> same FID); the
//               winner of a slot resolves the FID in the table (row index, expiry-timestamp bump) or queues it
//   2 insert  : absent FIDs get a row and are published with the lock-free cuckoo insert
//   3 sort    : stable LSD radix sort of (slot, position), 11 bits per pass (2 passes for 2 M occurrences):
//               the occurrences of a FID become one contiguous run in position order
//   4 runs    : run heads -> ordered run list (start, first position, resolved row)
//   5 reduce  : seg_reduce_kernel streams the sorted occurrences in 32-occurrence pieces; runs of <= 64
//               occurrences are summed in occurrence order (the CPU reference's order: bit-exact) and stored per run;
//               hot FIDs are cut into run-aligned 32-occurrence blocks, combined by 0-2 levels of 128-member tree
//               nodes (the depth follows the call's occurrence count) and a final in-order pass (deterministic,
//               pairwise-accurate; tests/reduce_order.py restates the order).  In the fused backward the runs of
//               <= kApplyRun (8) occurrences are left to the apply, which sums them itself
//   6 apply   : runs_apply_kernel applies the optimizer, one row per run: it sums a run of <= 8 occurrences from
//               the gradient rows (same order and arithmetic: same bits) and reads a longer run's sum from ugrad
#include <algorithm>
#include <cstring>

#include "rowops.cuh"

namespace mono {

// ==========================================================================================
// Stable LSD radix sort of (key, position), 11 bits per pass.
// Items travel as uint2 {key, position} (ONE 8-byte scattered store per item and pass); the first pass reads the
// bare keys (position = index).  Per pass: tile histograms (shared-memory atomics) -> column scan over the tiles
// -> stable scatter.  The scatter kernel ranks an item among the equal digits in front of it inside its tile
// with ballots (11 votes give the lane mask of equal digits; lanes are consecutive positions, so the count of
// lower lanes is the stable rank; one MATCH.ANY instead of the 11 votes measured slower over the two passes) and per-warp digit counters in shared memory; tiles are ordered by the scanned
// histograms, so no atomic ever decides an output position.
// ==========================================================================================
constexpr int kRadixBits = 11;
constexpr int kRadixBins = 1 << kRadixBits;
constexpr int kRadixIPT = 16;                         // items per thread
constexpr int kRadixTile = kThreads * kRadixIPT;      // 4096 items per block iteration
constexpr int kRadixWarps = kThreads / 32;

template <bool FIRST>
__device__ __forceinline__ uint2 radix_load(const void* __restrict__ in, int64_t i, int pre_shift) {
  if (FIRST) return make_uint2(static_cast<const uint32_t*>(in)[i] >> pre_shift, (uint32_t)i);
  return static_cast<const uint2*>(in)[i];
}

template <bool FIRST>
__global__ void __launch_bounds__(kThreads)
radix_hist_kernel(const void* __restrict__ in, int64_t n, int shift, int pre_shift, uint32_t* __restrict__ cnt /*[nblk][2048]*/,
                  int nblk) {
  __shared__ uint32_t h[kRadixBins];
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    for (int d = threadIdx.x; d < kRadixBins; d += kThreads) h[d] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blk * kRadixTile;
#pragma unroll
    for (int r = 0; r < kRadixIPT; ++r) {
      const int64_t i = base + r * kThreads + threadIdx.x;
      if (i < n) atomicAdd(&h[(radix_load<FIRST>(in, i, pre_shift).x >> shift) & (kRadixBins - 1)], 1u);
    }
    __syncthreads();
    for (int d = threadIdx.x; d < kRadixBins; d += kThreads) cnt[(size_t)blk * kRadixBins + d] = h[d];
    __syncthreads();
  }
}

// exclusive prefix over the tiles, per digit column (in place), and the digit totals.
// Block = 32 digit columns x 32 tile chunks.
__global__ void __launch_bounds__(1024)
radix_colscan_kernel(uint32_t* __restrict__ cnt, int nblk, uint32_t* __restrict__ dtot) {
  __shared__ uint32_t sums[32][33];
  const int dx = threadIdx.x & 31, ch = threadIdx.x >> 5;
  const int d = blockIdx.x * 32 + dx;
  const int per = (nblk + 31) / 32;
  const int t0 = min(nblk, ch * per), t1 = min(nblk, t0 + per);
  uint32_t s = 0;
  for (int t = t0; t < t1; ++t) s += cnt[(size_t)t * kRadixBins + d];
  sums[ch][dx] = s;
  __syncthreads();
  if (ch == 0) {
    uint32_t run = 0;
    for (int q = 0; q < 32; ++q) {
      const uint32_t v = sums[q][dx];
      sums[q][dx] = run;
      run += v;
    }
    dtot[d] = run;
  }
  __syncthreads();
  uint32_t run = sums[ch][dx];
  for (int t = t0; t < t1; ++t) {
    const uint32_t v = cnt[(size_t)t * kRadixBins + d];
    cnt[(size_t)t * kRadixBins + d] = run;
    run += v;
  }
}

template <bool FIRST>
__global__ void __launch_bounds__(kThreads, 4)
radix_scatter_kernel(const void* __restrict__ in, int64_t n, int shift, int pre_shift,
                     const uint32_t* __restrict__ goff /*[nblk][2048] scanned*/, const uint32_t* __restrict__ dtot,
                     int nblk, uint2* __restrict__ out) {
  __shared__ uint16_t wc[kRadixWarps][kRadixBins];   // per-warp digit counters, then exclusive warp offsets
  __shared__ uint32_t bbase[kRadixBins];             // global offset of (tile, digit)
  __shared__ uint32_t wsum[kRadixWarps];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  // exclusive scan of the 2048 digit totals; thread t keeps the bases of its digits q * 256 + t in registers
  uint32_t dbase[kRadixBins / kThreads];
  {
    uint32_t carry = 0;
#pragma unroll
    for (int q = 0; q < kRadixBins / kThreads; ++q) {
      const uint32_t v = dtot[q * kThreads + threadIdx.x];
      uint32_t x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) wsum[w] = x;
      __syncthreads();
      uint32_t off = 0, tot = 0;
#pragma unroll
      for (int ww = 0; ww < kRadixWarps; ++ww) {
        const uint32_t t = wsum[ww];
        if (ww < w) off += t;
        tot += t;
      }
      dbase[q] = carry + off + x - v;
      carry += tot;
      __syncthreads();
    }
  }
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    uint32_t* wz = reinterpret_cast<uint32_t*>(&wc[0][0]);
    for (int q = threadIdx.x; q < kRadixWarps * kRadixBins / 2; q += kThreads) wz[q] = 0;
    __syncthreads();
    // ---- phase 1: stable rank of every item among the equal digits of its warp's 512-item slice ----
    const int64_t wbeg = (int64_t)blk * kRadixTile + (int64_t)w * (kRadixTile / kRadixWarps);
    uint32_t dgv[kRadixIPT];   // all 16 digits first: 16 independent loads in flight (0xFFFFFFFF = past the end)
#pragma unroll
    for (int r = 0; r < kRadixIPT; ++r) {
      const int64_t i = wbeg + r * 32 + lane;
      dgv[r] = i < n ? (radix_load<FIRST>(in, i, pre_shift).x >> shift) & (kRadixBins - 1) : 0xFFFFFFFFu;
    }
#pragma unroll
    for (int r = 0; r < kRadixIPT; ++r) {  // afterwards dgv[r] = digit | rank << 16 (rank < 1024)
      const bool valid = dgv[r] != 0xFFFFFFFFu;
      const uint32_t dg = valid ? dgv[r] : 0u;
      uint32_t peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
      for (int b = 0; b < kRadixBits; ++b) {
        const uint32_t bal = __ballot_sync(0xffffffffu, (dg >> b) & 1u);
        peers &= ((dg >> b) & 1u) ? bal : ~bal;
      }
      const int leader = __ffs(peers) - 1;
      uint32_t old = 0;
      if (valid && lane == leader) {
        old = wc[w][dg];
        wc[w][dg] = (uint16_t)(old + __popc(peers));
      }
      old = __shfl_sync(0xffffffffu, old, max(leader, 0));
      if (valid) dgv[r] = dg | ((old + __popc(peers & lt)) << 16);
      __syncwarp();
    }
    __syncthreads();
    // ---- warp offsets per digit and the tile's global digit offsets ----
#pragma unroll
    for (int q = 0; q < kRadixBins / kThreads; ++q) {
      const int d = q * kThreads + threadIdx.x;
      uint32_t run = 0;
#pragma unroll
      for (int ww = 0; ww < kRadixWarps; ++ww) {
        const uint32_t v = wc[ww][d];
        wc[ww][d] = (uint16_t)run;
        run += v;
      }
      bbase[d] = goff[(size_t)blk * kRadixBins + d] + dbase[q];
    }
    __syncthreads();
    // ---- phase 2: scatter (digit and rank are in registers; the items are read again, 8 loads in flight) ----
#pragma unroll
    for (int h = 0; h < kRadixIPT; h += 8) {
      uint2 itv[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int64_t i = wbeg + (h + r) * 32 + lane;
        itv[r] = make_uint2(0u, 0u);
        if (dgv[h + r] != 0xFFFFFFFFu) itv[r] = radix_load<FIRST>(in, i, pre_shift);
      }
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const uint32_t v = dgv[h + r];
        if (v != 0xFFFFFFFFu) {
          const uint32_t dg = v & (kRadixBins - 1);
          out[bbase[dg] + wc[w][dg] + (v >> 16)] = itv[r];
        }
      }
    }
    __syncthreads();
  }
}

// ---- ordered run compaction: run j = j-th distinct key of the sorted array ----
__device__ __forceinline__ bool is_run_start(const uint2* __restrict__ sorted, int64_t i, int64_t n) {
  return i < n && (i == 0 || sorted[i].x != sorted[i - 1].x);
}

constexpr int kRunTile = kThreads * 8;

__global__ void __launch_bounds__(kThreads)
runs_count_kernel(const uint2* __restrict__ sorted, int64_t n, int nblk, uint32_t* __restrict__ blk_runs) {
  __shared__ uint32_t wc[kThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    uint32_t cnt = 0;
    for (int c = 0; c < kRunTile; c += kThreads)
      cnt += __popc(__ballot_sync(0xffffffffu, is_run_start(sorted, (int64_t)blk * kRunTile + c + threadIdx.x, n)));
    if (lane == 0) wc[w] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t t = 0;
      for (int ww = 0; ww < kThreads / 32; ++ww) t += wc[ww];
      blk_runs[blk] = t;
    }
    __syncthreads();
  }
}

// one block: exclusive scan of blk_runs, total -> n_runs, sentinel run_start[n_runs] = n
__global__ void __launch_bounds__(1024)
runs_scan_kernel(uint32_t* __restrict__ blk_runs, int nblk, uint32_t* __restrict__ n_runs,
                 uint32_t* __restrict__ run_start, int64_t n) {
  __shared__ uint32_t wsum[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int per = (nblk + 1023) / 1024;
  const int b = min(nblk, (int)threadIdx.x * per), e = min(nblk, b + per);
  uint32_t sum = 0;
  for (int i = b; i < e; ++i) sum += blk_runs[i];
  uint32_t x = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  if (w == 0) {
    uint32_t t = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    wsum[lane] = t;
  }
  __syncthreads();
  uint32_t run = (w ? wsum[w - 1] : 0) + x - sum;
  for (int i = b; i < e; ++i) {
    const uint32_t v = blk_runs[i];
    blk_runs[i] = run;
    run += v;
  }
  if (threadIdx.x == 1023) {
    *n_runs = wsum[31];
    run_start[wsum[31]] = (uint32_t)n;
  }
}

// run list: start (sorted index), first position, resolved row (when the claim parked it in the set), and per
// 32-occurrence piece the number of run heads in front of it (what seg_reduce_kernel indexes runs with)
__global__ void __launch_bounds__(kThreads)
runs_write_kernel(const uint2* __restrict__ sorted, int64_t n, int nblk, const uint32_t* __restrict__ blk_runs,
                  uint32_t* __restrict__ run_start, uint32_t* __restrict__ run_first_pos,
                  uint32_t* __restrict__ piece_run_base, uint32_t* __restrict__ run_of_sorted /* optional */,
                  const Entry* __restrict__ claim_set /* optional */, uint32_t* __restrict__ rowidx) {
  __shared__ uint32_t wc[kThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  constexpr int NW = kThreads / 32;
  constexpr int kPerWarp = kRunTile / NW;
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    const int64_t wbeg = (int64_t)blk * kRunTile + (int64_t)w * kPerWarp;
    uint32_t cnt = 0;
    for (int c = 0; c < kPerWarp; c += 32)
      cnt += __popc(__ballot_sync(0xffffffffu, is_run_start(sorted, wbeg + c + lane, n)));
    if (lane == 0) wc[w] = cnt;
    __syncthreads();
    uint32_t base = blk_runs[blk];
    for (int ww = 0; ww < w; ++ww) base += wc[ww];
    for (int c = 0; c < kPerWarp; c += 32) {
      const int64_t i = wbeg + c + lane;
      const bool st = is_run_start(sorted, i, n);
      const uint32_t bal = __ballot_sync(0xffffffffu, st);
      if (lane == 0 && wbeg + c < n) piece_run_base[(wbeg + c) >> 5] = base;
      if (st) {
        const uint32_t j = base + __popc(bal & ((1u << lane) - 1u));
        const uint2 it = sorted[i];
        run_start[j] = (uint32_t)i;
        run_first_pos[j] = it.y;
        if (claim_set) rowidx[j] = claim_set[it.x].row;
      }
      if (run_of_sorted && i < n) run_of_sorted[i] = base + __popc(bal & (0xffffffffu >> (31 - lane))) - 1;
      base += __popc(bal);
    }
    __syncthreads();
  }
}

static int radix_blocks(int64_t M) { return (int)((M + kRadixTile - 1) / kRadixTile); }
static int run_blocks(int64_t M) { return (int)((M + kRunTile - 1) / kRunTile); }
static int sort_passes(int bits) { return std::max(1, (bits + kRadixBits - 1) / kRadixBits); }

// stable LSD radix sort of (keys[i] >> pre_shift, i) over `bits` key bits, then the ordered run list (one run per
// distinct key; claim_set != null: the keys are its slots and each run's resolved row is gathered into w.rowidx).
// Everything stays on the stream; counts stay on the device.
static const uint2* sort_and_runs(const SortWs& w, const uint32_t* keys, int64_t M, int bits, int pre_shift,
                                  const Entry* claim_set, cudaStream_t s) {
  const int passes = sort_passes(bits);
  const int nb = radix_blocks(M);
  const void* in = keys;
  uint2* out = w.a;
  for (int p = 0; p < passes; ++p) {
    uint32_t* dt = w.dtot + kRadixBins * p;
    const int ps = p == 0 ? pre_shift : 0;
    if (p == 0) {
      radix_hist_kernel<true><<<resident_grid(radix_hist_kernel<true>, nb, 1), kThreads, 0, s>>>(in, M, 0, ps, w.cnt, nb);
      MONO_CHECK_LAUNCH();
    } else {
      radix_hist_kernel<false><<<resident_grid(radix_hist_kernel<false>, nb, 1), kThreads, 0, s>>>(in, M, kRadixBits * p, 0, w.cnt, nb);
      MONO_CHECK_LAUNCH();
    }
    radix_colscan_kernel<<<kRadixBins / 32, 1024, 0, s>>>(w.cnt, nb, dt);
    MONO_CHECK_LAUNCH();
    if (p == 0) {
      radix_scatter_kernel<true><<<resident_grid(radix_scatter_kernel<true>, nb, 1), kThreads, 0, s>>>(in, M, 0, ps, w.cnt, dt, nb, out);
      MONO_CHECK_LAUNCH();
    } else {
      radix_scatter_kernel<false><<<resident_grid(radix_scatter_kernel<false>, nb, 1), kThreads, 0, s>>>(in, M, kRadixBits * p, 0, w.cnt, dt, nb, out);
      MONO_CHECK_LAUNCH();
    }
    in = out;
    out = (out == w.a) ? w.b : w.a;
  }
  const uint2* sorted = static_cast<const uint2*>(in);
  const int nr = run_blocks(M);
  runs_count_kernel<<<resident_grid(runs_count_kernel, nr, 1), kThreads, 0, s>>>(sorted, M, nr, w.blk_runs);
  MONO_CHECK_LAUNCH();
  runs_scan_kernel<<<1, 1024, 0, s>>>(w.blk_runs, nr, w.n_runs, w.run_start, M);
  MONO_CHECK_LAUNCH();
  runs_write_kernel<<<resident_grid(runs_write_kernel, nr, 1), kThreads, 0, s>>>(
      sorted, M, nr, w.blk_runs, w.run_start, w.run_first_pos, w.piece_run_base, w.run_of_sorted, claim_set, w.rowidx);
  MONO_CHECK_LAUNCH();
  return sorted;
}

// ==========================================================================================
// gradient source and the per-row optimizer step
// ==========================================================================================
constexpr int kShortRun = 64;
// runs of at most kApplyRun occurrences are summed by runs_apply_kernel, kApplyStage gradient rows in flight per lane
constexpr int kApplyRun = 8;
constexpr int kApplyStage = 8;
static_assert(kApplyRun <= kShortRun, "the apply sums short runs only");

__global__ void __launch_bounds__(kThreads)
occ_row_kernel(const int32_t* __restrict__ row_offsets, int64_t n_rows, uint32_t* __restrict__ occ_row) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rows;
       r += (int64_t)gridDim.x * blockDim.x)
    for (int m = row_offsets[r]; m < row_offsets[r + 1]; ++m) occ_row[m] = (uint32_t)r;
}

struct BwdArgs {
  TableDev td;          // by value: lives in the kernel-parameter constant bank (uniform, free reads)
  const TableDev* t;    // device copy, for the generic apply_row path
  const int64_t* fids;
  const uint2* sorted;   // {scratch-set slot (sort key), occurrence position}, sorted by key, stable
  int64_t n;             // occurrences
  const uint32_t* n_runs;
  const uint32_t* run_start;
  const uint32_t* run_first_pos;
  const uint32_t* rowidx;       // per run (bit 31 = fresh)
  const uint32_t* occ_row;      // occurrence -> pooled row (null: identity)
  const int32_t* row_offsets;   // for MEAN (null: n == 1)
  int pooling;
  const float* pooled_grad;
  int64_t grad_stride;
  int grad_col;
  // parts call (run_pool_backward_parts): one table's occurrences are the sorted range [lo, n); each occurrence's
  // gradient row and MEAN divisor (0: none) come from the call's occurrence map, its run range from run_of_sorted
  int64_t lo;
  const float* const* occ_src;
  const float* occ_div;
  const uint32_t* run_of_sorted;
  const float* lr;              // device, slice learning rates of the table
  float* ugrad;                 // [runs][D] summed gradient of every run (= unique FID), run order
  float* scratch;               // alias of ugrad for the generic (multi-segment) apply path
};

// Where the gradient rows come from: copied out of the kernel parameters once per thread so that the
// inner loops do not re-read the constant bank (ncu showed LDCU stalls inside the unrolled loads).
struct GradSrc {
  const float* base;            // pooled_grad + grad_col + lane column, counted in row elements (T of the kernel)
  int64_t stride;
  const uint32_t* occ_row;
  const int32_t* row_offsets;
  const float* const* occ_src;  // parts call: gradient row (column included) of every occurrence; bf16 rows: a cast
                                // pointer to the row's bf16 elements
  const float* occ_div;         // parts call: MEAN divisor of every occurrence, 0 = none
  bool mean;
};
// T: the gradient row element; a bf16 pooled_grad is a cast pointer whose stride and column count bf16 elements
template <typename T>
__device__ __forceinline__ GradSrc make_grad_src(const BwdArgs& a, int c) {
  GradSrc g;
  g.base = reinterpret_cast<const float*>(reinterpret_cast<const T*>(a.pooled_grad) + a.grad_col + c);
  g.stride = a.grad_stride;
  g.occ_row = a.occ_row;
  g.row_offsets = a.row_offsets;
  g.occ_src = a.occ_src;
  g.occ_div = a.occ_div;
  g.mean = a.pooling == MONO_POOL_MEAN && (a.row_offsets != nullptr || a.occ_div != nullptr);
  return g;
}
// gradient row of occurrence m, from column c (the lane's; gs.base already holds it)
template <typename T>
__device__ __forceinline__ const T* occ_grad_src(const GradSrc& gs, uint32_t m, int c) {
  if (gs.occ_src) return reinterpret_cast<const T*>(gs.occ_src[m]) + c;
  return reinterpret_cast<const T*>(gs.base) + (size_t)(gs.occ_row ? gs.occ_row[m] : m) * gs.stride;
}
// MEAN divisor of occurrence m (gs.mean only; 0 = none)
__device__ __forceinline__ float occ_grad_div(const GradSrc& gs, uint32_t m) {
  if (gs.occ_div) return gs.occ_div[m];
  const uint32_t r = gs.occ_row ? gs.occ_row[m] : m;
  return (float)(gs.row_offsets[r + 1] - gs.row_offsets[r]);
}
__device__ __forceinline__ void add4(float4& a, const float4& b) {
  a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
}

// Row state prefetched BEFORE the gradient gather so that the w / optimizer-state reads overlap the
// random gradient-row reads (single-segment fast path).
struct RowPre {
  float4 w4, a4, b4;
  float b1p, b2p;
};

template <int G, int OPT>
__device__ __forceinline__ RowPre bwd_prefetch(const BwdArgs& a, uint32_t ri, int c) {
  RowPre p;
  p.w4 = p.a4 = p.b4 = make_float4(0.f, 0.f, 0.f, 0.f);
  p.b1p = p.b2p = 0.f;
  if (OPT < 0 || (ri & kFreshBit)) return p;
  const int D = a.td.dim;
  const uint32_t row = ri & ~kFreshBit;
  const float* __restrict__ w_row = a.td.emb + (size_t)row * a.td.emb_stride;
  const float* __restrict__ s_row = a.td.state + (size_t)row * a.td.state_stride;
  if (c < D) {
    p.w4 = *reinterpret_cast<const float4*>(w_row + c);
    if (OPT != MONO_OPT_SGD) p.a4 = *reinterpret_cast<const float4*>(s_row + c);
    if (OPT == MONO_OPT_FTRL || OPT == MONO_OPT_ADAM) p.b4 = *reinterpret_cast<const float4*>(s_row + D + c);
  }
  if (OPT == MONO_OPT_ADAM) {
    p.b1p = s_row[2 * D];
    p.b2p = s_row[2 * D + 1];
  }
  return p;
}

// Apply the optimizer to row `ri` with the summed gradient held in registers (one float4 per lane,
// dim <= 4*G).  OPT >= 0: single-segment table with that optimizer (compile-time specialised);
// OPT < 0: any segment mix, staged through scratch + apply_row.
template <int G, int OPT>
__device__ __forceinline__ void bwd_apply(const BwdArgs& a, uint32_t j, uint32_t ri, float4 g4, int c,
                                          RowPre pre) {
  const int D = a.td.dim;
  const uint32_t row = ri & ~kFreshBit;
  const bool fresh = (ri & kFreshBit) != 0;
  if (OPT >= 0) {
    const SegDev& s0 = a.td.segs[0];
    float* __restrict__ w_row = a.td.emb + (size_t)row * a.td.emb_stride;
    float* __restrict__ s_row = a.td.state + (size_t)row * a.td.state_stride;
    float lrt = a.lr[0];
    float4 w4 = pre.w4, a4 = pre.a4, b4 = pre.b4;
    float b1p = pre.b1p, b2p = pre.b2p;
    if (fresh) {  // the key is only needed to initialise a new row
      const int64_t key = a.fids[a.run_first_pos[j]];
      w4.x = init_emb_value(&a.td, s0, key, c); w4.y = init_emb_value(&a.td, s0, key, c + 1);
      w4.z = init_emb_value(&a.td, s0, key, c + 2); w4.w = init_emb_value(&a.td, s0, key, c + 3);
      a4.x = a4.y = a4.z = a4.w = init_state_value(s0, 0);
      b4.x = b4.y = b4.z = b4.w = init_state_value(s0, D);
      b1p = s0.p[0];
      b2p = s0.p[1];
    }
    if (OPT == MONO_OPT_ADAM) lrt = adam_lr(lrt, b1p, b2p);
    if (c < D) {
      const bool avx = c < (D & ~7);
      opt_elem_t<OPT>(s0.p, avx, lrt, g4.x, w4.x, a4.x, b4.x);
      opt_elem_t<OPT>(s0.p, avx, lrt, g4.y, w4.y, a4.y, b4.y);
      opt_elem_t<OPT>(s0.p, avx, lrt, g4.z, w4.z, a4.z, b4.z);
      opt_elem_t<OPT>(s0.p, avx, lrt, g4.w, w4.w, a4.w, b4.w);
      *reinterpret_cast<float4*>(w_row + c) = w4;
      if (OPT != MONO_OPT_SGD) *reinterpret_cast<float4*>(s_row + c) = a4;
      if (OPT == MONO_OPT_FTRL || OPT == MONO_OPT_ADAM) *reinterpret_cast<float4*>(s_row + D + c) = b4;
    }
    if (OPT == MONO_OPT_ADAM) {
      __syncwarp(Group<G>::mask());  // every lane has read the old powers (in the prefetch)
      if (Group<G>::gl() == 0) {
        s_row[2 * D] = __fmul_rn(b1p, s0.p[0]);
        s_row[2 * D + 1] = __fmul_rn(b2p, s0.p[1]);
      }
    }
  } else {
    float* sc = a.scratch + (size_t)j * D;
    if (c < D) *reinterpret_cast<float4*>(sc + c) = g4;
    __syncwarp(Group<G>::mask());
    apply_row<G, kOpOptimize>(a.t, row, a.fids[a.run_first_pos[j]], sc, a.lr, fresh);
  }
}

// destination of run j's summed row: ugrad[j], or (po.n != 0: the sharded backward's fused gradient
// exchange) row j of an owner-bucketed list whose part r lives in rank r's peer window.
__device__ __forceinline__ float* run_dst(float* ugrad, int n_parts, const int64_t* __restrict__ s_start,
                                          char* const* __restrict__ s_base, int64_t j, int D) {
  if (n_parts == 0) return ugrad + (size_t)j * D;
  const int r = peer_part(s_start, n_parts, j);
  return reinterpret_cast<float*>(s_base[r]) + (j - s_start[r]) * D;
}


// ==========================================================================================
// Gradient reduction over the sorted occurrence list (replaces the per-run-length-class kernels of round 1).
//
// The sorted list is cut into PIECES of 32 consecutive sorted occurrences; one lane group (G lanes, one 16-byte
// vector of the row per lane) owns one piece, a warp owns 32/G consecutive pieces.  Work is defined in UNITS:
//   * a SHORT run (<= kShortRun occurrences of one FID) is one unit, summed sequentially in occurrence
//     order = the CPU reference's order (bit-exact);
//   * a LONG run (> kShortRun) is cut into 32-occurrence BLOCKS aligned to the START OF THE RUN; each block is
//     one unit, summed sequentially; block sums are then combined over the block index by tree levels of
//     kTreeFan-member nodes (tree_level_kernel; as many levels as keep the final pass at <= kFinishMax terms for the
//     call's piece count) and the in-order final pass (long_finish_kernel).  The association depends on the run
//     length, on G (the node's lane-group split) and on the call's tree depth, nothing else: run-to-run bit-stable
//     whatever scratch-set slot the FID got, and pairwise-accurate (tests/reduce_order.py restates it;
//     tests/test_gpu_reduce_order.py checks it bit for bit).
// A group owns the units that START inside its piece and follows its last unit past the end of the piece (at most
// 63 occurrences); occurrences in front of the first unit start belong to the previous group's last unit.  Every
// group therefore streams 32 + <64 gradient rows whatever the run-length distribution is: hot FIDs of a Zipf
// batch (half of the occurrences) are plain 32-row units like everything else — no run-length classes, no
// work lists, no atomics, no device-side scheduling.
//
// Where results go (the optimizer is applied afterwards, by runs_apply_kernel):
//   SHORT unit  -> run_dst: the run's row of the local ugrad, or of the owner's peer window for the sharded backward.
//   LONG block  -> part[slot], slot = 2 * piece + (block 0 ? 1 : 0): at most one block of the run that covers the
//               piece start and at most one long-run head can START in a 32-occurrence piece, and block k + i of a
//               run starts exactly i pieces after block k.  The tree levels and the final pass therefore find
//               every operand by arithmetic on the slot index: meta[slot] = {run, block, #blocks, valid}.
// ==========================================================================================
constexpr int kPiece = 32;
constexpr int kTreeFan = 128;   // members summed by one tree node (in block order)
constexpr int kFinishMax = 512; // blocks / nodes the final pass may still have to add up per run

struct SegMeta {  // one per partial slot
  uint32_t run, blk, nblk, valid;
};

struct SegArgs {
  BwdArgs b;                        // gradient source, table, run list (run_start / rowidx / run_first_pos)
  const uint32_t* piece_run_base;   // [n_pieces]: number of run heads in front of piece p of the range
  float* part;                      // [2 * n_pieces][D]
  SegMeta* meta;                    // [2 * n_pieces]
  int64_t n_pieces;                 // pieces of the range [b.lo, b.n) of the sorted list
  int64_t piece0;                   // the range's first piece in the sorted list (b.lo / 32)
};

template <int EPL>
__device__ __forceinline__ uint32_t pick(const uint32_t (&v)[EPL], int comp) {
  uint32_t r = v[0];
#pragma unroll
  for (int c = 1; c < EPL; ++c)
    if (comp == c) r = v[c];
  return r;
}

// element `e` (0..31) of a 32-element chunk held EPL-per-lane by the G lanes of the group
template <int G>
__device__ __forceinline__ uint32_t chunk_elem(const uint32_t (&v)[32 / G], int e) {
  constexpr int EPL = 32 / G;
  const uint32_t mine = pick<EPL>(v, e % EPL);  // e is group-uniform: every lane selects the same component
  return __shfl_sync(Group<G>::mask(), mine, Group<G>::base() + e / EPL);
}

// 32 consecutive sorted items {key, position}, EPL per lane (lane gl holds items gl * EPL ..): vector loads
template <int G>
__device__ __forceinline__ void load_items(const uint2* __restrict__ src, int64_t first, int64_t n,
                                           uint32_t (&key)[32 / G], uint32_t (&pos)[32 / G]) {
  constexpr int EPL = 32 / G;
  const int64_t i0 = first + Group<G>::gl() * EPL;
  if (EPL >= 2 && i0 + EPL <= n) {
#pragma unroll
    for (int q = 0; q < EPL; q += 2) {
      const uint4 v = *reinterpret_cast<const uint4*>(src + i0 + q);
      key[q] = v.x; pos[q] = v.y;
      key[q + (EPL >= 2 ? 1 : 0)] = v.z; pos[q + (EPL >= 2 ? 1 : 0)] = v.w;
    }
  } else {
#pragma unroll
    for (int q = 0; q < EPL; ++q) {
      uint2 v = make_uint2(0u, 0u);
      if (i0 + q < n) v = src[i0 + q];
      key[q] = v.x;
      pos[q] = v.y;
    }
  }
}

// positions of the 4 consecutive elements e .. e+3 (e a multiple of 4, < 32) of a chunk held EPL-per-lane
template <int G>
__device__ __forceinline__ void fetch4(const uint32_t (&v)[32 / G], int e, uint32_t (&out)[4]) {
  constexpr int EPL = 32 / G;
  const uint32_t gmask = Group<G>::mask();
  const int gb = Group<G>::base();
  if (EPL == 4) {
#pragma unroll
    for (int u = 0; u < 4; ++u) out[u] = __shfl_sync(gmask, v[u % EPL], gb + e / 4);
  } else if (EPL == 8) {
    const bool hi = (e & 4) != 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) out[u] = __shfl_sync(gmask, hi ? v[(4 + u) % EPL] : v[u % EPL], gb + e / 8);
  } else if (EPL == 2) {
#pragma unroll
    for (int u = 0; u < 4; ++u) out[u] = __shfl_sync(gmask, v[u % EPL], gb + e / 2 + u / 2);
  } else {
#pragma unroll
    for (int u = 0; u < 4; ++u) out[u] = __shfl_sync(gmask, v[0], gb + e + u);
  }
}

// The reduction kernel: unit sums go to run_dst (short runs) / part (long-run blocks).
// Memory-level parallelism is what bounds it (a dependent random HBM round trip costs microseconds under load, so
// ~100 KB must be in flight per SM): the gradient rows of a group's stream are requested kStage = 16 at a time with cp.async
// (LDGSTS) into shared memory — every lane copies ITS 16-byte column slice of each row into a private slot, so nothing
// but the thread's own cp.async.wait orders the data and no register holds a row in flight — then the adds run in
// occurrence order out of shared memory.  3 blocks x 64 KB = 192 KB of gradient rows in flight per SM.

// G = lanes per group, VPL = 16-byte vectors of the row per lane (lane gl owns columns (gl + v * G) * 4 ..): VPL = 2 halves
// the warp instructions per occurrence (the kernel issues ~50 of them per occurrence at VPL = 1 and can be
// issue-bound) at the same bytes in flight (kStage / VPL rows of VPL vectors per thread).
// PLAIN = SUM pooling over identity occurrence rows (no CSR indirection, no MEAN divisor): compiled out.
// defer_short (the fused backward): the runs of at most kApplyRun occurrences are summed by runs_apply_kernel, which
// reads their gradient rows itself; this kernel skips their units, so a piece without any other unit costs its item
// loads and its meta stores only.
// T: the gradient row element (float; __nv_bfloat16 for bf16 parts: each lane stages its 4 elements, 8 bytes, in the
// first half of its 16-byte slot and widens them to fp32 when it reads the slot back).
template <typename T, int G, int VPL, bool PLAIN, bool AHEAD>
__device__ __forceinline__ void seg_reduce(const SegArgs& sa, const PeerOut& po, int defer_short) {
  __shared__ int64_t s_start[kMaxPeers + 1];
  __shared__ char* s_base[kMaxPeers];
  extern __shared__ float4 stage_raw[];        // [kStage][kThreads]: [slot][thread], conflict-free 16-byte accesses
  float4 (*stage)[kThreads] = reinterpret_cast<float4 (*)[kThreads]>(stage_raw);
  peer_starts(po, s_start, s_base);
  const int n_parts = po.n;
  constexpr int EPL = 32 / G;          // elements of a piece per lane
  constexpr int RPI = 32 / G;          // pieces per warp iteration
  constexpr int RS = kStage / VPL;     // gradient rows requested per stage
  const BwdArgs& a = sa.b;
  const int gl = Group<G>::gl(), grp = (threadIdx.x & 31) / G;
  const uint32_t gmask = Group<G>::mask();
  const int c = gl * 4;
  const int D = a.td.dim;
  bool in[VPL];
#pragma unroll
  for (int v = 0; v < VPL; ++v) in[v] = c + v * G * 4 < D;
  const int64_t M = a.n;
  const GradSrc gs = make_grad_src<T>(a, c);
  const uint32_t* __restrict__ run_start = a.run_start;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * RPI;
  for (int64_t p0 = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * RPI; p0 < sa.n_pieces; p0 += wstride) {
    const int64_t p = p0 + grp;
    if (p >= sa.n_pieces) continue;  // whole groups leave together: the shuffles below use the group mask only
    const int64_t base = (sa.piece0 + p) * kPiece;
    // ---- lane-parallel loads: the piece's sort keys and positions, the run index in front of the piece ----
    uint32_t pm0[EPL], sk[EPL];
    load_items<G>(a.sorted, base, M, sk, pm0);
    // AHEAD: the positions of the next two pieces too (a group may stream up to 63 occurrences past its piece), so the
    // continuation never waits for a dependent position load in front of its gradient-row request
    uint32_t pm1[AHEAD ? EPL : 1], pm2[AHEAD ? EPL : 1];
    if (AHEAD) {
      uint32_t skx[EPL];
      load_items<G>(a.sorted, base + kPiece, M, skx, reinterpret_cast<uint32_t (&)[EPL]>(pm1));
      load_items<G>(a.sorted, base + 2 * kPiece, M, skx, reinterpret_cast<uint32_t (&)[EPL]>(pm2));
    }
    uint32_t j0 = sa.piece_run_base[p];
    uint32_t sk_prev = __shfl_up_sync(gmask, sk[EPL - 1], 1, G);
    if (gl == 0) sk_prev = base > 0 ? a.sorted[base - 1].x : ~sk[0];
    uint32_t hb = 0;
#pragma unroll
    for (int q = 0; q < EPL; ++q) {
      const int64_t i = base + gl * EPL + q;
      const uint32_t before = q == 0 ? sk_prev : sk[q - 1];
      if (i < M && (i == 0 || sk[q] != before)) hb |= 1u << q;
    }
    uint32_t H = __reduce_or_sync(gmask, hb << (gl * EPL));  // run heads inside the piece
    // a range that starts inside the piece (parts call): the heads in front of it are another table's runs
    const bool lead_ok = base >= a.lo;
    if (!lead_ok) {
      const uint32_t foreign = (1u << (uint32_t)(a.lo - base)) - 1u;  // a.lo - base < 32: the range's first piece
      j0 += __popc(H & foreign);
      H &= ~foreign;
    }
    const int nheads = __popc(H);
    const int nvalid = (int)min((int64_t)kPiece, M - base);
    // run boundaries around the piece (three independent loads)
    const uint32_t rs_prev = j0 > 0 ? run_start[j0 - 1] : 0u;       // start of the run covering the piece start
    const uint32_t rs_0 = run_start[j0];                            // first head at / after the piece start
    const uint32_t rs_end = run_start[j0 + nheads];                 // end of the last run that starts in the piece
    // ---- units of this piece ----
    const int e_first = H ? __ffs(H) - 1 : nvalid;                  // leading occurrences belong to run j0 - 1
    uint32_t S = H;                                                  // unit starts
    int lead_o = -1;                                                 // start of the leading long-run block, if any
    uint32_t lead_k = 0, lead_nb = 0;
    if (lead_ok && e_first > 0 && rs_0 - rs_prev > (uint32_t)kShortRun) {
      const uint32_t into = (uint32_t)base - rs_prev;                // occurrences of that run in front of the piece
      const int o = (int)((kPiece - (into & (kPiece - 1))) & (kPiece - 1));
      if (o < e_first) {
        lead_o = o;
        lead_k = (into + o) / kPiece;
        lead_nb = (rs_0 - rs_prev + kPiece - 1) / kPiece;
        S |= 1u << o;
      }
    }
    const int e_last = nheads ? 31 - __clz(H) : -1;
    const uint32_t len_last = nheads ? rs_end - ((uint32_t)base + e_last) : 0u;
    const bool last_long = len_last > (uint32_t)kShortRun;
    int e_stop;  // end of the stream (exclusive), relative to the piece start; may exceed 32
    if (nheads) e_stop = last_long ? e_last + kPiece : (int)(rs_end - (uint32_t)base);
    else e_stop = lead_o >= 0 ? min(lead_o + kPiece, (int)(rs_0 - (uint32_t)base)) : 0;
    // slot bookkeeping: both slots of the piece are (in)validated by their owner, every call
    if (gl == 0) {
      SegMeta m0, m1;
      m0.run = j0 - 1; m0.blk = lead_k; m0.nblk = lead_nb; m0.valid = lead_o >= 0 ? 1u : 0u;
      m1.run = j0 + nheads - 1; m1.blk = 0; m1.nblk = (len_last + kPiece - 1) / kPiece; m1.valid = last_long ? 1u : 0u;
      *reinterpret_cast<uint4*>(sa.meta + 2 * p) = *reinterpret_cast<uint4*>(&m0);
      *reinterpret_cast<uint4*>(sa.meta + 2 * p + 1) = *reinterpret_cast<uint4*>(&m1);
    }
    // deferred units: SK = their elements inside the piece; the last run's continuation past the piece is deferred
    // with it, which ends the stream at that run's head
    uint32_t SK = 0;
    if (defer_short) {
      for (uint32_t rem = H; rem;) {
        const int h = __ffs(rem) - 1;
        rem &= rem - 1;
        const uint32_t end = rem ? (uint32_t)(__ffs(rem) - 1) : rs_end - (uint32_t)base;  // relative, exclusive
        if (end - (uint32_t)h <= (uint32_t)kApplyRun) {
          SK |= end >= (uint32_t)kPiece ? ~0u << h : ((1u << end) - 1u) & (~0u << h);
          if (end > (uint32_t)kPiece) e_stop = h;
        }
      }
    }
    const uint32_t SU = S & ~SK;  // starts of the units summed here
    if (SU == 0) continue;
    const int e_begin = __ffs(SU) - 1;

    float4 acc[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e0 = e_begin & ~(RS - 1); e0 < e_stop; e0 += RS) {
      if (e0 + RS <= kPiece && ((SK >> e0) & ((1u << RS) - 1u)) == ((1u << RS) - 1u)) continue;  // all deferred
      // ---- request: up to RS gradient rows, this lane's 16-byte slices of each ----
      // (the 4-element bodies are NOT unrolled 4x more: the kernel was instruction-fetch bound when they were)
#pragma unroll 1
      for (int b4 = 0; b4 < RS; b4 += 4) {
        const int eb = e0 + b4;
        if (eb >= e_stop) break;
        uint32_t m[4];
        if (eb < kPiece) {
          fetch4<G>(pm0, eb, m);
        } else if (AHEAD) {
          if (eb < 2 * kPiece) fetch4<G>(reinterpret_cast<const uint32_t (&)[EPL]>(pm1), eb - kPiece, m);
          else fetch4<G>(reinterpret_cast<const uint32_t (&)[EPL]>(pm2), eb - 2 * kPiece, m);
        } else {  // continuation past the piece: the positions straight from memory (same address in every lane)
#pragma unroll
          for (int u = 0; u < 4; ++u) m[u] = base + eb + u < M ? a.sorted[base + eb + u].y : 0u;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int e = eb + u;
          if (e >= e_begin && e < e_stop && !(e < kPiece && ((SK >> e) & 1u))) {
            const uint32_t r = (!PLAIN && gs.occ_row) ? gs.occ_row[m[u]] : m[u];
            const T* src = (!PLAIN && gs.occ_src) ? reinterpret_cast<const T*>(gs.occ_src[m[u]]) + c
                                                  : reinterpret_cast<const T*>(gs.base) + (size_t)r * gs.stride;
#pragma unroll
            for (int v = 0; v < VPL; ++v)
              if (in[v]) cp_async_row4(&stage[(b4 + u) * VPL + v][threadIdx.x], src + v * G * 4);
          }
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      // ---- consume in occurrence order ----
#pragma unroll 1
      for (int b4 = 0; b4 < RS; b4 += 4) {
        const int eb = e0 + b4;
        if (eb >= e_stop) break;
        // unit starts at eb + u, and at eb + u + 1 (=> eb + u ends a unit); no starts past the piece
        const uint32_t st4 = eb < kPiece ? (S >> eb) & 0xFu : 0u;
        const uint32_t nx4 = eb + 1 < kPiece ? (S >> (eb + 1)) & 0xFu : 0u;
        float fn[4] = {1.f, 1.f, 1.f, 1.f};
        if (!PLAIN && gs.mean) {  // MEAN pooling: the divisor of each row (positions fetched again: rare path)
          uint32_t m[4];
          if (eb < kPiece) {
            fetch4<G>(pm0, eb, m);
          } else {
#pragma unroll
            for (int u = 0; u < 4; ++u) m[u] = base + eb + u < M ? a.sorted[base + eb + u].y : 0u;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const uint32_t r = gs.occ_row ? gs.occ_row[m[u]] : m[u];
            fn[u] = gs.occ_div ? gs.occ_div[m[u]] : (float)(gs.row_offsets[r + 1] - gs.row_offsets[r]);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int e = eb + u;
          if (e < e_begin || e >= e_stop || (e < kPiece && ((SK >> e) & 1u))) continue;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in[v]) x = stage_row4<T>(&stage[(b4 + u) * VPL + v][threadIdx.x]);
            if (!PLAIN && gs.mean && fn[u] != 0.f) {
              x.x = __fdiv_rn(x.x, fn[u]); x.y = __fdiv_rn(x.y, fn[u]); x.z = __fdiv_rn(x.z, fn[u]); x.w = __fdiv_rn(x.w, fn[u]);
            }
            if ((st4 >> u) & 1u) acc[v] = x; else add4(acc[v], x);
          }
          if (!(e + 1 == e_stop || ((nx4 >> u) & 1u))) continue;
          // ---- a unit ends here ----
          const int hr = e < kPiece ? __popc(H & (0xFFFFFFFFu >> (31 - e))) : nheads;  // heads at or before e
          float* dst;
          if (hr == 0) dst = sa.part + (size_t)(2 * p) * D;                          // leading block of a long run
          else if (last_long && hr == nheads) dst = sa.part + (size_t)(2 * p + 1) * D;  // block 0 of a long run
          else dst = run_dst(a.ugrad, n_parts, s_start, s_base, (int64_t)j0 + hr - 1, D);  // a short run
#pragma unroll
          for (int v = 0; v < VPL; ++v)
            if (in[v]) *reinterpret_cast<float4*>(dst + c + v * G * 4) = acc[v];
        }
      }
    }
  }
}

template <int G, int VPL, bool PLAIN, bool AHEAD>
__global__ void __launch_bounds__(kThreads, 3)
seg_reduce_kernel(SegArgs sa, const PeerOut po, int defer_short) {
  seg_reduce<float, G, VPL, PLAIN, AHEAD>(sa, po, defer_short);
}

// bf16 gradient rows of a parts call (always through the occurrence map, so there is no PLAIN form)
template <int G, int VPL, bool AHEAD>
__global__ void __launch_bounds__(kThreads, 3)
bf16_seg_reduce_kernel(SegArgs sa, const PeerOut po, int defer_short) {
  seg_reduce<__nv_bfloat16, G, VPL, false, AHEAD>(sa, po, defer_short);
}

// One level of the fixed tree over the block index of the long runs: the slot of block k, k a multiple of
// kTreeFan * stride, receives (in place) the sum of the slots of blocks k, k + stride, ..., k + (kTreeFan - 1) * stride.
// A WARP owns a node: its 32 / G lane groups each sum a contiguous share (kTreeFan * G / 32 members, in block
// order, from 0, 16 requests in flight per lane), then the group sums are added in group order through shuffles —
// the association is a function of (run length, row width, tree depth) only, so results are run-to-run bit-stable.  (One lane group
// per node means 8 dependent stages of 16 loads: the hottest FIDs' chains become the kernel.)
template <int G>
__global__ void __launch_bounds__(kThreads)
tree_level_kernel(float* __restrict__ part, const SegMeta* __restrict__ meta, int64_t n_slots, uint32_t stride, int D) {
  extern __shared__ float4 stage_raw[];  // [kStage][kThreads]
  float4 (*stage)[kThreads] = reinterpret_cast<float4 (*)[kThreads]>(stage_raw);
  constexpr int NG = 32 / G;                 // lane groups per warp = slots scanned per warp iteration
  constexpr int PER = kTreeFan / NG;         // members per lane group
  static_assert(PER % 16 == 0 || PER == kTreeFan, "members per group must fill whole stages");
  const int gl = Group<G>::gl(), c = gl * 4, grp = (threadIdx.x & 31) / G;
  const bool in = c < D;
  const int lane = threadIdx.x & 31;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * 32;
  for (int64_t q0 = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * 32; q0 < n_slots; q0 += wstride) {
    // every lane inspects one slot; node heads are then processed one at a time by the whole warp
    SegMeta mine;
    mine.run = mine.blk = mine.nblk = mine.valid = 0;
    if (q0 + lane < n_slots) mine = meta[q0 + lane];
    const bool head = mine.valid && mine.blk % (kTreeFan * stride) == 0 && (uint64_t)mine.blk + stride < mine.nblk;
    uint32_t heads = __ballot_sync(0xFFFFFFFFu, head);
    while (heads) {
      const int src = __ffs(heads) - 1;       // the lane that saw this head
      heads &= heads - 1;
      const uint32_t blk = __shfl_sync(0xFFFFFFFFu, mine.blk, src);
      const uint32_t nblk = __shfl_sync(0xFFFFFFFFu, mine.nblk, src);
      const int64_t q = q0 + src;
      const int64_t piece = q >> 1;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      // member i of the node lives in slot q (i = 0) or 2 * (piece + i * stride): block k + i*stride starts i*stride pieces on
      for (int i0 = grp * PER; i0 < (grp + 1) * PER; i0 += 16) {
        if ((uint64_t)blk + (uint64_t)i0 * stride >= nblk) break;
#pragma unroll
        for (int u = 0; u < 16; ++u) {  // 16 UNCONDITIONAL requests (clamped to the node's own slot): all in flight together
          const int i = i0 + u;
          const bool ok = i > 0 && (uint64_t)blk + (uint64_t)i * stride < nblk;
          const size_t slot = ok ? (size_t)(2 * (piece + (int64_t)i * stride)) : (size_t)q;
          cp_async16(&stage[u][threadIdx.x], part + slot * D + (in ? c : 0));
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int u = 0; u < 16; ++u) {
          const int i = i0 + u;
          if ((uint64_t)blk + (uint64_t)i * stride < nblk) add4(acc, stage[u][threadIdx.x]);
        }
      }
      // group sums -> group 0, in group order
      float4 tot = acc;
#pragma unroll
      for (int g = 1; g < NG; ++g) {
        float4 o;
        o.x = __shfl_sync(0xFFFFFFFFu, acc.x, g * G + gl);
        o.y = __shfl_sync(0xFFFFFFFFu, acc.y, g * G + gl);
        o.z = __shfl_sync(0xFFFFFFFFu, acc.z, g * G + gl);
        o.w = __shfl_sync(0xFFFFFFFFu, acc.w, g * G + gl);
        if ((uint64_t)blk + (uint64_t)(g * PER) * stride < nblk) add4(tot, o);
      }
      __syncwarp();  // every group has read its members (slot q among them) before the node is overwritten
      if (grp == 0 && in) *reinterpret_cast<float4*>(part + (size_t)q * D + c) = tot;
    }
  }
}

// Long runs, last step: the head slot of a long run combines what the tree left (blocks 0, top, 2 * top, ... — at most
// kFinishMax of them, in order) and stores the run's summed row to run_dst.
template <int G>
__global__ void __launch_bounds__(kThreads)
long_finish_kernel(SegArgs sa, uint32_t top, const PeerOut po) {
  __shared__ int64_t s_start[kMaxPeers + 1];
  __shared__ char* s_base[kMaxPeers];
  extern __shared__ float4 stage_raw[];  // [kStage][kThreads]
  float4 (*stage)[kThreads] = reinterpret_cast<float4 (*)[kThreads]>(stage_raw);
  peer_starts(po, s_start, s_base);
  const BwdArgs& a = sa.b;
  const int gl = Group<G>::gl(), c = gl * 4;
  const int D = a.td.dim;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t p = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; p < sa.n_pieces; p += gstride) {
    const SegMeta m = sa.meta[2 * p + 1];
    if (!m.valid) continue;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < D) acc = *reinterpret_cast<const float4*>(sa.part + (size_t)(2 * p + 1) * D + c);
    for (uint32_t k0 = top; k0 < m.nblk; k0 += 16 * top) {
#pragma unroll
      for (int u = 0; u < 16; ++u) {  // 16 requests in flight (clamped to the head slot)
        const uint64_t k = (uint64_t)k0 + (uint64_t)u * top;
        const size_t slot = k < m.nblk ? (size_t)(2 * (p + (int64_t)k)) : (size_t)(2 * p + 1);
        cp_async16(&stage[u][threadIdx.x], sa.part + slot * D + (c < D ? c : 0));
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
      for (int u = 0; u < 16; ++u)
        if ((uint64_t)k0 + (uint64_t)u * top < m.nblk) add4(acc, stage[u][threadIdx.x]);
    }
    if (c < D) *reinterpret_cast<float4*>(run_dst(a.ugrad, po.n, s_start, s_base, m.run, D) + c) = acc;
  }
}

// Apply: group per run.  A run of at most kApplyRun occurrences is summed here: its positions, then its gradient
// rows, kApplyStage at a time with cp.async into per-thread shared-memory slots (as seg_reduce_kernel does), added
// in occurrence order from the first row with seg_reduce_kernel's arithmetic, so the bits are those of its unit.
// The row's w / state loads are issued first and overlap them.  A longer run reads ugrad[j] (long_finish_kernel).
// Summing here saves those runs' ugrad store and re-load (about 120 MB per C2 step).
// (A variant that handled two runs per group at a time needs 62 registers, which lowers occupancy.)
// The next run's row index and run bounds are read one iteration ahead.  prefetch != 0: its weight / state rows are
// also pulled into L2 meanwhile.
// T: the gradient row element, as in seg_reduce.
template <typename T, int G, int OPT>
__device__ __forceinline__ void runs_apply(const BwdArgs& a, int prefetch) {
  extern __shared__ float4 stage_raw[];  // [kApplyStage][kThreads]
  float4 (*stage)[kThreads] = reinterpret_cast<float4 (*)[kThreads]>(stage_raw);
  const int gl = Group<G>::gl();
  const int c = gl * 4;
  int64_t j_lo = 0, nr = *a.n_runs;
  if (a.run_of_sorted) {  // parts call: the runs of the sorted range [lo, n)
    j_lo = a.run_of_sorted[a.lo];
    nr = (int64_t)a.run_of_sorted[a.n - 1] + 1;
  }
  const int D = a.td.dim;
  const GradSrc gs = make_grad_src<T>(a, c);
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  int64_t j = j_lo + (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G;
  uint32_t ri_next = kEmptyRow, rs_next = 0, re_next = 0, p0_next = 0;
  if (j < nr) {
    ri_next = a.rowidx[j];
    rs_next = a.run_start[j];
    re_next = a.run_start[j + 1];
    p0_next = a.run_first_pos[j];
  }
  for (; j < nr; j += gstride) {
    const uint32_t ri = ri_next, rs = rs_next, re = re_next, p0 = p0_next;
    if (j + gstride < nr) {
      ri_next = a.rowidx[j + gstride];
      rs_next = a.run_start[j + gstride];
      re_next = a.run_start[j + gstride + 1];
      p0_next = a.run_first_pos[j + gstride];
      if (prefetch && OPT >= 0 && ri_next != kEmptyRow && !(ri_next & kFreshBit) && c < D) {
        const uint32_t row = ri_next & ~kFreshBit;
        prefetch_l2(a.td.emb + (size_t)row * a.td.emb_stride + c);
        if (OPT != MONO_OPT_SGD) {
          const float* s_row = a.td.state + (size_t)row * a.td.state_stride;
          prefetch_l2(s_row + c);
          if (OPT == MONO_OPT_FTRL || OPT == MONO_OPT_ADAM) prefetch_l2(s_row + D + c);
        }
      }
    }
    if (ri == kEmptyRow) continue;
    const RowPre pre = bwd_prefetch<G, OPT>(a, ri, c);
    float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (re - rs > (uint32_t)kApplyRun) {
      if (c < D) g4 = __ldcs(reinterpret_cast<const float4*>(a.ugrad + (size_t)j * D + c));
    } else {
      for (uint32_t k0 = rs; k0 < re; k0 += kApplyStage) {
        const int n = (int)min(re - k0, (uint32_t)kApplyStage);
        uint32_t m[kApplyStage];
#pragma unroll
        for (int u = 0; u < kApplyStage; ++u)  // the first position is p0: a one-occurrence run (most runs) has no hop
          m[u] = u >= n ? 0u : (u == 0 && k0 == rs) ? p0 : a.sorted[k0 + u].y;
#pragma unroll
        for (int u = 0; u < kApplyStage; ++u)
          if (u < n && c < D) cp_async_row4(&stage[u][threadIdx.x], occ_grad_src<T>(gs, m[u], c));
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int u = 0; u < kApplyStage; ++u) {
          if (u >= n) break;
          float4 x = stage_row4<T>(&stage[u][threadIdx.x]);
          if (gs.mean) {
            const float fn = occ_grad_div(gs, m[u]);
            if (fn != 0.f) {
              x.x = __fdiv_rn(x.x, fn); x.y = __fdiv_rn(x.y, fn); x.z = __fdiv_rn(x.z, fn); x.w = __fdiv_rn(x.w, fn);
            }
          }
          if (k0 == rs && u == 0) g4 = x; else add4(g4, x);
        }
      }
    }
    bwd_apply<G, OPT>(a, (uint32_t)j, ri, g4, c, pre);
  }
}

template <int G, int OPT>
__global__ void __launch_bounds__(kThreads) runs_apply_kernel(BwdArgs a, int prefetch) {
  runs_apply<float, G, OPT>(a, prefetch);
}

template <int G, int OPT>
__global__ void __launch_bounds__(kThreads) bf16_runs_apply_kernel(BwdArgs a, int prefetch) {
  runs_apply<__nv_bfloat16, G, OPT>(a, prefetch);
}

// run j of the sorted offsets -> destination row: out_rows + (sorted key << shift)
template <int G>
__global__ void __launch_bounds__(kThreads) runs_emit_kernel(BwdArgs a, int shift, float* __restrict__ out_rows) {
  const int gl = Group<G>::gl(), c = gl * 4;
  const int64_t nr = *a.n_runs;
  const int D = a.td.dim;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t j = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; j < nr; j += gstride) {
    if (c >= D) continue;
    const float4 g = __ldcs(reinterpret_cast<const float4*>(a.ugrad + (size_t)j * D + c));
    *reinterpret_cast<float4*>(out_rows + ((size_t)a.sorted[a.run_start[j]].x << shift) + c) = g;
  }
}


// Claim set entry (16 B, viewed as Entry): key = FID, ts = epoch of the call that claimed it (any other value =
// empty: the set is never cleared, engine.h ClaimSet), row = the FID's resolved table row (RESOLVE) or 0.
// Claimed entries never change during the kernel, so every read may be served by L1 (plain ld.global): the hot
// FIDs of a Zipf batch (8 % of the occurrences hit ONE slot) are answered per SM instead of serialising on one
// L2 slice.  A stale L1 line can only show "empty" for a slot that has been claimed meanwhile; the CAS then
// fails and returns the true entry.
// RESOLVE (single-GPU fused backward): the thread that wins a slot is the only one for its FID, so it also
// resolves the FID in the table right away — lane-level probe, expiry-timestamp bump
// (ref: entry.SetTimestamp(update_time), cuckoo_embedding_hash_table.cc:243), row index parked in the set
// entry; absent FIDs are queued (set slot) for claim_miss_kernel.  No separate resolve pass over the uniques.
// One table of a parts call: its occurrences are [occ_begin, occ_end) of the table-major concatenation, its FIDs
// are claimed in the set's slots [slot_base, slot_base + slots)
struct CallTable {
  int64_t occ_begin, occ_end;
  uint32_t slot_base, slots;
  int32_t table, pad;
};
// Linear scans over the call's tables: a multi-table merges slots of one config, so K is a handful (2-5 in Monolith
// models) and the regions array stays in L1.
__device__ __forceinline__ int call_table_of_occ(const CallTable* __restrict__ rg, int n, int64_t i) {
  int r = 0;
  while (r + 1 < n && i >= rg[r].occ_end) ++r;
  return r;
}
__device__ __forceinline__ int call_table_of_slot(const CallTable* __restrict__ rg, int n, uint32_t slot) {
  int r = 0;
  while (r + 1 < n && slot >= rg[r + 1].slot_base) ++r;
  return r;
}

struct ClaimResolve {
  const TableDev* t = nullptr;
  uint32_t update_ts = 0;
  uint32_t* miss_ctr = nullptr;
  uint32_t* miss_slots = nullptr;
  // parts call: occurrence i belongs to the call table whose [occ_begin, occ_end) holds it; it claims in that table's
  // region of the set and resolves in tables[table]; null: one region per owner (key mod N), table t
  const CallTable* regions = nullptr;
  int n_regions = 0;
};

template <bool RESOLVE, bool DUAL = false>
__global__ void __launch_bounds__(kThreads)
fid_claim_kernel(const int64_t* __restrict__ fids, int64_t n, Entry* set, uint32_t R, int N, uint32_t epoch,
                 uint32_t* __restrict__ slot_of, uint32_t* __restrict__ owner_cnt /* [N], [256] = overflow */,
                 ClaimResolve cr, int prefetch) {
  __shared__ uint32_t cnt[256];
  for (int d = threadIdx.x; d < 256; d += blockDim.x) cnt[d] = 0;
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  // the chain per occurrence is FID -> set entry (-> CAS -> table bucket for a winner), one HBM latency per dependent
  // round trip: the NEXT occurrence's FID is requested one iteration ahead, which takes it off the chain
  // ... and so are (prefetch != 0) its scratch-set slot and, for RESOLVE, its first table bucket: both are pulled into
  // L2 while this iteration's chain runs, so the next iteration's two dependent reads are L2 hits.
  int64_t key_next = i < n ? __ldg(fids + i) : 0;
  const Entry* pf_buckets = nullptr;
  uint32_t pf_nb = 0;
  if (RESOLVE && prefetch) {
    pf_buckets = cr.t->buckets;
    pf_nb = cr.t->num_buckets;
  }
  for (; i < n; i += stride) {
    const int64_t key = key_next;
    if (i + stride < n) {
      key_next = __ldg(fids + i + stride);
      if (prefetch && !cr.regions) {
        const uint32_t o_n = N == 1 ? 0u : (uint32_t)((uint64_t)key_next % (uint64_t)N);
        prefetch_l2(set + o_n * R + __umulhi((uint32_t)(mix64((uint64_t)key_next) >> 24), R));
        if (RESOLVE) {
          uint32_t b1, b2;
          bucket_pair(key_next, pf_nb, b1, b2);
          prefetch_l2(pf_buckets + (size_t)b1 * kBucketSlots);
        }
      }
    }
    const uint32_t owner = N == 1 ? 0u : (uint32_t)((uint64_t)key % (uint64_t)N);
    uint32_t base = owner * R;
    const TableDev* tk = cr.t;
    if (cr.regions) {
      const CallTable& rg = cr.regions[call_table_of_occ(cr.regions, cr.n_regions, i)];
      base = rg.slot_base;
      R = rg.slots;
      tk = cr.t + rg.table;
    }
    uint32_t idx = __umulhi((uint32_t)(mix64((uint64_t)key) >> 24), R);
    uint32_t found = 0xFFFFFFFFu;
    bool won = false;
    for (uint32_t probes = 0; probes < R; ++probes) {
      Entry* p = set + base + idx;
      Entry e = ld_entry(p);  // L1-cacheable
      while (e.ts != epoch) {  // empty as far as we can see: claim it (CAS against what we saw)
        Entry ne;
        ne.key = key;
        ne.row = kEmptyRow;
        ne.ts = epoch;
        const Entry old = cas_entry_old(p, e, ne);
        if (old.key == e.key && old.row == e.row && old.ts == e.ts) {
          won = true;
          e = ne;
        } else {
          e = old;  // somebody else changed it: the true entry (claimed this epoch, or a different stale one)
        }
      }
      if (e.key == key) {
        found = base + idx;
        break;
      }
      idx = idx + 1 == R ? 0 : idx + 1;
    }
    if (found == 0xFFFFFFFFu) {  // region full (owner skew): the host retries with larger regions
      owner_cnt[256] = 1;
      found = base;
      won = false;
    }
    slot_of[i] = found;
    if (won) {
      atomicAdd(&cnt[owner], 1u);
      if (RESOLVE) {
        Entry* slot = nullptr;
        const uint32_t row = probe_lane_slot<DUAL>(tk, key, &slot);
        if (row != kEmptyRow) {
          slot->ts = cr.update_ts;
          set[found].row = row;
        } else {
          cr.miss_slots[atomicAdd(cr.miss_ctr, 1u)] = found;
        }
      }
    }
  }
  __syncthreads();
  for (int d = threadIdx.x; d < N; d += blockDim.x)
    if (cnt[d]) atomicAdd(owner_cnt + d, cnt[d]);
}

// FIDs the claim found absent from the table (each exactly once): take a row (free list first, then the bump
// allocator), publish {fid, row, ts} with the lock-free cuckoo insert and park row | fresh in the set entry.
__global__ void __launch_bounds__(kThreads)
claim_miss_kernel(const TableDev* __restrict__ tables, Entry* set, const uint32_t* __restrict__ miss_ctr,
                  const uint32_t* __restrict__ miss_slots, uint32_t update_ts,
                  const CallTable* __restrict__ regions /* parts call: the slot's table; null: tables[0] */, int n_regions) {
  const int64_t n = (int64_t)*miss_ctr;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t sl = miss_slots[q];
    const TableDev* t = regions ? tables + regions[call_table_of_slot(regions, n_regions, sl)].table : tables;
    // admission filter: the backward hands every distinct FID once per step (count 1), as the reference's
    // deduplicated optimize does; a FID below its slot's threshold gets no row (its run is skipped by the apply)
    if (should_be_filtered(t, ld_entry_cg(set + sl).key, 1u)) continue;
    const uint32_t ticket = atomicAdd(t->ctrs + kCtrMiss, 1u);
    const uint32_t fc = t->ctrs[kCtrFree];  // stable during this kernel (finalize updates it)
    const uint32_t row = ticket < fc ? t->free_list[fc - 1 - ticket] : t->ctrs[kCtrBump] + (ticket - fc);
    if (row >= t->row_cap) {
      atomicOr(t->ctrs + kCtrError, 2u);
      continue;  // the set entry keeps kEmptyRow: the run is skipped by the apply pass
    }
    Entry e;
    e.key = ld_entry_cg(set + sl).key;
    e.row = row;
    e.ts = update_ts;
    cuckoo_insert(t, e);
    set[sl].row = row | kFreshBit;
  }
}


// ==========================================================================================
// host side
// ==========================================================================================
static const PeerOut no_peer = {};  // n == 0: the reduce writes the local ugrad buffer

// Optional parts of the pipeline scratch (scratch_plan)
enum : unsigned {
  kPartK0 = 1, kPartRowIdx = 2, kPartMiss = 4, kPartOcc = 8, kPartRunOfSorted = 16, kPartUGrad = 32,
  kPartOccMap = 64  // parts call: concatenated FIDs, gradient row and MEAN divisor of every occurrence
};

// Layout of the pipeline scratch for M occurrences of dim D sorted on `bits` key bits: one 256-byte aligned region
// per part, the optional ones only when `parts` asks for them.  base == nullptr only sizes it (.bytes).
static BwdScratch scratch_plan(int64_t M, int D, int bits, unsigned parts, char* base) {
  size_t off = 0;
  auto take = [&](size_t bytes, unsigned part = 0) -> void* {
    if (part && !(parts & part)) return nullptr;
    const uintptr_t p = reinterpret_cast<uintptr_t>(base) + off;
    off = (off + bytes + 255) & ~(size_t)255;
    return reinterpret_cast<void*>(p);
  };
  const size_t m4 = 4 * (size_t)M;
  BwdScratch w;
  w.n_pieces = (M + kPiece - 1) / kPiece;
  w.k0 = (uint32_t*)take(m4, kPartK0);
  w.sort.a = (uint2*)take(8 * (size_t)M);
  w.sort.b = (uint2*)take(8 * (size_t)M);
  w.sort.cnt = (uint32_t*)take(4 * (size_t)kRadixBins * radix_blocks(M));
  w.ctr = (uint32_t*)take(kCtrBytes);
  w.sort.dtot = (uint32_t*)take(4 * (size_t)kRadixBins * sort_passes(bits));  // right behind the counters
  w.sort.n_runs = w.ctr + kCtrRuns;
  w.sort.blk_runs = (uint32_t*)take(4 * (size_t)run_blocks(M));
  w.sort.run_start = (uint32_t*)take(m4 + 4);
  w.sort.run_first_pos = (uint32_t*)take(m4);
  w.sort.rowidx = (uint32_t*)take(m4, kPartRowIdx);
  w.miss = (uint32_t*)take(m4, kPartMiss);
  w.sort.run_of_sorted = (uint32_t*)take(m4, kPartRunOfSorted);
  w.occ = (uint32_t*)take(m4, kPartOcc);
  w.sort.piece_run_base = (uint32_t*)take(4 * (size_t)w.n_pieces);
  w.part = (float*)take(sizeof(float) * 2 * (size_t)w.n_pieces * D);
  w.meta = (SegMeta*)take(sizeof(SegMeta) * 2 * (size_t)w.n_pieces);
  w.ugrad = (float*)take(sizeof(float) * (size_t)M * D, kPartUGrad);
  w.fids = (int64_t*)take(8 * (size_t)M, kPartOccMap);
  w.occ_src = (const float**)take(sizeof(float*) * (size_t)M, kPartOccMap);
  w.occ_div = (float*)take(m4, kPartOccMap);
  w.sorted = nullptr;
  w.bytes = off;
  return w;
}

// The reduce reads and writes gradient rows as 4-element vectors (16 bytes; 8 of bf16 rows, elem_bytes = 2), one
// per lane of a group of at most 32 lanes.
static void check_grad_rows(const char* who, int D, const float* pooled_grad = nullptr, int64_t grad_stride = 0,
                            int grad_col = 0, const float* out_rows = nullptr, int elem_bytes = 4) {
  if ((D & 3) || D > 128) throw ArgError(std::string(who) + " needs dim % 4 == 0 and dim <= 128");
  const uintptr_t amask = 4 * (uintptr_t)elem_bytes - 1;
  if ((grad_stride & 3) || (grad_col & 3) || (reinterpret_cast<uintptr_t>(pooled_grad) & amask) ||
      (reinterpret_cast<uintptr_t>(out_rows) & amask))
    throw ArgError(std::string(who) + " needs " + std::to_string(4 * elem_bytes) + "-byte aligned rows");
}

// One table's share of a parts call: the sorted range [lo, hi) and whether any of its parts pools by MEAN
struct SortedRange {
  int64_t lo, hi;
  bool mean;
};

// Arguments of a reduce over the plan's sorted list: the gradient rows of pooled_grad (row_offsets != null: CSR
// rows, occurrence -> row mapped into w.occ first), per-run sums to ugrad (or the peer windows of the launch).
// range != null (parts call): only the sorted range of one table, gradient rows from the plan's occurrence map.
static SegArgs seg_args(const BwdScratch& w, int64_t M, int D, const float* pooled_grad, int64_t grad_stride,
                        int grad_col, const int32_t* row_offsets, int64_t n_rows, int pooling, float* ugrad,
                        cudaStream_t s, const SortedRange* range = nullptr) {
  SegArgs sa;
  std::memset(&sa, 0, sizeof(sa));
  BwdArgs& a = sa.b;
  a.td.dim = D;
  a.sorted = w.sorted;
  a.n = M;
  a.n_runs = w.sort.n_runs;
  a.run_start = w.sort.run_start;
  a.run_first_pos = w.sort.run_first_pos;
  a.row_offsets = row_offsets;
  a.pooling = pooling;
  a.pooled_grad = pooled_grad;
  a.grad_stride = grad_stride;
  a.grad_col = grad_col;
  a.ugrad = ugrad;
  sa.piece_run_base = w.sort.piece_run_base;
  sa.part = w.part;
  sa.meta = w.meta;
  sa.n_pieces = w.n_pieces;
  if (range) {
    a.n = range->hi;
    a.lo = range->lo;
    a.pooling = range->mean ? MONO_POOL_MEAN : MONO_POOL_SUM;
    a.occ_src = w.occ_src;
    a.occ_div = w.occ_div;
    a.run_of_sorted = w.sort.run_of_sorted;
    sa.piece0 = range->lo / kPiece;
    sa.n_pieces = (range->hi + kPiece - 1) / kPiece - sa.piece0;
    sa.piece_run_base += sa.piece0;
  }
  if (row_offsets) {
    occ_row_kernel<<<resident_grid(occ_row_kernel, n_rows, kThreads), kThreads, 0, s>>>(row_offsets, n_rows, w.occ);
    MONO_CHECK_LAUNCH();
    a.occ_row = w.occ;
  }
  return sa;
}

constexpr size_t kStageBytes = sizeof(float4) * kStage * kThreads;
// BF16: bf16_seg_reduce_kernel<GL, VPL, AHEAD> (PLAIN is then false)
template <int GL, int VPL, bool PLAIN, bool AHEAD, bool BF16>
static void launch_seg2(const SegArgs& sa, const PeerOut& po, bool defer_short, cudaStream_t s) {
  void (*const kern)(SegArgs, const PeerOut, int) =
      BF16 ? bf16_seg_reduce_kernel<GL, VPL, AHEAD> : seg_reduce_kernel<GL, VPL, PLAIN, AHEAD>;
  static bool attr_set = false;
  if (!attr_set) {
    MONO_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStageBytes));
    attr_set = true;
  }
  kern<<<resident_grid(kern, sa.n_pieces, (kThreads / 32) * (32 / GL), kThreads, kStageBytes), kThreads, kStageBytes,
         s>>>(sa, po, defer_short ? 1 : 0);
  MONO_CHECK_LAUNCH();
}
template <int GL, int VPL, bool PLAIN, bool BF16 = false>
static void launch_seg(const SegArgs& sa, const PeerOut& po, bool defer_short, cudaStream_t s) {
  if (knob(KNOB_SEG_AHEAD)) launch_seg2<GL, VPL, PLAIN, true, BF16>(sa, po, defer_short, s);
  else launch_seg2<GL, VPL, PLAIN, false, BF16>(sa, po, defer_short, s);
}

// per-run gradient sums -> run_dst (a.ugrad, or the owners' peer windows).  defer_short: runs_apply_kernel follows
// and sums the runs of at most kApplyRun occurrences itself, so only the longer runs' sums are stored.
// bf16: the gradient rows are bf16 (parts call); the tree and finish kernels add fp32 partials either way.
static void launch_reduce(const SegArgs& sa, int G, const PeerOut& po, bool defer_short, cudaStream_t s,
                          bool bf16 = false) {
  const int64_t nr = sa.n_pieces;
  if (nr <= 0) return;
  // the tree depth follows the range's occurrence count (the whole list but for one table of a parts call)
  const int64_t np = (sa.b.n - sa.b.lo + kPiece - 1) / kPiece;
  int levels = 0;
  uint64_t top = 1;
  while ((uint64_t)np > top * kFinishMax) {  // the final pass adds up to kFinishMax nodes per run, 16 loads in flight
    top *= kTreeFan;
    ++levels;
  }
  const int D = sa.b.td.dim;
  const bool plain = sa.b.occ_row == nullptr && sa.b.occ_src == nullptr &&
                     !(sa.b.pooling == MONO_POOL_MEAN && sa.b.row_offsets != nullptr);
  const bool two = knob(KNOB_SEG_VPL) == 2;
#define SEG_G(GG)                                                                                                   \
  do {                                                                                                              \
    static bool attr_set = false;                                                                                   \
    if (!attr_set) {                                                                                                \
      MONO_CUDA(cudaFuncSetAttribute(tree_level_kernel<GG>, cudaFuncAttributeMaxDynamicSharedMemorySize,            \
                                     (int)kStageBytes));                                                            \
      MONO_CUDA(cudaFuncSetAttribute(long_finish_kernel<GG>, cudaFuncAttributeMaxDynamicSharedMemorySize,           \
                                     (int)kStageBytes));                                                            \
      attr_set = true;                                                                                              \
    }                                                                                                               \
    if (two && GG >= 8) {                                                                                           \
      if (bf16) launch_seg<(GG >= 8 ? GG / 2 : GG), (GG >= 8 ? 2 : 1), false, true>(sa, po, defer_short, s);        \
      else if (plain) launch_seg<(GG >= 8 ? GG / 2 : GG), (GG >= 8 ? 2 : 1), true>(sa, po, defer_short, s);         \
      else launch_seg<(GG >= 8 ? GG / 2 : GG), (GG >= 8 ? 2 : 1), false>(sa, po, defer_short, s);                   \
    } else {                                                                                                        \
      if (bf16) launch_seg<GG, 1, false, true>(sa, po, defer_short, s);                                             \
      else if (plain) launch_seg<GG, 1, true>(sa, po, defer_short, s);                                              \
      else launch_seg<GG, 1, false>(sa, po, defer_short, s);                                                        \
    }                                                                                                               \
    uint32_t stride = 1;                                                                                            \
    for (int l = 0; l < levels; ++l, stride *= kTreeFan) {                                                          \
      tree_level_kernel<GG><<<resident_grid(tree_level_kernel<GG>, 2 * nr, kThreads, kThreads, kStageBytes),        \
                              kThreads, kStageBytes, s>>>(sa.part, sa.meta, 2 * nr, stride, D);                     \
      MONO_CHECK_LAUNCH();                                                                                          \
    }                                                                                                               \
    long_finish_kernel<GG><<<resident_grid(long_finish_kernel<GG>, nr, kThreads / GG, kThreads, kStageBytes),      \
                             kThreads, kStageBytes, s>>>(sa, (uint32_t)top, po);                                    \
    MONO_CHECK_LAUNCH();                                                                                            \
  } while (0)
  switch (G) {
    case 4: SEG_G(4); break;
    case 8: SEG_G(8); break;
    case 16: SEG_G(16); break;
    default: SEG_G(32); break;
  }
#undef SEG_G
}

static int bits_for(uint64_t cap) {
  int bits = 0;
  while (((uint64_t)1 << bits) < cap) ++bits;
  return bits;
}

// the register-resident apply exists for the four vectorised optimizers; anything else: store + generic apply_row
static int apply_opt_sel(const HostTable& ht) {
  const int opt_sel = (ht.segs.size() == 1 && ht.segs[0].opt_type <= MONO_OPT_ADAM) ? ht.segs[0].opt_type : -1;
  return opt_sel;
}

// the optimizer step of every run of the reduce's range (M: its occurrence count, sizes the grid); bf16: bf16
// gradient rows (parts call)
static void launch_apply(const BwdArgs& a, int G, int opt_sel, int64_t M, cudaStream_t s, bool bf16 = false) {
  const int pf = knob(KNOB_APPLY_PF);
  constexpr size_t smem = sizeof(float4) * kApplyStage * kThreads;
  static_assert(smem <= 48 * 1024, "runs_apply_kernel's stage fits the default dynamic shared memory limit");
#define BWD2(GG, OO)                                                                                              \
  do {                                                                                                            \
    void (*const kern)(BwdArgs, int) = bf16 ? bf16_runs_apply_kernel<GG, OO> : runs_apply_kernel<GG, OO>;         \
    kern<<<resident_grid(kern, M, kThreads / GG, kThreads, smem), kThreads, smem, s>>>(a, pf);                    \
    MONO_CHECK_LAUNCH();                                                                                          \
  } while (0)
#define BWD(GG)                                                         \
  switch (opt_sel) {                                                    \
    case MONO_OPT_SGD: BWD2(GG, MONO_OPT_SGD); break;                   \
    case MONO_OPT_ADAGRAD: BWD2(GG, MONO_OPT_ADAGRAD); break;           \
    case MONO_OPT_FTRL: BWD2(GG, MONO_OPT_FTRL); break;                 \
    case MONO_OPT_ADAM: BWD2(GG, MONO_OPT_ADAM); break;                 \
    default: BWD2(GG, -1); break;                                       \
  }
  switch (G) {
    case 4: BWD(4); break;
    case 8: BWD(8); break;
    case 16: BWD(16); break;
    default: BWD(32); break;
  }
#undef BWD2
#undef BWD
}

void run_pool_backward(mono_mtable* mt, int k, const int64_t* fids_dev, int64_t n_fids,
                       const int32_t* row_offsets, int64_t n_rows, int pooling,
                       const float* pooled_grad, int64_t grad_stride, int grad_col,
                       const float* lr_host, int64_t update_time, cudaStream_t s) {
  mt->note_insert(s);
  if (n_fids <= 0) return;
  if (n_fids > ((int64_t)1 << 30)) throw ArgError("more than 2^30 fids in one call");
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("pool_backward: SUM or MEAN");
  HostTable& ht = mt->tables[k];
  const int D = ht.dim;
  check_grad_rows("pool_backward", D, pooled_grad, grad_stride, grad_col);
  const int64_t M = n_fids;
  ensure_capacity(mt, k, (uint64_t)M, s);
  upload_tables(mt, s);
  CallSeg sg;
  sg.id_begin = 0;
  sg.id_end = M;
  sg.val_off = 0;
  sg.table = k;
  sg.lr_off = 0;
  CallBlob cb = stage_call(mt, &sg, 1, lr_host, ht.slices, s);
  const int G = pick_group(D);

  // ---- scratch ----
  const uint32_t cap = claim_set_slots(M);
  const int bits = bits_for(cap);
  const unsigned parts = kPartK0 | kPartRowIdx | kPartMiss | (row_offsets ? kPartOcc : 0u) | kPartUGrad;
  BwdScratch w = scratch_plan(M, D, bits, parts, nullptr);
  w = scratch_plan(M, D, bits, parts, (char*)mt->ws_a.get(w.bytes, s));
  uint32_t epoch = 0;
  Entry* set = (Entry*)mt->claim_set.get(sizeof(Entry) * (size_t)cap, s, &epoch);
  MONO_CUDA(cudaMemsetAsync(w.ctr, 0, kCtrBytes, s));

  // 1 claim: k0[i] = set slot of occurrence i; the winner of a slot resolves its FID in the table (row parked in
  //   the set entry, expiry timestamp bumped) or queues it as absent
  uint32_t* miss_ctr = w.ctr + kCtrMisses;
  ClaimResolve cr{};
  cr.t = mt->d_tables + k;
  cr.update_ts = (uint32_t)update_time;
  cr.miss_ctr = miss_ctr;
  cr.miss_slots = w.miss;
  if (knob(KNOB_CLAIM_DUAL))
    fid_claim_kernel<true, true><<<resident_grid(fid_claim_kernel<true, true>, M, kThreads), kThreads, 0, s>>>(
        fids_dev, M, set, cap, 1, epoch, w.k0, w.ctr + kCtrOwners, cr, knob(KNOB_CLAIM_PF));
  else
    fid_claim_kernel<true><<<resident_grid(fid_claim_kernel<true>, M, kThreads), kThreads, 0, s>>>(
        fids_dev, M, set, cap, 1, epoch, w.k0, w.ctr + kCtrOwners, cr, knob(KNOB_CLAIM_PF));
  MONO_CHECK_LAUNCH();
  // 2 absent FIDs: allocate a row + lock-free insert (few in steady state; the count stays on the device)
  claim_miss_kernel<<<resident_grid(claim_miss_kernel, std::min<int64_t>(M, (int64_t)device_sms() * 2 * kThreads), kThreads), kThreads, 0, s>>>(
      mt->d_tables + k, set, miss_ctr, w.miss, (uint32_t)update_time, nullptr, 0);
  MONO_CHECK_LAUNCH();
  launch_upsert_finalize(mt, cb, miss_ctr, (uint32_t)update_time, s);
  // 3 stable LSD radix sort of (slot, position)  +  4 ordered run list (with each run's resolved row)
  w.sorted = sort_and_runs(w.sort, w.k0, M, bits, 0, set, s);
  // 5 reduce
  SegArgs sa = seg_args(w, M, D, pooled_grad, grad_stride, grad_col, row_offsets, n_rows, pooling, w.ugrad, s);
  BwdArgs& a = sa.b;
  a.td = ht.dev;  // descriptor is current: ensure_capacity / upload_tables ran above
  a.t = mt->d_tables + k;
  a.fids = fids_dev;
  a.rowidx = w.sort.rowidx;
  a.lr = cb.lr;
  a.scratch = a.ugrad;
  launch_reduce(sa, G, no_peer, true, s);
  // 6 apply: one streaming pass over the runs — row index, summed gradient, w / optimizer state of every distinct FID
  launch_apply(a, G, apply_opt_sel(ht), M, s);
  ht.issued_total += (uint64_t)M;
  ht.max_update_ts = std::max<int64_t>(ht.max_update_ts, update_time);
  request_snapshot(mt, k, s);
}

// ---- fused backward over many parts (features) of several tables in one call ----
// A part as the occurrence map kernel sees it (parts ordered table-major, part order inside a table)
struct PartDev {
  const int64_t* fids;
  const int32_t* row_offsets;   // null: one FID per row
  const float* rows;            // gradient rows, column included
  int64_t stride;
  int64_t occ_begin;            // first occurrence in the table-major concatenation
  int64_t row_begin;            // first row in the concatenation of the parts' rows
  int32_t mean;                 // CSR MEAN: terms divided by the row's n
  int32_t seq_len;              // FIRSTN: L (0 for SUM / MEAN)
  int32_t dim, pad;             // the table's dim: FIRSTN positions are dim floats apart
};

// One thread per row of the concatenated parts: the row's occurrences get their FID, gradient row and MEAN divisor.
// Occurrence j of a FIRSTN row reads position j of the row for j < L and zero_row (128 floats of +0.0) beyond it,
// as ScatterGrad's FIRSTN branch leaves such a FID's gradient at its zero fill (fused_embedding_to_layout.h:334-340).
__global__ void __launch_bounds__(kThreads)
parts_occ_kernel(const PartDev* __restrict__ parts, int n_parts, int64_t n_rows, int64_t* __restrict__ fids_out,
                 const float** __restrict__ src_out, float* __restrict__ div_out, const float* __restrict__ zero_row) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_parts - 1;  // the last part whose rows start at or before r
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (parts[mid].row_begin <= r) lo = mid;
      else hi = mid - 1;
    }
    const PartDev& p = parts[lo];
    const int64_t lr = r - p.row_begin;
    int64_t b = lr, e = lr + 1;
    if (p.row_offsets) {
      b = p.row_offsets[lr];
      e = p.row_offsets[lr + 1];
    }
    const float* src = p.rows + lr * p.stride;
    const float dv = p.mean ? (float)(e - b) : 0.f;
    for (int64_t m = b; m < e; ++m) {
      fids_out[p.occ_begin + m] = p.fids[m];
      const int64_t j = m - b;
      src_out[p.occ_begin + m] = !p.seq_len ? src : j < p.seq_len ? src + j * p.dim : zero_row;
      div_out[p.occ_begin + m] = dv;
    }
  }
}

// The occurrences of all parts of one table are one batch (part order, then occurrence order): the claim set gets one
// region per table, so one claim, one sort and one run list serve every table and leave each table's occurrences as
// one contiguous sorted range; the reduce and the apply then run once per table over its range, with its row width,
// optimizer and tree depth.  Everything is checked before the first device operation.
// bf16: every part's rows_dev is bf16 storage (stride and col in bf16 elements); each term is widened to fp32 first.
void run_pool_backward_parts(mono_mtable* mt, const mono_pool_part* parts, int n_parts, const float* lr_host,
                             int64_t update_time, cudaStream_t s, bool bf16) {
  const int K = (int)mt->tables.size();
  if (n_parts < 0 || n_parts > MONO_MAX_POOL_PARTS) throw ArgError("pool_backward_parts: bad part count");
  if ((n_parts > 0 && !parts) || !lr_host) throw ArgError("pool_backward_parts: null argument");
  std::vector<int64_t> per_table(K, 0);
  std::vector<char> mean(K, 0);
  int64_t M = 0, n_rows = 0;
  for (int i = 0; i < n_parts; ++i) {
    const mono_pool_part& p = parts[i];
    if (p.table < 0 || p.table >= K) throw ArgError("pool_backward_parts: bad table index");
    if (p.pooling != MONO_POOL_SUM && p.pooling != MONO_POOL_MEAN && p.pooling != MONO_POOL_FIRSTN)
      throw ArgError("pool_backward_parts: SUM, MEAN or FIRSTN");
    if (p.n_fids < 0 || p.n_rows < 0) throw ArgError("pool_backward_parts: negative count");
    check_firstn("pool_backward_parts", p);
    if (!p.row_offsets_dev && p.n_rows != p.n_fids)
      throw ArgError("pool_backward_parts: n_rows must equal n_fids without offsets");
    if (p.n_fids > 0 && (!p.fids_dev || !p.rows_dev)) throw ArgError("pool_backward_parts: null argument");
    check_grad_rows("pool_backward_parts", mt->tables[p.table].dim, p.rows_dev, p.stride, p.col, nullptr,
                    bf16 ? 2 : 4);
    M += p.n_fids;
    if (M > ((int64_t)1 << 30)) throw ArgError("pool_backward_parts: more than 2^30 occurrences in one call");
    if (p.n_fids == 0) continue;
    per_table[p.table] += p.n_fids;
    n_rows += p.n_rows;
    if (p.pooling == MONO_POOL_MEAN && p.row_offsets_dev) mean[p.table] = 1;
  }
  mt->note_insert(s);
  if (M == 0) return;
  // call tables in table order, each with its occurrence range, claim region and learning rates
  std::vector<CallTable> ct;
  std::vector<CallSeg> segs;
  uint64_t cap = 0;
  int64_t occ = 0;
  int n_lr = 0, Dmax = 4;
  for (int k = 0; k < K; ++k) {
    const int lr_off = n_lr;
    n_lr += mt->tables[k].slices;
    if (!per_table[k]) continue;
    CallTable c;
    c.occ_begin = occ;
    c.occ_end = occ + per_table[k];
    c.slot_base = (uint32_t)cap;
    c.slots = claim_set_slots(per_table[k]);
    c.table = k;
    c.pad = 0;
    ct.push_back(c);
    CallSeg sg;
    sg.id_begin = c.occ_begin;
    sg.id_end = c.occ_end;
    sg.val_off = 0;
    sg.table = k;
    sg.lr_off = lr_off;
    segs.push_back(sg);
    cap += c.slots;
    occ = c.occ_end;
    Dmax = std::max(Dmax, mt->tables[k].dim);
  }
  if (cap > ((uint64_t)1 << 31)) throw ArgError("pool_backward_parts: claim set over 2^31 slots");
  const size_t ct_off = (sizeof(PartDev) * (size_t)n_parts + 15) & ~(size_t)15;
  if (ct_off + sizeof(CallTable) * ct.size() > StageRing::kBlockBytes)
    throw ArgError("pool_backward_parts: too many parts and tables for one call descriptor");
  // the parts, table-major
  std::vector<PartDev> pd;
  std::vector<int64_t> occ_at(K), row_at(K);
  {
    int64_t o = 0, r = 0;
    for (int k = 0; k < K; ++k) {
      occ_at[k] = o;
      row_at[k] = r;
      for (int i = 0; i < n_parts; ++i)
        if (parts[i].table == k && parts[i].n_fids > 0) {
          o += parts[i].n_fids;
          r += parts[i].n_rows;
        }
    }
  }
  for (int k = 0; k < K; ++k)
    for (int i = 0; i < n_parts; ++i) {
      const mono_pool_part& p = parts[i];
      if (p.table != k || p.n_fids == 0) continue;
      PartDev d;
      d.fids = p.fids_dev;
      d.row_offsets = p.row_offsets_dev;
      d.rows = p.rows_dev + p.col;
      d.stride = p.stride;
      d.occ_begin = occ_at[k];
      d.row_begin = row_at[k];
      d.mean = p.pooling == MONO_POOL_MEAN && p.row_offsets_dev ? 1 : 0;
      d.seq_len = p.pooling == MONO_POOL_FIRSTN ? p.max_seq_len : 0;
      d.dim = mt->tables[k].dim;
      if (bf16) {  // parts_occ_kernel steps in floats: half as many floats as bf16 elements (stride, dim % 4 == 0)
        d.rows = reinterpret_cast<const float*>(reinterpret_cast<const __nv_bfloat16*>(p.rows_dev) + p.col);
        d.stride = p.stride / 2;
        d.dim = d.dim / 2;
      }
      d.pad = 0;
      pd.push_back(d);
      occ_at[k] += p.n_fids;
      row_at[k] += p.n_rows;
    }

  for (const CallTable& c : ct) ensure_capacity(mt, c.table, (uint64_t)(c.occ_end - c.occ_begin), s);
  upload_tables(mt, s);
  CallBlob cb = stage_call(mt, segs.data(), (int)segs.size(), lr_host, n_lr, s);
  const int rb = mt->ring.acquire();
  std::memcpy(mt->ring.h(rb), pd.data(), sizeof(PartDev) * pd.size());
  std::memcpy(mt->ring.h(rb) + ct_off, ct.data(), sizeof(CallTable) * ct.size());
  mt->ring.commit(rb, ct_off + sizeof(CallTable) * ct.size(), s);
  const PartDev* d_parts = reinterpret_cast<const PartDev*>(mt->ring.d(rb));
  const CallTable* d_ct = reinterpret_cast<const CallTable*>(mt->ring.d(rb) + ct_off);
  const int T = (int)ct.size();

  // ---- scratch ----
  const int bits = bits_for(cap);
  const unsigned sparts = kPartK0 | kPartRowIdx | kPartMiss | kPartRunOfSorted | kPartUGrad | kPartOccMap;
  BwdScratch w = scratch_plan(M, Dmax, bits, sparts, nullptr);
  w = scratch_plan(M, Dmax, bits, sparts, (char*)mt->ws_a.get(w.bytes, s));
  uint32_t epoch = 0;
  Entry* set = (Entry*)mt->claim_set.get(sizeof(Entry) * (size_t)cap, s, &epoch);
  MONO_CUDA(cudaMemsetAsync(w.ctr, 0, kCtrBytes, s));

  // 0 occurrence map: FIDs, gradient row and MEAN divisor of every occurrence, table-major
  parts_occ_kernel<<<resident_grid(parts_occ_kernel, n_rows, kThreads), kThreads, 0, s>>>(
      d_parts, (int)pd.size(), n_rows, w.fids, w.occ_src, w.occ_div, mt->zero_row);
  MONO_CHECK_LAUNCH();
  // 1 claim in the occurrence's table region, resolve in that table  +  2 absent FIDs  (as run_pool_backward)
  uint32_t* miss_ctr = w.ctr + kCtrMisses;
  ClaimResolve cr{};
  cr.t = mt->d_tables;
  cr.update_ts = (uint32_t)update_time;
  cr.miss_ctr = miss_ctr;
  cr.miss_slots = w.miss;
  cr.regions = d_ct;
  cr.n_regions = T;
  if (knob(KNOB_CLAIM_DUAL))
    fid_claim_kernel<true, true><<<resident_grid(fid_claim_kernel<true, true>, M, kThreads), kThreads, 0, s>>>(
        w.fids, M, set, (uint32_t)cap, 1, epoch, w.k0, w.ctr + kCtrOwners, cr, knob(KNOB_CLAIM_PF));
  else
    fid_claim_kernel<true><<<resident_grid(fid_claim_kernel<true>, M, kThreads), kThreads, 0, s>>>(
        w.fids, M, set, (uint32_t)cap, 1, epoch, w.k0, w.ctr + kCtrOwners, cr, knob(KNOB_CLAIM_PF));
  MONO_CHECK_LAUNCH();
  claim_miss_kernel<<<resident_grid(claim_miss_kernel, std::min<int64_t>(M, (int64_t)device_sms() * 2 * kThreads), kThreads), kThreads, 0, s>>>(
      mt->d_tables, set, miss_ctr, w.miss, (uint32_t)update_time, d_ct, T);
  MONO_CHECK_LAUNCH();
  launch_upsert_finalize(mt, cb, miss_ctr, (uint32_t)update_time, s);
  // 3 sort + 4 run list, once: slots are table-major, so each table's runs are one contiguous range
  w.sorted = sort_and_runs(w.sort, w.k0, M, bits, 0, set, s);
  // 5 reduce + 6 apply, per table over its range
  for (int q = 0; q < T; ++q) {
    const int k = ct[q].table;
    HostTable& ht = mt->tables[k];
    const int64_t Mk = ct[q].occ_end - ct[q].occ_begin;
    const SortedRange rg = {ct[q].occ_begin, ct[q].occ_end, mean[k] != 0};
    SegArgs sa = seg_args(w, M, ht.dim, nullptr, 0, 0, nullptr, 0, MONO_POOL_SUM, w.ugrad, s, &rg);
    BwdArgs& a = sa.b;
    a.td = ht.dev;
    a.t = mt->d_tables + k;
    a.fids = w.fids;
    a.rowidx = w.sort.rowidx;
    a.lr = cb.lr + segs[q].lr_off;
    a.scratch = a.ugrad;
    const int G = pick_group(ht.dim);
    launch_reduce(sa, G, no_peer, true, s, bf16);
    launch_apply(a, G, apply_opt_sel(ht), Mk, s, bf16);
    ht.issued_total += (uint64_t)Mk;
    ht.max_update_ts = std::max<int64_t>(ht.max_update_ts, update_time);
    request_snapshot(mt, k, s);
  }
}

// Deterministic replacement of the float-atomic scatter of pooled-row gradients
// (ref: FusedGatherGradKernel, map_id_to_embedding.cu.cc:75-118; ScatterGrad,
// fused_embedding_to_layout.h:286-347): out_rows[offs[m] : +dim] = sum over the occurrences m with that
// offset of pooled_grad[row(m)] (or /n for MEAN), in the reduce's order (occurrence order for <= 64
// occurrences).  Rows of out_rows that no occurrence points at are left untouched.
// bf16: pooled_grad is a cast pointer to bf16 rows (grad_stride and grad_col count bf16 elements); the reduce
// widens them exactly and the sums, the tree and out_rows stay fp32 (bf16_seg_reduce_kernel, then the same kernels).
void run_scatter_rows(int device, const int32_t* offs_dev, int64_t M, int dim, const int32_t* row_offsets,
                      int64_t n_rows, int pooling, const float* pooled_grad, int64_t grad_stride,
                      int grad_col, float* out_rows, int64_t total_floats, cudaStream_t s, bool bf16) {
  MONO_CUDA(cudaSetDevice(device));
  if (M <= 0) return;
  if (M >= ((int64_t)1 << 31) || total_floats >= ((int64_t)1 << 31)) throw ArgError("scatter_rows: sizes exceed 2^31");
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("scatter_rows: SUM or MEAN");
  if (bf16) {  // bf16 pooled gradient rows (8-byte aligned), fp32 destination rows (16-byte aligned)
    check_grad_rows("scatter_rows", dim, pooled_grad, grad_stride, grad_col, nullptr, 2);
    check_grad_rows("scatter_rows", dim, nullptr, 0, 0, out_rows);
  } else {
    check_grad_rows("scatter_rows", dim, pooled_grad, grad_stride, grad_col, out_rows);
  }
  const int D = dim;
  // offsets are multiples of 4 floats (16-byte aligned rows; every dim in the fused buffer is a multiple
  // of 4): drop the two zero bits from the sort key
  const int shift = 2;
  int bits = 1;
  while (((int64_t)1 << bits) < ((total_floats >> shift) + 1)) ++bits;
  const unsigned parts = (row_offsets ? kPartOcc : 0u) | kPartUGrad;
  BwdScratch w = scratch_plan(M, D, bits, parts, nullptr);
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, w.bytes, s));
  w = scratch_plan(M, D, bits, parts, ws);
  MONO_CUDA(cudaMemsetAsync(w.ctr, 0, kCtrBytes, s));
  // the offsets are the sort keys (read-only: the first pass copies them out)
  w.sorted = sort_and_runs(w.sort, reinterpret_cast<const uint32_t*>(offs_dev), M, bits, shift, nullptr, s);
  const SegArgs sa = seg_args(w, M, D, pooled_grad, grad_stride, grad_col, row_offsets, n_rows, pooling, w.ugrad, s);
  const int G = pick_group(D);
  launch_reduce(sa, G, no_peer, false, s, bf16);
#define EMIT(GG)                                                                                              \
  runs_emit_kernel<GG><<<resident_grid(runs_emit_kernel<GG>, M, kThreads / GG), kThreads, 0, s>>>(sa.b, shift, out_rows); \
  MONO_CHECK_LAUNCH()
  switch (G) {
    case 4: EMIT(4); break;
    case 8: EMIT(8); break;
    case 16: EMIT(16); break;
    default: EMIT(32); break;
  }
#undef EMIT
  MONO_CUDA(cudaFreeAsync(ws, s));
}

// ==========================================================================================
// Owner grouping: ONE grouping of a batch's FID occurrences shared by the forward (dedup + bucket by
// owner for the exchange) and the backward (deterministic per-FID gradient reduction) of the sharded
// step.  Functionally FusedReorderByIndices (ref: fused_reorder_by_indices.cc:38-123) for a single id
// list, except that the order of the distinct FIDs inside a shard is the engine's (scratch-set slot
// order), not first-occurrence order; mono_reorder_by_indices is the bit-exact op.
//
// The scratch set is split into N regions of R slots and a FID lives in region owner(fid) = fid mod N
// (linear probing wraps inside the region).  Sorting the occurrences by slot therefore yields the runs
// (one per distinct FID) already bucketed by owner: no separate partition pass, and a run's index IS its
// position in the bucketed unique list.  The per-owner distinct counts fall out of the claim kernel (one
// count per successful insert), i.e. after the FIRST kernel: they are copied to the host on a side
// stream while the sort still runs, so the host can size and enqueue the exchange without idling the GPU.
// ==========================================================================================
// bucketed unique list and the per-occurrence row offsets: run j (slot order == owner-bucketed order)
__global__ void __launch_bounds__(kThreads)
group_emit_kernel(const int64_t* __restrict__ fids, const uint2* __restrict__ sorted,
                  const uint32_t* __restrict__ run_of_sorted, const uint32_t* __restrict__ run_first_pos,
                  const uint32_t* __restrict__ n_runs, int64_t n, int dim, int32_t* __restrict__ occ_offset,
                  int64_t* __restrict__ uniq_out) {
  const int64_t t0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = t0; i < n; i += stride) occ_offset[sorted[i].y] = (int32_t)(run_of_sorted[i] * (uint32_t)dim);
  const int64_t nr = *n_runs;
  for (int64_t j = t0; j < nr; j += stride) uniq_out[j] = fids[run_first_pos[j]];
}

mono_grouping* grouping_create(int device) {
  auto g = new mono_grouping();
  g->device = device;
  return g;
}

void grouping_destroy(mono_grouping* g) {
  if (!g) return;
  cudaSetDevice(g->device);
  cudaDeviceSynchronize();
  g->ws.release();
  g->claim_set.release();
  if (g->h_counts) cudaFreeHost(g->h_counts);
  if (g->ev_claimed) cudaEventDestroy(g->ev_claimed);
  if (g->ev_copied) cudaEventDestroy(g->ev_copied);
  if (g->side) cudaStreamDestroy(g->side);
  delete g;
}

void grouping_build(mono_grouping* g, const int64_t* fids_dev, int64_t M, int N, int dim,
                    int64_t* uniq_out, int32_t* occ_offset_out, int32_t* shard_counts_host,
                    int64_t* n_unique_host, cudaStream_t s) {
  MONO_CUDA(cudaSetDevice(g->device));
  if (N <= 0 || N > 256) throw ArgError("grouping: num_shards must be in [1, 256]");
  if (M < 0 || M >= ((int64_t)1 << 29)) throw ArgError("grouping: bad occurrence count");
  if (dim <= 0) throw ArgError("grouping: dim must be positive");
  check_grad_rows("grouping", dim);
  g->M = M;
  g->dim = dim;
  g->plan = BwdScratch{};
  if (M == 0) {
    if (!shard_counts_host) throw ArgError("grouping: the device-driven step needs a non-empty batch");
    for (int n = 0; n < N; ++n) shard_counts_host[n] = 0;
    if (n_unique_host) *n_unique_host = 0;
    return;
  }
  if (!g->h_counts) {
    MONO_CUDA(cudaHostAlloc((void**)&g->h_counts, 4 * 260, cudaHostAllocDefault));
    MONO_CUDA(cudaStreamCreateWithFlags(&g->side, cudaStreamNonBlocking));
    MONO_CUDA(cudaEventCreateWithFlags(&g->ev_claimed, cudaEventDisableTiming));
    MONO_CUDA(cudaEventCreateWithFlags(&g->ev_copied, cudaEventDisableTiming));
  }
  const uint64_t cap0 = claim_set_slots(M);
  for (int attempt = 0; attempt < 2; ++attempt) {
    // attempt 0: the regions share 2M slots (load <= 0.5 for hash-balanced owners);
    // attempt 1 (a region overflowed: heavily skewed owners): every region can hold all M FIDs.
    const uint64_t cap = attempt == 0 ? cap0 : cap0 * (uint64_t)N;
    if (cap > ((uint64_t)1 << 31)) throw ArgError("grouping: FID owners too skewed for this batch size");
    const uint32_t R = (uint32_t)(cap / (uint64_t)N);
    const int bits = bits_for(cap);
    const unsigned parts = kPartK0 | kPartRunOfSorted | kPartOcc;  // occ: reduce()'s CSR map
    BwdScratch w = scratch_plan(M, dim, bits, parts, nullptr);
    w = scratch_plan(M, dim, bits, parts, (char*)g->ws.get(w.bytes, s));
    uint32_t epoch = 0;
    Entry* set = (Entry*)g->claim_set.get(sizeof(Entry) * (size_t)cap, s, &epoch);
    uint32_t* owner_cnt = w.ctr + kCtrOwners;
    MONO_CUDA(cudaMemsetAsync(w.ctr, 0, kCtrBytes, s));
    ClaimResolve cr0;
    std::memset(&cr0, 0, sizeof(cr0));
    fid_claim_kernel<false><<<resident_grid(fid_claim_kernel<false>, M, kThreads), kThreads, 0, s>>>(
        fids_dev, M, set, R, N, epoch, w.k0, owner_cnt, cr0, knob(KNOB_CLAIM_PF));
    MONO_CHECK_LAUNCH();
    // counts -> host on the side stream, while the sort below keeps the GPU busy.  Device-driven callers
    // (shard_counts_host == nullptr: xstep.cu) never read them on the host: nothing waits, the per-owner counts stay
    // in owner_cnt and a region overflow is left in owner_cnt[256] for the caller to check later.
    const bool host_counts = shard_counts_host != nullptr;
    if (host_counts) {
      MONO_CUDA(cudaEventRecord(g->ev_claimed, s));
      MONO_CUDA(cudaStreamWaitEvent(g->side, g->ev_claimed, 0));
      MONO_CUDA(cudaMemcpyAsync(g->h_counts, owner_cnt, 4 * 257, cudaMemcpyDeviceToHost, g->side));
      MONO_CUDA(cudaEventRecord(g->ev_copied, g->side));
    }
    w.sorted = sort_and_runs(w.sort, w.k0, M, bits, 0, nullptr, s);
    group_emit_kernel<<<resident_grid(group_emit_kernel, M, kThreads), kThreads, 0, s>>>(
        fids_dev, w.sorted, w.sort.run_of_sorted, w.sort.run_first_pos, w.sort.n_runs, M, dim, occ_offset_out, uniq_out);
    MONO_CHECK_LAUNCH();
    if (host_counts) {
      MONO_CUDA(cudaEventSynchronize(g->ev_copied));
      if (g->h_counts[256] != 0) continue;  // region overflow: redo with full-size regions
      int64_t total = 0;
      for (int n = 0; n < N; ++n) {
        shard_counts_host[n] = (int32_t)g->h_counts[n];
        total += g->h_counts[n];
      }
      if (n_unique_host) *n_unique_host = total;
    }
    g->plan = w;
    return;
  }
  throw ArgError("grouping: scratch set overflow (internal)");
}

static void grouping_reduce_impl(mono_grouping* g, const float* pooled_grad, int64_t grad_stride, int grad_col,
                                 const int32_t* row_offsets, int64_t n_rows, int pooling, float* out_rows,
                                 const PeerOut& po, cudaStream_t s) {
  MONO_CUDA(cudaSetDevice(g->device));
  const int64_t M = g->M;
  const int D = g->dim;
  if (M <= 0) return;
  if (!g->plan.sorted) throw ArgError("grouping_reduce before grouping_build");
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("grouping_reduce: SUM or MEAN");
  check_grad_rows("grouping_reduce", D, pooled_grad, grad_stride, grad_col, po.n == 0 ? out_rows : nullptr);
  // runs are already in the bucketed order: the sums are written in place
  const SegArgs sa = seg_args(g->plan, M, D, pooled_grad, grad_stride, grad_col, row_offsets, n_rows, pooling,
                              out_rows, s);
  launch_reduce(sa, pick_group(D), po, false, s);
}

// out_rows[u] = summed gradient of the u-th distinct FID of the bucketed list (ref: ScatterGrad)
void grouping_reduce(mono_grouping* g, const float* pooled_grad, int64_t grad_stride, int grad_col,
                     const int32_t* row_offsets, int64_t n_rows, int pooling, float* out_rows, cudaStream_t s) {
  grouping_reduce_impl(g, pooled_grad, grad_stride, grad_col, row_offsets, n_rows, pooling, out_rows, no_peer, s);
}

// same, fused with the gradient exchange of the sharded backward: the row of the u-th distinct FID is stored
// into the window of the rank that owns it (replaces the gradient all-to-all, ref:
// distributed_ps_sync.py:531-573); the NVLink stores overlap the reduction, run by run.
void grouping_reduce_push(mono_grouping* g, const float* pooled_grad, int64_t grad_stride, int grad_col,
                          const int32_t* row_offsets, int64_t n_rows, int pooling, const PeerOut& po,
                          cudaStream_t s) {
  if (po.n <= 0) throw ArgError("grouping_reduce_push without a peer window");
  grouping_reduce_impl(g, pooled_grad, grad_stride, grad_col, row_offsets, n_rows, pooling, nullptr, po, s);
}

}  // namespace mono
