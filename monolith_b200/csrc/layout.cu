// layout.cu — pooling from already-looked-up row buffers (the sync all-to-all path) and the generic
// fused layout op.
//
//  * gather_pool / gather_pool_grad: FusedGatherKernel / FusedGatherGradKernel
//    (ref: RT/ops/map_id_to_embedding.cu.cc:30-118) fused with the per-row SUM / MEAN pool.
//    The reference assigns one THREAD per output float; here a lane group moves 16-byte vectors.
//  * embedding_to_layout / _grad: MonolithEmbeddingToLayoutV3-5 (ref: RT/ops/fused_embedding_to_layout
//    .{h,cc,cu.cc}).  The reference GPU kernel runs one thread per (sample, slice task) with a scalar
//    loop over dim (cu.cc:53-78,96-194); here one lane group per (sample, output slice), lanes across
//    dim, terms accumulated in the CPU reference's order (deterministic forward).
#include <algorithm>
#include <cstring>
#include <vector>

#include "engine.h"
#include "rowelem.cuh"

namespace mono {

// T: element type of the pooled rows (float, or bf16 for the *_bf16 calls); the fused row buffer is always fp32 and
// every add and division runs in fp32, so a bf16 element is the fp32 result rounded once.
template <typename T, int G>
__device__ __forceinline__ void gather_pool(const float* __restrict__ fused, const int32_t* __restrict__ emb_offset,
                                            const int32_t* __restrict__ row_offsets, int64_t n_rows, int dim,
                                            int pooling, T* __restrict__ out, int64_t out_stride, int out_col) {
  const int gl = Group<G>::gl();
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  const bool src_vec = (dim & 3) == 0 && (reinterpret_cast<uintptr_t>(fused) & 15) == 0;
  for (int64_t r = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; r < n_rows; r += gstride) {
    const int64_t b = row_offsets ? row_offsets[r] : r;
    const int64_t e = row_offsets ? row_offsets[r + 1] : r + 1;
    const int n = (int)(e - b);
    const float fn = (float)n;
    T* dst = out + r * out_stride + out_col;
    // 4 elements per vector store: 16 bytes of fp32, 8 of bf16
    const bool dst_vec = src_vec && (reinterpret_cast<uintptr_t>(dst) & (4 * sizeof(T) - 1)) == 0;
    if (dst_vec) {
      for (int c = gl * 4; c < dim; c += G * 4) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < n; ++j) {
          // rows of a multi-table fused buffer start at arbitrary float offsets when some table's dim
          // is not a multiple of 4: vector load only when this row is 16-byte aligned
          const float* src = fused + emb_offset[b + j] + c;
          float4 x;
          if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
            x = __ldg(reinterpret_cast<const float4*>(src));
          } else {
            x.x = __ldg(src); x.y = __ldg(src + 1); x.z = __ldg(src + 2); x.w = __ldg(src + 3);
          }
          if (pooling == MONO_POOL_MEAN) {
            x.x = __fdiv_rn(x.x, fn); x.y = __fdiv_rn(x.y, fn);
            x.z = __fdiv_rn(x.z, fn); x.w = __fdiv_rn(x.w, fn);
          }
          if (j == 0) acc = x;
          else {
            acc.x = __fadd_rn(acc.x, x.x); acc.y = __fadd_rn(acc.y, x.y);
            acc.z = __fadd_rn(acc.z, x.z); acc.w = __fadd_rn(acc.w, x.w);
          }
        }
        store_row4(dst + c, acc);
      }
    } else {
      for (int c = gl; c < dim; c += G) {
        float acc = 0.f;
        for (int j = 0; j < n; ++j) {
          float x = __ldg(fused + emb_offset[b + j] + c);
          if (pooling == MONO_POOL_MEAN) x = __fdiv_rn(x, fn);
          acc = j == 0 ? x : __fadd_rn(acc, x);
        }
        dst[c] = to_row_elem(acc, dst);
      }
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads)
gather_pool_kernel(const float* __restrict__ fused, const int32_t* __restrict__ emb_offset,
                   const int32_t* __restrict__ row_offsets, int64_t n_rows, int dim, int pooling,
                   float* __restrict__ out, int64_t out_stride, int out_col) {
  gather_pool<float, G>(fused, emb_offset, row_offsets, n_rows, dim, pooling, out, out_stride, out_col);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
bf16_gather_pool_kernel(const float* __restrict__ fused, const int32_t* __restrict__ emb_offset,
                        const int32_t* __restrict__ row_offsets, int64_t n_rows, int dim, int pooling,
                        __nv_bfloat16* __restrict__ out, int64_t out_stride, int out_col) {
  gather_pool<__nv_bfloat16, G>(fused, emb_offset, row_offsets, n_rows, dim, pooling, out, out_stride, out_col);
}

// One occurrence per output row (row_offsets == NULL: FusedGatherKernel proper) with 16-byte aligned rows:
// the same two-phase shape as the table lookup (ops.cu lookup_kernel): a lane fetches one offset
// (32 coalesced, independent loads per warp), then G lanes move one row with 128-bit accesses, 4 rows in
// flight per lane before the first store.  Pooling over a single row is the identity for SUM and MEAN.
// T = bf16: the same fp32 loads, one 8-byte streaming store of 4 rounded elements per lane.
template <typename T, int G>
__device__ __forceinline__ void gather_rows(const float* __restrict__ fused, const int32_t* __restrict__ emb_offset,
                                            int64_t n_rows, int dim, T* __restrict__ out, int64_t out_stride,
                                            int out_col) {
  constexpr int RPI = 32 / G, ITERS = G, UNR = 4;
  const int lane = threadIdx.x & 31, gl = Group<G>::gl(), grp = lane / G;
  const int c = gl * 4;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * 32;
  for (int64_t wbase = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * 32; wbase < n_rows;
       wbase += wstride) {
    const int64_t i = wbase + lane;
    const int32_t off = i < n_rows ? __ldg(emb_offset + i) : 0;
#pragma unroll
    for (int it0 = 0; it0 < ITERS; it0 += UNR) {
      float4 x[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int32_t o = __shfl_sync(0xffffffffu, off, (it0 + u) * RPI + grp);
        x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (wbase + (it0 + u) * RPI + grp < n_rows && c < dim) {
          const float* src = fused + o + c;
          // rows of a multi-table fused buffer may start at any float offset
          x[u] = (o & 3) == 0 ? __ldg(reinterpret_cast<const float4*>(src))
                              : make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3));
        }
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int64_t ir = wbase + (it0 + u) * RPI + grp;
        if (ir < n_rows && c < dim) stcs_row4(out + ir * out_stride + out_col + c, x[u]);
      }
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads, 4)
gather_rows_kernel(const float* __restrict__ fused, const int32_t* __restrict__ emb_offset, int64_t n_rows,
                   int dim, float* __restrict__ out, int64_t out_stride, int out_col) {
  gather_rows<float, G>(fused, emb_offset, n_rows, dim, out, out_stride, out_col);
}

template <int G>
__global__ void __launch_bounds__(kThreads, 4)
bf16_gather_rows_kernel(const float* __restrict__ fused, const int32_t* __restrict__ emb_offset, int64_t n_rows,
                        int dim, __nv_bfloat16* __restrict__ out, int64_t out_stride, int out_col) {
  gather_rows<__nv_bfloat16, G>(fused, emb_offset, n_rows, dim, out, out_stride, out_col);
}

// grad_fused[offset[m] : +dim] += g_row   (float atomics: several occurrences may share a row,
// exactly like the reference's FusedGatherGradKernel atomicAdd, map_id_to_embedding.cu.cc:75-118)
// T = bf16: the pooled gradient is widened exactly, then divided and added in fp32.
template <typename T, int G>
__device__ __forceinline__ void gather_pool_grad(const T* __restrict__ pooled_grad, int64_t grad_stride, int grad_col,
                                                 const int32_t* __restrict__ emb_offset,
                                                 const int32_t* __restrict__ row_offsets, int64_t n_rows, int dim,
                                                 int pooling, float* __restrict__ grad_fused) {
  const int gl = Group<G>::gl();
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t r = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; r < n_rows; r += gstride) {
    const int64_t b = row_offsets ? row_offsets[r] : r;
    const int64_t e = row_offsets ? row_offsets[r + 1] : r + 1;
    const int n = (int)(e - b);
    const float fn = (float)n;
    const T* g = pooled_grad + r * grad_stride + grad_col;
    for (int c = gl; c < dim; c += G) {
      float x = row_elem_f32(__ldg(g + c));
      if (pooling == MONO_POOL_MEAN) x = __fdiv_rn(x, fn);
      for (int j = 0; j < n; ++j) atomicAdd(grad_fused + emb_offset[b + j] + c, x);
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads)
gather_pool_grad_kernel(const float* __restrict__ pooled_grad, int64_t grad_stride, int grad_col,
                        const int32_t* __restrict__ emb_offset, const int32_t* __restrict__ row_offsets,
                        int64_t n_rows, int dim, int pooling, float* __restrict__ grad_fused) {
  gather_pool_grad<float, G>(pooled_grad, grad_stride, grad_col, emb_offset, row_offsets, n_rows, dim, pooling,
                             grad_fused);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
bf16_gather_pool_grad_kernel(const __nv_bfloat16* __restrict__ pooled_grad, int64_t grad_stride, int grad_col,
                             const int32_t* __restrict__ emb_offset, const int32_t* __restrict__ row_offsets,
                             int64_t n_rows, int dim, int pooling, float* __restrict__ grad_fused) {
  gather_pool_grad<__nv_bfloat16, G>(pooled_grad, grad_stride, grad_col, emb_offset, row_offsets, n_rows, dim, pooling,
                                     grad_fused);
}

static int pick_group(int dim) {
  int v = (dim + 3) / 4, g = 4;
  while (g < v && g < 32) g <<= 1;
  return g;
}

void launch_gather_pool(const float* fused_emb, const int32_t* emb_offset, const int32_t* row_offsets,
                        int64_t n_rows, int dim, int pooling, float* out, int64_t out_stride,
                        int out_col, cudaStream_t s) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("gather_pool: SUM or MEAN");
  // One occurrence per output row: MEAN is x / 1, the identity, except that the division would replace a NaN's payload
  // with the canonical NaN.  Pool as SUM (a copy), so every width keeps all 32 bits, as gather_rows_kernel does.
  if (row_offsets == nullptr) pooling = MONO_POOL_SUM;
  const int G = pick_group(dim);
  if (row_offsets == nullptr && (dim & 3) == 0 && dim <= 4 * G && (out_stride & 3) == 0 && (out_col & 3) == 0 &&
      ((reinterpret_cast<uintptr_t>(fused_emb) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
#define GR(GG) gather_rows_kernel<GG><<<resident_grid(gather_rows_kernel<GG>, n_rows, kThreads), kThreads, 0, s>>>( \
      fused_emb, emb_offset, n_rows, dim, out, out_stride, out_col)
    switch (G) { case 4: GR(4); break; case 8: GR(8); break; case 16: GR(16); break; default: GR(32); }
#undef GR
    MONO_CHECK_LAUNCH();
    return;
  }
  const int grid = grid_for(n_rows, kThreads / G);
#define GP(GG) gather_pool_kernel<GG><<<grid, kThreads, 0, s>>>(fused_emb, emb_offset, row_offsets, n_rows, dim, pooling, out, out_stride, out_col)
  switch (G) { case 4: GP(4); break; case 8: GP(8); break; case 16: GP(16); break; default: GP(32); }
#undef GP
  MONO_CHECK_LAUNCH();
}

void launch_gather_pool_grad(const float* pooled_grad, int64_t grad_stride, int grad_col,
                             const int32_t* emb_offset, const int32_t* row_offsets, int64_t n_rows,
                             int dim, int pooling, float* grad_fused, cudaStream_t s) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("gather_pool_grad: SUM or MEAN");
  const int G = std::min(32, std::max(4, pick_group(dim * 4)));  // one float per lane
  const int grid = grid_for(n_rows, kThreads / G);
#define GG_(GG) gather_pool_grad_kernel<GG><<<grid, kThreads, 0, s>>>(pooled_grad, grad_stride, grad_col, emb_offset, row_offsets, n_rows, dim, pooling, grad_fused)
  switch (G) { case 4: GG_(4); break; case 8: GG_(8); break; case 16: GG_(16); break; default: GG_(32); }
#undef GG_
  MONO_CHECK_LAUNCH();
}

// bf16 pooled rows: launch_gather_pool's rules, with 8-byte aligned output rows for the row copy
void launch_gather_pool_bf16(const float* fused_emb, const int32_t* emb_offset, const int32_t* row_offsets,
                             int64_t n_rows, int dim, int pooling, __nv_bfloat16* out, int64_t out_stride,
                             int out_col, cudaStream_t s) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("gather_pool: SUM or MEAN");
  if (row_offsets == nullptr) pooling = MONO_POOL_SUM;
  const int G = pick_group(dim);
  if (row_offsets == nullptr && (dim & 3) == 0 && dim <= 4 * G && (out_stride & 3) == 0 && (out_col & 3) == 0 &&
      (reinterpret_cast<uintptr_t>(fused_emb) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0) {
#define BR(GG) bf16_gather_rows_kernel<GG><<<resident_grid(bf16_gather_rows_kernel<GG>, n_rows, kThreads), kThreads, 0, \
      s>>>(fused_emb, emb_offset, n_rows, dim, out, out_stride, out_col)
    switch (G) { case 4: BR(4); break; case 8: BR(8); break; case 16: BR(16); break; default: BR(32); }
#undef BR
    MONO_CHECK_LAUNCH();
    return;
  }
  const int grid = grid_for(n_rows, kThreads / G);
#define BP(GG) bf16_gather_pool_kernel<GG><<<grid, kThreads, 0, s>>>(fused_emb, emb_offset, row_offsets, n_rows, dim, \
      pooling, out, out_stride, out_col)
  switch (G) { case 4: BP(4); break; case 8: BP(8); break; case 16: BP(16); break; default: BP(32); }
#undef BP
  MONO_CHECK_LAUNCH();
}

void launch_gather_pool_grad_bf16(const __nv_bfloat16* pooled_grad, int64_t grad_stride, int grad_col,
                                  const int32_t* emb_offset, const int32_t* row_offsets, int64_t n_rows, int dim,
                                  int pooling, float* grad_fused, cudaStream_t s) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("gather_pool_grad: SUM or MEAN");
  const int G = std::min(32, std::max(4, pick_group(dim * 4)));
  const int grid = grid_for(n_rows, kThreads / G);
#define BG(GG) bf16_gather_pool_grad_kernel<GG><<<grid, kThreads, 0, s>>>(pooled_grad, grad_stride, grad_col, \
      emb_offset, row_offsets, n_rows, dim, pooling, grad_fused)
  switch (G) { case 4: BG(4); break; case 8: BG(8); break; case 16: BG(16); break; default: BG(32); }
#undef BG
  MONO_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------------------
// generic layout op
// ------------------------------------------------------------------------------------------
struct LayoutArgs {
  float* const* emb_ptrs;       // [n_emb] (forward: read; backward: atomically accumulated)
  const int32_t* emb_strides;   // [n_emb] PtrWrapper.offset
  const uint64_t* fid_offset;
  int64_t total_fid;
  const int32_t* feature_offset;
  int total_feature;
  const uint32_t* nfl_offset;
  int total_nfl;
  int batch_size;
  const mono_slice_task* tasks;  // device copy
  const int32_t* chain_start;    // [n_chains + 1]
  int n_chains;
  float* const* out_ptrs;
};

// ref: GetFeatureInfo, fused_embedding_to_layout.h:62-76
__device__ __forceinline__ void feature_info(const LayoutArgs& a, int nfl_idx, bool* shared, int* off,
                                             int* num) {
  const uint32_t enc = a.nfl_offset[nfl_idx];
  *shared = enc >> 31;
  *off = enc & 0x7fffffff;
  if (nfl_idx < a.total_nfl - 1) *num = (int)(a.nfl_offset[nfl_idx + 1] & 0x7fffffff) - *off;
  else *num = a.total_feature - *off;
}

__device__ __forceinline__ void fid_range(const LayoutArgs& a, int feature_idx, int* start, int* num) {
  *start = a.feature_offset[feature_idx];
  *num = feature_idx < a.total_feature - 1 ? a.feature_offset[feature_idx + 1] - *start
                                           : (int)a.total_fid - *start;
}

// Forward.  A "chain" is the list of slice tasks that write the same destination (length 1 except
// for ADDN outputs, where the reference sums the slices in config order:
// ForwardTaskRunImpl, fused_embedding_to_layout.cc:468-540).
// T: element type of the outputs (a.out_ptrs point at T storage; out_row_stride and out_col count T elements).
template <typename T, int G>
__device__ __forceinline__ void layout_fwd(const LayoutArgs& a) {
  const int gl = Group<G>::gl();
  const int64_t total = (int64_t)a.n_chains * a.batch_size;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t u = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; u < total; u += gstride) {
    const int ch = (int)(u / a.batch_size);
    const int b = (int)(u % a.batch_size);
    const int t0 = a.chain_start[ch], t1 = a.chain_start[ch + 1];
    const mono_slice_task first = a.tasks[t0];
    T* dst = reinterpret_cast<T* const*>(a.out_ptrs)[first.out_tensor] + (int64_t)b * first.out_row_stride +
             first.out_col;
    if (first.pooling == MONO_POOL_FIRSTN) {
      // out[seq_idx, :] = row of the seq_idx-th fid (zeros past the end)
      bool shared; int off, num;
      feature_info(a, first.nfl_idx, &shared, &off, &num);
      int start = 0, fnum = 0;
      if (num) fid_range(a, shared ? off : off + b, &start, &fnum);
      for (int q = 0; q < first.max_seq_len; ++q) {
        const float* src = nullptr;
        if (q < fnum) {
          const uint64_t fo = a.fid_offset[start + q];
          const int i1 = (int)(fo >> 32), i2 = (int)(fo & 0xffffffffu);
          src = a.emb_ptrs[i1] + (int64_t)i2 * a.emb_strides[i1] + first.slice_start;
        }
        for (int c = gl; c < first.dim; c += G) dst[q * first.dim + c] = to_row_elem(src ? src[c] : 0.0f, dst);
      }
      continue;
    }
    for (int c = gl; c < first.dim; c += G) {
      float acc = 0.0f;
      bool init = true;  // first term assigns (OptimizedSumpooling, cc:26-59)
      for (int ti = t0; ti < t1; ++ti) {
        const mono_slice_task tk = a.tasks[ti];
        bool shared; int off, num;
        feature_info(a, tk.nfl_idx, &shared, &off, &num);
        if (!num) continue;
        int start, fnum;
        fid_range(a, shared ? off : off + b, &start, &fnum);
        const float fn = (float)fnum;
        // shared + ADDN pools into a temporary first, then adds the temporary (cc:486-505)
        const bool via_tmp = shared && tk.accumulate;
        float tmp = 0.0f;
        bool tinit = true;
        for (int f = 0; f < fnum; ++f) {
          const uint64_t fo = a.fid_offset[start + f];
          const int i1 = (int)(fo >> 32), i2 = (int)(fo & 0xffffffffu);
          float x = a.emb_ptrs[i1][(int64_t)i2 * a.emb_strides[i1] + tk.slice_start + c];
          if (tk.pooling == MONO_POOL_MEAN) x = __fdiv_rn(x, fn);
          if (via_tmp) {
            tmp = tinit ? x : __fadd_rn(tmp, x);
            tinit = false;
          } else if (tk.accumulate) {
            acc = __fadd_rn(acc, x);  // ADDN rows start from zero and every term accumulates
          } else {
            acc = init ? x : __fadd_rn(acc, x);
            init = false;
          }
        }
        if (via_tmp) acc = __fadd_rn(acc, tmp);
      }
      dst[c] = to_row_elem(acc, dst);
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads) layout_fwd_kernel(LayoutArgs a) {
  layout_fwd<float, G>(a);
}

template <int G>
__global__ void __launch_bounds__(kThreads) bf16_layout_fwd_kernel(LayoutArgs a) {
  layout_fwd<__nv_bfloat16, G>(a);
}

// Backward: ScatterGrad (ref: fused_embedding_to_layout.h:286-347) with float atomics, as the
// reference GPU kernel does (BackwardBatchKernel, cu.cc:337-381).
// T: element type of the output gradients, widened exactly; the division and the atomics run in fp32.
template <typename T, int G>
__device__ __forceinline__ void layout_bwd(const LayoutArgs& a, int n_tasks) {
  const int gl = Group<G>::gl();
  const int64_t total = (int64_t)n_tasks * a.batch_size;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t u = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; u < total; u += gstride) {
    const int ti = (int)(u / a.batch_size);
    const int b = (int)(u % a.batch_size);
    const mono_slice_task tk = a.tasks[ti];
    bool shared; int off, num;
    feature_info(a, tk.nfl_idx, &shared, &off, &num);
    if (!num) continue;
    int start, fnum;
    fid_range(a, shared ? off : off + b, &start, &fnum);
    const T* g = reinterpret_cast<T* const*>(a.out_ptrs)[tk.out_tensor] + (int64_t)b * tk.out_row_stride + tk.out_col;
    const float fn = (float)fnum;
    for (int f = 0; f < fnum; ++f) {
      if (tk.pooling == MONO_POOL_FIRSTN && f >= tk.max_seq_len) break;
      const uint64_t fo = a.fid_offset[start + f];
      const int i1 = (int)(fo >> 32), i2 = (int)(fo & 0xffffffffu);
      float* dst = a.emb_ptrs[i1] + (int64_t)i2 * a.emb_strides[i1] + tk.slice_start;
      for (int c = gl; c < tk.dim; c += G) {
        float x = row_elem_f32(tk.pooling == MONO_POOL_FIRSTN ? g[f * tk.dim + c] : g[c]);
        if (tk.pooling == MONO_POOL_MEAN) x = __fdiv_rn(x, fn);
        atomicAdd(dst + c, x);
      }
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads) layout_bwd_kernel(LayoutArgs a, int n_tasks) {
  layout_bwd<float, G>(a, n_tasks);
}

template <int G>
__global__ void __launch_bounds__(kThreads) bf16_layout_bwd_kernel(LayoutArgs a, int n_tasks) {
  layout_bwd<__nv_bfloat16, G>(a, n_tasks);
}

// Host-side checks of the tasks: the kernels index with every field unchecked.
void check_layout_tasks(const mono_slice_task* tasks, int n_tasks, int total_nfl) {
  if (n_tasks <= 0) return;
  if (tasks == nullptr) throw ArgError("layout: tasks is null");
  for (int i = 0; i < n_tasks; ++i) {
    const mono_slice_task& t = tasks[i];
    if (t.nfl_idx < 0 || t.nfl_idx >= total_nfl) throw ArgError("layout: task nfl_idx outside [0, total_nfl)");
    if (t.dim <= 0) throw ArgError("layout: task dim must be positive");
    if (t.slice_start < 0 || t.out_col < 0 || t.out_tensor < 0)
      throw ArgError("layout: task slice_start, out_col and out_tensor must be >= 0");
    if (t.pooling != MONO_POOL_SUM && t.pooling != MONO_POOL_MEAN && t.pooling != MONO_POOL_FIRSTN)
      throw ArgError("layout: task pooling must be SUM, MEAN or FIRSTN");
    int64_t width = t.dim;
    if (t.pooling == MONO_POOL_FIRSTN) {
      if (t.max_seq_len <= 0) throw ArgError("layout: FIRSTN task needs max_seq_len >= 1");
      if (t.accumulate) throw ArgError("layout: FIRSTN task cannot accumulate (ADDN)");
      width *= t.max_seq_len;
    }
    if ((int64_t)t.out_row_stride < (int64_t)t.out_col + width)
      throw ArgError("layout: task out_row_stride < out_col + dim (+ max_seq_len * dim for FIRSTN)");
  }
}

// the bf16 twins of layout_fwd_kernel / layout_bwd_kernel at lane-group width G
template <int G>
static void launch_bf16_layout(bool backward, int grid, const LayoutArgs& a, int n_tasks, cudaStream_t s) {
  if (backward) bf16_layout_bwd_kernel<G><<<grid, kThreads, 0, s>>>(a, n_tasks);
  else bf16_layout_fwd_kernel<G><<<grid, kThreads, 0, s>>>(a);
}

void launch_layout(bool backward, float* const* emb_ptrs_dev, const int32_t* emb_strides_dev,
                   int n_emb, const uint64_t* fid_offset, int64_t total_fid,
                   const int32_t* feature_offset, int total_feature, const uint32_t* nfl_offset,
                   int total_nfl, int batch_size, const mono_slice_task* tasks_host, int n_tasks,
                   float* const* out_ptrs_dev, cudaStream_t s, bool bf16) {
  (void)n_emb;
  if (n_tasks <= 0 || batch_size <= 0) return;
  // chains: consecutive grouping of tasks by destination (accumulate tasks with equal destination)
  std::vector<mono_slice_task> ordered;
  std::vector<int32_t> chain_start;
  std::vector<char> used(n_tasks, 0);
  for (int i = 0; i < n_tasks; ++i) {
    if (used[i]) continue;
    chain_start.push_back((int32_t)ordered.size());
    ordered.push_back(tasks_host[i]);
    used[i] = 1;
    if (tasks_host[i].accumulate) {
      for (int j = i + 1; j < n_tasks; ++j) {
        const mono_slice_task& o = tasks_host[j];
        if (!used[j] && o.accumulate && o.out_tensor == tasks_host[i].out_tensor &&
            o.out_col == tasks_host[i].out_col) {
          if (o.dim != tasks_host[i].dim) throw ArgError("ADDN slices must have equal dims");
          ordered.push_back(o);
          used[j] = 1;
        }
      }
    }
  }
  chain_start.push_back((int32_t)ordered.size());
  const int n_chains = (int)chain_start.size() - 1;
  int max_dim = 1;
  for (auto& t : ordered) max_dim = std::max(max_dim, t.dim);

  const size_t tb = sizeof(mono_slice_task) * ordered.size();
  const size_t cb = sizeof(int32_t) * chain_start.size();
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, tb + cb + 64, s));
  MONO_CUDA(cudaMemcpyAsync(ws, ordered.data(), tb, cudaMemcpyHostToDevice, s));
  MONO_CUDA(cudaMemcpyAsync(ws + ((tb + 15) & ~(size_t)15), chain_start.data(), cb, cudaMemcpyHostToDevice, s));
  LayoutArgs a;
  a.emb_ptrs = emb_ptrs_dev;
  a.emb_strides = emb_strides_dev;
  a.fid_offset = fid_offset;
  a.total_fid = total_fid;
  a.feature_offset = feature_offset;
  a.total_feature = total_feature;
  a.nfl_offset = nfl_offset;
  a.total_nfl = total_nfl;
  a.batch_size = batch_size;
  a.tasks = reinterpret_cast<const mono_slice_task*>(ws);
  a.chain_start = reinterpret_cast<const int32_t*>(ws + ((tb + 15) & ~(size_t)15));
  a.n_chains = n_chains;
  a.out_ptrs = out_ptrs_dev;
  int G = 4;
  while (G < max_dim && G < 32) G <<= 1;  // one float per lane
  const int64_t units = (int64_t)(backward ? (int)ordered.size() : n_chains) * batch_size;
  const int grid = grid_for(units, kThreads / G);
  if (bf16) {
    switch (G) {
      case 4: launch_bf16_layout<4>(backward, grid, a, (int)ordered.size(), s); break;
      case 8: launch_bf16_layout<8>(backward, grid, a, (int)ordered.size(), s); break;
      case 16: launch_bf16_layout<16>(backward, grid, a, (int)ordered.size(), s); break;
      default: launch_bf16_layout<32>(backward, grid, a, (int)ordered.size(), s); break;
    }
  } else if (!backward) {
    switch (G) {
      case 4: layout_fwd_kernel<4><<<grid, kThreads, 0, s>>>(a); break;
      case 8: layout_fwd_kernel<8><<<grid, kThreads, 0, s>>>(a); break;
      case 16: layout_fwd_kernel<16><<<grid, kThreads, 0, s>>>(a); break;
      default: layout_fwd_kernel<32><<<grid, kThreads, 0, s>>>(a); break;
    }
  } else {
    const int nt = (int)ordered.size();
    switch (G) {
      case 4: layout_bwd_kernel<4><<<grid, kThreads, 0, s>>>(a, nt); break;
      case 8: layout_bwd_kernel<8><<<grid, kThreads, 0, s>>>(a, nt); break;
      case 16: layout_bwd_kernel<16><<<grid, kThreads, 0, s>>>(a, nt); break;
      default: layout_bwd_kernel<32><<<grid, kThreads, 0, s>>>(a, nt); break;
    }
  }
  MONO_CHECK_LAUNCH();
  MONO_CUDA(cudaFreeAsync(ws, s));
  // `ordered` / `chain_start` are pageable sources of async copies: wait for them
  MONO_CUDA(cudaStreamSynchronize(s));
}

}  // namespace mono
