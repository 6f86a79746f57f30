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
// SCALED (scaled_ kernels): x * *scale in fp32 before the MEAN division (FusedGatherGradKernel's input * scale).
template <typename T, int G, bool SCALED = false>
__device__ __forceinline__ void gather_pool_grad(const T* __restrict__ pooled_grad, int64_t grad_stride, int grad_col,
                                                 const int32_t* __restrict__ emb_offset,
                                                 const int32_t* __restrict__ row_offsets, int64_t n_rows, int dim,
                                                 int pooling, float* __restrict__ grad_fused,
                                                 const float* __restrict__ scale = nullptr) {
  const int gl = Group<G>::gl();
  const float gscale = SCALED ? *scale : 1.f;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t r = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; r < n_rows; r += gstride) {
    const int64_t b = row_offsets ? row_offsets[r] : r;
    const int64_t e = row_offsets ? row_offsets[r + 1] : r + 1;
    const int n = (int)(e - b);
    const float fn = (float)n;
    const T* g = pooled_grad + r * grad_stride + grad_col;
    for (int c = gl; c < dim; c += G) {
      float x = row_elem_f32(__ldg(g + c));
      if (SCALED) x = __fmul_rn(x, gscale);
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

template <int G>
__global__ void __launch_bounds__(kThreads)
scaled_gather_pool_grad_kernel(const float* __restrict__ pooled_grad, int64_t grad_stride, int grad_col,
                               const int32_t* __restrict__ emb_offset, const int32_t* __restrict__ row_offsets,
                               int64_t n_rows, int dim, int pooling, float* __restrict__ grad_fused,
                               const float* __restrict__ scale) {
  gather_pool_grad<float, G, true>(pooled_grad, grad_stride, grad_col, emb_offset, row_offsets, n_rows, dim, pooling,
                                   grad_fused, scale);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
scaled_bf16_gather_pool_grad_kernel(const __nv_bfloat16* __restrict__ pooled_grad, int64_t grad_stride, int grad_col,
                                    const int32_t* __restrict__ emb_offset, const int32_t* __restrict__ row_offsets,
                                    int64_t n_rows, int dim, int pooling, float* __restrict__ grad_fused,
                                    const float* __restrict__ scale) {
  gather_pool_grad<__nv_bfloat16, G, true>(pooled_grad, grad_stride, grad_col, emb_offset, row_offsets, n_rows, dim,
                                           pooling, grad_fused, scale);
}

// The kernel of an fp32 / bf16 pair for pooled rows of element type T
template <typename T, class F32, class BF16>
static constexpr auto by_elem(F32 f32, BF16 bf16) {
  if constexpr (std::is_same<T, float>::value) return f32;
  else return bf16;
}

template <typename T>
void launch_gather_pool(const float* fused_emb, const int32_t* emb_offset, const int32_t* row_offsets,
                        int64_t n_rows, int dim, int pooling, T* out, int64_t out_stride, int out_col,
                        cudaStream_t s) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("gather_pool: SUM or MEAN");
  // One occurrence per output row: MEAN is x / 1, the identity, except that the division would replace a NaN's payload
  // with the canonical NaN.  Pool as SUM (a copy), so every width keeps all 32 bits, as gather_rows_kernel does.
  if (row_offsets == nullptr) pooling = MONO_POOL_SUM;
  const int G = pick_group(dim);
  // the row copy stores 4 elements per lane: 16-byte aligned fp32 output rows, 8-byte aligned bf16 ones
  const bool rows = row_offsets == nullptr && (dim & 3) == 0 && dim <= 4 * G && (out_stride & 3) == 0 &&
                    (out_col & 3) == 0 && (reinterpret_cast<uintptr_t>(fused_emb) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(out) & (4 * sizeof(T) - 1)) == 0;
  by_group(G, [&](auto g) {
    constexpr int GG = decltype(g)::value;
    if (rows) {
      const auto kern = by_elem<T>(gather_rows_kernel<GG>, bf16_gather_rows_kernel<GG>);
      kern<<<resident_grid(kern, n_rows, kThreads), kThreads, 0, s>>>(fused_emb, emb_offset, n_rows, dim, out,
                                                                      out_stride, out_col);
    } else {
      const auto kern = by_elem<T>(gather_pool_kernel<GG>, bf16_gather_pool_kernel<GG>);
      kern<<<grid_for(n_rows, kThreads / G), kThreads, 0, s>>>(fused_emb, emb_offset, row_offsets, n_rows, dim,
                                                              pooling, out, out_stride, out_col);
    }
  });
  MONO_CHECK_LAUNCH();
}

template <typename T>
void launch_gather_pool_grad(const T* pooled_grad, int64_t grad_stride, int grad_col, const int32_t* emb_offset,
                             const int32_t* row_offsets, int64_t n_rows, int dim, int pooling, float* grad_fused,
                             cudaStream_t s, const float* grad_scale) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN) throw ArgError("gather_pool_grad: SUM or MEAN");
  const int G = pick_group(dim * 4);  // one float per lane
  by_group(G, [&](auto g) {
    constexpr int GG = decltype(g)::value;
    if (grad_scale) {
      const auto kern = by_elem<T>(scaled_gather_pool_grad_kernel<GG>, scaled_bf16_gather_pool_grad_kernel<GG>);
      kern<<<grid_for(n_rows, kThreads / G), kThreads, 0, s>>>(pooled_grad, grad_stride, grad_col, emb_offset,
                                                              row_offsets, n_rows, dim, pooling, grad_fused,
                                                              grad_scale);
      return;
    }
    const auto kern = by_elem<T>(gather_pool_grad_kernel<GG>, bf16_gather_pool_grad_kernel<GG>);
    kern<<<grid_for(n_rows, kThreads / G), kThreads, 0, s>>>(pooled_grad, grad_stride, grad_col, emb_offset,
                                                            row_offsets, n_rows, dim, pooling, grad_fused);
  });
  MONO_CHECK_LAUNCH();
}

// ---- pooling of received rows over the parts of a sharded step (ShardedStep.step_parts) ----
// A part as the kernels below see it: blockIdx.y serves one part; offs points at the grouping's row offset of the
// part's first occurrence, so offs[m] is the row of the part's occurrence m (row_offsets index the part's own FIDs).
struct GatherPart {
  const int32_t* offs;
  const int32_t* row_offsets;  // null: one occurrence per row
  int64_t n_rows;
  void* out;                   // T rows of the launch
  int64_t out_stride;
  int32_t out_col, pooling;    // pooling: SUM or MEAN (gather_pool_parts_kernel)
  int32_t seq_len, pad;        // FIRSTN: L (gather_seq_parts_kernel)
};

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, 4)
gather_rows_parts_kernel(const float* __restrict__ rows_in, int dim, const GatherPart* __restrict__ parts) {
  const GatherPart& p = parts[blockIdx.y];
  gather_rows<T, G>(rows_in, p.offs, p.n_rows, dim, reinterpret_cast<T*>(p.out), p.out_stride, p.out_col);
}

template <typename T, int G>
__global__ void __launch_bounds__(kThreads)
gather_pool_parts_kernel(const float* __restrict__ rows_in, int dim, const GatherPart* __restrict__ parts) {
  const GatherPart& p = parts[blockIdx.y];
  gather_pool<T, G>(rows_in, p.offs, p.row_offsets, p.n_rows, dim, p.pooling, reinterpret_cast<T*>(p.out),
                    p.out_stride, p.out_col);
}

// FIRSTN: one lane group per position slot q = r * L + j; position j < n_r is the row of the row's j-th occurrence,
// the rest are +0.0 (as lookup_seq_kernel writes them).  rows_in is 16-byte aligned and dim % 4 == 0.
template <typename T, int G>
__global__ void __launch_bounds__(kThreads)
gather_seq_parts_kernel(const float* __restrict__ rows_in, int dim, const GatherPart* __restrict__ parts) {
  const GatherPart& p = parts[blockIdx.y];
  const int gl = Group<G>::gl();
  const int64_t L = p.seq_len, n_slots = p.n_rows * L;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  T* const out = reinterpret_cast<T*>(p.out) + p.out_col;
  for (int64_t q = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; q < n_slots; q += gstride) {
    const int64_t r = q / L, j = q - r * L;
    int64_t b = r, e = r + 1;
    if (p.row_offsets) {
      b = p.row_offsets[r];
      e = p.row_offsets[r + 1];
    }
    const float* src = j < e - b ? rows_in + p.offs[b + j] : nullptr;
    T* dst = out + r * p.out_stride + j * dim;
    const bool vec = (reinterpret_cast<uintptr_t>(dst) & (4 * sizeof(T) - 1)) == 0;
    for (int c = gl * 4; c < dim; c += G * 4) {
      const float4 x = src ? __ldg(reinterpret_cast<const float4*>(src + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (vec) {
        stcs_row4(dst + c, x);
      } else {
        const float a[4] = {x.x, x.y, x.z, x.w};
        for (int w = 0; w < 4; ++w) dst[c + w] = to_row_elem(a[w], dst);
      }
    }
  }
}

// The kernels of the parts pooling: the row copy (aligned one-FID parts), the pooling kernel, the FirstN kernel
enum GatherKind { kGatherRows, kGatherPool, kGatherSeq, kGatherKinds };

// One launch of a parts pooling kernel over ny parts
template <typename T, int G>
static void launch_gather_parts_kind(int kind, int64_t work, unsigned ny, const float* rows_in, int D,
                                     const GatherPart* parts, cudaStream_t s) {
  if (kind == kGatherRows) {
    const auto kern = gather_rows_parts_kernel<T, G>;
    kern<<<dim3(resident_grid(kern, work, kThreads), ny), kThreads, 0, s>>>(rows_in, D, parts);
  } else if (kind == kGatherPool) {
    const auto kern = gather_pool_parts_kernel<T, G>;
    kern<<<dim3(grid_for(work, kThreads / G), ny), kThreads, 0, s>>>(rows_in, D, parts);
  } else {
    const auto kern = gather_seq_parts_kernel<T, G>;
    kern<<<dim3(resident_grid(kern, work, kThreads / G), ny), kThreads, 0, s>>>(rows_in, D, parts);
  }
  MONO_CHECK_LAUNCH();
}

// Every SUM / MEAN part pooled exactly as launch_gather_pool pools it alone (the row copy for an aligned one-FID part,
// the pooling kernel otherwise), every FIRSTN part by gather_seq_parts_kernel; the parts served by the same kernel share
// one launch, one grid row per part, their arguments in one staged array.
template <typename T>
void launch_gather_pool_parts(mono_mtable* mt, int k, const float* rows_in, const int32_t* occ_offset,
                              const mono_pool_part* parts, int n_parts, cudaStream_t s) {
  const int D = mt->tables[k].dim;
  if ((reinterpret_cast<uintptr_t>(rows_in) & 15) != 0) throw ArgError("gather_pool_parts: 16-byte aligned rows_in");
  const int G = pick_group(D);
  std::vector<GatherPart> by_kind[kGatherKinds];
  int64_t work[kGatherKinds] = {0, 0, 0};
  int order[kGatherKinds], n_kinds = 0;  // kinds in order of first use
  int64_t occ = 0;
  for (int i = 0; i < n_parts; ++i) {
    const mono_pool_part& p = parts[i];
    GatherPart g;
    g.offs = occ_offset + occ;
    g.row_offsets = p.row_offsets_dev;
    g.n_rows = p.n_rows;
    g.out = p.rows_dev;
    g.out_stride = p.stride;
    g.out_col = p.col;
    // one occurrence per row: MEAN is x / 1, pooled as SUM (a copy), as launch_gather_pool does
    g.pooling = p.row_offsets_dev ? p.pooling : MONO_POOL_SUM;
    g.seq_len = p.pooling == MONO_POOL_FIRSTN ? p.max_seq_len : 0;
    g.pad = 0;
    occ += p.n_fids;
    if (p.n_rows == 0) continue;
    const bool rows = p.row_offsets_dev == nullptr && D <= 4 * G && (p.stride & 3) == 0 && (p.col & 3) == 0 &&
                      (reinterpret_cast<uintptr_t>(p.rows_dev) & (4 * sizeof(T) - 1)) == 0;
    const int kind = g.seq_len ? kGatherSeq : rows ? kGatherRows : kGatherPool;
    if (by_kind[kind].empty()) order[n_kinds++] = kind;
    by_kind[kind].push_back(g);
    work[kind] = std::max(work[kind], kind == kGatherSeq ? p.n_rows * p.max_seq_len : p.n_rows);
  }
  if (n_kinds == 0) return;
  const int rb = mt->ring.acquire();
  static_assert(sizeof(GatherPart) * MONO_MAX_POOL_PARTS <= StageRing::kBlockBytes, "the parts fit one staged block");
  size_t off = 0;
  const GatherPart* d[kGatherKinds];
  for (int q = 0; q < n_kinds; ++q) {
    const auto& v = by_kind[order[q]];
    std::memcpy(mt->ring.h(rb) + off, v.data(), sizeof(GatherPart) * v.size());
    d[order[q]] = reinterpret_cast<const GatherPart*>(mt->ring.d(rb) + off);
    off += sizeof(GatherPart) * v.size();
  }
  mt->ring.commit(rb, off, s);
  by_group(G, [&](auto g) {
    for (int q = 0; q < n_kinds; ++q) {
      const int kind = order[q];
      launch_gather_parts_kind<T, decltype(g)::value>(kind, work[kind], (unsigned)by_kind[kind].size(), rows_in, D,
                                                      d[kind], s);
    }
  });
}

template void launch_gather_pool_parts<float>(mono_mtable*, int, const float*, const int32_t*, const mono_pool_part*,
                                              int, cudaStream_t);
template void launch_gather_pool_parts<__nv_bfloat16>(mono_mtable*, int, const float*, const int32_t*,
                                                      const mono_pool_part*, int, cudaStream_t);
template void launch_gather_pool<float>(const float*, const int32_t*, const int32_t*, int64_t, int, int, float*,
                                        int64_t, int, cudaStream_t);
template void launch_gather_pool<__nv_bfloat16>(const float*, const int32_t*, const int32_t*, int64_t, int, int,
                                                __nv_bfloat16*, int64_t, int, cudaStream_t);
template void launch_gather_pool_grad<float>(const float*, int64_t, int, const int32_t*, const int32_t*, int64_t,
                                             int, int, float*, cudaStream_t, const float*);
template void launch_gather_pool_grad<__nv_bfloat16>(const __nv_bfloat16*, int64_t, int, const int32_t*,
                                                     const int32_t*, int64_t, int, int, float*, cudaStream_t,
                                                     const float*);

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
// S: element type of the embedding lists (float, or __half for the f16in_ kernels, widened exactly at the load).
template <typename T, int G, typename S = float>
__device__ __forceinline__ void layout_fwd(const LayoutArgs& a) {
  const S* const* emb = reinterpret_cast<const S* const*>(a.emb_ptrs);
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
        const S* src = nullptr;
        if (q < fnum) {
          const uint64_t fo = a.fid_offset[start + q];
          const int i1 = (int)(fo >> 32), i2 = (int)(fo & 0xffffffffu);
          src = emb[i1] + (int64_t)i2 * a.emb_strides[i1] + first.slice_start;
        }
        for (int c = gl; c < first.dim; c += G)
          dst[q * first.dim + c] = to_row_elem(src ? row_elem_f32(src[c]) : 0.0f, dst);
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
          float x = row_elem_f32(emb[i1][(int64_t)i2 * a.emb_strides[i1] + tk.slice_start + c]);
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

// fp16 embedding lists (rows a transfer_float16 server sent), fp32 or bf16 outputs
template <int G>
__global__ void __launch_bounds__(kThreads) f16in_layout_fwd_kernel(LayoutArgs a) {
  layout_fwd<float, G, __half>(a);
}

template <int G>
__global__ void __launch_bounds__(kThreads) f16in_bf16_layout_fwd_kernel(LayoutArgs a) {
  layout_fwd<__nv_bfloat16, G, __half>(a);
}

// Backward: ScatterGrad (ref: fused_embedding_to_layout.h:286-347) with float atomics, as the
// reference GPU kernel does (BackwardBatchKernel, cu.cc:337-381).
// T: element type of the output gradients, widened exactly; the division and the atomics run in fp32.
// SCALED (scaled_ kernels): each gradient element times *scale in fp32 before the MEAN division
// (layout_tensors_grad_scale * grad, ref: distribution_ops.py:544-550).
template <typename T, int G, bool SCALED = false>
__device__ __forceinline__ void layout_bwd(const LayoutArgs& a, int n_tasks, const float* scale = nullptr) {
  const int gl = Group<G>::gl();
  const float gscale = SCALED ? *scale : 1.f;
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
        if (SCALED) x = __fmul_rn(x, gscale);
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

template <int G>
__global__ void __launch_bounds__(kThreads) scaled_layout_bwd_kernel(LayoutArgs a, int n_tasks, const float* scale) {
  layout_bwd<float, G, true>(a, n_tasks, scale);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
scaled_bf16_layout_bwd_kernel(LayoutArgs a, int n_tasks, const float* scale) {
  layout_bwd<__nv_bfloat16, G, true>(a, n_tasks, scale);
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

void launch_layout(bool backward, float* const* emb_ptrs_dev, const int32_t* emb_strides_dev,
                   int n_emb, const uint64_t* fid_offset, int64_t total_fid,
                   const int32_t* feature_offset, int total_feature, const uint32_t* nfl_offset,
                   int total_nfl, int batch_size, const mono_slice_task* tasks_host, int n_tasks,
                   float* const* out_ptrs_dev, cudaStream_t s, bool bf16, const float* grad_scale, bool f16_in) {
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
  const int nt = (int)ordered.size();
  const int64_t units = (int64_t)(backward ? nt : n_chains) * batch_size;
  const int grid = grid_for(units, kThreads / G);
  by_group(G, [&](auto g) {
    constexpr int GG = decltype(g)::value;
    if (!backward && f16_in && !bf16) f16in_layout_fwd_kernel<GG><<<grid, kThreads, 0, s>>>(a);
    else if (!backward && f16_in) f16in_bf16_layout_fwd_kernel<GG><<<grid, kThreads, 0, s>>>(a);
    else if (!backward && !bf16) layout_fwd_kernel<GG><<<grid, kThreads, 0, s>>>(a);
    else if (!backward) bf16_layout_fwd_kernel<GG><<<grid, kThreads, 0, s>>>(a);
    else if (grad_scale && !bf16) scaled_layout_bwd_kernel<GG><<<grid, kThreads, 0, s>>>(a, nt, grad_scale);
    else if (grad_scale) scaled_bf16_layout_bwd_kernel<GG><<<grid, kThreads, 0, s>>>(a, nt, grad_scale);
    else if (!bf16) layout_bwd_kernel<GG><<<grid, kThreads, 0, s>>>(a, nt);
    else bf16_layout_bwd_kernel<GG><<<grid, kThreads, 0, s>>>(a, nt);
  });
  MONO_CHECK_LAUNCH();
  MONO_CUDA(cudaFreeAsync(ws, s));
  // `ordered` / `chain_start` are pageable sources of async copies: wait for them
  MONO_CUDA(cudaStreamSynchronize(s));
}

// One rounding of fp32 values to fp16 (nearest even): the layout gradient a transfer_float16 worker sends to its
// servers.  4 elements per thread where the pointers allow 16-byte loads, else one.
__global__ void __launch_bounds__(kThreads) round_to_f16_kernel(const float* __restrict__ src, int64_t n,
                                                                 __half* __restrict__ dst, int vec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec) {
    const int64_t n4 = n / 4;
    for (int64_t t = t0; t < n4; t += stride)
      store_row4(dst + 4 * t, reinterpret_cast<const float4*>(src)[t]);
    for (int64_t i = 4 * n4 + t0; i < n; i += stride) dst[i] = __float2half_rn(src[i]);
  } else {
    for (int64_t i = t0; i < n; i += stride) dst[i] = __float2half_rn(src[i]);
  }
}

void launch_round_to_f16(const float* src, int64_t n, __half* dst, cudaStream_t s) {
  if (n <= 0) return;
  const int vec = ((uintptr_t)src % 16 == 0 && (uintptr_t)dst % 8 == 0) ? 1 : 0;
  round_to_f16_kernel<<<grid_for(vec ? (n + 3) / 4 : n, kThreads), kThreads, 0, s>>>(src, n, dst, vec);
  MONO_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------------------
// ReduceSum / ReduceMean / FusedReduceAndSplitGPU (ref: RT/ops/reduce_op.cc:29-89,124-180,232-330,
// reduce_op.cu.cc:290-378): per-occurrence rows pooled per sample and cut into slices.  The reference GPU kernel
// runs one thread per output element with a dependent scalar load chain (cu.cc:308-316); here one lane group per
// (feature, sample), lanes across the slice's columns, occurrence rows staged kRsStage at a time with cp.async and
// added strictly in occurrence order.  Every group handles exactly one (feature, sample): the block scheduler hands
// out blocks as SMs free up, so a long row holds up only its own block (a row cannot be split without changing the
// order of its adds).
// ------------------------------------------------------------------------------------------
struct RsFeat {
  const int32_t* splits;
  float* rows;
  int64_t n_rows, row_stride;
  int32_t pooling, slice0, n_slices;
};
struct RsSlice {
  void* ptr;       // T rows of the slice (forward: written; grad: read)
  int64_t stride;  // T elements between samples
  int32_t dim, col;  // col: first column of the slice in the feature's rows
};
struct RsArgs {
  const RsFeat* feats;
  const RsSlice* slices;
  const int32_t* order;  // the features of this launch's lane-group width
  int64_t units;         // features of this launch x batch
  int64_t batch;
  int32_t* bad;          // optional malformed-splits flag
};

constexpr int kRsStage = 8;  // occurrence rows in flight per lane (8 x 16 B x 256 threads = 32 KB per block)

__device__ __forceinline__ void rs_cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void rs_cp_async4(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}

// Sample b's occurrences [*lo, *lo + n) of feature f.  A range outside [0, n_rows] or decreasing is empty; it, and
// splits that do not start at 0 or end at n_rows, raise the flag.
__device__ __forceinline__ int rs_range(const RsFeat& f, int64_t b, int64_t batch, int32_t* bad, int* lo) {
  int l = __ldg(f.splits + b), h = __ldg(f.splits + b + 1);
  const bool ok = l >= 0 && h >= l && h <= f.n_rows;
  if (bad && (!ok || (b == 0 && l != 0) || (b == batch - 1 && h != f.n_rows))) *bad = 1;
  if (!ok) l = h = 0;
  *lo = l;
  return h - l;
}

// ReduceMeanOp's factor: float multiply = 1.0 / static_cast<float>(count) (reduce_op.cc:81, :172), a double
// division rounded to float; n == 0 gives +inf
__device__ __forceinline__ float rs_mean_factor(int n) { return __double2float_rn(__drcp_rn((double)(float)n)); }

__device__ __forceinline__ float4 rs_load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 rs_load4(const __nv_bfloat16* p) {
  return widen_bf16x4(*reinterpret_cast<const uint2*>(p));
}

// A lane owns 4 columns of a slice per pass: c .. c + 3 when the slice's rows allow 16-byte source and 4-element
// destination accesses, else c, c + G, c + 2G, c + 3G (odd dims, 1-column slices, unaligned columns).
template <typename T>
__device__ __forceinline__ bool rs_vec(const RsFeat& f, const RsSlice& sl, const T* tower_row) {
  return ((sl.dim | sl.col) & 3) == 0 && (f.row_stride & 3) == 0 && (reinterpret_cast<uintptr_t>(f.rows) & 15) == 0 &&
         (sl.stride & 3) == 0 && (reinterpret_cast<uintptr_t>(tower_row) & (4 * sizeof(T) - 1)) == 0;
}

// The occurrence rows of one sum: get() is the address of the current occurrence's column c, advance() moves on
struct RsStridedRows {  // rows row_stride floats apart (ReduceSum)
  const float* p;
  int64_t stride;
  __device__ __forceinline__ const float* get() const { return p; }
  __device__ __forceinline__ void advance() { p += stride; }
};
struct RsOffsetRows {  // rows at float offsets (FillWithOffsetMapGradient)
  const float* base;   // the gradient buffer plus column c
  const int64_t* off;  // the occurrences' float offsets, in occurrence order
  __device__ __forceinline__ const float* get() const { return base + *off; }
  __device__ __forceinline__ void advance() { ++off; }
};

// +0.0 + row_0 + row_1 + ... + row_{n-1}, strictly in that order, for the 4 columns a lane owns (c .. c + 3 when vec,
// else c, c + G, c + 2G, c + 3G below dim), the rows staged kRsStage at a time through the lane's slot of `stage`
template <int G, class Rows>
__device__ __forceinline__ float4 rs_sum_rows(float4 (*stage)[kThreads], float* slot, Rows rows, int n, int c, int dim,
                                              bool vec) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);  // ReduceSumOp's zero-filled output (reduce_op.cc:44)
  for (int j0 = 0; j0 < n; j0 += kRsStage) {
    const int m = min(kRsStage, n - j0);
    for (int k = 0; k < m; ++k, rows.advance()) {
      const float* p = rows.get();
      if (vec) {
        rs_cp_async16(slot + k * kThreads * 4, p);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (c + i * G < dim) rs_cp_async4(slot + k * kThreads * 4 + i, p + i * G);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    for (int k = 0; k < m; ++k) {
      const float4 x = stage[k][threadIdx.x];
      acc.x = __fadd_rn(acc.x, x.x); acc.y = __fadd_rn(acc.y, x.y);
      acc.z = __fadd_rn(acc.z, x.z); acc.w = __fadd_rn(acc.w, x.w);
    }
  }
  return acc;
}

template <typename T, int G>
__device__ __forceinline__ void reduce_split_fwd(const RsArgs& a) {
  __shared__ float4 stage[kRsStage][kThreads];
  const int64_t u = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G;
  if (u >= a.units) return;
  const RsFeat f = a.feats[a.order[u / a.batch]];
  const int64_t b = u % a.batch;
  int lo;
  const int n = rs_range(f, b, a.batch, a.bad, &lo);
  const int gl = Group<G>::gl();
  const float* occ = f.rows + (int64_t)lo * f.row_stride;
  const int64_t rstride = f.row_stride;
  for (int s = f.slice0; s < f.slice0 + f.n_slices; ++s) {
    const RsSlice sl = a.slices[s];
    T* dst = reinterpret_cast<T*>(sl.ptr) + b * sl.stride;
    const bool vec = rs_vec(f, sl, reinterpret_cast<T*>(sl.ptr));
    const int step = vec ? 1 : G;
    float* slot = reinterpret_cast<float*>(&stage[0][threadIdx.x]);
    for (int c = vec ? gl * 4 : gl; c < sl.dim; c += 4 * G) {
      float4 acc = rs_sum_rows<G>(stage, slot, RsStridedRows{occ + sl.col + c, rstride}, n, c, sl.dim, vec);
      if (f.pooling == MONO_POOL_MEAN) {
        const float mult = rs_mean_factor(n);
        acc.x = __fmul_rn(acc.x, mult); acc.y = __fmul_rn(acc.y, mult);
        acc.z = __fmul_rn(acc.z, mult); acc.w = __fmul_rn(acc.w, mult);
      }
      if (vec) {
        store_row4(dst + c, acc);
      } else {
        dst[c] = to_row_elem(acc.x, dst);
        if (c + step < sl.dim) dst[c + step] = to_row_elem(acc.y, dst);
        if (c + 2 * step < sl.dim) dst[c + 2 * step] = to_row_elem(acc.z, dst);
        if (c + 3 * step < sl.dim) dst[c + 3 * step] = to_row_elem(acc.w, dst);
      }
    }
  }
}

// Every occurrence row of sample b gets b's slice gradients: copied (SUM) or times the forward's factor (MEAN).
// SCALED (scaled_ kernels): each gradient element times *scale in fp32 where it is loaded, before the MEAN factor.
template <typename T, int G, bool SCALED = false>
__device__ __forceinline__ void reduce_split_bwd(const RsArgs& a, const float* scale = nullptr) {
  const int64_t u = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G;
  if (u >= a.units) return;
  const RsFeat f = a.feats[a.order[u / a.batch]];
  const int64_t b = u % a.batch;
  int lo;
  const int n = rs_range(f, b, a.batch, a.bad, &lo);
  if (n == 0) return;
  const float mult = rs_mean_factor(n);
  const bool mean = f.pooling == MONO_POOL_MEAN;
  const float gscale = SCALED ? *scale : 1.f;
  const int gl = Group<G>::gl();
  float* occ = f.rows + (int64_t)lo * f.row_stride;
  for (int s = f.slice0; s < f.slice0 + f.n_slices; ++s) {
    const RsSlice sl = a.slices[s];
    const T* g = reinterpret_cast<const T*>(sl.ptr) + b * sl.stride;
    const bool vec = rs_vec(f, sl, reinterpret_cast<const T*>(sl.ptr));
    for (int c = vec ? gl * 4 : gl; c < sl.dim; c += 4 * G) {
      float* dst = occ + sl.col + c;
      if (vec) {
        float4 x = rs_load4(g + c);
        if (SCALED) {
          x.x = __fmul_rn(x.x, gscale); x.y = __fmul_rn(x.y, gscale);
          x.z = __fmul_rn(x.z, gscale); x.w = __fmul_rn(x.w, gscale);
        }
        if (mean) {
          x.x = __fmul_rn(x.x, mult); x.y = __fmul_rn(x.y, mult);
          x.z = __fmul_rn(x.z, mult); x.w = __fmul_rn(x.w, mult);
        }
        for (int j = 0; j < n; ++j) *reinterpret_cast<float4*>(dst + (int64_t)j * f.row_stride) = x;
      } else {
        float x[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          x[i] = c + i * G < sl.dim ? row_elem_f32(g[c + i * G]) : 0.f;
          if (SCALED) x[i] = __fmul_rn(x[i], gscale);
          if (mean) x[i] = __fmul_rn(x[i], mult);
        }
        for (int j = 0; j < n; ++j) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (c + i * G < sl.dim) dst[(int64_t)j * f.row_stride + i * G] = x[i];
        }
      }
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads, 4) reduce_split_fwd_kernel(RsArgs a) {
  reduce_split_fwd<float, G>(a);
}

template <int G>
__global__ void __launch_bounds__(kThreads, 4) bf16_reduce_split_fwd_kernel(RsArgs a) {
  reduce_split_fwd<__nv_bfloat16, G>(a);
}

template <int G>
__global__ void __launch_bounds__(kThreads) reduce_split_bwd_kernel(RsArgs a) {
  reduce_split_bwd<float, G>(a);
}

template <int G>
__global__ void __launch_bounds__(kThreads) bf16_reduce_split_bwd_kernel(RsArgs a) {
  reduce_split_bwd<__nv_bfloat16, G>(a);
}

// the two above with every gradient element multiplied by *scale (the _scaled calls' grad_scale_dev)
template <int G>
__global__ void __launch_bounds__(kThreads) scaled_reduce_split_bwd_kernel(RsArgs a, const float* scale) {
  reduce_split_bwd<float, G, true>(a, scale);
}

template <int G>
__global__ void __launch_bounds__(kThreads) scaled_bf16_reduce_split_bwd_kernel(RsArgs a, const float* scale) {
  reduce_split_bwd<__nv_bfloat16, G, true>(a, scale);
}

// Host-side checks of the records: the kernels index with every field unchecked.
void check_reduce_split(const mono_reduce_feature* feats, int F) {
  if (F < 0 || F > (1 << 20)) throw ArgError("reduce_and_split: num_features outside [0, 2^20]");
  if (F > 0 && feats == nullptr) throw ArgError("reduce_and_split: features is null");
  for (int i = 0; i < F; ++i) {
    const mono_reduce_feature& f = feats[i];
    if (f.batch_size < 0 || f.batch_size > INT32_MAX - 1)
      throw ArgError("reduce_and_split: batch_size outside [0, 2^31 - 2]");
    if (f.batch_size != feats[0].batch_size) throw ArgError("reduce_and_split: features with different batch sizes");
    if (f.dim <= 0) throw ArgError("reduce_and_split: dim must be positive");
    if (f.n_rows < 0 || f.n_rows > INT32_MAX) throw ArgError("reduce_and_split: n_rows outside [0, 2^31 - 1]");
    if (f.row_stride < f.dim) throw ArgError("reduce_and_split: row_stride < dim");
    if (f.batch_size > 0 && (f.splits_dev == nullptr || (f.rows_dev == nullptr && f.n_rows > 0)))
      throw ArgError("reduce_and_split: null splits or rows");
    if (f.pooling != MONO_POOL_SUM && f.pooling != MONO_POOL_MEAN)
      throw ArgError("reduce_and_split: pooling must be SUM or MEAN");
    if (f.n_slices <= 0 || f.slices == nullptr) throw ArgError("reduce_and_split: a feature needs slices");
    int64_t cols = 0;
    for (int s = 0; s < f.n_slices; ++s) {
      const mono_reduce_slice& sl = f.slices[s];
      if (sl.dim <= 0) throw ArgError("reduce_and_split: slice dim must be positive");
      if (sl.stride < sl.dim) throw ArgError("reduce_and_split: slice stride < slice dim");
      if (sl.out_dev == nullptr && f.batch_size > 0) throw ArgError("reduce_and_split: null slice pointer");
      cols += sl.dim;
    }
    if (cols != f.dim) throw ArgError("reduce_and_split: slice dims must add up to dim");
  }
  if (F > 0 && (int64_t)F * feats[0].batch_size > ((int64_t)1 << 33))
    throw ArgError("reduce_and_split: features x batch_size over 2^33");
}

template <typename T>
void launch_reduce_split(bool backward, const mono_reduce_feature* feats, int F, int32_t* bad_dev, cudaStream_t s,
                         const float* grad_scale) {
  if (bad_dev) MONO_CUDA(cudaMemsetAsync(bad_dev, 0, sizeof(int32_t), s));
  const int64_t B = F > 0 ? feats[0].batch_size : 0;
  if (F == 0 || B == 0) return;
  // staged tables: features, slices, then the features ordered by lane-group width
  int S = 0;
  for (int i = 0; i < F; ++i) S += feats[i].n_slices;
  const size_t fb = sizeof(RsFeat) * F, sb = sizeof(RsSlice) * S, ob = sizeof(int32_t) * F;
  const size_t o_sl = (fb + 15) & ~(size_t)15, o_ord = (o_sl + sb + 15) & ~(size_t)15, bytes = o_ord + ob;
  std::vector<char> h(bytes);
  RsFeat* hf = reinterpret_cast<RsFeat*>(h.data());
  RsSlice* hs = reinterpret_cast<RsSlice*>(h.data() + o_sl);
  int32_t* ho = reinterpret_cast<int32_t*>(h.data() + o_ord);
  std::vector<int> width(F);
  int count[4] = {0, 0, 0, 0};  // features per width 4, 8, 16, 32
  for (int i = 0, s0 = 0; i < F; ++i) {
    const mono_reduce_feature& f = feats[i];
    hf[i] = RsFeat{f.splits_dev, f.rows_dev, f.n_rows, f.row_stride, f.pooling, s0, f.n_slices};
    int col = 0, widest = 0;
    for (int j = 0; j < f.n_slices; ++j, ++s0) {
      hs[s0] = RsSlice{f.slices[j].out_dev, f.slices[j].stride, f.slices[j].dim, col};
      col += f.slices[j].dim;
      widest = std::max(widest, f.slices[j].dim);
    }
    width[i] = pick_group(widest);  // 4 columns per lane
    ++count[__builtin_ctz(width[i]) - 2];
  }
  int start[5] = {0, 0, 0, 0, 0};
  for (int w = 0; w < 4; ++w) start[w + 1] = start[w] + count[w];
  int fill[4] = {start[0], start[1], start[2], start[3]};
  for (int i = 0; i < F; ++i) ho[fill[__builtin_ctz(width[i]) - 2]++] = i;

  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, bytes, s));
  // a pageable H2D copy is staged by the driver before the call returns: h may go out of scope after it
  MONO_CUDA(cudaMemcpyAsync(ws, h.data(), bytes, cudaMemcpyHostToDevice, s));
  for (int w = 0; w < 4; ++w) {
    if (count[w] == 0) continue;
    RsArgs a;
    a.feats = reinterpret_cast<const RsFeat*>(ws);
    a.slices = reinterpret_cast<const RsSlice*>(ws + o_sl);
    a.order = reinterpret_cast<const int32_t*>(ws + o_ord) + start[w];
    a.units = (int64_t)count[w] * B;
    a.batch = B;
    a.bad = bad_dev;
    by_group(4 << w, [&](auto g) {
      constexpr int GG = decltype(g)::value;
      const int64_t grid = (a.units + kThreads / GG - 1) / (kThreads / GG);
      if (!backward) by_elem<T>(reduce_split_fwd_kernel<GG>, bf16_reduce_split_fwd_kernel<GG>)
                         <<<(unsigned)grid, kThreads, 0, s>>>(a);
      else if (grad_scale) by_elem<T>(scaled_reduce_split_bwd_kernel<GG>, scaled_bf16_reduce_split_bwd_kernel<GG>)
                               <<<(unsigned)grid, kThreads, 0, s>>>(a, grad_scale);
      else by_elem<T>(reduce_split_bwd_kernel<GG>, bf16_reduce_split_bwd_kernel<GG>)
               <<<(unsigned)grid, kThreads, 0, s>>>(a);
    });
    MONO_CHECK_LAUNCH();
  }
  MONO_CUDA(cudaFreeAsync(ws, s));
}

template void launch_reduce_split<float>(bool, const mono_reduce_feature*, int, int32_t*, cudaStream_t,
                                         const float*);
template void launch_reduce_split<__nv_bfloat16>(bool, const mono_reduce_feature*, int, int32_t*, cudaStream_t,
                                                 const float*);

// ------------------------------------------------------------------------------------------
// FillWithOffsetMap and its gradient (ref: RT/ops/unique_mapping_ops.cc:204-329): the n rows of one parameter server,
// row t of table k(t) (pos_split) with dims[k] floats, packed in row order, and each row's unique key pos[t], whose
// occurrences sit at value_offset[value_offset_split[pos[t]] ..].  The forward is the ReduceSum gradient's broadcast
// copy and the gradient the ReduceSum forward's sequential sum (rs_sum_rows), with occurrence rows addressed through
// value_offset instead of a row stride.  The forward runs over occurrences so that a hot key's copies spread over
// the grid; the gradient keeps one lane group per row, its adds in occurrence order.
// ------------------------------------------------------------------------------------------
struct FoStage {
  int64_t* split;  // [K + 1] pos_split
  int64_t* base;   // [K]     float offset of table k's first row in the packed rows
  int32_t* dims;   // [K]
};

struct FoArgs {
  const int64_t* pos;
  int64_t n;                  // rows
  int K;
  FoStage st;
  const int64_t* value_offset;
  const int64_t* value_offset_split;
  int64_t num_unique;
  int32_t* bad;
};

// table of row t: the last k with split[k] <= t
__device__ __forceinline__ int fo_table(const int64_t* __restrict__ split, int K, int64_t t) {
  int lo = 0, hi = K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (split[mid] <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// row t: its table, dim and first float in the packed rows; false (and bad = 1) for a pos outside [0, num_unique)
__device__ __forceinline__ bool fo_row(const FoArgs& a, int64_t t, int* dim, int64_t* row, int64_t* occ_lo,
                                       int64_t* occ_n) {
  const int k = a.K > 1 ? fo_table(a.st.split, a.K, t) : 0;
  *dim = a.st.dims[k];
  *row = a.st.base[k] + (t - a.st.split[k]) * *dim;
  const int64_t p = a.pos[t];
  if (p < 0 || p >= a.num_unique) {
    *a.bad = 1;
    *occ_lo = *occ_n = 0;
    return false;
  }
  *occ_lo = a.value_offset_split[p];
  *occ_n = a.value_offset_split[p + 1] - *occ_lo;
  return true;
}

// The forward's occurrences are spread over the whole grid, so that a hot key's copies run in parallel: a three-pass
// scan of the rows' occurrence counts (tile sums of kFillRows rows, one block over the tile sums, the rows' starts),
// then one lane group per occurrence, which finds its row by binary search over the starts.
constexpr int kFillRows = 4 * kThreads;

// tile_occ[b] = occurrences of tile b's rows
__global__ void __launch_bounds__(kThreads) fill_count_kernel(FoArgs a, int64_t n_tiles, int64_t* __restrict__ tile_occ) {
  __shared__ int64_t wsum[kThreads / 32];
  for (int64_t b = blockIdx.x; b < n_tiles; b += gridDim.x) {
    int64_t sum = 0;
    for (int i = threadIdx.x; i < kFillRows; i += kThreads) {
      const int64_t t = b * kFillRows + i;
      if (t >= a.n) break;
      int dim;
      int64_t row, lo, n;
      fo_row(a, t, &dim, &row, &lo, &n);
      sum += n;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
      int64_t tot = 0;
      for (int w = 0; w < kThreads / 32; ++w) tot += wsum[w];
      tile_occ[b] = tot;
    }
    __syncthreads();
  }
}

// one block: in-place exclusive scan of v[0, n), v[n] = the total
__global__ void __launch_bounds__(1024) fill_scan_kernel(int64_t* __restrict__ v, int64_t n) {
  __shared__ int64_t wsum[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t per = (n + 1023) / 1024;
  const int64_t b = min(n, (int64_t)threadIdx.x * per), e = min(n, b + per);
  int64_t sum = 0;
  for (int64_t i = b; i < e; ++i) sum += v[i];
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
  for (int64_t i = b; i < e; ++i) {
    const int64_t c = v[i];
    v[i] = run;
    run += c;
  }
  if (threadIdx.x == 1023) v[n] = wsum[31];
}

// occ_start[t] = tile_off[tile of t] + occurrences of the rows before t in its tile; occ_start[n] = the total
__global__ void __launch_bounds__(kThreads)
fill_rows_kernel(FoArgs a, int64_t n_tiles, const int64_t* __restrict__ tile_off, int64_t* __restrict__ occ_start) {
  constexpr int R = kFillRows / kThreads;  // rows per thread: thread i owns rows R i .. R i + R - 1 of the tile
  __shared__ int64_t wsum[kThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int64_t b = blockIdx.x; b < n_tiles; b += gridDim.x) {
    const int64_t t0 = b * kFillRows;
    int64_t cnt[R], sum = 0;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t t = t0 + threadIdx.x * R + r;
      cnt[r] = 0;
      if (t < a.n) {
        int dim;
        int64_t row, lo;
        fo_row(a, t, &dim, &row, &lo, &cnt[r]);
      }
      sum += cnt[r];
    }
    int64_t x = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    int64_t run = tile_off[b] + x - sum;
    for (int ww = 0; ww < w; ++ww) run += wsum[ww];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int64_t t = t0 + threadIdx.x * R + r;
      if (t < a.n) occ_start[t] = run;
      run += cnt[r];
    }
    if (b == n_tiles - 1 && threadIdx.x == 0) occ_start[a.n] = tile_off[n_tiles];
    __syncthreads();
  }
}

// one lane group per occurrence q: the row t whose occurrences hold q (the last t with occ_start[t] <= q), copied
// to the occurrence's offset.  T: element type of the server's rows, float or __half (widened exactly where loaded).
template <typename T, int G>
__device__ __forceinline__ void fill_copy(const FoArgs& a, const int64_t* __restrict__ occ_start,
                                          const T* __restrict__ value, float* __restrict__ buffer) {
  const int gl = Group<G>::gl();
  const int64_t total = occ_start[a.n];
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t q = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; q < total; q += gstride) {
    int64_t lo = 0, hi = a.n - 1;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (occ_start[mid] <= q) lo = mid; else hi = mid - 1;
    }
    const int k = a.K > 1 ? fo_table(a.st.split, a.K, lo) : 0;
    const int dim = a.st.dims[k];
    const T* src = value + a.st.base[k] + (lo - a.st.split[k]) * dim;
    float* dst = buffer + a.value_offset[a.value_offset_split[a.pos[lo]] + (q - occ_start[lo])];
    for (int c = gl; c < dim; c += G) dst[c] = row_elem_f32(__ldg(src + c));
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads)
fill_copy_kernel(FoArgs a, const int64_t* __restrict__ occ_start, const float* __restrict__ value,
                 float* __restrict__ buffer) {
  fill_copy<float, G>(a, occ_start, value, buffer);
}

// mono_fill_with_offset_map_f16: fp16 server rows
template <int G>
__global__ void __launch_bounds__(kThreads)
f16_fill_copy_kernel(FoArgs a, const int64_t* __restrict__ occ_start, const __half* __restrict__ value,
                     float* __restrict__ buffer) {
  fill_copy<__half, G>(a, occ_start, value, buffer);
}

// one lane group per row: out row t = +0.0 + g[o_1 ..] + g[o_2 ..] + ... over its key's occurrences, in order.
// T: element type of the output rows, float or __half (the fp32 sum rounded once where it is stored).
template <typename T, int G>
__device__ __forceinline__ void fill_grad(const FoArgs& a, const float* __restrict__ grad, T* __restrict__ out) {
  __shared__ float4 stage[kRsStage][kThreads];
  const int64_t t = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G;
  if (t >= a.n) return;
  int dim;
  int64_t row, lo, n;
  fo_row(a, t, &dim, &row, &lo, &n);
  const int gl = Group<G>::gl();
  float* slot = reinterpret_cast<float*>(&stage[0][threadIdx.x]);
  for (int c = gl; c < dim; c += 4 * G) {
    const float4 acc = rs_sum_rows<G>(stage, slot, RsOffsetRows{grad + c, a.value_offset + lo}, (int)n, c, dim, false);
    T* dst = out + row + c;
    dst[0] = to_row_elem(acc.x, dst);
    if (c + G < dim) dst[G] = to_row_elem(acc.y, dst);
    if (c + 2 * G < dim) dst[2 * G] = to_row_elem(acc.z, dst);
    if (c + 3 * G < dim) dst[3 * G] = to_row_elem(acc.w, dst);
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads, 4)
fill_grad_kernel(FoArgs a, const float* __restrict__ grad, float* __restrict__ out) {
  fill_grad<float, G>(a, grad, out);
}

// mono_fill_with_offset_map_grad_f16: fp16 output rows
template <int G>
__global__ void __launch_bounds__(kThreads, 4)
f16_fill_grad_kernel(FoArgs a, const float* __restrict__ grad, __half* __restrict__ out) {
  fill_grad<__half, G>(a, grad, out);
}

// Host-side checks and the staged tables; returns the packed rows' float count
static int64_t fill_setup(const int64_t* pos_split_host, int K, const int32_t* dims_host, std::vector<char>* h,
                          size_t* o_base, size_t* o_dims, int* max_dim) {
  if (K <= 0) throw ArgError("fill_with_offset_map: num_tables must be positive");
  if (pos_split_host[0] != 0) throw ArgError("fill_with_offset_map: pos_split must start at 0");
  int64_t floats = 0;
  *max_dim = 1;
  const size_t o_split = 0;
  *o_base = (sizeof(int64_t) * (K + 1) + 15) & ~(size_t)15;
  *o_dims = *o_base + sizeof(int64_t) * K;
  h->assign(*o_dims + sizeof(int32_t) * K, 0);
  int64_t* split = reinterpret_cast<int64_t*>(h->data() + o_split);
  int64_t* base = reinterpret_cast<int64_t*>(h->data() + *o_base);
  int32_t* dims = reinterpret_cast<int32_t*>(h->data() + *o_dims);
  for (int k = 0; k < K; ++k) {
    if (pos_split_host[k + 1] < pos_split_host[k]) throw ArgError("fill_with_offset_map: pos_split must not decrease");
    if (dims_host[k] <= 0) throw ArgError("fill_with_offset_map: dims must be positive");
    base[k] = floats;
    floats += (pos_split_host[k + 1] - pos_split_host[k]) * dims_host[k];
    *max_dim = std::max(*max_dim, dims_host[k]);
  }
  std::memcpy(split, pos_split_host, sizeof(int64_t) * (K + 1));
  std::memcpy(dims, dims_host, sizeof(int32_t) * K);
  if (pos_split_host[K] > ((int64_t)1 << 30)) throw ArgError("fill_with_offset_map: more than 2^30 rows in one call");
  return floats;
}

void run_fill_offset_map(bool grad, int device, const int64_t* pos_dev, const int64_t* pos_split_host, int K,
                         const int32_t* dims_host, const float* src_dev, int64_t src_len,
                         const int64_t* value_offset_dev, const int64_t* value_offset_split_dev, int64_t num_unique,
                         float* dst_dev, int32_t* bad_dev, cudaStream_t s, bool f16) {
  std::vector<char> h;
  size_t o_base, o_dims;
  int max_dim;
  const int64_t floats = fill_setup(pos_split_host, K, dims_host, &h, &o_base, &o_dims, &max_dim);
  const char* who = grad ? "fill_with_offset_map_gradient" : "fill_with_offset_map";
  if (num_unique < 0 || num_unique > ((int64_t)1 << 30))
    throw ArgError(std::string(who) + ": num_unique must be in [0, 2^30]");
  // ref: FillWithOffsetMapOp's value size check, unique_mapping_ops.cc:233-235 (a longer value is accepted)
  if (!grad && src_len < floats)
    throw ArgError("fill_with_offset_map: Value size doesn't match expected size. expected: " + std::to_string(floats) +
                   ", actual: " + std::to_string(src_len));
  const int64_t n = pos_split_host[K];
  if (n > 0 && !(pos_dev && src_dev && value_offset_dev && value_offset_split_dev && dst_dev))
    throw ArgError(std::string(who) + ": null argument");
  MONO_CUDA(cudaSetDevice(device));
  const size_t o_bad = (h.size() + 15) & ~(size_t)15, o_occ = o_bad + 16;
  const int64_t n_tiles = (n + kFillRows - 1) / kFillRows;
  const size_t bytes = o_occ + (grad ? 0 : sizeof(int64_t) * (n_tiles + 1 + n + 1));
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, bytes, s));
  // a pageable H2D copy is staged by the driver before the call returns: h may go out of scope after it
  MONO_CUDA(cudaMemcpyAsync(ws, h.data(), h.size(), cudaMemcpyHostToDevice, s));
  MONO_CUDA(cudaMemsetAsync(ws + o_bad, 0, 16, s));
  FoArgs a;
  a.pos = pos_dev;
  a.n = n;
  a.K = K;
  a.st.split = reinterpret_cast<int64_t*>(ws);
  a.st.base = reinterpret_cast<int64_t*>(ws + o_base);
  a.st.dims = reinterpret_cast<int32_t*>(ws + o_dims);
  a.value_offset = value_offset_dev;
  a.value_offset_split = value_offset_split_dev;
  a.num_unique = num_unique;
  a.bad = reinterpret_cast<int32_t*>(ws + o_bad);
  if (n > 0) {
    if (grad) {
      by_group(pick_group(max_dim), [&](auto g) {
        constexpr int GG = decltype(g)::value;
        const unsigned grid = (unsigned)((n + kThreads / GG - 1) / (kThreads / GG));
        if (f16)
          f16_fill_grad_kernel<GG><<<grid, kThreads, 0, s>>>(a, src_dev, reinterpret_cast<__half*>(dst_dev));
        else
          fill_grad_kernel<GG><<<grid, kThreads, 0, s>>>(a, src_dev, dst_dev);
      });
      MONO_CHECK_LAUNCH();
    } else {
      int64_t* tile_off = reinterpret_cast<int64_t*>(ws + o_occ);
      int64_t* occ_start = tile_off + n_tiles + 1;
      fill_count_kernel<<<grid_for(n_tiles, 1), kThreads, 0, s>>>(a, n_tiles, tile_off);
      MONO_CHECK_LAUNCH();
      fill_scan_kernel<<<1, 1024, 0, s>>>(tile_off, n_tiles);
      MONO_CHECK_LAUNCH();
      fill_rows_kernel<<<grid_for(n_tiles, 1), kThreads, 0, s>>>(a, n_tiles, tile_off, occ_start);
      MONO_CHECK_LAUNCH();
      // the occurrence count is on the device: one resident wave, grid-stride
      by_group(pick_group(max_dim * 4), [&](auto g) {  // one element per lane
        constexpr int GG = decltype(g)::value;
        if (f16)
          f16_fill_copy_kernel<GG><<<resident_grid(f16_fill_copy_kernel<GG>, INT32_MAX, 1), kThreads, 0, s>>>(
              a, occ_start, reinterpret_cast<const __half*>(src_dev), dst_dev);
        else
          fill_copy_kernel<GG><<<resident_grid(fill_copy_kernel<GG>, INT32_MAX, 1), kThreads, 0, s>>>(a, occ_start,
                                                                                                      src_dev, dst_dev);
      });
      MONO_CHECK_LAUNCH();
    }
  }
  if (bad_dev) MONO_CUDA(cudaMemcpyAsync(bad_dev, a.bad, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  MONO_CUDA(cudaFreeAsync(ws, s));
}

}  // namespace mono
