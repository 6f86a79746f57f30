// clip.cu — the global L2 norm of a list of gradient tensors and the ClipByGlobalNorm scale, on the device
// (ref: GlobalL2Reduce, RT/ops/global_norm.cu.cc; the scale rule of ClipByGlobalNorm, clip_by_global_norm.h:42-49).
// The reference sums fp32 squares with float atomics across blocks, so its bits vary from run to run.  Here every
// square is exact in fp64 and the fp64 sum has one fixed association, a function of the tensors' sizes only (not of
// the grid, the SM count or timing), stated in include/mono_emb.h at mono_global_norm:
//   chunks of kNormChunk elements that never cross a tensor boundary; thread t of kNormThreads adds the squares of
//   the chunk's elements t + kNormThreads * i, in increasing i, from +0.0; then s[t] += s[t + h] for
//   h = kNormThreads / 2 ... 1.  The chunk partials, in (tensor, chunk) order, are reduced by the same rule until one
//   value is left.
// Two launches: norm_partials_kernel (one block per chunk, grid-stride), then norm_combine_kernel (one block: the
// levels of the partials' reduction, the sqrt and the scale).  Nothing returns to the host.
#include <cuda_bf16.h>

#include <cstring>
#include <vector>

#include "engine.h"

namespace mono {

constexpr int kNormThreads = 256;
constexpr int kNormChunk = 8192;
constexpr int kNormPer = kNormChunk / kNormThreads;  // elements of a chunk per thread
static_assert(kNormThreads == kThreads, "one block shape for the engine's kernels");

struct NormTensor {
  const void* data;
  int64_t n;
  int64_t chunk0;  // first chunk of the tensor in (tensor, chunk) order
  int32_t dtype;   // MONO_DTYPE_F32 | MONO_DTYPE_BF16
  int32_t pad;
};

// s[t] += s[t + h] for h = kNormThreads / 2 ... 1; returns s[0] in thread 0
__device__ __forceinline__ double tree_sum(double v, double* s) {
  s[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int h = kNormThreads / 2; h >= 1; h >>= 1) {
    if ((int)threadIdx.x < h) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + h]);
    __syncthreads();
  }
  const double r = s[0];
  __syncthreads();  // s is reused by the caller's next chunk
  return r;
}

__device__ __forceinline__ float elem_f32(const void* p, int32_t dtype, int64_t i) {
  return dtype == MONO_DTYPE_BF16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i])
                                  : static_cast<const float*>(p)[i];
}

// One block per chunk (grid-stride).  The chunk is staged into shared memory as fp32 with 16-byte loads when the
// chunk start is 16-byte aligned (the scalar loop otherwise, and for the ragged tail), so that every thread then
// reads exactly the elements t + kNormThreads * i that the fixed order gives it.  Elements past the tensor's end are
// staged as +0.0: adding +0.0 to a sum of squares (>= +0.0, inf or NaN) leaves its bits unchanged.
__global__ void __launch_bounds__(kNormThreads)
norm_partials_kernel(const NormTensor* __restrict__ tensors, int n_tensors, int64_t n_chunks,
                     double* __restrict__ partials) {
  __shared__ float4 stage4[kNormChunk / 4];
  __shared__ double red[kNormThreads];
  float* stage = reinterpret_cast<float*>(stage4);
  for (int64_t q = blockIdx.x; q < n_chunks; q += gridDim.x) {
    int lo = 0, hi = n_tensors - 1;  // the last tensor whose chunks start at or before q
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tensors[mid].chunk0 <= q) lo = mid;
      else hi = mid - 1;
    }
    const NormTensor tn = tensors[lo];
    const int64_t first = (q - tn.chunk0) * kNormChunk;
    const int len = (int)min((int64_t)kNormChunk, tn.n - first);
    if (tn.dtype == MONO_DTYPE_BF16) {
      const __nv_bfloat16* src = static_cast<const __nv_bfloat16*>(tn.data) + first;
      if (len == kNormChunk && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
#pragma unroll
        for (int k = 0; k < kNormChunk / 8 / kNormThreads; ++k) {
          const int v = threadIdx.x + k * kNormThreads;
          const uint4 w = __ldcs(s4 + v);
          const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {  // bf16 -> fp32 is the bit pattern shifted into the high half: exact
            stage[8 * v + 2 * j] = __uint_as_float(u[j] << 16);
            stage[8 * v + 2 * j + 1] = __uint_as_float(u[j] & 0xFFFF0000u);
          }
        }
      } else {
        for (int i = threadIdx.x; i < kNormChunk; i += kNormThreads)
          stage[i] = i < len ? __bfloat162float(src[i]) : 0.f;
      }
    } else {
      const float* src = static_cast<const float*>(tn.data) + first;
      if (len == kNormChunk && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
        for (int k = 0; k < kNormChunk / 4 / kNormThreads; ++k) {
          const int v = threadIdx.x + k * kNormThreads;
          stage4[v] = __ldcs(s4 + v);
        }
      } else {
        for (int i = threadIdx.x; i < kNormChunk; i += kNormThreads) stage[i] = i < len ? src[i] : 0.f;
      }
    }
    __syncthreads();
    double acc = 0.0;
#pragma unroll
    for (int i = 0; i < kNormPer; ++i) {
      const double x = (double)stage[threadIdx.x + i * kNormThreads];
      acc = __dadd_rn(acc, __dmul_rn(x, x));  // the square of an fp32 value is exact in fp64
    }
    const double r = tree_sum(acc, red);  // its trailing barrier also frees `stage` for the next chunk
    if (threadIdx.x == 0) partials[q] = r;
  }
}

// One block: the partials reduced level by level by the chunk rule (in place: chunk q of a level is written to
// slot q, which lies in chunk 0 of that level, already read), then norm = sqrtf((float)sum) and the scale.
__global__ void __launch_bounds__(kNormThreads)
norm_combine_kernel(double* __restrict__ partials, int64_t n, float clip_norm, float* __restrict__ norm_out,
                    float* __restrict__ scale_out) {
  __shared__ double red[kNormThreads];
  while (n > 1) {
    const int64_t m = (n + kNormChunk - 1) / kNormChunk;
    for (int64_t q = 0; q < m; ++q) {
      double acc = 0.0;
#pragma unroll 4
      for (int i = 0; i < kNormPer; ++i) {
        const int64_t k = q * kNormChunk + threadIdx.x + (int64_t)i * kNormThreads;
        if (k < n) acc = __dadd_rn(acc, partials[k]);
      }
      const double r = tree_sum(acc, red);
      if (threadIdx.x == 0) partials[q] = r;
      __syncthreads();
    }
    n = m;
  }
  if (threadIdx.x == 0) {
    const double sum = n == 1 ? partials[0] : 0.0;
    const float norm = sqrtf((float)sum);
    *norm_out = norm;
    // ClipByGlobalNorm: scale only when the norm exceeds clip_norm (a NaN norm compares false: scale 1; an infinite
    // norm gives clip_norm / inf = +0.0)
    if (scale_out) *scale_out = norm > clip_norm ? __fdiv_rn(clip_norm, norm) : 1.0f;
  }
}

void check_global_norm(const mono_norm_tensor* tensors, int n_tensors, float clip_norm, const float* norm_dev,
                       const float* scale_dev) {
  if (n_tensors < 0 || n_tensors > MONO_MAX_NORM_TENSORS) throw ArgError("global_norm: n_tensors outside [0, 4096]");
  if (n_tensors > 0 && !tensors) throw ArgError("global_norm: tensors is null");
  if (!norm_dev) throw ArgError("global_norm: norm_dev is null");
  if (!(clip_norm >= 0.f) || clip_norm == INFINITY) throw ArgError("global_norm: clip_norm must be finite and >= 0");
  if (clip_norm > 0.f && !scale_dev) throw ArgError("global_norm: clip_norm > 0 needs scale_dev");
  for (int i = 0; i < n_tensors; ++i) {
    const mono_norm_tensor& t = tensors[i];
    if (t.n < 0) throw ArgError("global_norm: negative tensor size");
    if (t.n > 0 && !t.data_dev) throw ArgError("global_norm: null tensor data");
    if (t.dtype != MONO_DTYPE_F32 && t.dtype != MONO_DTYPE_BF16) throw ArgError("global_norm: unknown dtype");
  }
}

void launch_global_norm(const mono_norm_tensor* tensors, int n_tensors, float clip_norm, float* norm_dev,
                        float* scale_dev, cudaStream_t s) {
  std::vector<NormTensor> h;
  int64_t chunks = 0;
  for (int i = 0; i < n_tensors; ++i) {
    const mono_norm_tensor& t = tensors[i];
    if (t.n == 0) continue;  // no chunks: leaving it out keeps the search over tensors that own chunks
    h.push_back(NormTensor{t.data_dev, t.n, chunks, t.dtype, 0});
    chunks += (t.n + kNormChunk - 1) / kNormChunk;
  }
  const size_t tb = (sizeof(NormTensor) * h.size() + 15) & ~(size_t)15;
  char* ws = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&ws, tb + sizeof(double) * (size_t)std::max<int64_t>(chunks, 1), s));
  double* partials = reinterpret_cast<double*>(ws + tb);
  if (chunks > 0) {
    // a pageable H2D copy is staged by the driver before the call returns: h may go out of scope after it
    MONO_CUDA(cudaMemcpyAsync(ws, h.data(), sizeof(NormTensor) * h.size(), cudaMemcpyHostToDevice, s));
    const int grid = (int)std::min<int64_t>(chunks, resident_grid(norm_partials_kernel, chunks, 1, kNormThreads));
    norm_partials_kernel<<<grid, kNormThreads, 0, s>>>(reinterpret_cast<const NormTensor*>(ws), (int)h.size(), chunks,
                                                        partials);
    MONO_CHECK_LAUNCH();
  }
  norm_combine_kernel<<<1, kNormThreads, 0, s>>>(partials, chunks, clip_norm, norm_dev,
                                                 clip_norm > 0.f ? scale_dev : nullptr);
  MONO_CHECK_LAUNCH();
  MONO_CUDA(cudaFreeAsync(ws, s));
}

}  // namespace mono
