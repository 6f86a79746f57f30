// rowelem.cuh — element types of the rows handed in or back by the caller: float, bf16 (the *_bf16 calls) or fp16
// (the *_f16 calls).  Shared by ops.cu, bwd.cu (through rowops.cuh) and layout.cu.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "engine.h"

namespace mono {

// A lane moves 4 consecutive elements of a row (16 bytes of fp32, 8 of bf16); every add, division and optimizer
// step runs in fp32.  bf16 -> fp32 is exact; fp32 -> bf16 rounds to nearest even.
__device__ __forceinline__ float4 widen_bf16x4(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
// fp16 -> fp32 is exact; fp32 -> fp16 rounds to nearest even (__float2half_rn): beyond the fp16 range to +-inf, below
// half the smallest fp16 subnormal to +-0, the sign of zero kept.
__device__ __forceinline__ float4 widen_f16x4(uint2 u) {
  const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  const __half2 v = __halves2half2(__float2half_rn(lo), __float2half_rn(hi));
  return *reinterpret_cast<const uint32_t*>(&v);
}
// the 4 elements a lane staged with cp_async_row4, as fp32
template <typename T>
__device__ __forceinline__ float4 stage_row4(const float4* slot) { return *slot; }
template <>
__device__ __forceinline__ float4 stage_row4<__nv_bfloat16>(const float4* slot) {
  return widen_bf16x4(*reinterpret_cast<const uint2*>(slot));
}
// streaming store of 4 elements (dst aligned to 4 elements)
__device__ __forceinline__ void stcs_row4(float* dst, const float4& x) { __stcs(reinterpret_cast<float4*>(dst), x); }
__device__ __forceinline__ void stcs_row4(__nv_bfloat16* dst, const float4& x) {
  __stcs(reinterpret_cast<uint2*>(dst), make_uint2(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w)));
}
__device__ __forceinline__ void stcs_row4(__half* dst, const float4& x) {
  __stcs(reinterpret_cast<uint2*>(dst), make_uint2(pack_f16x2(x.x, x.y), pack_f16x2(x.z, x.w)));
}
// plain (write-back) store of 4 elements (dst aligned to 4 elements)
__device__ __forceinline__ void store_row4(float* dst, const float4& x) { *reinterpret_cast<float4*>(dst) = x; }
__device__ __forceinline__ void store_row4(__nv_bfloat16* dst, const float4& x) {
  *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w));
}
__device__ __forceinline__ void store_row4(__half* dst, const float4& x) {
  *reinterpret_cast<uint2*>(dst) = make_uint2(pack_f16x2(x.x, x.y), pack_f16x2(x.z, x.w));
}
__device__ __forceinline__ float to_row_elem(float x, const float*) { return x; }
__device__ __forceinline__ __nv_bfloat16 to_row_elem(float x, const __nv_bfloat16*) { return __float2bfloat16_rn(x); }
__device__ __forceinline__ __half to_row_elem(float x, const __half*) { return __float2half_rn(x); }
// one element of a row as fp32 (exact)
__device__ __forceinline__ float row_elem_f32(float x) { return x; }
__device__ __forceinline__ float row_elem_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float row_elem_f32(__half x) { return __half2float(x); }

}  // namespace mono
