// Scalar building blocks of the quantisers, shared by quant.cu and kvcache8.cu: 16-bit <-> fp32 conversions and the INT8 /
// e4m3 rounding instructions.
#pragma once
#include <cstdint>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace sab {

template <typename T>
__device__ __forceinline__ float to_f(T v);
template <>
__device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ int8_t cvt_rni_sat_s8(float x) {  // csrc/numeric_conversion.cuh:144-148
  int r;
  asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(r) : "f"(x));
  return static_cast<int8_t>(r);
}
__device__ __forceinline__ uint32_t pack_e4m3x4_q(float a, float b, float c, float d) {
  uint32_t r;
  asm("{\n\t.reg .b16 lo, hi;\n\t"
      "cvt.rn.satfinite.e4m3x2.f32 lo, %2, %1;\n\t"
      "cvt.rn.satfinite.e4m3x2.f32 hi, %4, %3;\n\t"
      "mov.b32 %0, {lo, hi};\n\t}"
      : "=r"(r)
      : "f"(a), "f"(b), "f"(c), "f"(d));
  return r;
}

}  // namespace sab
