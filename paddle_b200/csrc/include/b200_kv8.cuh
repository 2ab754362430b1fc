// 8-bit KV cache (int8 / fp8 e4m3) element conversions shared by the cache write, decode and paged prefill kernels.
// Quantize (static per-KV-head scales, the block_multihead_attention cache-KV rules): y = (max_bound * quant_scale) * x in fp32;
// int8 rounds with rint (round_type 0) or roundf (1) and then clamps to [min_bound, max_bound]; e4m3 clamps first and then
// converts round-to-nearest-even.  Dequantize: q * dequant_scale.  Every int8 and every e4m3 value is exact in fp32, fp16 and bf16.
#pragma once
#include <cuda_fp8.h>

#include "b200_common.cuh"

namespace b200 {
namespace kv8 {

struct I8 {};     // tag types: the cache element formats
struct E4M3 {};

template <typename KV> __device__ __forceinline__ uint8_t quantize(float x, float a, int round_type, float lo, float hi);
template <> __device__ __forceinline__ uint8_t quantize<I8>(float x, float a, int round_type, float lo, float hi) {
  float y = __fmul_rn(a, x);
  y = round_type == 0 ? rintf(y) : roundf(y);
  y = fmaxf(fminf(y, hi), lo);
  return (uint8_t)(int8_t)(int)y;
}
template <> __device__ __forceinline__ uint8_t quantize<E4M3>(float x, float a, int round_type, float lo, float hi) {
  const float y = fmaxf(fminf(__fmul_rn(a, x), hi), lo);
  return (uint8_t)__nv_cvt_float_to_fp8(y, __NV_SATFINITE, __NV_E4M3);
}

// the 16 cache values of one 16-byte load -> fp32, exactly
template <typename KV> __device__ __forceinline__ void to_float16(const uint4& raw, float (&f)[16]);
template <> __device__ __forceinline__ void to_float16<I8>(const uint4& raw, float (&f)[16]) {
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t u = w[i] ^ 0x80808080u;   // int8 b -> b + 128 in [0, 255]; 2^23 + that byte is exact, minus 2^23 + 128 gives b
#pragma unroll
    for (int e = 0; e < 4; ++e) f[i * 4 + e] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7440u + e)) - 8388736.f;
  }
}
template <> __device__ __forceinline__ void to_float16<E4M3>(const uint4& raw, float (&f)[16]) {
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] >> (16 * e)), __NV_E4M3);
      const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&h));
      f[i * 4 + e * 2] = v.x;
      f[i * 4 + e * 2 + 1] = v.y;
    }
}

}  // namespace kv8
}  // namespace b200
