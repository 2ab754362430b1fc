// Quantizing write of the new K / V rows into a paged int8 / fp8 (e4m3) KV cache, for prefill and decode rows alike, in one launch.
//
// Parity (behaviour): the static cache-KV quantization of block_multihead_attention (QuantHelperFunc in
// paddle/phi/kernels/fusion/gpu/mmha_util.cu.h), extended to e4m3; the rules are in include/b200_kv8.cuh.
//
// The rows are read in place from the packed qkv [T, (H + 2 Hkv) * 128].  Token t belongs to the last sequence i with cu_q[i] <= t; its
// position is (seq_lens_encoder[i] > 0 ? 0 : seq_lens_decoder[i]) + t - cu_q[i], and it goes to block block_tables[i, pos / block_size],
// row pos % block_size.  Everything is found on the device: no host read of the lengths.  Grid (T, ceil(Hkv / 2)), 4 warps: warp w
// writes the K (w < 2) or V row of KV head 2 blockIdx.y + (w & 1), 4 elements per lane.
//
// prologue_write_kernel is the same one-launch write with block_multihead_attention's qkv prologue folded in (int32 dequantization, bias,
// rotary; parity: DequantKernel, the bias add, GQA(Neox)VariableLengthRotaryKernel and CacheKernel in
// paddle/phi/kernels/fusion/gpu/block_attn.h), for 16-bit caches too; out_quant_kernel is the op's out_scale output quantization.
#include <cuda.h>

#include <algorithm>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"

namespace b200 {
namespace kvq {

constexpr int D = 128;

template <typename T, typename KV>
__global__ void __launch_bounds__(128) cache_write_kernel(const T* __restrict__ qkv, int64_t row_stride, uint8_t* __restrict__ kc,
                                                         uint8_t* __restrict__ vc, const int* __restrict__ cu_q, const int* __restrict__ enc,
                                                         const int* __restrict__ dec, const int* __restrict__ block_tables, int b, int max_blocks,
                                                         int block_size, int h, int hkv, const float* __restrict__ k_qs,
                                                         const float* __restrict__ v_qs, int round_type, float max_bound, float min_bound) {
  const int t = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y * 2 + (warp & 1), is_v = warp >> 1;
  if (head >= hkv || t >= __ldg(cu_q + b)) return;   // rows past the last sequence are padding
  int lo = 0, hi = b - 1;                            // last sequence whose first row is <= t (empty sequences share their successor's)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(cu_q + mid) <= t) lo = mid; else hi = mid - 1;
  }
  const int pos = (__ldg(enc + lo) > 0 ? 0 : __ldg(dec + lo)) + t - __ldg(cu_q + lo);
  const int blk = __ldg(block_tables + (int64_t)lo * max_blocks + pos / block_size);
  const T* src = qkv + (int64_t)t * row_stride + (int64_t)(h + is_v * hkv + head) * D + lane * 4;
  const float a = max_bound * __ldg((is_v ? v_qs : k_qs) + head);
  const uint2 raw = *reinterpret_cast<const uint2*>(src);
  const T* x = reinterpret_cast<const T*>(&raw);
  uint32_t packed = 0;
#pragma unroll
  for (int e = 0; e < 4; ++e) packed |= (uint32_t)kv8::quantize<KV>(to_f(x[e]), a, round_type, min_bound, max_bound) << (8 * e);
  uint8_t* dst = (is_v ? vc : kc) + (((int64_t)blk * hkv + head) * block_size + pos % block_size) * D + lane * 4;
  *reinterpret_cast<uint32_t*>(dst) = packed;
}

// ---- the same write with the qkv prologue of block_multihead_attention folded in ------------------------------------------------------
// Per element of every new packed row, in this order (each arrow a rounding to T):
//   int32 rows (IN = int32_t): x = float(qkv[c]) * col_scale[c] -> T;   bias: x = x + bias[c] -> T;
//   rotary on the Q and K heads (ROPE kInterleaved: pairs (2i, 2i + 1); kNeox: pairs (i, i + 64)), with cos / sin fp32 [S, rope_stride]
//   read at the token's position p, column i < 64:  l' = l c - r s,  r' = r c + l s  (every product and sum rounded to fp32, no FMA) -> T.
// The processed row is written to `out` (nullptr: not written; it may be qkv itself), and its K / V heads go to the cache: a 16-bit copy
// (KV = T) or the 8-bit quantization of cache_write_kernel.  Grid (T, ceil((H + 2 Hkv) / 16)), 128 threads: 8 per head; thread j of a
// head owns columns [8j, 8j + 8) and [64 + 8j, 64 + 8j + 8), so a neox pair never leaves its thread and an interleaved pair sits in one
// vector.  Every load and store is 16 bytes wide (8 bytes for an 8-bit cache row).
enum RopeStyle : int { kNoRope = 0, kInterleaved = 1, kNeox = 2 };

template <typename T> __device__ __forceinline__ float round_to(float x) { return to_f(from_f<T>(x)); }

// 8 consecutive elements -> fp32 values of T
template <typename T> __device__ __forceinline__ void load8(const T* p, const float*, float* f) {
  const Vec16<T> v = ld16(p);
#pragma unroll
  for (int e = 0; e < 8; ++e) f[e] = to_f(v.v[e]);
}
template <typename T> __device__ __forceinline__ void load8(const int32_t* p, const float* scale, float* f) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int4 q = *reinterpret_cast<const int4*>(p + 4 * h);
    const float4 s = __ldg(reinterpret_cast<const float4*>(scale + 4 * h));
    f[4 * h + 0] = round_to<T>(__fmul_rn((float)q.x, s.x));
    f[4 * h + 1] = round_to<T>(__fmul_rn((float)q.y, s.y));
    f[4 * h + 2] = round_to<T>(__fmul_rn((float)q.z, s.z));
    f[4 * h + 3] = round_to<T>(__fmul_rn((float)q.w, s.w));
  }
}

__device__ __forceinline__ void rotate(float& l, float& r, float c, float s) {
  const float nl = __fsub_rn(__fmul_rn(l, c), __fmul_rn(r, s));
  r = __fadd_rn(__fmul_rn(r, c), __fmul_rn(l, s));
  l = nl;
}

template <typename T, typename IN, typename KV, int ROPE>
__global__ void __launch_bounds__(128) prologue_write_kernel(const IN* qkv, int64_t row_stride, T* out, int64_t out_stride, uint8_t* __restrict__ kc,
                                                            uint8_t* __restrict__ vc, const int* __restrict__ cu_q, const int* __restrict__ enc,
                                                            const int* __restrict__ dec, const int* __restrict__ block_tables, int b, int max_blocks,
                                                            int block_size, int h, int hkv, const float* __restrict__ col_scale,
                                                            const T* __restrict__ bias, const float* __restrict__ cos_t,
                                                            const float* __restrict__ sin_t, int rope_stride, const float* __restrict__ k_qs,
                                                            const float* __restrict__ v_qs, int round_type, float max_bound, float min_bound) {
  const int t = blockIdx.x, head = blockIdx.y * 16 + (threadIdx.x >> 3), j = threadIdx.x & 7;
  if (head >= h + 2 * hkv || (out == nullptr && head < h) || t >= __ldg(cu_q + b)) return;   // rows past the last sequence are padding
  int lo = 0, hi = b - 1;                                     // last sequence whose first row is <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(cu_q + mid) <= t) lo = mid; else hi = mid - 1;
  }
  const int pos = (__ldg(enc + lo) > 0 ? 0 : __ldg(dec + lo)) + t - __ldg(cu_q + lo);
  const int c0 = head * D + j * 8;
  float x[16];                                                // columns c0 .. c0 + 7, then c0 + 64 .. c0 + 71
  load8<T>(qkv + (int64_t)t * row_stride + c0, col_scale + c0, x);
  load8<T>(qkv + (int64_t)t * row_stride + c0 + 64, col_scale + c0 + 64, x + 8);
  if (bias != nullptr) {
    const Vec16<T> b0 = ld16(bias + c0), b1 = ld16(bias + c0 + 64);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      x[e] = round_to<T>(__fadd_rn(x[e], to_f(b0.v[e])));
      x[8 + e] = round_to<T>(__fadd_rn(x[8 + e], to_f(b1.v[e])));
    }
  }
  if (ROPE != kNoRope && head < h + hkv) {
    const float* cr = cos_t + (int64_t)pos * rope_stride;
    const float* sr = sin_t + (int64_t)pos * rope_stride;
    if (ROPE == kInterleaved) {                               // column 8j + 2m (+ 64) pairs with the next one and uses entry 4j + m (+ 32)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const float4 c = __ldg(reinterpret_cast<const float4*>(cr + 32 * k + 4 * j));
        const float4 s = __ldg(reinterpret_cast<const float4*>(sr + 32 * k + 4 * j));
        rotate(x[8 * k + 0], x[8 * k + 1], c.x, s.x);
        rotate(x[8 * k + 2], x[8 * k + 3], c.y, s.y);
        rotate(x[8 * k + 4], x[8 * k + 5], c.z, s.z);
        rotate(x[8 * k + 6], x[8 * k + 7], c.w, s.w);
      }
    } else {                                                  // column 8j + m pairs with 64 + 8j + m and uses entry 8j + m
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const float4 c = __ldg(reinterpret_cast<const float4*>(cr + 8 * j + 4 * k));
        const float4 s = __ldg(reinterpret_cast<const float4*>(sr + 8 * j + 4 * k));
        rotate(x[4 * k + 0], x[8 + 4 * k + 0], c.x, s.x);
        rotate(x[4 * k + 1], x[8 + 4 * k + 1], c.y, s.y);
        rotate(x[4 * k + 2], x[8 + 4 * k + 2], c.z, s.z);
        rotate(x[4 * k + 3], x[8 + 4 * k + 3], c.w, s.w);
      }
    }
  }
  Vec16<T> y[2];
#pragma unroll
  for (int e = 0; e < 16; ++e) y[e >> 3].v[e & 7] = from_f<T>(x[e]);
  if (out != nullptr) {
    st16(out + (int64_t)t * out_stride + c0, y[0]);
    st16(out + (int64_t)t * out_stride + c0 + 64, y[1]);
  }
  if (head < h) return;
  const int is_v = head >= h + hkv, kvh = head - h - is_v * hkv;
  const int blk = __ldg(block_tables + (int64_t)lo * max_blocks + pos / block_size);
  uint8_t* dst = (is_v ? vc : kc) + (((int64_t)blk * hkv + kvh) * block_size + pos % block_size) * D * (int64_t)sizeof(KV) + j * 8 * sizeof(KV);
  if constexpr (sizeof(KV) == 2) {
    st16(reinterpret_cast<T*>(dst), y[0]);
    st16(reinterpret_cast<T*>(dst) + 64, y[1]);
  } else {
    const float a = max_bound * __ldg((is_v ? v_qs : k_qs) + kvh);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      uint2 packed = make_uint2(0u, 0u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        packed.x |= (uint32_t)kv8::quantize<KV>(to_f(y[k].v[e]), a, round_type, min_bound, max_bound) << (8 * e);
        packed.y |= (uint32_t)kv8::quantize<KV>(to_f(y[k].v[4 + e]), a, round_type, min_bound, max_bound) << (8 * e);
      }
      *reinterpret_cast<uint2*>(dst + 64 * k) = packed;
    }
  }
}

// ---- output quantization: [rows, cols] T -> int8 / e4m3 -------------------------------------------------------------------------------
// y = x (shift / smooth: y = (x + shift[c]) -> T, then y * smooth[c] -> T), stored as kv8::quantize(y, a = max_bound * out_scale).
// 8 elements per thread and step: one 16-byte load and one 8-byte store.
template <typename T, typename KV>
__global__ void __launch_bounds__(256) out_quant_kernel(const T* __restrict__ x, uint8_t* __restrict__ y, int64_t n8, int cols,
                                                       const T* __restrict__ shift, const T* __restrict__ smooth, float a, int round_type,
                                                       float min_bound, float max_bound) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
    const Vec16<T> v = ld16_stream(x + i * 8);
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = to_f(v.v[e]);
    if (shift != nullptr) {
      const int c = (int)((i * 8) % cols);
      const Vec16<T> sh = ld16(shift + c), sm = ld16(smooth + c);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = round_to<T>(__fmul_rn(round_to<T>(__fadd_rn(f[e], to_f(sh.v[e]))), to_f(sm.v[e])));
    }
    uint2 packed = make_uint2(0u, 0u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      packed.x |= (uint32_t)kv8::quantize<KV>(f[e], a, round_type, min_bound, max_bound) << (8 * e);
      packed.y |= (uint32_t)kv8::quantize<KV>(f[4 + e], a, round_type, min_bound, max_bound) << (8 * e);
    }
    *reinterpret_cast<uint2*>(y + i * 8) = packed;
  }
}

}  // namespace kvq

namespace {

int prologue_write(const PagedKvWriteArgs& a, cudaStream_t s) {
  using namespace kvq;
  if (a.d != D || (a.dtype != kBF16 && a.dtype != kF16) || (a.kv_dtype != a.dtype && a.kv_dtype != kI8 && a.kv_dtype != kE4M3) ||
      (a.qkv_int32 && a.col_scale == nullptr) || a.rope < kNoRope || a.rope > kNeox)
    return 1;
  if (a.t == 0 || a.b == 0) return 0;
  dim3 grid(a.t, (a.h + 2 * a.hkv + 15) / 16);
  auto launch = [&](auto tag_t, auto tag_in, auto tag_kv, auto tag_rope) {
    using T = decltype(tag_t);
    using IN = decltype(tag_in);
    using KV = decltype(tag_kv);
    prologue_write_kernel<T, IN, KV, decltype(tag_rope)::value><<<grid, 128, 0, s>>>(
        reinterpret_cast<const IN*>(a.qkv), a.row_stride, reinterpret_cast<T*>(a.out), a.out_stride, reinterpret_cast<uint8_t*>(a.k_cache),
        reinterpret_cast<uint8_t*>(a.v_cache), a.cu_q, a.enc, a.dec, a.block_tables, a.b, a.max_blocks, a.block_size, a.h, a.hkv, a.col_scale,
        reinterpret_cast<const T*>(a.bias), a.rope_cos, a.rope_sin, a.rope_stride, a.k_quant_scales, a.v_quant_scales, a.round_type,
        a.max_bound, a.min_bound);
  };
  auto by_rope = [&](auto tag_t, auto tag_in, auto tag_kv) {
    if (a.rope == kNoRope) launch(tag_t, tag_in, tag_kv, std::integral_constant<int, kNoRope>());
    else if (a.rope == kInterleaved) launch(tag_t, tag_in, tag_kv, std::integral_constant<int, kInterleaved>());
    else launch(tag_t, tag_in, tag_kv, std::integral_constant<int, kNeox>());
  };
  auto by_kv = [&](auto tag_t, auto tag_in) {
    if (a.kv_dtype == kI8) by_rope(tag_t, tag_in, kv8::I8());
    else if (a.kv_dtype == kE4M3) by_rope(tag_t, tag_in, kv8::E4M3());
    else by_rope(tag_t, tag_in, tag_t);
  };
  auto by_in = [&](auto tag_t) {
    if (a.qkv_int32) by_kv(tag_t, int32_t()); else by_kv(tag_t, tag_t);
  };
  if (a.dtype == kBF16) by_in(__nv_bfloat16()); else by_in(__half());
  return B200_LAUNCH_RESULT();
}

}  // namespace

int paged_kv_cache_write(const PagedKvWriteArgs& a, cudaStream_t s) {
  using namespace kvq;
  if (a.qkv_int32 || a.out != nullptr || a.col_scale != nullptr || a.bias != nullptr || a.rope != kNoRope || a.kv_dtype == a.dtype)
    return prologue_write(a, s);
  if (a.d != D || (a.dtype != kBF16 && a.dtype != kF16) || (a.kv_dtype != kI8 && a.kv_dtype != kE4M3)) return 1;
  if (a.t == 0 || a.b == 0) return 0;
  dim3 grid(a.t, (a.hkv + 1) / 2);
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    cache_write_kernel<T, KV><<<grid, 128, 0, s>>>(reinterpret_cast<const T*>(a.qkv), a.row_stride, reinterpret_cast<uint8_t*>(a.k_cache),
                                                   reinterpret_cast<uint8_t*>(a.v_cache), a.cu_q, a.enc, a.dec, a.block_tables, a.b, a.max_blocks,
                                                   a.block_size, a.h, a.hkv, a.k_quant_scales, a.v_quant_scales, a.round_type, a.max_bound,
                                                   a.min_bound);
  };
  if (a.dtype == kBF16) {
    if (a.kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (a.kv_dtype == kI8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  return B200_LAUNCH_RESULT();
}

int attention_out_quant(const OutQuantArgs& a, cudaStream_t s) {
  using namespace kvq;
  if ((a.dtype != kBF16 && a.dtype != kF16) || (a.out_dtype != kI8 && a.out_dtype != kE4M3) || a.cols % 8 != 0 ||
      ((a.shift == nullptr) != (a.smooth == nullptr)))
    return 1;
  const int64_t n8 = a.rows * a.cols / 8;
  if (n8 == 0) return 0;
  const int blocks = (int)std::min<int64_t>((n8 + 255) / 256, 132 * 16);
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    out_quant_kernel<T, decltype(tag_kv)><<<blocks, 256, 0, s>>>(reinterpret_cast<const T*>(a.x), reinterpret_cast<uint8_t*>(a.y), n8, a.cols,
                                                                 reinterpret_cast<const T*>(a.shift), reinterpret_cast<const T*>(a.smooth),
                                                                 a.scale, a.round_type, a.min_bound, a.max_bound);
  };
  if (a.dtype == kBF16) {
    if (a.out_dtype == kI8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (a.out_dtype == kI8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  return B200_LAUNCH_RESULT();
}

}  // namespace b200
