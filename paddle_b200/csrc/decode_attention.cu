// Single-token decode attention against a contiguous KV cache (serving path of FusedMultiTransformer /
// masked_multihead_attention).  HBM-bound: every cached key / value row is read exactly once with 16-byte loads.
//
// Parity (behaviour): masked_multihead_attention (paddle/phi/kernels/fusion/gpu/masked_multihead_attention_kernel.cu).
//
// Layout: q [B, H, D]; k_cache / v_cache [B, Hkv, S_max, D] (the two halves of paddle's cache_kv [2, B, H, S_max, D]);
// lens[b] = number of valid cached positions (the new token already written).  Grid = (splits, H, B): every CTA owns a
// contiguous range of positions; thread t handles positions t, t+128, ... with a private online softmax (m, l, acc[D]);
// the CTA combines its threads through shared memory and writes one partial (m, l, acc) per split; a second tiny kernel
// merges the splits.  D = 128, fp16 / bf16.
//
// Paged caches (block_multihead_attention, paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu): with `block_tables`
// [B, max_blocks] the caches are [num_blocks, Hkv, block_size, D] and position p of sequence b lives in block block_tables[b, p / block_size]
// at row p % block_size - one table lookup per cached row, the rest of the kernel is unchanged.
//
// Paged int8 / fp8 e4m3 caches (decode_split_q8_kernel): the same walk over 8-bit rows, dequantized with per-KV-head scales.
#include <cuda.h>
#include <cstdio>

#include "include/b200_common.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"

namespace b200 {
namespace decode {

constexpr int D = 128, kThreads = 128;

// Combine the CTA's per-thread online-softmax partials (m, l, acc) and write this split's partial (m, l, acc * v_scale).
__device__ __forceinline__ void split_epilogue(float m, float l, const float (&acc)[D], float* red, float (*sacc)[D + 1], float* __restrict__ part_acc,
                                               float* __restrict__ part_ml, int h, int splits, float v_scale) {
  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  // CTA-wide maximum, then every thread rescales its partial to it
  red[tid] = m;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (tid < o) red[tid] = fmaxf(red[tid], red[tid + o]);
    __syncthreads();
  }
  const float mg = red[0];
  __syncthreads();
  const float f = (m == -INFINITY) ? 0.f : exp2f(m - mg);
  l *= f;
  red[tid] = l;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (tid < o) red[tid] += red[tid + o];
    __syncthreads();
  }
  const float lg = red[0];
  // sum the 128 per-thread accumulators: 4 rounds of 32 threads' vectors through shared memory, thread t owns output dim t
  float out = 0.f;
  for (int r = 0; r < kThreads / 32; ++r) {
    __syncthreads();
    if ((tid >> 5) == r) {
#pragma unroll
      for (int i = 0; i < D; ++i) sacc[tid & 31][i] = acc[i] * f;
    }
    __syncthreads();
#pragma unroll 8
    for (int j = 0; j < 32; ++j) out += sacc[j][tid];
  }
  const int64_t pi = ((int64_t)b * h + head) * splits + split;
  part_acc[pi * D + tid] = out * v_scale;
  if (tid == 0) { part_ml[pi * 2] = mg; part_ml[pi * 2 + 1] = lg; }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) decode_split_kernel(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
                                                                const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                float* __restrict__ part_ml, int h, int hkv, int smax, int splits, float scale_log2,
                                                                const int* __restrict__ block_tables, int max_blocks, int block_size) {
  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (h / hkv);
  const int len = block_tables ? min(lens[b], max_blocks * block_size) : min(lens[b], smax);
  const int per = (len + splits - 1) / splits;
  const int p0 = split * per, p1 = min(len, p0 + per);
  __shared__ float sq[D];
  __shared__ float red[kThreads];
  __shared__ float sacc[32][D + 1];           // one slice of the cross-thread reduction at a time
  const int tid = threadIdx.x;
  sq[tid] = to_f(q[((int64_t)b * h + head) * D + tid]) * scale_log2;
  __syncthreads();
  const T* kbase = kc + ((int64_t)b * hkv + kvh) * (int64_t)smax * D;
  const T* vbase = vc + ((int64_t)b * hkv + kvh) * (int64_t)smax * D;
  const int* bt = block_tables ? block_tables + (int64_t)b * max_blocks : nullptr;
  // element offset of cached position `pos` of this (sequence, kv head)
  auto row_off = [&](int pos) -> int64_t {
    if (!bt) return (int64_t)pos * D;
    const int blk = bt[pos / block_size];
    return (((int64_t)blk * hkv + kvh) * block_size + pos % block_size) * D;
  };
  if (bt) { kbase = kc; vbase = vc; }
  float m = -INFINITY, l = 0.f;
  float acc[D];
#pragma unroll
  for (int i = 0; i < D; ++i) acc[i] = 0.f;
  for (int pos = p0 + tid; pos < p1; pos += kThreads) {
    const int64_t roff = row_off(pos);
    const Vec16<T>* kr = reinterpret_cast<const Vec16<T>*>(kbase + roff);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      const Vec16<T> kv = ld16(reinterpret_cast<const T*>(kr + c));
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(to_f(kv.v[e]), sq[c * 8 + e], s);
    }
    const float m_new = fmaxf(m, s);
    const float alpha = exp2f(m - m_new), pv = exp2f(s - m_new);
    l = l * alpha + pv;
    const Vec16<T>* vr = reinterpret_cast<const Vec16<T>*>(vbase + roff);
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      const Vec16<T> vv = ld16(reinterpret_cast<const T*>(vr + c));
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[c * 8 + e] = fmaf(acc[c * 8 + e], alpha, pv * to_f(vv.v[e]));
    }
    m = m_new;
  }
  split_epilogue(m, l, acc, red, sacc, part_acc, part_ml, h, splits, 1.f);
}

// Paged 8-bit caches (KV = kv8::I8 / kv8::E4M3): one 16-byte load carries 16 elements.  The K dequant scale is folded into sq, the V
// dequant scale is applied once to the split's partial output; with power-of-two scales the result is bit-identical to
// decode_split_kernel on a 16-bit cache holding the dequantized values.
template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) decode_split_q8_kernel(const T* __restrict__ q, const uint8_t* __restrict__ kc, const uint8_t* __restrict__ vc,
                                                                   const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                   float* __restrict__ part_ml, int h, int hkv, int splits, float scale_log2,
                                                                   const float* __restrict__ k_dq, const float* __restrict__ v_dq,
                                                                   const int* __restrict__ block_tables, int max_blocks, int block_size) {
  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (h / hkv);
  const int len = min(lens[b], max_blocks * block_size);
  const int per = (len + splits - 1) / splits;
  const int p0 = split * per, p1 = min(len, p0 + per);
  __shared__ float sq[D];
  __shared__ float red[kThreads];
  __shared__ float sacc[32][D + 1];
  const int tid = threadIdx.x;
  sq[tid] = to_f(q[((int64_t)b * h + head) * D + tid]) * scale_log2 * __ldg(k_dq + kvh);
  __syncthreads();
  const int* bt = block_tables + (int64_t)b * max_blocks;
  float m = -INFINITY, l = 0.f;
  float acc[D];
#pragma unroll
  for (int i = 0; i < D; ++i) acc[i] = 0.f;
  for (int pos = p0 + tid; pos < p1; pos += kThreads) {
    const int64_t roff = (((int64_t)bt[pos / block_size] * hkv + kvh) * block_size + pos % block_size) * D;
    const uint4* kr = reinterpret_cast<const uint4*>(kc + roff);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < D / 16; ++c) {
      float kf[16];
      kv8::to_float16<KV>(kr[c], kf);
#pragma unroll
      for (int e = 0; e < 16; e += 4) {   // re-read q from shared memory every row: 128 q registers on top of acc would spill
        float4 qv;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(qv.x), "=f"(qv.y), "=f"(qv.z), "=f"(qv.w)
                     : "r"((uint32_t)__cvta_generic_to_shared(sq + c * 16 + e)));
        s = fmaf(kf[e], qv.x, s);
        s = fmaf(kf[e + 1], qv.y, s);
        s = fmaf(kf[e + 2], qv.z, s);
        s = fmaf(kf[e + 3], qv.w, s);
      }
    }
    const float m_new = fmaxf(m, s);
    const float alpha = exp2f(m - m_new), pv = exp2f(s - m_new);
    l = l * alpha + pv;
    const uint4* vr = reinterpret_cast<const uint4*>(vc + roff);
#pragma unroll
    for (int c = 0; c < D / 16; ++c) {
      float vf[16];
      kv8::to_float16<KV>(vr[c], vf);
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[c * 16 + e] = fmaf(acc[c * 16 + e], alpha, pv * vf[e]);
    }
    m = m_new;
  }
  split_epilogue(m, l, acc, red, sacc, part_acc, part_ml, h, splits, __ldg(v_dq + kvh));
}

template <typename T>
__global__ void __launch_bounds__(D) decode_merge_kernel(const float* __restrict__ part_acc, const float* __restrict__ part_ml, T* __restrict__ out,
                                                         int splits) {
  const int64_t bh = blockIdx.x;
  const int tid = threadIdx.x;
  float mg = -INFINITY;
  for (int s = 0; s < splits; ++s) mg = fmaxf(mg, part_ml[(bh * splits + s) * 2]);
  float l = 0.f, o = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float ms = part_ml[(bh * splits + s) * 2];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - mg);
    l += part_ml[(bh * splits + s) * 2 + 1] * f;
    o += part_acc[(bh * splits + s) * D + tid] * f;
  }
  out[bh * D + tid] = from_f<T>(l > 0.f ? o / l : 0.f);
}

}  // namespace decode

int decode_attention_splits(int b, int h, int smax) {
  // enough CTAs to fill the machine, at least 256 positions per split
  int splits = (2 * sm_count() + b * h - 1) / (b * h);
  const int max_by_len = (smax + 255) / 256;
  if (splits > max_by_len) splits = max_by_len;
  return splits < 1 ? 1 : (splits > 64 ? 64 : splits);
}

int decode_attention(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml, int b,
                     int h, int hkv, int smax, int d, int splits, float scale, int dtype, cudaStream_t s, const int* block_tables, int max_blocks,
                     int block_size) {
  using namespace decode;
  if (d != D || h % hkv || (dtype != kBF16 && dtype != kF16)) return 1;
  if (block_tables && (max_blocks <= 0 || block_size <= 0)) return 1;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  if (dtype == kBF16) {
    decode_split_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k_cache, (const __nv_bfloat16*)v_cache, lens,
                                                                   part_acc, part_ml, h, hkv, smax, splits, sl2, block_tables, max_blocks, block_size);
    decode_merge_kernel<__nv_bfloat16><<<b * h, D, 0, s>>>(part_acc, part_ml, (__nv_bfloat16*)out, splits);
  } else {
    decode_split_kernel<__half><<<grid, kThreads, 0, s>>>((const __half*)q, (const __half*)k_cache, (const __half*)v_cache, lens, part_acc, part_ml, h, hkv,
                                                           smax, splits, sl2, block_tables, max_blocks, block_size);
    decode_merge_kernel<__half><<<b * h, D, 0, s>>>(part_acc, part_ml, (__half*)out, splits);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

int decode_attention_paged_q8(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml,
                              int b, int h, int hkv, int d, int splits, float scale, int dtype, int kv_dtype, const float* k_dq, const float* v_dq,
                              const int* block_tables, int max_blocks, int block_size, cudaStream_t s) {
  using namespace decode;
  if (d != D || h % hkv || (dtype != kBF16 && dtype != kF16) || (kv_dtype != kI8 && kv_dtype != kE4M3)) return 1;
  if (!block_tables || !k_dq || !v_dq || max_blocks <= 0 || block_size <= 0) return 1;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    decode_split_q8_kernel<T, decltype(tag_kv)><<<grid, kThreads, 0, s>>>((const T*)q, (const uint8_t*)k_cache, (const uint8_t*)v_cache, lens,
                                                                          part_acc, part_ml, h, hkv, splits, sl2, k_dq, v_dq, block_tables,
                                                                          max_blocks, block_size);
    decode_merge_kernel<T><<<b * h, D, 0, s>>>(part_acc, part_ml, (T*)out, splits);
  };
  if (dtype == kBF16) {
    if (kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (kv_dtype == kI8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

}  // namespace b200
