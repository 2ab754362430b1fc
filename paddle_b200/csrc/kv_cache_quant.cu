// Quantizing write of the new K / V rows into a paged int8 / fp8 (e4m3) KV cache, for prefill and decode rows alike, in one launch.
//
// Parity (behaviour): the static cache-KV quantization of block_multihead_attention (QuantHelperFunc in
// paddle/phi/kernels/fusion/gpu/mmha_util.cu.h), extended to e4m3; the rules are in include/b200_kv8.cuh.
//
// The rows are read in place from the packed qkv [T, (H + 2 Hkv) * 128].  Token t belongs to the last sequence i with cu_q[i] <= t; its
// position is (seq_lens_encoder[i] > 0 ? 0 : seq_lens_decoder[i]) + t - cu_q[i], and it goes to block block_tables[i, pos / block_size],
// row pos % block_size.  Everything is found on the device: no host read of the lengths.  Grid (T, ceil(Hkv / 2)), 4 warps: warp w
// writes the K (w < 2) or V row of KV head 2 blockIdx.y + (w & 1), 4 elements per lane.
#include <cuda.h>

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

}  // namespace kvq

int paged_kv_cache_write(const PagedKvWriteArgs& a, cudaStream_t s) {
  using namespace kvq;
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
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

}  // namespace b200
