// Sliding-window attention over the KV cache for serving: the windowed instantiations of the single-token decode, verify-row and paged
// prefill kernels.  The query at absolute position i sees key j iff i - W < j <= i (W keys including itself), the mask of models trained
// with a local window (Mistral, Phi-3) and a way to bound a sequence's KV memory.
//
// The kernel bodies are the unwindowed kernels' own (include/b200_decode_attention.cuh, include/b200_attention_fwd.cuh) instantiated with
// WINDOW = true; only the key range and the left edge of the mask change:
// - decode: a split covers positions [max(0, len - W), len), so a call touches min(len, W) rows per query;
// - verify: the splits cover the key tiles from the one holding past - W + 1, and row r of token j masks keys below past + j - W + 1;
// - prefill: a 128-row query tile starts at key tile max(0, m0 + past - W + 1) / 128 and masks each row's left edge, and the work list
//   counts only those key tiles, so a long chunk costs O(n W) instead of O(n^2).
// Keys below the lowest bound of a CTA's rows are never loaded and their block-table entries never read (the TMA producer fetches the
// window's first block in their place and the tile's V rows below the window are zeroed), so blocks wholly below the window may hold
// NaN or belong to another sequence.
#include <cuda.h>
#include <algorithm>
#include <type_traits>

#include "include/b200_attention_fwd.cuh"
#include "include/b200_common.cuh"
#include "include/b200_decode_attention.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"

namespace b200 {
namespace window {

// 192 registers: left to itself ptxas stops the bf16 D = 128 instantiation at 168 with a small spill; two CTAs per SM either way
template <typename T, int D>
__global__ void __maxnreg__(192) decode_split_window_kernel(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
                                                                              const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                              float* __restrict__ part_ml, int h, int hkv, int smax, int splits,
                                                                              float scale_log2, const int* __restrict__ block_tables, int max_blocks,
                                                                              int block_size, int window) {
  decode::decode_split<T, D, true>(q, kc, vc, lens, part_acc, part_ml, h, hkv, smax, splits, scale_log2, block_tables, max_blocks, block_size, window);
}

template <typename T, typename KV>
__global__ void __launch_bounds__(decode::kThreads) decode_split_q8_window_kernel(const T* __restrict__ q, const uint8_t* __restrict__ kc,
                                                                                 const uint8_t* __restrict__ vc, const int* __restrict__ lens,
                                                                                 float* __restrict__ part_acc, float* __restrict__ part_ml, int h,
                                                                                 int hkv, int splits, float scale_log2, const float* __restrict__ k_dq,
                                                                                 const float* __restrict__ v_dq, const int* __restrict__ block_tables,
                                                                                 int max_blocks, int block_size, int window) {
  decode::decode_split_q8<T, KV, true>(q, kc, vc, lens, part_acc, part_ml, h, hkv, splits, scale_log2, k_dq, v_dq, block_tables, max_blocks, block_size,
                                       window);
}

template <typename T, int D>
__global__ void __launch_bounds__(D) decode_merge_window_kernel(const float* __restrict__ part_acc, const float* __restrict__ part_ml, T* __restrict__ out,
                                                                int splits) {
  decode::decode_merge<T, D>(part_acc, part_ml, out, splits);
}

struct MultiParams : decode_multi::Params {
  int window;
};

template <typename T, typename KV, int D>
__global__ void __launch_bounds__(decode_multi::kThreads) multi_split_window_kernel(const __grid_constant__ MultiParams p) {
  decode_multi::multi_split<T, KV, D, true>(p, p.window);
}

template <typename T, int D>
__global__ void __launch_bounds__(D) multi_merge_window_kernel(const __grid_constant__ MultiParams p) { decode_multi::multi_merge<T, D>(p); }

__global__ void __launch_bounds__(1024) paged_work_window_kernel(const int* __restrict__ n_q, const int* __restrict__ past, int b, int slots,
                                                                 int* scratch, int2* work, int window) {
  attn::paged_work<true>(n_q, past, b, slots, scratch, work, window);
}

template <typename T, typename KV, int D>
__global__ void __launch_bounds__(std::is_same<KV, T>::value ? attn::kThreads : attn::kThreadsQ8, 1)
fwd_window_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                  const attn::WindowParams<std::conditional_t<std::is_same<KV, T>::value, attn::PagedParams, attn::QuantPagedParams>> p) {
  attn::fwd_body<T, false, true, KV, D, true>(map_q, map_k, map_v, p);
}

}  // namespace window

int decode_attention_window(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml,
                            int b, int h, int hkv, int smax, int d, int splits, float scale, int dtype, cudaStream_t s, const int* block_tables,
                            int max_blocks, int block_size, int window) {
  using namespace window;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_d) {
    using T = decltype(tag_t);
    constexpr int D = decltype(tag_d)::value;
    decode_split_window_kernel<T, D><<<grid, decode::kThreads, 0, s>>>((const T*)q, (const T*)k_cache, (const T*)v_cache, lens, part_acc, part_ml, h, hkv,
                                                                       smax, splits, sl2, block_tables, max_blocks, block_size, window);
    decode_merge_window_kernel<T, D><<<b * h, D, 0, s>>>(part_acc, part_ml, (T*)out, splits);
  };
  if (dtype == kBF16) {
    if (d == 128) launch(__nv_bfloat16(), HeadDim<128>()); else launch(__nv_bfloat16(), HeadDim<64>());
  } else {
    if (d == 128) launch(__half(), HeadDim<128>()); else launch(__half(), HeadDim<64>());
  }
  return B200_LAUNCH_RESULT();
}

int decode_attention_paged_q8_window(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc,
                                     float* part_ml, int b, int h, int hkv, int splits, float scale, int dtype, int kv_dtype, const float* k_dq,
                                     const float* v_dq, const int* block_tables, int max_blocks, int block_size, int window, cudaStream_t s) {
  using namespace window;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    decode_split_q8_window_kernel<T, decltype(tag_kv)><<<grid, decode::kThreads, 0, s>>>((const T*)q, (const uint8_t*)k_cache, (const uint8_t*)v_cache,
                                                                                         lens, part_acc, part_ml, h, hkv, splits, sl2, k_dq, v_dq,
                                                                                         block_tables, max_blocks, block_size, window);
    decode_merge_window_kernel<T, 128><<<b * h, 128, 0, s>>>(part_acc, part_ml, (T*)out, splits);
  };
  if (dtype == kBF16) {
    if (kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (kv_dtype == kI8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  return B200_LAUNCH_RESULT();
}

int decode_attention_paged_multi_window(const decode_multi::Params& p, const PagedMultiArgs& a, cudaStream_t s) {
  using namespace window;
  MultiParams wp;
  static_cast<decode_multi::Params&>(wp) = p;
  wp.window = a.window;
  const dim3 grid(a.splits, a.hkv, a.b), mgrid(decode_multi::kRows, a.hkv, a.b);
  auto launch = [&](auto tag_t, auto tag_kv, auto tag_d) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    constexpr int D = decltype(tag_d)::value;
    constexpr int smem = decode_multi::Smem<!std::is_same<T, KV>::value, D>::kBytes;
    set_max_dynamic_smem<multi_split_window_kernel<T, KV, D>>(smem);
    multi_split_window_kernel<T, KV, D><<<grid, decode_multi::kThreads, smem, s>>>(wp);
    multi_merge_window_kernel<T, D><<<mgrid, D, 0, s>>>(wp);
  };
  if (a.dtype == kBF16) {
    if (a.d == 64) launch(__nv_bfloat16(), __nv_bfloat16(), HeadDim<64>());
    else if (a.kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8(), HeadDim<128>());
    else if (a.kv_dtype == kE4M3) launch(__nv_bfloat16(), kv8::E4M3(), HeadDim<128>());
    else launch(__nv_bfloat16(), __nv_bfloat16(), HeadDim<128>());
  } else {
    if (a.d == 64) launch(__half(), __half(), HeadDim<64>());
    else if (a.kv_dtype == kI8) launch(__half(), kv8::I8(), HeadDim<128>());
    else if (a.kv_dtype == kE4M3) launch(__half(), kv8::E4M3(), HeadDim<128>());
    else launch(__half(), __half(), HeadDim<128>());
  }
  return B200_LAUNCH_RESULT();
}

int attention_paged_prefill_window(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const attn::PagedParams& p,
                                   const PagedAttnArgs& a, int slots, cudaStream_t s) {
  using namespace window;
  attn::WindowParams<attn::PagedParams> wp;
  static_cast<attn::PagedParams&>(wp) = p;
  wp.window = a.window;
  paged_work_window_kernel<<<1, 1024, 0, s>>>(a.n_q, a.past, a.b, slots, a.scratch + 2 * slots, reinterpret_cast<int2*>(a.scratch), a.window);
  dim3 grid(a.h, slots);
  auto launch = [&](auto tag_t, auto tag_d) {
    using T = decltype(tag_t);
    constexpr int D = decltype(tag_d)::value;
    set_max_dynamic_smem<fwd_window_kernel<T, T, D>>(attn::kSmemBytes<D>);
    fwd_window_kernel<T, T, D><<<grid, attn::kThreads, attn::kSmemBytes<D>, s>>>(mq, mk, mv, wp);
  };
  if (a.dtype == kBF16) {
    if (a.d == 128) launch(__nv_bfloat16(), HeadDim<128>()); else launch(__nv_bfloat16(), HeadDim<64>());
  } else {
    if (a.d == 128) launch(__half(), HeadDim<128>()); else launch(__half(), HeadDim<64>());
  }
  return B200_LAUNCH_RESULT();
}

int attention_paged_prefill_window(const CUtensorMap& mq, const attn::QuantPagedParams& p, const PagedAttnArgs& a, int slots, cudaStream_t s) {
  using namespace window;
  attn::WindowParams<attn::QuantPagedParams> wp;
  static_cast<attn::QuantPagedParams&>(wp) = p;
  wp.window = a.window;
  paged_work_window_kernel<<<1, 1024, 0, s>>>(a.n_q, a.past, a.b, slots, a.scratch + 2 * slots, reinterpret_cast<int2*>(a.scratch), a.window);
  dim3 grid(a.h, slots);
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    set_max_dynamic_smem<fwd_window_kernel<T, KV, 128>>(attn::SMEM_BYTES);
    fwd_window_kernel<T, KV, 128><<<grid, attn::kThreadsQ8, attn::SMEM_BYTES, s>>>(mq, mq, mq, wp);
  };
  const bool i8 = a.kv_dtype == kI8;
  if (a.dtype == kBF16) {
    if (i8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (i8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  return B200_LAUNCH_RESULT();
}

}  // namespace b200
