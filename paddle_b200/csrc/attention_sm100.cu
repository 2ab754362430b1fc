// Flash-attention forward for sm_90a (head_dim 128, and 64 in attention_d64_sm100.cu; bf16/fp16): S = Q K^T and O += P V run on
// wgmma tensor cores, K/V tiles streamed by TMA (4-D maps straight over the strided [B,S,H,D] views of a packed QKV tensor, so no
// q/k/v split copies), online softmax on the accumulator fragment in registers, and P never leaves registers: the S fragment of a
// thread IS the A-operand fragment of the P V MMA once packed to 16 bits.  Hand-written PTX; no CUTLASS, no library attention.
//
// Parity (behaviour): paddle.nn.functional.flash_attention / scaled_dot_product_attention
// (python/paddle/nn/functional/flash_attention.py -> phi flash_attn kernels calling the flash-attention library).
//
// CTA = 128 query rows of one (batch, head): two MMA warpgroups of 64 rows each (warps 0-7) walk the key tiles with their own running
// (max, sum) and O accumulator; nothing is exchanged between them, so one warpgroup's softmax runs under the other's MMAs.  Warp 8 is
// the TMA producer (Q once, K and V double-buffered with separate barriers so that S of a tile can start before its V has landed).
//
// PAGED instantiation (prefill / chunked prefill for serving): the queries are the new tokens of each sequence, read in place from the
// packed qkv rows, and K / V come straight from the block-table KV cache [num_blocks, Hkv, block_size, D].  A CTA takes one (sequence,
// 128-row query tile) from a work list built on the device (heaviest tiles first) and walks only its own sequence's key tiles up to the
// bottom-right causal limit.  A 128-key tile is assembled from {64 d, min(block_size, 64) rows} boxes, each at a 1024-byte multiple of
// the tile, so the 128B-swizzled shared tile is byte-for-byte what one dense box would have written and the MMA code is unchanged.
//
// PAGED at head_dim 64 (16-bit caches): a 128-row x 64-d tile is one 128-byte swizzle span (16 KB), so Q, K and V are one "half" each:
// S = Q K^T takes 4 k-steps, P V is one n = 64 wgmma per 16 keys, and the boxes land at the same 1024-byte placements.
//
// PAGED over 8-bit caches (KV = kv8::I8 / kv8::E4M3; q and o stay fp16 / bf16): a converter warpgroup (warps 8-11, 384 threads) takes
// the TMA producer's place for K and V.  Its threads read the 8-bit rows through the block table with 16-byte loads, convert them
// exactly to 16 bits and store them into the same swizzled K / V tiles, then fence.proxy.async and arrive on the tiles' mbarriers; keys
// past the sequence are written as zeros, so stale or NaN cache rows never reach the MMAs.  The K dequant scale is folded into the exp2
// scale and the V dequant scale into the epilogue's 1 / l, so the MMA and softmax code is the 16-bit kernel's.
//
// PAGED with a sliding window W (window > 0, fwd_window_kernel): row i sees keys (i - W, i].  A 128-row query tile starts at key tile
// max(0, m0 + past - W + 1) / 128 and masks each row's left edge, and the work list counts only those key tiles, so a long chunk costs
// O(n W) instead of O(n^2).  Keys below the lowest bound of a CTA's rows are never loaded and their block-table entries never read (the
// TMA producer fetches the window's first block in their place and the tile's V rows below the window are zeroed), so blocks wholly
// below the window may hold NaN or belong to another sequence.
//
// Dense at head_dim 64 (training, attention_d64_sm100.cu): the same CTA and tiles with every operand tile one 64-wide d chunk, so the
// producer issues one box for Q and K and two for V per tile.
//
// The kernel bodies live in include/b200_attention_fwd.cuh.
#include <cuda.h>
#include <algorithm>
#include <cstdio>
#include <type_traits>

#include "include/b200_attention_fwd.cuh"
#include "include/b200_common.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace attn {
using namespace ptx;

// ---------------------------------------------------------------------------------------------- host side
// 4-D map {d, s, h, b} over a strided [B,S,H,D] view (strides in elements), box {128 bytes of d, rows, 1, 1}: 64 d of the 16-bit
// operands, 32 d of the backward's fp32 dQ accumulator (kF32)
bool make_map4(CUtensorMap* out, const void* ptr, int d, int s, int h, int b, int64_t ss, int64_t sh, int64_t sb, uint32_t box_rows, int dtype) {
  const uint64_t es = dtype == kF32 ? 4 : 2;
  const uint64_t dims[4] = {(uint64_t)d, (uint64_t)s, (uint64_t)h, (uint64_t)b};
  const uint64_t strides[3] = {(uint64_t)ss * es, (uint64_t)sh * es, (uint64_t)sb * es};
  const uint32_t box[4] = {(uint32_t)(128 / es), box_rows, 1, 1};
  const CUtensorMapDataType type = dtype == kBF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                  : (dtype == kF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  return encode_tensor_map(out, type, 4, ptr, dims, strides, box, "attention");
}

__global__ void __launch_bounds__(1024) paged_work_kernel(const int* __restrict__ n_q, const int* __restrict__ past, int b, int slots,
                                                          int* scratch, int2* work) {
  paged_work<false>(n_q, past, b, slots, scratch, work, 0);
}

// The sliding-window paged kernels: the windowed prefill takes the larger WindowParams and the work list the window as one more
// argument, so they are kernels of their own; the unwindowed kernels keep their smaller parameters, which their code depends on.
template <typename T, typename KV, int D>
__global__ void __launch_bounds__(std::is_same<KV, T>::value ? kThreads : kThreadsQ8, 1)
fwd_window_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                  const WindowParams<std::conditional_t<std::is_same<KV, T>::value, PagedParams, QuantPagedParams>> p) {
  fwd_body<T, false, true, KV, D, true>(map_q, map_k, map_v, p);
}

__global__ void __launch_bounds__(1024) paged_work_window_kernel(const int* __restrict__ n_q, const int* __restrict__ past, int b, int slots,
                                                                 int* scratch, int2* work, int window) {
  paged_work<true>(n_q, past, b, slots, scratch, work, window);
}

}  // namespace attn

int attention_fwd_supported(const AttnArgs& a) {
  if ((a.d != 128 && a.d != 64) || (a.dtype != kBF16 && a.dtype != kF16)) return 0;
  if (a.h % a.hk) return 0;
  const int64_t* st[3] = {a.q_strides, a.k_strides, a.v_strides};
  for (auto s : st)
    for (int i = 0; i < 3; ++i)
      if (s[i] % 8) return 0;                    // TMA strides: multiples of 16 bytes
  if ((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v) | reinterpret_cast<uintptr_t>(a.o)) & 15) return 0;
  if (a.o_strides[0] % 8 || a.o_strides[1] % 8 || a.o_strides[2] % 8) return 0;
  return 1;
}

int attention_fwd(const AttnArgs& a, cudaStream_t s) {
  if (!attention_fwd_supported(a)) return 1;
  if (a.colmask && a.mask_tiles) return attention_fwd_flashmask(a, nullptr, s);
  return a.d == 64 ? attention_fwd_d64(a, s) : attn::fwd_dense<attn::HD>(a, s);
}

int attention_paged_prefill_slots(int t, int b) { return (t + attn::BM - 1) / attn::BM + b; }
int attention_paged_prefill_scratch_ints(int t, int b) { return 3 * attention_paged_prefill_slots(t, b) + b + 1; }

int attention_paged_prefill_supported(const PagedAttnArgs& a) {
  if ((a.d != 128 && !(a.d == 64 && a.kv_dtype == -1)) || (a.dtype != kBF16 && a.dtype != kF16)) return 0;   // head_dim 64: 16-bit caches
  if (a.kv_dtype != -1 && ((a.kv_dtype != kI8 && a.kv_dtype != kE4M3) || !a.k_dq || !a.v_dq)) return 0;
  if (a.hk <= 0 || a.h % a.hk) return 0;
  if (a.block_size != 16 && a.block_size != 32 && a.block_size != 64 && a.block_size != 128 && a.block_size != 256) return 0;
  if (a.q_strides[0] % 8 || a.q_strides[1] % 8 || a.o_strides[0] % 8 || a.o_strides[1] % 8) return 0;   // 16-byte rows
  if ((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k_cache) | reinterpret_cast<uintptr_t>(a.v_cache) |
       reinterpret_cast<uintptr_t>(a.o)) & 15) return 0;
  return 1;
}

int attention_paged_prefill(const PagedAttnArgs& a, cudaStream_t s) {
  using namespace attn;
  if (!attention_paged_prefill_supported(a)) return 1;
  if (a.t == 0 || a.b == 0) return 0;
  const int slots = attention_paged_prefill_slots(a.t, a.b);
  const int64_t blk = (int64_t)a.block_size * a.d;
  const uint32_t rows = (uint32_t)std::min(a.block_size, 64);
  CUtensorMap mq, mk, mv;
  // q: {d, token, head, 1} over the strided [T, H, D] view; caches: {d, row in block, kv head, block}
  if (!make_map4(&mq, a.q, a.d, a.t, a.h, 1, a.q_strides[0], a.q_strides[1], a.q_strides[0] * a.t, BM, a.dtype)) return 2;
  if (a.kv_dtype != -1) {   // 8-bit caches: no tensor maps over them (the converter warpgroup reads them)
    mk = mv = mq;
  } else {
    if (!make_map4(&mk, a.k_cache, a.d, a.block_size, a.hk, a.num_blocks, a.d, blk, blk * a.hk, rows, a.dtype)) return 2;
    if (!make_map4(&mv, a.v_cache, a.d, a.block_size, a.hk, a.num_blocks, a.d, blk, blk * a.hk, rows, a.dtype)) return 2;
  }
  int2* work = reinterpret_cast<int2*>(a.scratch);
  int* keys = a.scratch + 2 * slots;
  if (a.window > 0) paged_work_window_kernel<<<1, 1024, 0, s>>>(a.n_q, a.past, a.b, slots, keys, work, a.window);
  else paged_work_kernel<<<1, 1024, 0, s>>>(a.n_q, a.past, a.b, slots, keys, work);
  dim3 grid(a.h, slots);   // every head of the heaviest tile is dispatched first
  auto launch = [&](auto tag_t, auto tag_kv, auto tag_d) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    constexpr int D = decltype(tag_d)::value;
    constexpr bool Q8 = !std::is_same<T, KV>::value;
    constexpr int threads = Q8 ? kThreadsQ8 : kThreads;
    constexpr uint32_t smem = kSmemBytes<D>;
    using P = std::conditional_t<Q8, QuantPagedParams, PagedParams>;
    WindowParams<P> p = {};
    p.b = a.b; p.sq = a.t; p.sk = 0; p.h = a.h; p.hk = a.hk;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    p.causal = 1; p.causal_off = 0;
    p.o = a.o; p.lse = a.lse;
    p.o_sb = 0; p.o_ss = a.o_strides[0]; p.o_sh = a.o_strides[1];
    p.colmask = nullptr; p.mask_heads = 1;
    p.work = work; p.cu_q = a.cu_q; p.n_q = a.n_q; p.past = a.past;
    p.block_tables = a.block_tables; p.max_blocks = a.max_blocks; p.block_size = a.block_size;
    if constexpr (Q8) {
      p.k_cache = reinterpret_cast<const uint8_t*>(a.k_cache); p.v_cache = reinterpret_cast<const uint8_t*>(a.v_cache);
      p.k_dq = a.k_dq; p.v_dq = a.v_dq;
    }
    p.window = a.window;
    if (a.window > 0) {
      set_max_dynamic_smem<fwd_window_kernel<T, KV, D>>(smem);
      fwd_window_kernel<T, KV, D><<<grid, threads, smem, s>>>(mq, mk, mv, p);
    } else {
      set_max_dynamic_smem<fwd_kernel<T, false, true, KV, D>>(smem);
      fwd_kernel<T, false, true, KV, D><<<grid, threads, smem, s>>>(mq, mk, mv, static_cast<const P&>(p));
    }
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

}  // namespace b200
