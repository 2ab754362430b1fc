// Single-token decode attention against a contiguous KV cache (serving path of FusedMultiTransformer /
// masked_multihead_attention).  HBM-bound: every cached key / value row is read exactly once with 16-byte loads.
//
// Parity (behaviour): masked_multihead_attention (paddle/phi/kernels/fusion/gpu/masked_multihead_attention_kernel.cu).
//
// Layout: q [B, H, D]; k_cache / v_cache [B, Hkv, S_max, D] (the two halves of paddle's cache_kv [2, B, H, S_max, D]);
// lens[b] = number of valid cached positions (the new token already written).  Grid = (splits, H, B): every CTA owns a
// contiguous range of positions; thread t handles positions t, t+128, ... with a private online softmax (m, l, acc[D]);
// the CTA combines its threads through shared memory and writes one partial (m, l, acc) per split; a second tiny kernel
// merges the splits.  D = 128 or 64 (a template argument), fp16 / bf16.
//
// Paged caches (block_multihead_attention, paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu): with `block_tables`
// [B, max_blocks] the caches are [num_blocks, Hkv, block_size, D] and position p of sequence b lives in block block_tables[b, p / block_size]
// at row p % block_size - one table lookup per cached row, the rest of the kernel is unchanged.
//
// Paged int8 / fp8 e4m3 caches (decode_split_q8_kernel, D = 128): the same walk over 8-bit rows, dequantized with per-KV-head scales.
//
// Sliding window (window > 0): the same kernels over the last `window` positions (see include/b200_decode_attention.cuh).
//
// The kernel bodies live in include/b200_decode_attention.cuh.
#include <cuda.h>
#include <cstdio>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_decode_attention.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"

namespace b200 {
namespace decode {

template <typename T, int D>
__global__ void __launch_bounds__(kThreads) decode_split_kernel(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
                                                                const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                float* __restrict__ part_ml, int h, int hkv, int smax, int splits, float scale_log2,
                                                                const int* __restrict__ block_tables, int max_blocks, int block_size) {
  decode_split<T, D, false>(q, kc, vc, lens, part_acc, part_ml, h, hkv, smax, splits, scale_log2, block_tables, max_blocks, block_size, 0);
}

template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) decode_split_q8_kernel(const T* __restrict__ q, const uint8_t* __restrict__ kc, const uint8_t* __restrict__ vc,
                                                                   const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                   float* __restrict__ part_ml, int h, int hkv, int splits, float scale_log2,
                                                                   const float* __restrict__ k_dq, const float* __restrict__ v_dq,
                                                                   const int* __restrict__ block_tables, int max_blocks, int block_size) {
  decode_split_q8<T, KV, false>(q, kc, vc, lens, part_acc, part_ml, h, hkv, splits, scale_log2, k_dq, v_dq, block_tables, max_blocks, block_size, 0);
}

// The sliding-window decode kernels take the window as one more argument, so they are kernels of their own; the unwindowed kernels keep
// their smaller argument lists.  Their splits are merged by decode_merge_kernel.
// 192 registers: left to itself ptxas stops the bf16 D = 128 instantiation at 168 with a small spill; two CTAs per SM either way
template <typename T, int D>
__global__ void __maxnreg__(192) decode_split_window_kernel(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
                                                            const int* __restrict__ lens, float* __restrict__ part_acc, float* __restrict__ part_ml,
                                                            int h, int hkv, int smax, int splits, float scale_log2,
                                                            const int* __restrict__ block_tables, int max_blocks, int block_size, int window) {
  decode_split<T, D, true>(q, kc, vc, lens, part_acc, part_ml, h, hkv, smax, splits, scale_log2, block_tables, max_blocks, block_size, window);
}

template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) decode_split_q8_window_kernel(const T* __restrict__ q, const uint8_t* __restrict__ kc,
                                                                          const uint8_t* __restrict__ vc, const int* __restrict__ lens,
                                                                          float* __restrict__ part_acc, float* __restrict__ part_ml, int h, int hkv,
                                                                          int splits, float scale_log2, const float* __restrict__ k_dq,
                                                                          const float* __restrict__ v_dq, const int* __restrict__ block_tables,
                                                                          int max_blocks, int block_size, int window) {
  decode_split_q8<T, KV, true>(q, kc, vc, lens, part_acc, part_ml, h, hkv, splits, scale_log2, k_dq, v_dq, block_tables, max_blocks, block_size,
                               window);
}

template <typename T, int D>
__global__ void __launch_bounds__(D) decode_merge_kernel(const float* __restrict__ part_acc, const float* __restrict__ part_ml, T* __restrict__ out,
                                                         int splits) {
  decode_merge<T, D>(part_acc, part_ml, out, splits);
}

}  // namespace decode

// Multi-token paged decode: the few new tokens of each sequence (the verify rows of speculative decoding) over its long cached prefix.
// Grid = (splits, Hkv, B).  A CTA owns every query row of one (sequence, KV head): n_q tokens x G = H / Hkv heads, packed into one 64-row
// tile (row r = token r / G, head kvh * G + r % G), so each cached K / V row is read from HBM once per call.  Its 4 warps own 16 rows each
// and run mma.sync m16n8k16 (fp32 accumulate): S = Q K^T over 64-key tiles, P kept in registers as the A operand of P V.  K / V tiles come
// through the block table by cp.async 16-byte copies, three stages deep; keys at or past the sequence's length are zero-filled without
// reading their table entry, so NaN in a recycled block never reaches the MMAs.  Masking is bottom-right causal: token j sees keys
// < past + j + 1.  Each split writes an unnormalized partial (m, l, acc) per row; multi_merge_kernel combines them like decode_merge_kernel.
// 8-bit caches are copied raw and converted exactly to 16 bits in shared memory; K's dequant scale joins the softmax scale and V's scales
// the split's partial, so with power-of-two scales the result is bit-identical to the 16-bit kernel on the dequantized cache.
// D = 128, or 64 on 16-bit caches: the same 64-row tile, with half the k-steps of S and half the output columns.
// Sliding window (WINDOW, p.window > 0): see include/b200_decode_attention.cuh; the splits are merged by the same multi_merge_kernel.
namespace decode_multi {

template <typename T, typename KV, int D, bool WINDOW>
__global__ void __launch_bounds__(kThreads) multi_split_kernel(const __grid_constant__ Params p) { multi_split<T, KV, D, WINDOW>(p, p.window); }

template <typename T, int D>
__global__ void __launch_bounds__(D) multi_merge_kernel(const Params p) { multi_merge<T, D>(p); }

}  // namespace decode_multi

// Shared-prefix decode ("cascade" decode): single-token decode rows of sequences whose leading blocks are the same physical blocks.
// The host turns the groups into a task list.  A prefix task packs up to 64 / G members of one group (G = H / Hkv query heads per KV
// head; row r = member r / G, head kvh * G + r % G) into one 64-row tile and reads the group's prefix keys [0, prefix_len) through the
// first member's table, with no mask: every prefix key is visible to every member.  A suffix task holds one member's G rows and reads its
// own keys [prefix_len, len).  Both are split over their keys and write unnormalized partials (m, l, acc) at their own rows of one
// [Hkv, rows] buffer; shared_merge_kernel combines every partial of a member's row and writes the output in place.  The split kernel is
// decode_multi's tile loop (cp.async three stages deep through the block table, mma.sync m16n8k16 with P in registers, zero-filled keys
// past the end whose table entries are never read, exact 8-bit conversion in shared memory with K's scale in the softmax scale and V's
// in the partial) with the shared-prefix key range, row packing and partial layout.
namespace decode_shared {

using decode_multi::kRows;
using decode_multi::kThreads;
constexpr int D = 128;

struct Params {
  const void* q; const void* k_cache; const void* v_cache;
  void* out; float* part_acc; float* part_ml;
  const int* block_tables; const int* cu_q; const int* lens; const int* group_seqs;
  const int* tasks; const int* members;   // kTaskInts per task, kMemberInts per member (see PagedSharedArgs)
  const float* k_dq; const float* v_dq;
  int64_t q_st, q_sh, o_st;
  int h, hkv, rows, max_blocks, block_size;
  float scale_log2;
};

template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) shared_split_kernel(const Params p) { decode_multi::multi_split<T, KV, D, false, true>(p); }

// grid (members, Hkv), D threads: one member's G rows of one KV head.  A member that breaks the group contract - its first
// prefix_len / block_size table entries differ from the group's first member's, or prefix_len is not below its length or the first
// member's - gets NaN rows.
template <typename T>
__global__ void __launch_bounds__(D) shared_merge_kernel(const Params p) {
  const int* mi = p.members + (int64_t)blockIdx.x * kSharedMemberInts;
  const int kvh = blockIdx.y, tid = threadIdx.x, g_size = p.h / p.hkv;
  const int pt0 = mi[0], slot = mi[1], st0 = mi[2], first = mi[3], plen = mi[4], b = mi[5];
  bool bad = p.lens[b] - 1 < plen || p.lens[first] - 1 < plen;
  const int* bt_b = p.block_tables + (int64_t)b * p.max_blocks;
  const int* bt_f = p.block_tables + (int64_t)first * p.max_blocks;
  for (int j = tid; j < plen / p.block_size; j += D) bad |= bt_b[j] != bt_f[j];
  bad = __syncthreads_or(bad);
  T* out = reinterpret_cast<T*>(p.out) + (int64_t)p.cu_q[b] * p.o_st + (int64_t)kvh * g_size * D + tid;
  const int np = p.tasks[pt0 * kSharedTaskInts + 6], ns = p.tasks[st0 * kSharedTaskInts + 6];
  const int64_t kb = (int64_t)kvh * p.rows;
  for (int hq = 0; hq < g_size; ++hq) {
    if (bad) { out[hq * D] = from_f<T>(__int_as_float(0x7fc00000)); continue; }
    float mg = -INFINITY;
    for (int s = 0; s < np + ns; ++s) {
      const int64_t row = kb + (s < np ? p.tasks[(pt0 + s) * kSharedTaskInts + 7] + slot : p.tasks[(st0 + s - np) * kSharedTaskInts + 7]) + hq;
      mg = fmaxf(mg, p.part_ml[row * 2]);
    }
    float l = 0.f, o = 0.f;
    for (int s = 0; s < np + ns; ++s) {
      const int64_t row = kb + (s < np ? p.tasks[(pt0 + s) * kSharedTaskInts + 7] + slot : p.tasks[(st0 + s - np) * kSharedTaskInts + 7]) + hq;
      const float ms = p.part_ml[row * 2];
      if (ms == -INFINITY) continue;                         // an empty partial: its acc was never written
      const float f = exp2f(ms - mg);
      l += p.part_ml[row * 2 + 1] * f;
      o += p.part_acc[row * D + tid] * f;
    }
    out[hq * D] = from_f<T>(l > 0.f ? o / l : 0.f);
  }
}

}  // namespace decode_shared

int decode_attention_splits(int b, int h, int smax) {
  // enough CTAs to fill the machine, at least 256 positions per split
  int splits = (2 * sm_count() + b * h - 1) / (b * h);
  const int max_by_len = (smax + 255) / 256;
  if (splits > max_by_len) splits = max_by_len;
  return splits < 1 ? 1 : (splits > 64 ? 64 : splits);
}

int decode_attention(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml, int b,
                     int h, int hkv, int smax, int d, int splits, float scale, int dtype, cudaStream_t s, const int* block_tables, int max_blocks,
                     int block_size, int window) {
  using namespace decode;
  if ((d != 128 && d != 64) || h % hkv || (dtype != kBF16 && dtype != kF16)) return 1;
  if (block_tables && (max_blocks <= 0 || block_size <= 0)) return 1;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_d) {
    using T = decltype(tag_t);
    constexpr int D = decltype(tag_d)::value;
    if (window > 0)
      decode_split_window_kernel<T, D><<<grid, kThreads, 0, s>>>((const T*)q, (const T*)k_cache, (const T*)v_cache, lens, part_acc, part_ml, h, hkv,
                                                                 smax, splits, sl2, block_tables, max_blocks, block_size, window);
    else
      decode_split_kernel<T, D><<<grid, kThreads, 0, s>>>((const T*)q, (const T*)k_cache, (const T*)v_cache, lens, part_acc, part_ml, h, hkv, smax,
                                                          splits, sl2, block_tables, max_blocks, block_size);
    decode_merge_kernel<T, D><<<b * h, D, 0, s>>>(part_acc, part_ml, (T*)out, splits);
  };
  if (dtype == kBF16) {
    if (d == 128) launch(__nv_bfloat16(), HeadDim<128>()); else launch(__nv_bfloat16(), HeadDim<64>());
  } else {
    if (d == 128) launch(__half(), HeadDim<128>()); else launch(__half(), HeadDim<64>());
  }
  return B200_LAUNCH_RESULT();
}

int decode_attention_paged_q8(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml,
                              int b, int h, int hkv, int d, int splits, float scale, int dtype, int kv_dtype, const float* k_dq, const float* v_dq,
                              const int* block_tables, int max_blocks, int block_size, cudaStream_t s, int window) {
  using namespace decode;
  if (d != 128 || h % hkv || (dtype != kBF16 && dtype != kF16) || (kv_dtype != kI8 && kv_dtype != kE4M3)) return 1;
  if (!block_tables || !k_dq || !v_dq || max_blocks <= 0 || block_size <= 0) return 1;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    if (window > 0)
      decode_split_q8_window_kernel<T, KV><<<grid, kThreads, 0, s>>>((const T*)q, (const uint8_t*)k_cache, (const uint8_t*)v_cache, lens, part_acc,
                                                                     part_ml, h, hkv, splits, sl2, k_dq, v_dq, block_tables, max_blocks, block_size,
                                                                     window);
    else
      decode_split_q8_kernel<T, KV><<<grid, kThreads, 0, s>>>((const T*)q, (const uint8_t*)k_cache, (const uint8_t*)v_cache, lens, part_acc, part_ml,
                                                              h, hkv, splits, sl2, k_dq, v_dq, block_tables, max_blocks, block_size);
    decode_merge_kernel<T, 128><<<b * h, 128, 0, s>>>(part_acc, part_ml, (T*)out, splits);
  };
  if (dtype == kBF16) {
    if (kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (kv_dtype == kI8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  return B200_LAUNCH_RESULT();
}

int decode_attention_paged_multi(const PagedMultiArgs& a, cudaStream_t s) {
  using namespace decode_multi;
  if ((a.d != 128 && a.d != 64) || (a.d == 64 && a.kv_dtype != -1) || a.hkv <= 0 || a.h % a.hkv || a.h / a.hkv > kRows || (a.dtype != kBF16 && a.dtype != kF16)) return 1;
  if (a.kv_dtype != -1 && ((a.kv_dtype != kI8 && a.kv_dtype != kE4M3) || !a.k_dq || !a.v_dq)) return 1;
  if (a.max_blocks <= 0 || a.block_size <= 0 || a.splits < 1) return 1;
  if (a.q_st % 8 || a.q_sh % 8 || a.o_st % 8 || ((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k_cache) |
                                                  reinterpret_cast<uintptr_t>(a.v_cache)) & 15)) return 1;
  if (a.b == 0) return 0;
  Params p;
  p.q = a.q; p.k_cache = a.k_cache; p.v_cache = a.v_cache; p.out = a.out; p.part_acc = a.part_acc; p.part_ml = a.part_ml;
  p.block_tables = a.block_tables; p.cu_q = a.cu_q; p.n_q = a.n_q; p.past = a.past; p.k_dq = a.k_dq; p.v_dq = a.v_dq;
  p.q_st = a.q_st; p.q_sh = a.q_sh; p.o_st = a.o_st;
  p.h = a.h; p.hkv = a.hkv; p.splits = a.splits; p.max_blocks = a.max_blocks; p.block_size = a.block_size;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.window = a.window;
  const dim3 grid(a.splits, a.hkv, a.b), mgrid(kRows, a.hkv, a.b);
  auto launch = [&](auto tag_t, auto tag_kv, auto tag_d) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    constexpr int D = decltype(tag_d)::value;
    constexpr int smem = Smem<!std::is_same<T, KV>::value, D>::kBytes;
    auto run = [&](auto tag_w) {
      constexpr bool W = decltype(tag_w)::value;
      set_max_dynamic_smem<multi_split_kernel<T, KV, D, W>>(smem);
      multi_split_kernel<T, KV, D, W><<<grid, kThreads, smem, s>>>(p);
    };
    if (a.window > 0) run(std::true_type()); else run(std::false_type());
    multi_merge_kernel<T, D><<<mgrid, D, 0, s>>>(p);
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

int decode_attention_paged_shared(const PagedSharedArgs& a, cudaStream_t s) {
  using namespace decode_shared;
  if (a.d != D || a.hkv <= 0 || a.h % a.hkv || a.h / a.hkv > kRows || (a.dtype != kBF16 && a.dtype != kF16)) return 1;
  if (a.kv_dtype != -1 && ((a.kv_dtype != kI8 && a.kv_dtype != kE4M3) || !a.k_dq || !a.v_dq)) return 1;
  if (a.max_blocks <= 0 || a.block_size <= 0 || a.n_tasks < 0 || a.n_members < 0) return 1;
  if (a.q_st % 8 || a.q_sh % 8 || a.o_st % 8 || ((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k_cache) |
                                                  reinterpret_cast<uintptr_t>(a.v_cache)) & 15)) return 1;
  if (a.n_members == 0) return 0;
  Params p;
  p.q = a.q; p.k_cache = a.k_cache; p.v_cache = a.v_cache; p.out = a.out; p.part_acc = a.part_acc; p.part_ml = a.part_ml;
  p.block_tables = a.block_tables; p.cu_q = a.cu_q; p.lens = a.lens; p.group_seqs = a.group_seqs; p.tasks = a.tasks; p.members = a.members;
  p.k_dq = a.k_dq; p.v_dq = a.v_dq;
  p.q_st = a.q_st; p.q_sh = a.q_sh; p.o_st = a.o_st;
  p.h = a.h; p.hkv = a.hkv; p.rows = a.rows; p.max_blocks = a.max_blocks; p.block_size = a.block_size;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  const dim3 grid(a.n_tasks, a.hkv), mgrid(a.n_members, a.hkv);
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    constexpr int smem = decode_multi::Smem<!std::is_same<T, KV>::value, D>::kBytes;
    set_max_dynamic_smem<shared_split_kernel<T, KV>>(smem);
    shared_split_kernel<T, KV><<<grid, kThreads, smem, s>>>(p);
    shared_merge_kernel<T><<<mgrid, D, 0, s>>>(p);
  };
  if (a.dtype == kBF16) {
    if (a.kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8());
    else if (a.kv_dtype == kE4M3) launch(__nv_bfloat16(), kv8::E4M3());
    else launch(__nv_bfloat16(), __nv_bfloat16());
  } else {
    if (a.kv_dtype == kI8) launch(__half(), kv8::I8());
    else if (a.kv_dtype == kE4M3) launch(__half(), kv8::E4M3());
    else launch(__half(), __half());
  }
  return B200_LAUNCH_RESULT();
}

}  // namespace b200
