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
// The kernel bodies live in include/b200_decode_attention.cuh, shared with the sliding-window kernels of attention_window.cu.
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
namespace decode_multi {

template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) multi_split_kernel(const Params p) { multi_split<T, KV, 128>(p); }

template <typename T>
__global__ void __launch_bounds__(128) multi_merge_kernel(const Params p) { multi_merge<T, 128>(p); }

}  // namespace decode_multi

// Verify rows at head_dim 64 (16-bit caches): decode_multi's split and merge bodies at D = 64, in kernels of their own so that the
// head_dim 128 kernels keep their names and code.
namespace decode_verify64 {

struct Params : decode_multi::Params {};

template <typename T>
__global__ void __launch_bounds__(decode_multi::kThreads) multi_split_kernel(const __grid_constant__ Params p) { decode_multi::multi_split<T, T, 64>(p); }

template <typename T>
__global__ void __launch_bounds__(64) multi_merge_kernel(const __grid_constant__ Params p) { decode_multi::multi_merge<T, 64>(p); }

}  // namespace decode_verify64

// Shared-prefix decode ("cascade" decode): single-token decode rows of sequences whose leading blocks are the same physical blocks.
// The host turns the groups into a task list.  A prefix task packs up to 64 / G members of one group (G = H / Hkv query heads per KV
// head; row r = member r / G, head kvh * G + r % G) into one 64-row tile and reads the group's prefix keys [0, prefix_len) through the
// first member's table, with no mask: every prefix key is visible to every member.  A suffix task holds one member's G rows and reads its
// own keys [prefix_len, len).  Both are split over their keys and write unnormalized partials (m, l, acc) at their own rows of one
// [Hkv, rows] buffer; shared_merge_kernel combines every partial of a member's row and writes the output in place.  The tile loop is
// decode_multi's (cp.async three stages deep through the block table, mma.sync m16n8k16 with P in registers, zero-filled keys past the
// end whose table entries are never read, exact 8-bit conversion in shared memory with K's scale in the softmax scale and V's in the
// partial); only the key range, the row packing and the partial layout differ, so its helpers are reused and its kernels are untouched.
namespace decode_shared {

using decode_multi::BN;
using decode_multi::kRows;
using decode_multi::kStages;
using decode_multi::kThreads;
constexpr int D = 128, kTile16 = decode_multi::kTile16<D>, kTile8 = decode_multi::kTile8<D>;

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
__global__ void __launch_bounds__(kThreads) shared_split_kernel(const Params p) {
  constexpr bool Q8 = !std::is_same<T, KV>::value;
  using S = decode_multi::Smem<Q8, D>;
  const int* task = p.tasks + (int64_t)blockIdx.x * kSharedTaskInts;
  const int kvh = blockIdx.y;
  const int tb = task[0], m0 = task[1], cnt = task[2], lo = task[3], split = task[5], splits = task[6];
  const int g_size = p.h / p.hkv, nrows = cnt * g_size;
  const int cap = p.max_blocks * p.block_size, len_tb = p.lens[tb];
  // prefix: keys below prefix_len, never past the reference member's cached ones (a bad group is NaN-ed by the merge); suffix: up to len
  const int hi = task[4] >= 0 ? min(min(task[4], len_tb - 1), cap) : min(len_tb, cap);
  const int ntiles = hi > lo ? (hi - lo + BN - 1) / BN : 0, per = (ntiles + splits - 1) / splits;
  const int t0 = split * per, t1 = min(ntiles, t0 + per);
  const int64_t pbase = (int64_t)kvh * p.rows + task[7];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (t0 >= t1) {                                            // no keys: an empty partial (the merge skips it)
    for (int r = tid; r < nrows; r += kThreads) { p.part_ml[(pbase + r) * 2] = -INFINITY; p.part_ml[(pbase + r) * 2 + 1] = 0.f; }
    return;
  }
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  const int* bt = p.block_tables + (int64_t)tb * p.max_blocks;

  // Q tile: rows past nrows are zero
#pragma unroll
  for (int i = 0; i < kRows * D / 8 / kThreads; ++i) {
    const int row = i * (kThreads / 16) + (tid >> 4), c = tid & 15;
    const bool ok = row < nrows;
    const T* src = reinterpret_cast<const T*>(p.q);
    if (ok) src += (int64_t)p.cu_q[p.group_seqs[m0 + row / g_size]] * p.q_st + (int64_t)(kvh * g_size + row % g_size) * p.q_sh + c * 8;
    decode_multi::cp_async16(sbase + decode_multi::swz<D>(row, c), src, ok);
  }
  // K / V rows of key tile `tile` (keys lo + tile * 64 ...) into stage `st`; keys at or past hi are zero-filled
  auto load_kv = [&](int tile, int st) {
    constexpr int kEl = Q8 ? 16 : 8;
    constexpr int kChunks = D / kEl;
#pragma unroll
    for (int i = 0; i < BN * kChunks / kThreads; ++i) {
      const int row = i * (kThreads / kChunks) + tid / kChunks, c = tid % kChunks;
      const int pos = lo + tile * BN + row;
      const bool ok = pos < hi;
      int64_t off = 0;
      if (ok) off = (((int64_t)bt[pos / p.block_size] * p.hkv + kvh) * p.block_size + pos % p.block_size) * D + c * kEl;
      if constexpr (Q8) {
        const uint32_t dst = sbase + S::kRaw + st * 2 * kTile8 + row * D + c * 16;
        decode_multi::cp_async16(dst, reinterpret_cast<const uint8_t*>(p.k_cache) + off, ok);
        decode_multi::cp_async16(dst + kTile8, reinterpret_cast<const uint8_t*>(p.v_cache) + off, ok);
      } else {
        const uint32_t dst = sbase + S::kKV + st * 2 * kTile16 + decode_multi::swz<D>(row, c);
        decode_multi::cp_async16(dst, reinterpret_cast<const T*>(p.k_cache) + off, ok);
        decode_multi::cp_async16(dst + kTile16, reinterpret_cast<const T*>(p.v_cache) + off, ok);
      }
    }
  };
  load_kv(t0, 0);
  decode_multi::cp_async_commit();
  if (t0 + 1 < t1) load_kv(t0 + 1, 1);
  decode_multi::cp_async_commit();

  float qk_scale = p.scale_log2, v_scale = 1.f;
  if constexpr (Q8) { qk_scale *= __ldg(p.k_dq + kvh); v_scale = __ldg(p.v_dq + kvh); }
  const bool active = warp * 16 < nrows;
  const int r_lo = warp * 16 + (lane >> 2);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float acc[D / 8][4];
#pragma unroll
  for (int n = 0; n < D / 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  uint32_t qf[D / 16][4];

  for (int t = t0; t < t1; ++t) {
    const int st = (t - t0) % kStages;
    decode_multi::cp_async_wait<1>();
    __syncthreads();
    if (t + 2 < t1) load_kv(t + 2, (st + 2) % kStages);
    decode_multi::cp_async_commit();
    if (t == t0 && active) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) decode_multi::ldsm_x4(qf[kk], sbase + decode_multi::swz<D>(warp * 16 + (lane & 15), kk * 2 + (lane >> 4)));
    }
    uint32_t kv16 = sbase + S::kKV + st * 2 * kTile16;
    if constexpr (Q8) {
      kv16 = sbase + S::kKV;
#pragma unroll
      for (int i = 0; i < 2 * BN * (D / 16) / kThreads; ++i) {
        const int id = i * kThreads + tid, kv = id / (BN * 8), row = (id / 8) % BN, c = id % 8;
        const uint4 raw = *reinterpret_cast<const uint4*>(smem + S::kRaw + st * 2 * kTile8 + kv * kTile8 + row * D + c * 16);
        float f[16];
        kv8::to_float16<KV>(raw, f);
        uint32_t w[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) w[e] = pack2<T>(f[2 * e], f[2 * e + 1]);
        uint8_t* dst = smem + S::kKV + kv * kTile16;
        *reinterpret_cast<uint4*>(dst + decode_multi::swz<D>(row, 2 * c)) = make_uint4(w[0], w[1], w[2], w[3]);
        *reinterpret_cast<uint4*>(dst + decode_multi::swz<D>(row, 2 * c + 1)) = make_uint4(w[4], w[5], w[6], w[7]);
      }
      __syncthreads();
    }
    if (active) {
      float s[BN / 8][4];
#pragma unroll
      for (int n = 0; n < BN / 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
        for (int np = 0; np < BN / 16; ++np) {
          uint32_t bf[4];
          decode_multi::ldsm_x4(bf, kv16 + decode_multi::swz<D>(np * 16 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1)));
          decode_multi::mma16816<T>(s[2 * np], qf[kk], bf[0], bf[1]);
          decode_multi::mma16816<T>(s[2 * np + 1], qf[kk], bf[2], bf[3]);
        }
      }
      // every row sees every key below hi: only the zero-filled keys of the last tile are masked
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int n = 0; n < BN / 8; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = lo + t * BN + n * 8 + 2 * (lane & 3) + e;
            float& v = s[n][hh * 2 + e];
            v = key < hi ? v * qk_scale : -INFINITY;
            mx = fmaxf(mx, v);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[hh], mx);
        const float base = m_new == -INFINITY ? 0.f : m_new;
        const float alpha = exp2f(m[hh] - base);
        float sum = 0.f;
#pragma unroll
        for (int n = 0; n < BN / 8; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = s[n][hh * 2 + e];
            v = exp2f(v - base);
            sum += v;
          }
        l[hh] = l[hh] * alpha + sum;
        m[hh] = m_new;
#pragma unroll
        for (int n = 0; n < D / 8; ++n) { acc[n][hh * 2] *= alpha; acc[n][hh * 2 + 1] *= alpha; }
      }
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        const uint32_t pa[4] = {pack2<T>(s[2 * kk][0], s[2 * kk][1]), pack2<T>(s[2 * kk][2], s[2 * kk][3]),
                                pack2<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]), pack2<T>(s[2 * kk + 1][2], s[2 * kk + 1][3])};
#pragma unroll
        for (int np = 0; np < D / 16; ++np) {
          uint32_t bf[4];
          decode_multi::ldsm_x4_t(bf, kv16 + kTile16 + decode_multi::swz<D>(kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), np * 2 + (lane >> 4)));
          decode_multi::mma16816<T>(acc[2 * np], pa, bf[0], bf[1]);
          decode_multi::mma16816<T>(acc[2 * np + 1], pa, bf[2], bf[3]);
        }
      }
    }
  }
  decode_multi::cp_async_wait<0>();
  if (!active) return;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float lq = l[hh];
    lq += __shfl_xor_sync(0xffffffffu, lq, 1);
    lq += __shfl_xor_sync(0xffffffffu, lq, 2);
    const int r = r_lo + hh * 8;
    if (r >= nrows) continue;
    float* pa = p.part_acc + (pbase + r) * D + 2 * (lane & 3);
#pragma unroll
    for (int n = 0; n < D / 8; ++n) *reinterpret_cast<float2*>(pa + n * 8) = make_float2(acc[n][hh * 2] * v_scale, acc[n][hh * 2 + 1] * v_scale);
    if ((lane & 3) == 0) { p.part_ml[(pbase + r) * 2] = m[hh]; p.part_ml[(pbase + r) * 2 + 1] = lq; }
  }
}

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
  if (window > 0)
    return decode_attention_window(q, k_cache, v_cache, lens, out, part_acc, part_ml, b, h, hkv, smax, d, splits, scale, dtype, s, block_tables, max_blocks,
                                   block_size, window);
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_d) {
    using T = decltype(tag_t);
    constexpr int D = decltype(tag_d)::value;
    decode_split_kernel<T, D><<<grid, kThreads, 0, s>>>((const T*)q, (const T*)k_cache, (const T*)v_cache, lens, part_acc, part_ml, h, hkv, smax, splits,
                                                        sl2, block_tables, max_blocks, block_size);
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
  if (window > 0)
    return decode_attention_paged_q8_window(q, k_cache, v_cache, lens, out, part_acc, part_ml, b, h, hkv, splits, scale, dtype, kv_dtype, k_dq, v_dq,
                                            block_tables, max_blocks, block_size, window, s);
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    decode_split_q8_kernel<T, decltype(tag_kv)><<<grid, kThreads, 0, s>>>((const T*)q, (const uint8_t*)k_cache, (const uint8_t*)v_cache, lens,
                                                                          part_acc, part_ml, h, hkv, splits, sl2, k_dq, v_dq, block_tables,
                                                                          max_blocks, block_size);
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
  if (a.window > 0) return decode_attention_paged_multi_window(p, a, s);
  const dim3 grid(a.splits, a.hkv, a.b), mgrid(kRows, a.hkv, a.b);
  if (a.d == 64) {
    auto launch64 = [&](auto tag_t) {
      using T = decltype(tag_t);
      constexpr int smem = Smem<false, 64>::kBytes;
      decode_verify64::Params p64;
      static_cast<Params&>(p64) = p;
      set_max_dynamic_smem<decode_verify64::multi_split_kernel<T>>(smem);
      decode_verify64::multi_split_kernel<T><<<grid, kThreads, smem, s>>>(p64);
      decode_verify64::multi_merge_kernel<T><<<mgrid, 64, 0, s>>>(p64);
    };
    if (a.dtype == kBF16) launch64(__nv_bfloat16()); else launch64(__half());
    return B200_LAUNCH_RESULT();
  }
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    constexpr int smem = Smem<!std::is_same<T, KV>::value, 128>::kBytes;
    set_max_dynamic_smem<multi_split_kernel<T, KV>>(smem);
    multi_split_kernel<T, KV><<<grid, kThreads, smem, s>>>(p);
    multi_merge_kernel<T><<<mgrid, 128, 0, s>>>(p);
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
