// Flash-attention forward for sm_90a (head_dim 128, bf16/fp16): S = Q K^T and O += P V run on wgmma tensor cores, K/V tiles streamed
// by TMA (4-D maps straight over the strided [B,S,H,D] views of a packed QKV tensor, so no q/k/v split copies), online softmax on the
// accumulator fragment in registers, and P never leaves registers: the S fragment of a thread IS the A-operand fragment of the P V MMA
// once packed to 16 bits.  Hand-written PTX; no CUTLASS, no library attention.
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
// PAGED over 8-bit caches (KV = kv8::I8 / kv8::E4M3; q and o stay fp16 / bf16): a converter warpgroup (warps 8-11, 384 threads) takes
// the TMA producer's place for K and V.  Its threads read the 8-bit rows through the block table with 16-byte loads, convert them
// exactly to 16 bits and store them into the same swizzled K / V tiles, then fence.proxy.async and arrive on the tiles' mbarriers; keys
// past the sequence are written as zeros, so stale or NaN cache rows never reach the MMAs.  The K dequant scale is folded into the exp2
// scale and the V dequant scale into the epilogue's 1 / l, so the MMA and softmax code is the 16-bit kernel's.
#include <cuda.h>
#include <algorithm>
#include <cstdio>
#include <string>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace attn {
using namespace ptx;

constexpr int BM = 128, BN = 128, HD = 128;
constexpr int kThreads = 288;   // warps 0-7: two MMA / softmax warpgroups, warp 8: TMA producer
constexpr int kThreadsQ8 = 384; // 8-bit paged caches: warps 8-11 convert K / V (warp 8 lane 0 also loads Q)
constexpr uint32_t TILE_BYTES = 128 * 128 * 2;   // 32 KB: every operand tile (Q, K, V)
constexpr uint32_t HALF_BYTES = TILE_BYTES / 2;  // one 64-wide K-block of a tile
constexpr uint32_t SMEM_BYTES = 5 * TILE_BYTES + 1024 /*align*/ + 256 /*barriers*/;   // Q, 2x K, 2x V

template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
  const __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}

struct Params {
  int b, sq, sk, h, hk;
  float scale_log2;
  int causal, causal_off;     // key j is visible to query i iff j <= i + causal_off
  void* o;
  float* lse;
  int64_t o_sb, o_ss, o_sh;   // element strides of the output [B,S,H,D]
  const int4* colmask;        // [b, mask_heads, sk] row ranges hidden from every key column (nullptr: none)
  int mask_heads;
};
// The paged instantiation's parameters (the dense ones keep the smaller Params: a different kernel-parameter block changes their code).
// sq is the number of packed token rows, b the number of sequences.
struct PagedParams : Params {
  const int2* work;           // [gridDim.y] {sequence, query tile}; sequence < 0: spare CTA
  const int* cu_q;            // [b] first packed row of each sequence's new tokens
  const int* n_q;             // [b] new tokens (0: not a prefill sequence)
  const int* past;            // [b] tokens already cached before them
  const int* block_tables;    // [b, max_blocks]
  int max_blocks, block_size;
};
// 8-bit paged caches: the caches are read by the converter warpgroup, not through tensor maps.
struct QuantPagedParams : PagedParams {
  const uint8_t* k_cache;     // [num_blocks, hk, block_size, D]
  const uint8_t* v_cache;
  const float* k_dq;          // [hk] dequant scales
  const float* v_dq;
};

__device__ __forceinline__ void st_shared_zero16(uint32_t addr) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(addr), "r"(0) : "memory");
}

// MASKED: column-wise row-range mask (flashmask / varlen) compiled in; the dense instantiation carries none of its code or registers
// PAGED: queries = new tokens of each sequence, K / V read through the block table (see the file header); always causal, never MASKED
// KV: the cache element type; kv8::I8 / kv8::E4M3 (PAGED only) select the converter warpgroup and QuantPagedParams
template <typename T, bool MASKED, bool PAGED = false, typename KV = T>
__global__ void __launch_bounds__(std::is_same<KV, T>::value ? kThreads : kThreadsQ8, 1)
fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
           const std::conditional_t<PAGED, std::conditional_t<std::is_same<KV, T>::value, PagedParams, QuantPagedParams>, Params> p) {
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr bool Q8 = !std::is_same<KV, T>::value;
  static_assert(!Q8 || (PAGED && !MASKED), "8-bit caches are paged only");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  auto sK = [&](int s) { return base + (1 + s) * TILE_BYTES; };
  auto sV = [&](int s) { return base + (3 + s) * TILE_BYTES; };
  const uint32_t bars = base + 5 * TILE_BYTES;
  const uint32_t q_full = bars;
  auto k_full = [&](int s) { return bars + 8u * (1 + s); };
  auto v_full = [&](int s) { return bars + 8u * (3 + s); };
  auto k_empty = [&](int s) { return bars + 8u * (5 + s); };    // 8 warp arrivals
  auto v_empty = [&](int s) { return bars + 8u * (7 + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int m_tile, head, batch, sk, causal_off, nrows, q0 = 0;
  if constexpr (PAGED) {
    const int2 w = p.work[blockIdx.y];
    if (w.x < 0) return;                                      // spare CTA: the grid is an upper bound on the work list
    batch = w.x; m_tile = w.y; head = blockIdx.x;
    q0 = __ldg(p.cu_q + batch);
    nrows = __ldg(p.n_q + batch);
    causal_off = __ldg(p.past + batch);
    sk = causal_off + nrows;
  } else {
    m_tile = (int)gridDim.x - 1 - (int)blockIdx.x;          // long (late) rows first under the causal mask
    head = blockIdx.y; batch = blockIdx.z;
    sk = p.sk; causal_off = p.causal_off; nrows = p.sq;
  }
  const int kv_head = head / (p.h / p.hk);
  const int m0 = m_tile * BM;
  int n_tiles = (sk + BN - 1) / BN;
  if (p.causal) {                                            // always set for PAGED
    const int last_key = min(sk - 1, m0 + BM - 1 + causal_off);
    n_tiles = last_key < 0 ? 0 : min(n_tiles, last_key / BN + 1);
  }

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_q);
    if constexpr (!Q8) {
      tma_prefetch_desc(&map_k);
      tma_prefetch_desc(&map_v);
    }
    mbar_init(q_full, 1);
    constexpr uint32_t kv_arrivals = Q8 ? 4 : 1;   // converter warps, or the producer's expect_tx
    for (int s = 0; s < 2; ++s) {
      mbar_init(k_full(s), kv_arrivals); mbar_init(v_full(s), kv_arrivals); mbar_init(k_empty(s), 8); mbar_init(v_empty(s), 8);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (Q8 ? warp >= 8 : warp == 8) {
    if constexpr (Q8) {
      if (n_tiles > 0) {
        // ================= converter warpgroup: thread c of 8 takes d [16c, 16c + 16) of key rows (tid / 8) + 16 i, i < 8 =================
        const int tid = threadIdx.x - 256, c = tid & 7, r0 = tid >> 3;
        if (tid == 0) {
          mbar_expect_tx(q_full, TILE_BYTES);
          tma_load_4d(sQ, &map_q, q_full, 0, q0 + m0, head, 0);
          tma_load_4d(sQ + HALF_BYTES, &map_q, q_full, 64, q0 + m0, head, 0);
        }
        const int bsz = p.block_size, bshift = __ffs(bsz) - 1;
        const int* bt = p.block_tables + (int64_t)batch * p.max_blocks;
        const int64_t blk_stride = (int64_t)p.hk * bsz * HD;
        const uint8_t* kcache = p.k_cache + (int64_t)kv_head * bsz * HD + c * 16;
        const uint8_t* vcache = p.v_cache + (int64_t)kv_head * bsz * HD + c * 16;
        // 16 converted values (16-byte chunks 2c, 2c + 1 of a 128-column row) -> the swizzled 16-bit tile row at `row_addr`
        auto store_row = [&](const uint4& raw, uint32_t row_addr, int r) {
          float f[16];
          kv8::to_float16<KV>(raw, f);
          uint32_t w[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) w[i] = pack2<T>(f[2 * i], f[2 * i + 1]);
#pragma unroll
          for (int hc = 0; hc < 2; ++hc)
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(row_addr + ((((2 * c + hc) & 7) ^ (r & 7)) << 4)),
                         "r"(w[4 * hc]), "r"(w[4 * hc + 1]), "r"(w[4 * hc + 2]), "r"(w[4 * hc + 3]) : "memory");
        };
        for (int j = 0; j < n_tiles; ++j) {
          const int s = j & 1;
          const uint32_t ph = ((j >> 1) & 1) ^ 1;
          uint4 kr[8], vr[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // both tiles' loads in flight before the first wait
            const int key = j * BN + i * 16 + r0;
            kr[i] = vr[i] = make_uint4(0, 0, 0, 0);
            if (key < sk) {
              const int64_t off = __ldg(bt + (key >> bshift)) * blk_stride + (int64_t)(key & (bsz - 1)) * HD;
              kr[i] = __ldg(reinterpret_cast<const uint4*>(kcache + off));
              vr[i] = __ldg(reinterpret_cast<const uint4*>(vcache + off));
            }
          }
          mbar_wait(k_empty(s), ph);
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // K tile: key rows of 128 bytes, d-half c / 4 at HALF_BYTES
            const int r = i * 16 + r0;
            store_row(kr[i], sK(s) + (c >> 2) * HALF_BYTES + r * 128, r);
          }
          fence_proxy_async();           // generic-proxy stores before the wgmma (async proxy) reads them
          __syncwarp();
          if (lane == 0) mbar_arrive(k_full(s));
          mbar_wait(v_empty(s), ph);
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // V tile: 64-key blocks at HALF_BYTES, d-halves 8192 B apart
            const int r = i * 16 + r0;
            store_row(vr[i], sV(s) + (r >> 6) * HALF_BYTES + (c >> 2) * 8192 + (r & 63) * 128, r);
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(v_full(s));
        }
      }
    } else if constexpr (PAGED) {
      if (n_tiles > 0) {
        // ================= TMA producer, paged: lane l loads box l % C of K half / V d-half l / C =================
        const int bsz = p.block_size, R = min(bsz, 64), C = BN / R;   // C boxes of R key rows per 128-key K half and per 64-d V half
        const int* bt = p.block_tables + (int64_t)batch * p.max_blocks;
        const int last_blk = __ldg(bt + (sk - 1) / bsz);            // table entries past the sequence are never read
        const int c = lane % C, half = lane / C;
        if (lane == 0) {
          mbar_expect_tx(q_full, TILE_BYTES);
          tma_load_4d(sQ, &map_q, q_full, 0, q0 + m0, head, 0);
          tma_load_4d(sQ + HALF_BYTES, &map_q, q_full, 64, q0 + m0, head, 0);
        }
        for (int j = 0; j < n_tiles; ++j) {
          const int s = j & 1, key = j * BN + c * R;
          const uint32_t ph = ((j >> 1) & 1) ^ 1;
          // keys past the sequence come from a valid block (masked in S, zeroed in V) so every tile carries the same bytes
          const int blk = lane < 2 * C ? (key < sk ? __ldg(bt + key / bsz) : last_blk) : 0;
          const int row = key % bsz;
          mbar_wait(k_empty(s), ph);
          if (lane == 0) mbar_expect_tx(k_full(s), TILE_BYTES);
          __syncwarp();
          if (lane < 2 * C) tma_load_4d(sK(s) + half * HALF_BYTES + c * R * 128, &map_k, k_full(s), half * 64, row, kv_head, blk);
          mbar_wait(v_empty(s), ph);
          if (lane == 0) mbar_expect_tx(v_full(s), TILE_BYTES);
          __syncwarp();
          if (lane < 2 * C)
            tma_load_4d(sV(s) + (c * R / 64) * HALF_BYTES + half * 8192 + (c * R % 64) * 128, &map_v, v_full(s), half * 64, row, kv_head, blk);
        }
      }
    } else if (lane == 0 && n_tiles > 0) {
      // ================= TMA producer =================
      mbar_expect_tx(q_full, TILE_BYTES);
      tma_load_4d(sQ, &map_q, q_full, 0, m0, head, batch);
      tma_load_4d(sQ + HALF_BYTES, &map_q, q_full, 64, m0, head, batch);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j & 1, n0 = j * BN;
        const uint32_t ph = ((j >> 1) & 1) ^ 1;
        mbar_wait(k_empty(s), ph);
        mbar_expect_tx(k_full(s), TILE_BYTES);
        tma_load_4d(sK(s), &map_k, k_full(s), 0, n0, kv_head, batch);               // box {64 d, 128 keys}: K-major B operand
        tma_load_4d(sK(s) + HALF_BYTES, &map_k, k_full(s), 64, n0, kv_head, batch);
        mbar_wait(v_empty(s), ph);
        mbar_expect_tx(v_full(s), TILE_BYTES);
#pragma unroll
        for (int kb = 0; kb < 2; ++kb)                                              // box {64 d, 64 keys}: MN-major B operand
#pragma unroll
          for (int i = 0; i < 2; ++i)
            tma_load_4d(sV(s) + kb * HALF_BYTES + i * 8192, &map_v, v_full(s), i * 64, n0 + kb * 64, kv_head, batch);
      }
    }
  } else {
    // ================= MMA + softmax + epilogue: warpgroup wg owns query rows [64 wg, 64 wg + 64) =================
    const int wg = warp >> 2, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: rl and rl + 8
    float scale_log2 = p.scale_log2;
    if constexpr (Q8) scale_log2 *= __ldg(p.k_dq + kv_head);  // S is computed on the quantized K
    float o_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o_acc[i] = 0.f;
    float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};   // l_i: this thread's share of the row sum (reduced over the quad at the end)
    if (n_tiles > 0) mbar_wait(q_full, 0);
    for (int j = 0; j < n_tiles; ++j) {
      const int s = j & 1, ph = (j >> 1) & 1;
      float sv[BN / 2];
      mbar_wait(k_full(s), ph);
      wgmma_fence_regs(sv);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss_n128<BF16, 0, 0>(sv, make_smem_desc(sQ + kb * HALF_BYTES + wg * 8192 + k * 32, 16, 1024),
                                    make_smem_desc(sK(s) + kb * HALF_BYTES + k * 32, 16, 1024), (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sv);
      __syncwarp();
      if (lane == 0) mbar_arrive(k_empty(s));
      // ---- masks (raw logits; the softmax scale is folded into the exp2 FFMA) ----
      const bool edge = PAGED ? (j * BN + BN > sk) || (j * BN + BN - 1 > m0 + causal_off)
                              : (j * BN + BN > p.sk) || (p.causal && j * BN + BN - 1 > m0 + p.causal_off);
      if (edge) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + rl + h * 8;
          const int lim = (p.causal ? min(sk - 1, row + causal_off) : sk - 1) - j * BN;   // last visible key, tile-relative
#pragma unroll
          for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (jn * 8 + 2 * q + e > lim) sv[jn * 4 + h * 2 + e] = -INFINITY;
        }
      }
      if constexpr (MASKED) {     // flashmask / varlen: key column j hides the query rows [lt_start, lt_end) and [ut_start, ut_end)
        const int4* cm = p.colmask + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.sk;
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = j * BN + jn * 8 + 2 * q + e;
            if (key < p.sk) {
              const int4 m = __ldg(cm + key);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int row = m0 + rl + h * 8;
                if ((row >= m.x && row < m.y) || (row >= m.z && row < m.w)) sv[jn * 4 + h * 2 + e] = -INFINITY;
              }
            }
          }
      }
      // ---- online softmax: a row lives in the four lanes of a quad ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn) mx = fmaxf(mx, fmaxf(sv[jn * 4 + h * 2], sv[jn * 4 + h * 2 + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float m_new = fmaxf(m_i[h], mx * scale_log2);     // scale > 0
        if (m_new == -INFINITY) m_new = 0.f;                // fully masked so far: keep exp2 finite
        const float alpha = ex2(m_i[h] - m_new);
        m_i[h] = m_new;
        float sum = 0.f;
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pv = ex2(fmaf(sv[jn * 4 + h * 2 + e], scale_log2, -m_new));
            sv[jn * 4 + h * 2 + e] = pv;
            sum += pv;
          }
        l_i[h] = l_i[h] * alpha + sum;
#pragma unroll
        for (int jn = 0; jn < HD / 8; ++jn) { o_acc[jn * 4 + h * 2] *= alpha; o_acc[jn * 4 + h * 2 + 1] *= alpha; }
      }
      // ---- P as A fragments: 16-key step ks = accumulator column groups 2 ks and 2 ks + 1 ----
      uint32_t pa[BN / 16][4];
#pragma unroll
      for (int ks = 0; ks < BN / 16; ++ks) {
        pa[ks][0] = pack2<T>(sv[ks * 8 + 0], sv[ks * 8 + 1]);
        pa[ks][1] = pack2<T>(sv[ks * 8 + 2], sv[ks * 8 + 3]);
        pa[ks][2] = pack2<T>(sv[ks * 8 + 4], sv[ks * 8 + 5]);
        pa[ks][3] = pack2<T>(sv[ks * 8 + 6], sv[ks * 8 + 7]);
      }
      mbar_wait(v_full(s), ph);
      if constexpr (PAGED && !Q8) {   // (the converter writes zeros past the sequence)
        if (j * BN + BN > sk) {   // V rows past the sequence hold stale cache contents (possibly NaN) and P = 0 does not cancel NaN: zero them
          const int tid = threadIdx.x & 127;
          for (int e = (sk - j * BN) * 16 + tid; e < BN * 16; e += 128) {   // 16-byte chunks: key row e / 16, d-half (e / 8) & 1
            const int r = e >> 4;
            st_shared_zero16(sV(s) + (r >> 6) * HALF_BYTES + ((e >> 3) & 1) * 8192 + (r & 63) * 128 + (e & 7) * 16);
          }
          fence_proxy_async();                    // generic-proxy stores before this warpgroup's wgmma reads them
          named_bar_sync(1 + wg, 128);
        }
      }
      wgmma_fence_regs(o_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BN / 16; ++ks)     // V tile MN-major: 64-key block ks / 4, 16 key rows = 2048 B per step, 64-wide d chunks 8192 B apart
        wgmma_rs_n128<BF16, 1>(o_acc, pa[ks], make_smem_desc(sV(s) + (ks >> 2) * HALF_BYTES + (ks & 3) * 2048, 8192, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o_acc);
#pragma unroll
      for (int ks = 0; ks < BN / 16; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(pa[ks][i])::"memory");   // read asynchronously until the wait above
      __syncwarp();
      if (lane == 0) mbar_arrive(v_empty(s));
    }
    // ---- epilogue ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_i[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      float inv = l > 0.f ? 1.f / l : 0.f;
      if constexpr (Q8) inv *= __ldg(p.v_dq + kv_head);   // O is accumulated on the quantized V
      const int row = m0 + rl + h * 8;
      if (row < nrows) {
        T* orow = reinterpret_cast<T*>(p.o) + (PAGED ? 0 : (int64_t)batch * p.o_sb) + (int64_t)(q0 + row) * p.o_ss + (int64_t)head * p.o_sh;
#pragma unroll
        for (int jn = 0; jn < HD / 8; ++jn)
          *reinterpret_cast<uint32_t*>(orow + jn * 8 + 2 * q) = pack2<T>(o_acc[jn * 4 + h * 2] * inv, o_acc[jn * 4 + h * 2 + 1] * inv);
        if (q == 0 && p.lse) p.lse[((int64_t)(PAGED ? 0 : batch) * p.h + head) * p.sq + q0 + row] = l > 0.f ? (m_i[h] + log2f(l)) * 0.69314718055994531f : -INFINITY;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 4-D map {d, s, h, b} over a strided [B,S,H,D] view (strides in elements), box {64, rows, 1, 1}, 128B swizzle
static bool make_map4(CUtensorMap* out, const void* ptr, int d, int s, int h, int b, int64_t ss, int64_t sh, int64_t sb, uint32_t box_rows, int dtype) {
  bind_primary_context();
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_last_error(__FILE__, __LINE__, "cuTensorMapEncodeTiled unavailable"); return false; }
  cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)s, (cuuint64_t)h, (cuuint64_t)b};
  cuuint64_t strides[3] = {(cuuint64_t)ss * 2, (cuuint64_t)sh * 2, (cuuint64_t)sb * 2};
  cuuint32_t box[4] = {64, box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(out, dtype == kBF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr),
                   dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error(__FILE__, __LINE__, ("cuTensorMapEncodeTiled (attention) failed: " + std::to_string((int)r)).c_str());
    return false;
  }
  return true;
}

// Work list of the paged kernel: one (sequence, 128-row query tile) per slot, sorted by key tiles (heaviest first, ties in sequence
// order) so a long prefix starts early instead of running alone at the end; slots past the list get sequence -1.  One CTA; the
// O(tiles^2) ranking is a few hundred thousand compares at the largest batches, well under the attention it schedules.
// scratch: int32 [slots] key-tile counts followed by [b + 1] tile offsets.
__global__ void __launch_bounds__(1024) paged_work_kernel(const int* __restrict__ n_q, const int* __restrict__ past, int b, int slots,
                                                          int* scratch, int2* work) {
  int* keys = scratch;
  int* start = scratch + slots;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < b; ++i) { start[i] = acc; acc += (max(n_q[i], 0) + BM - 1) / BM; }
    start[b] = acc;
  }
  __syncthreads();
  const int n = min(start[b], slots);
  auto seq_of = [&](int w) {   // last sequence whose first tile is <= w (sequences without tiles share their successor's offset)
    int lo = 0, hi = b - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (start[mid] <= w) lo = mid; else hi = mid - 1;
    }
    return lo;
  };
  for (int w = threadIdx.x; w < n; w += blockDim.x) {
    const int sq = seq_of(w), m0 = (w - start[sq]) * BM;
    keys[w] = (past[sq] + min(n_q[sq] - 1, m0 + BM - 1)) / BN + 1;   // key tiles up to the causal limit of the tile's last row
  }
  __syncthreads();
  for (int w = threadIdx.x; w < slots; w += blockDim.x) {
    if (w < n) {
      const int kw = keys[w];
      int rank = 0;
      for (int u = 0; u < n; ++u) {
        const int ku = keys[u];
        rank += (ku > kw) || (ku == kw && u < w);
      }
      const int sq = seq_of(w);
      work[rank] = make_int2(sq, w - start[sq]);
    } else {
      work[w] = make_int2(-1, -1);
    }
  }
}

}  // namespace attn

int attention_fwd_supported(const AttnArgs& a) {
  if (a.d != 128 || (a.dtype != kBF16 && a.dtype != kF16)) return 0;
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
  using namespace attn;
  if (!attention_fwd_supported(a)) return 1;
  CUtensorMap mq, mk, mv;
  // strides arrays are (batch, seq, head)
  if (!make_map4(&mq, a.q, a.d, a.sq, a.h, a.b, a.q_strides[1], a.q_strides[2], a.q_strides[0], BM, a.dtype)) return 2;
  if (!make_map4(&mk, a.k, a.d, a.sk, a.hk, a.b, a.k_strides[1], a.k_strides[2], a.k_strides[0], BN, a.dtype)) return 2;
  if (!make_map4(&mv, a.v, a.d, a.sk, a.hk, a.b, a.v_strides[1], a.v_strides[2], a.v_strides[0], 64, a.dtype)) return 2;
  Params p;
  p.b = a.b; p.sq = a.sq; p.sk = a.sk; p.h = a.h; p.hk = a.hk;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.causal = a.causal; p.causal_off = a.sk - a.sq;
  p.o = a.o; p.lse = a.lse;
  p.o_sb = a.o_strides[0]; p.o_ss = a.o_strides[1]; p.o_sh = a.o_strides[2];
  p.colmask = reinterpret_cast<const int4*>(a.colmask);
  p.mask_heads = a.mask_heads > 0 ? a.mask_heads : 1;
  dim3 grid((a.sq + BM - 1) / BM, a.h, a.b);
  static bool attr_bf = false, attr_h = false;
  static bool attr_bf_m = false, attr_h_m = false;
  if (a.dtype == kBF16 && !p.colmask) {
    auto kern = fwd_kernel<__nv_bfloat16, false>;
    if (!attr_bf) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_bf = true; }
    kern<<<grid, kThreads, SMEM_BYTES, s>>>(mq, mk, mv, p);
  } else if (a.dtype == kBF16) {
    auto kern = fwd_kernel<__nv_bfloat16, true>;
    if (!attr_bf_m) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_bf_m = true; }
    kern<<<grid, kThreads, SMEM_BYTES, s>>>(mq, mk, mv, p);
  } else if (!p.colmask) {
    auto kern = fwd_kernel<__half, false>;
    if (!attr_h) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_h = true; }
    kern<<<grid, kThreads, SMEM_BYTES, s>>>(mq, mk, mv, p);
  } else {
    auto kern = fwd_kernel<__half, true>;
    if (!attr_h_m) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_h_m = true; }
    kern<<<grid, kThreads, SMEM_BYTES, s>>>(mq, mk, mv, p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

int attention_paged_prefill_slots(int t, int b) { return (t + attn::BM - 1) / attn::BM + b; }
int attention_paged_prefill_scratch_ints(int t, int b) { return 3 * attention_paged_prefill_slots(t, b) + b + 1; }

int attention_paged_prefill_supported(const PagedAttnArgs& a) {
  if (a.d != 128 || (a.dtype != kBF16 && a.dtype != kF16)) return 0;
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
  int2* work = reinterpret_cast<int2*>(a.scratch);
  if (a.kv_dtype != -1) {   // 8-bit caches: no tensor maps over them (the converter warpgroup reads them)
    paged_work_kernel<<<1, 1024, 0, s>>>(a.n_q, a.past, a.b, slots, a.scratch + 2 * slots, work);
    QuantPagedParams p = {};
    p.b = a.b; p.sq = a.t; p.sk = 0; p.h = a.h; p.hk = a.hk;
    p.scale_log2 = a.scale * 1.4426950408889634f;
    p.causal = 1; p.causal_off = 0;
    p.o = a.o; p.lse = a.lse;
    p.o_sb = 0; p.o_ss = a.o_strides[0]; p.o_sh = a.o_strides[1];
    p.colmask = nullptr; p.mask_heads = 1;
    p.work = work; p.cu_q = a.cu_q; p.n_q = a.n_q; p.past = a.past;
    p.block_tables = a.block_tables; p.max_blocks = a.max_blocks; p.block_size = a.block_size;
    p.k_cache = reinterpret_cast<const uint8_t*>(a.k_cache); p.v_cache = reinterpret_cast<const uint8_t*>(a.v_cache);
    p.k_dq = a.k_dq; p.v_dq = a.v_dq;
    dim3 grid(a.h, slots);
    auto launch = [&](auto kern, bool& attr) {
      if (!attr) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr = true; }
      kern<<<grid, kThreadsQ8, SMEM_BYTES, s>>>(mq, mq, mq, p);
    };
    static bool attr[4] = {};
    const bool i8 = a.kv_dtype == kI8;
    if (a.dtype == kBF16) {
      if (i8) launch(fwd_kernel<__nv_bfloat16, false, true, kv8::I8>, attr[0]); else launch(fwd_kernel<__nv_bfloat16, false, true, kv8::E4M3>, attr[1]);
    } else {
      if (i8) launch(fwd_kernel<__half, false, true, kv8::I8>, attr[2]); else launch(fwd_kernel<__half, false, true, kv8::E4M3>, attr[3]);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
    return 0;
  }
  if (!make_map4(&mk, a.k_cache, a.d, a.block_size, a.hk, a.num_blocks, a.d, blk, blk * a.hk, rows, a.dtype)) return 2;
  if (!make_map4(&mv, a.v_cache, a.d, a.block_size, a.hk, a.num_blocks, a.d, blk, blk * a.hk, rows, a.dtype)) return 2;
  paged_work_kernel<<<1, 1024, 0, s>>>(a.n_q, a.past, a.b, slots, a.scratch + 2 * slots, work);
  PagedParams p = {};
  p.b = a.b; p.sq = a.t; p.sk = 0; p.h = a.h; p.hk = a.hk;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  p.causal = 1; p.causal_off = 0;
  p.o = a.o; p.lse = a.lse;
  p.o_sb = 0; p.o_ss = a.o_strides[0]; p.o_sh = a.o_strides[1];
  p.colmask = nullptr; p.mask_heads = 1;
  p.work = work; p.cu_q = a.cu_q; p.n_q = a.n_q; p.past = a.past;
  p.block_tables = a.block_tables; p.max_blocks = a.max_blocks; p.block_size = a.block_size;
  dim3 grid(a.h, slots);   // every head of the heaviest tile is dispatched first
  static bool attr_bf = false, attr_h = false;
  if (a.dtype == kBF16) {
    auto kern = fwd_kernel<__nv_bfloat16, false, true>;
    if (!attr_bf) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_bf = true; }
    kern<<<grid, kThreads, SMEM_BYTES, s>>>(mq, mk, mv, p);
  } else {
    auto kern = fwd_kernel<__half, false, true>;
    if (!attr_h) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_h = true; }
    kern<<<grid, kThreads, SMEM_BYTES, s>>>(mq, mk, mv, p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

}  // namespace b200
