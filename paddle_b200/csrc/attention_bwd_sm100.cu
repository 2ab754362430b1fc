// Flash-attention backward for sm_90a (head_dim 128, bf16/fp16), wgmma + TMA, in two kernels that share no atomics:
//
//   dkv_kernel: one CTA owns a 128-key K/V tile of one (batch, kv head) - 64 keys per MMA warpgroup - and walks the 64-row query tiles
//     that can see it (and, under GQA, every query head of the group).  It computes the TRANSPOSED tiles S^T = K Q^T and dP^T = V dO^T
//     (accumulator row = key), so that P^T and dS^T, packed to 16 bits, are already the register A fragments of dV += P^T dO and
//     dK += dS^T Q: nothing is staged in shared memory and the dV / dK accumulators stay in registers across the whole loop.
//   dq_kernel: one CTA owns 128 query rows of one (batch, head) - 64 per warpgroup - and walks the 64-key tiles it can see: S = Q K^T,
//     dP = dO V^T (accumulator row = query), dS packed in registers is the A fragment of dQ += dS K.  Every dQ element is written once,
//     by one thread, in a fixed order: the result is bitwise reproducible without turn-taking and dQ needs no fp32 atomics.
//   Recomputing S and dP in the second kernel costs 2 of 7 GEMMs; in exchange no tile is transposed through shared memory and the
//     register budget of each kernel holds its accumulators without spilling.
// The K and Q tiles are consumed K-major (S) and MN-major (dQ, dK) from one copy by choice of descriptor.
//
// Parity (behaviour): flash_attn_grad (paddle/phi/kernels/gpu/flash_attn_grad_kernel.cu -> flash-attention library).
#include <cuda.h>
#include <cstdio>
#include <string>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace attn_bwd {
using namespace ptx;

constexpr int HD = 128;
constexpr int kThreads = 288;      // dq_kernel: warps 0-7 two MMA warpgroups, warp 8 TMA producer
constexpr int kThreadsDkv = 384;   // dkv_kernel: warpgroup 0 = producer (warp 0) giving its registers to the MMA warpgroups 1 and 2
constexpr uint32_t BIG_BYTES = 128 * 128 * 2;     // a 128-row tile: two 64-wide d halves [half][row][128 B swizzled]
constexpr uint32_t BIG_HALF = BIG_BYTES / 2;
constexpr uint32_t SMALL_BYTES = 64 * 128 * 2;    // a 64-row tile, same structure
constexpr uint32_t SMALL_HALF = SMALL_BYTES / 2;
constexpr uint32_t SMEM_BYTES = 2 * BIG_BYTES + 4 * SMALL_BYTES + 1024 + 256;   // two resident 128-row tiles + two double-buffered 64-row tiles

template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
  const __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ void keep_regs(uint32_t (&a)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(a[i][j])::"memory");
}

struct Params {
  int b, sq, sk, h, hk;
  float scale, scale_log2;
  int causal, causal_off;
  const float* lse;      // [B,H,Sq] natural log
  const float* delta;    // [B,H,Sq]
  float* dq;             // fp32 [B,Sq,H,D]: every element is written
  void* dk;              // [B,Sk,Hk,D] with element strides (dkv_sb, dkv_ss, dkv_sh): may be slices of a packed dQKV tensor
  void* dv;
  int64_t dkv_sb, dkv_ss, dkv_sh;
  int64_t dq_sb, dq_ss, dq_sh;   // element strides of the fp32 dQ [B,Sq,H,D] (may be laid out seq-major)
  const int4* colmask;   // [b, mask_heads, sk] hidden row ranges per key column (see AttnArgs::colmask); nullptr: none
  int mask_heads;
};

// resident tile (128 rows) in slot 0 / 1, streamed tiles (64 rows): operand a in slots [0, 2), operand b in slots [2, 4)
struct Smem {
  uint32_t base;
  __device__ uint32_t big(int i) const { return base + i * BIG_BYTES; }
  __device__ uint32_t small(int i) const { return base + 2 * BIG_BYTES + i * SMALL_BYTES; }
  __device__ uint32_t bar(int i) const { return base + 2 * BIG_BYTES + 4 * SMALL_BYTES + 8u * i; }
};

template <typename T, bool MASKED>
__global__ void __launch_bounds__(kThreadsDkv, 1)
dkv_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
           const __grid_constant__ CUtensorMap map_do, const Params p) {
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr int BN = 128, BQ = 64;
  extern __shared__ uint8_t smem_raw[];
  const Smem sm{(smem_u32(smem_raw) + 1023u) & ~1023u};
  const uint32_t sK = sm.big(0), sV = sm.big(1);
  auto sQ = [&](int s) { return sm.small(s); };
  auto sDO = [&](int s) { return sm.small(2 + s); };
  const uint32_t kv_full = sm.bar(0);
  auto qdo_full = [&](int s) { return sm.bar(1 + s); };
  auto qdo_empty = [&](int s) { return sm.bar(3 + s); };     // 8 warp arrivals

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x, kv_head = blockIdx.y, batch = blockIdx.z;
  const int n0 = n_tile * BN;
  const int group = p.h / p.hk;
  const int num_m = (p.sq + BQ - 1) / BQ;
  int m_first = 0;
  if (p.causal) {                       // first query row that can see key n0 + BN - 1 or an earlier one of the tile: i >= n0 - causal_off
    const int r0 = max(0, n0 - p.causal_off);
    m_first = min(num_m, r0 / BQ);
  }
  const int tiles_per_head = num_m - m_first;
  const int total = tiles_per_head * group;    // iteration it -> (query head = kv_head*group + it / tiles_per_head, m tile = m_first + it % tiles_per_head)

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v); tma_prefetch_desc(&map_do);
    mbar_init(kv_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(qdo_full(s), 1); mbar_init(qdo_empty(s), 8); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dealloc<40>();
    if (warp == 0 && lane == 0 && total > 0) {
      // ================= TMA producer =================
      mbar_expect_tx(kv_full, 2 * BIG_BYTES);
      tma_load_4d(sK, &map_k, kv_full, 0, n0, kv_head, batch);
      tma_load_4d(sK + BIG_HALF, &map_k, kv_full, 64, n0, kv_head, batch);
      tma_load_4d(sV, &map_v, kv_full, 0, n0, kv_head, batch);
      tma_load_4d(sV + BIG_HALF, &map_v, kv_full, 64, n0, kv_head, batch);
      for (int it = 0; it < total; ++it) {
        const int s = it & 1;
        const int head = kv_head * group + it / tiles_per_head;
        const int m0 = (m_first + it % tiles_per_head) * BQ;
        mbar_wait(qdo_empty(s), ((it >> 1) & 1) ^ 1);
        mbar_expect_tx(qdo_full(s), 2 * SMALL_BYTES);
        tma_load_4d(sQ(s), &map_q, qdo_full(s), 0, m0, head, batch);
        tma_load_4d(sQ(s) + SMALL_HALF, &map_q, qdo_full(s), 64, m0, head, batch);
        tma_load_4d(sDO(s), &map_do, qdo_full(s), 0, m0, head, batch);
        tma_load_4d(sDO(s) + SMALL_HALF, &map_do, qdo_full(s), 64, m0, head, batch);
      }
    }
  } else {
    // ================= MMA warpgroups: wg owns keys [64 wg, 64 wg + 64) of the tile; accumulator row = key, column = query =================
    reg_alloc<232>();
    const int wg = (warp >> 2) - 1, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // tile-relative key rows rl and rl + 8
    constexpr float kLog2e = 1.4426950408889634f;
    float dv_acc[HD / 2], dk_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) { dv_acc[i] = 0.f; dk_acc[i] = 0.f; }
    if (total > 0) mbar_wait(kv_full, 0);
    for (int it = 0; it < total; ++it) {
      const int s = it & 1;
      const int head = kv_head * group + it / tiles_per_head;
      const int m0 = (m_first + it % tiles_per_head) * BQ;
      const int64_t stat0 = ((int64_t)batch * p.h + head) * p.sq;
      mbar_wait(qdo_full(s), (it >> 1) & 1);
      float st[BQ / 2], dpt[BQ / 2];
      wgmma_fence_regs(st);
      wgmma_fence_regs(dpt);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_ss_n64<BF16, 0, 0>(st, make_smem_desc(sK + kb * BIG_HALF + wg * 8192 + k * 32, 16, 1024),
                                   make_smem_desc(sQ(s) + kb * SMALL_HALF + k * 32, 16, 1024), (kb | k) != 0);      // S^T = K Q^T
          wgmma_ss_n64<BF16, 0, 0>(dpt, make_smem_desc(sV + kb * BIG_HALF + wg * 8192 + k * 32, 16, 1024),
                                   make_smem_desc(sDO(s) + kb * SMALL_HALF + k * 32, 16, 1024), (kb | k) != 0);     // dP^T = V dO^T
        }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(st);
      wgmma_fence_regs(dpt);
      int4 cm[2];
      if constexpr (MASKED) {
        const int4* cmp = p.colmask + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.sk;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int key = n0 + rl + h * 8;
          cm[h] = key < p.sk ? __ldg(cmp + key) : make_int4(0, 0, 0, 0);
        }
      }
      // P^T = exp2(S^T scale - lse[query]), dS^T = P^T (dP^T - delta[query]) scale, packed as A fragments (16-query step ks = column groups 2 ks, 2 ks + 1)
      uint32_t pa[BQ / 16][4], dsa[BQ / 16][4];
#pragma unroll
      for (int jn = 0; jn < BQ / 8; ++jn) {
        float pv[4], ds[4];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = m0 + jn * 8 + 2 * q + e;      // query
          const bool row_ok = row < p.sq;
          const float lse2 = row_ok ? __ldg(p.lse + stat0 + row) * kLog2e : 0.f;
          const float dl = row_ok ? __ldg(p.delta + stat0 + row) : 0.f;
          const int lim = p.causal ? min(p.sk - 1, row + p.causal_off) : p.sk - 1;   // last visible key of this query row
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int key = n0 + rl + h * 8;
            float x = ex2(fmaf(st[jn * 4 + h * 2 + e], p.scale_log2, -lse2));
            if (!row_ok || key > lim) x = 0.f;
            if constexpr (MASKED) {
              if ((row >= cm[h].x && row < cm[h].y) || (row >= cm[h].z && row < cm[h].w)) x = 0.f;
            }
            pv[h * 2 + e] = x;
            ds[h * 2 + e] = x * (dpt[jn * 4 + h * 2 + e] - dl) * p.scale;
          }
        }
        pa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(pv[0], pv[1]);
        pa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(pv[2], pv[3]);
        dsa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(ds[0], ds[1]);
        dsa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(ds[2], ds[3]);
      }
      wgmma_fence_regs(dv_acc);
      wgmma_fence_regs(dk_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BQ / 16; ++ks) {   // B = dO / Q tile read MN-major (N = head dim): 16 query rows = 2048 B per step, d halves SMALL_HALF apart
        wgmma_rs_n128<BF16, 1>(dv_acc, pa[ks], make_smem_desc(sDO(s) + ks * 2048, SMALL_HALF, 1024), 1);   // dV += P^T dO
        wgmma_rs_n128<BF16, 1>(dk_acc, dsa[ks], make_smem_desc(sQ(s) + ks * 2048, SMALL_HALF, 1024), 1);   // dK += dS^T Q
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dv_acc);
      wgmma_fence_regs(dk_acc);
      keep_regs(pa);
      keep_regs(dsa);
      __syncwarp();
      if (lane == 0) mbar_arrive(qdo_empty(s));
    }
    // epilogue: dV, dK rows (accumulator row = key)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = n0 + rl + h * 8;
      if (key >= p.sk) continue;
      const int64_t kv_off = (int64_t)batch * p.dkv_sb + (int64_t)key * p.dkv_ss + (int64_t)kv_head * p.dkv_sh;
      T* dv_row = reinterpret_cast<T*>(p.dv) + kv_off;
      T* dk_row = reinterpret_cast<T*>(p.dk) + kv_off;
#pragma unroll
      for (int jn = 0; jn < HD / 8; ++jn) {
        *reinterpret_cast<uint32_t*>(dv_row + jn * 8 + 2 * q) = pack2<T>(dv_acc[jn * 4 + h * 2], dv_acc[jn * 4 + h * 2 + 1]);
        *reinterpret_cast<uint32_t*>(dk_row + jn * 8 + 2 * q) = pack2<T>(dk_acc[jn * 4 + h * 2], dk_acc[jn * 4 + h * 2 + 1]);
      }
    }
  }
}

template <typename T, bool MASKED>
__global__ void __launch_bounds__(kThreads, 1)
dq_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
          const __grid_constant__ CUtensorMap map_do, const Params p) {
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr int BM = 128, BK = 64;
  extern __shared__ uint8_t smem_raw[];
  const Smem sm{(smem_u32(smem_raw) + 1023u) & ~1023u};
  const uint32_t sQ = sm.big(0), sDO = sm.big(1);
  auto sK = [&](int s) { return sm.small(s); };
  auto sV = [&](int s) { return sm.small(2 + s); };
  const uint32_t qdo_full = sm.bar(0);
  auto kv_full = [&](int s) { return sm.bar(1 + s); };
  auto kv_empty = [&](int s) { return sm.bar(3 + s); };     // 8 warp arrivals

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = (int)gridDim.x - 1 - (int)blockIdx.x;   // long (late) rows first under the causal mask
  const int head = blockIdx.y, batch = blockIdx.z;
  const int kv_head = head / (p.h / p.hk);
  const int m0 = m_tile * BM;
  int n_tiles = (p.sk + BK - 1) / BK;
  if (p.causal) {
    const int last_key = min(p.sk - 1, m0 + BM - 1 + p.causal_off);
    n_tiles = last_key < 0 ? 0 : min(n_tiles, last_key / BK + 1);
  }

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_k); tma_prefetch_desc(&map_v); tma_prefetch_desc(&map_do);
    mbar_init(qdo_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 8); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0 && n_tiles > 0) {
      // ================= TMA producer =================
      mbar_expect_tx(qdo_full, 2 * BIG_BYTES);
      tma_load_4d(sQ, &map_q, qdo_full, 0, m0, head, batch);
      tma_load_4d(sQ + BIG_HALF, &map_q, qdo_full, 64, m0, head, batch);
      tma_load_4d(sDO, &map_do, qdo_full, 0, m0, head, batch);
      tma_load_4d(sDO + BIG_HALF, &map_do, qdo_full, 64, m0, head, batch);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j & 1, n0 = j * BK;
        mbar_wait(kv_empty(s), ((j >> 1) & 1) ^ 1);
        mbar_expect_tx(kv_full(s), 2 * SMALL_BYTES);
        tma_load_4d(sK(s), &map_k, kv_full(s), 0, n0, kv_head, batch);
        tma_load_4d(sK(s) + SMALL_HALF, &map_k, kv_full(s), 64, n0, kv_head, batch);
        tma_load_4d(sV(s), &map_v, kv_full(s), 0, n0, kv_head, batch);
        tma_load_4d(sV(s) + SMALL_HALF, &map_v, kv_full(s), 64, n0, kv_head, batch);
      }
    }
  } else {
    // ================= MMA warpgroups: wg owns query rows [64 wg, 64 wg + 64); accumulator row = query, column = key / head dim =================
    const int wg = warp >> 2, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    constexpr float kLog2e = 1.4426950408889634f;
    float dq_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq_acc[i] = 0.f;
    float lse2[2], dl[2];
    int lim[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + rl + h * 8;
      row_ok[h] = row < p.sq;
      const int64_t stat = ((int64_t)batch * p.h + head) * p.sq + row;
      lse2[h] = row_ok[h] ? p.lse[stat] * kLog2e : 0.f;
      dl[h] = row_ok[h] ? p.delta[stat] : 0.f;
      lim[h] = p.causal ? min(p.sk - 1, row + p.causal_off) : p.sk - 1;
    }
    const int4* cmp = MASKED ? p.colmask + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.sk : nullptr;
    (void)cmp;
    if (n_tiles > 0) mbar_wait(qdo_full, 0);
    for (int j = 0; j < n_tiles; ++j) {
      const int s = j & 1, n0 = j * BK;
      mbar_wait(kv_full(s), (j >> 1) & 1);
      float sv[BK / 2], dpv[BK / 2];
      wgmma_fence_regs(sv);
      wgmma_fence_regs(dpv);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_ss_n64<BF16, 0, 0>(sv, make_smem_desc(sQ + kb * BIG_HALF + wg * 8192 + k * 32, 16, 1024),
                                   make_smem_desc(sK(s) + kb * SMALL_HALF + k * 32, 16, 1024), (kb | k) != 0);      // S = Q K^T
          wgmma_ss_n64<BF16, 0, 0>(dpv, make_smem_desc(sDO + kb * BIG_HALF + wg * 8192 + k * 32, 16, 1024),
                                   make_smem_desc(sV(s) + kb * SMALL_HALF + k * 32, 16, 1024), (kb | k) != 0);      // dP = dO V^T
        }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sv);
      wgmma_fence_regs(dpv);
      uint32_t dsa[BK / 16][4];
#pragma unroll
      for (int jn = 0; jn < BK / 8; ++jn) {
        float ds[4];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = n0 + jn * 8 + 2 * q + e;
          int4 m = make_int4(0, 0, 0, 0);
          if constexpr (MASKED) { if (key < p.sk) m = __ldg(cmp + key); }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m0 + rl + h * 8;
            float x = ex2(fmaf(sv[jn * 4 + h * 2 + e], p.scale_log2, -lse2[h]));
            if (!row_ok[h] || key > lim[h]) x = 0.f;
            if constexpr (MASKED) {
              if ((row >= m.x && row < m.y) || (row >= m.z && row < m.w)) x = 0.f;
            }
            ds[h * 2 + e] = x * (dpv[jn * 4 + h * 2 + e] - dl[h]) * p.scale;
          }
        }
        dsa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(ds[0], ds[1]);
        dsa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(ds[2], ds[3]);
      }
      wgmma_fence_regs(dq_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BK / 16; ++ks)     // B = K tile read MN-major (N = head dim): 16 key rows = 2048 B per step
        wgmma_rs_n128<BF16, 1>(dq_acc, dsa[ks], make_smem_desc(sK(s) + ks * 2048, SMALL_HALF, 1024), 1);   // dQ += dS K
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dq_acc);
      keep_regs(dsa);
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty(s));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + rl + h * 8;
      if (!row_ok[h]) continue;
      float* dst = p.dq + (int64_t)batch * p.dq_sb + (int64_t)row * p.dq_ss + (int64_t)head * p.dq_sh;
#pragma unroll
      for (int jn = 0; jn < HD / 8; ++jn)
        *reinterpret_cast<float2*>(dst + jn * 8 + 2 * q) = make_float2(dq_acc[jn * 4 + h * 2], dq_acc[jn * 4 + h * 2 + 1]);
    }
  }
}

// delta[b,h,s] = sum_d dO[b,s,h,d] * O[b,s,h,d]   (one warp per row; O and dO share the element strides (sb, ss, sh), d contiguous)
template <typename T>
__global__ void delta_kernel(const T* __restrict__ o, const T* __restrict__ d_o, float* __restrict__ delta, int64_t rows, int sq, int h,
                             int64_t sb, int64_t ss, int64_t sh) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // row = (b*sq + s)*h + head
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int64_t bs = row / h;
  const int head = (int)(row - bs * h);
  const int64_t bb = bs / sq;
  const int sidx = (int)(bs - bb * sq);
  const int64_t off = bb * sb + (int64_t)sidx * ss + (int64_t)head * sh + lane * 4;
  const uint2 a = *reinterpret_cast<const uint2*>(o + off);
  const uint2 b = *reinterpret_cast<const uint2*>(d_o + off);
  const T* pa = reinterpret_cast<const T*>(&a);
  const T* pb = reinterpret_cast<const T*>(&b);
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) acc += to_f(pa[i]) * to_f(pb[i]);
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o2);
  if (lane == 0) delta[(bb * h + head) * sq + sidx] = acc;
}

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
    set_last_error(__FILE__, __LINE__, ("cuTensorMapEncodeTiled (attention bwd) failed: " + std::to_string((int)r)).c_str());
    return false;
  }
  return true;
}
}  // namespace attn_bwd

int attention_bwd(const AttnBwdArgs& a, cudaStream_t s) {
  using namespace attn_bwd;
  if (!attention_fwd_supported(a.fwd)) return 1;
  const AttnArgs& f = a.fwd;
  if (a.dq_strides[0] % 2 || a.dq_strides[1] % 2 || a.dq_strides[2] % 2 || (reinterpret_cast<uintptr_t>(a.dq) & 7)) return 1;   // float2 stores
  if (a.dkv_strides[0] % 2 || a.dkv_strides[1] % 2 || a.dkv_strides[2] % 2) return 1;
  // every operand as a 128-row box map (the resident tile of a kernel) and as a 64-row box map (the streamed tile of the other kernel)
  CUtensorMap mq[2], mk[2], mv[2], mdo[2];
  for (int i = 0; i < 2; ++i) {
    const uint32_t rows = i ? 64 : 128;
    if (!make_map4(&mq[i], f.q, f.d, f.sq, f.h, f.b, f.q_strides[1], f.q_strides[2], f.q_strides[0], rows, f.dtype)) return 2;
    if (!make_map4(&mk[i], f.k, f.d, f.sk, f.hk, f.b, f.k_strides[1], f.k_strides[2], f.k_strides[0], rows, f.dtype)) return 2;
    if (!make_map4(&mv[i], f.v, f.d, f.sk, f.hk, f.b, f.v_strides[1], f.v_strides[2], f.v_strides[0], rows, f.dtype)) return 2;
    if (!make_map4(&mdo[i], a.d_o, f.d, f.sq, f.h, f.b, a.o_strides[1], a.o_strides[2], a.o_strides[0], rows, f.dtype)) return 2;
  }
  const int64_t rows = (int64_t)f.b * f.sq * f.h;
  const int wpb = 8;
  if (f.dtype == kBF16)
    delta_kernel<__nv_bfloat16><<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, s>>>((const __nv_bfloat16*)f.o, (const __nv_bfloat16*)a.d_o, a.delta, rows, f.sq, f.h,
                                                                                     a.o_strides[0], a.o_strides[1], a.o_strides[2]);
  else
    delta_kernel<__half><<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, s>>>((const __half*)f.o, (const __half*)a.d_o, a.delta, rows, f.sq, f.h, a.o_strides[0], a.o_strides[1], a.o_strides[2]);
  Params p;
  p.b = f.b; p.sq = f.sq; p.sk = f.sk; p.h = f.h; p.hk = f.hk;
  p.scale = f.scale; p.scale_log2 = f.scale * 1.4426950408889634f;
  p.causal = f.causal; p.causal_off = f.sk - f.sq;
  p.colmask = reinterpret_cast<const int4*>(f.colmask);
  p.mask_heads = f.mask_heads > 0 ? f.mask_heads : 1;
  p.lse = f.lse; p.delta = a.delta; p.dq = a.dq; p.dk = a.dk; p.dv = a.dv;
  p.dkv_sb = a.dkv_strides[0]; p.dkv_ss = a.dkv_strides[1]; p.dkv_sh = a.dkv_strides[2];
  p.dq_sb = a.dq_strides[0]; p.dq_ss = a.dq_strides[1]; p.dq_sh = a.dq_strides[2];
  const dim3 grid_kv((f.sk + 127) / 128, f.hk, f.b), grid_q((f.sq + 127) / 128, f.h, f.b);
  static bool attr_set[8] = {false, false, false, false, false, false, false, false};
  auto go = [&](auto kern, int slot, dim3 grid, int threads, const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const CUtensorMap& d_o) {
    if (!attr_set[slot]) { B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES)); attr_set[slot] = true; }
    kern<<<grid, threads, SMEM_BYTES, s>>>(q, k, v, d_o, p);
  };
  if (f.dtype == kBF16) {
    if (p.colmask) { go(dkv_kernel<__nv_bfloat16, true>, 0, grid_kv, kThreadsDkv, mq[1], mk[0], mv[0], mdo[1]); go(dq_kernel<__nv_bfloat16, true>, 1, grid_q, kThreads, mq[0], mk[1], mv[1], mdo[0]); }
    else { go(dkv_kernel<__nv_bfloat16, false>, 2, grid_kv, kThreadsDkv, mq[1], mk[0], mv[0], mdo[1]); go(dq_kernel<__nv_bfloat16, false>, 3, grid_q, kThreads, mq[0], mk[1], mv[1], mdo[0]); }
  } else {
    if (p.colmask) { go(dkv_kernel<__half, true>, 4, grid_kv, kThreadsDkv, mq[1], mk[0], mv[0], mdo[1]); go(dq_kernel<__half, true>, 5, grid_q, kThreads, mq[0], mk[1], mv[1], mdo[0]); }
    else { go(dkv_kernel<__half, false>, 6, grid_kv, kThreadsDkv, mq[1], mk[0], mv[0], mdo[1]); go(dq_kernel<__half, false>, 7, grid_q, kThreads, mq[0], mk[1], mv[1], mdo[0]); }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

}  // namespace b200
