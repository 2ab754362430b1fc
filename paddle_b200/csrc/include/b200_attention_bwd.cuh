// Bodies of the flash-attention backward kernels (see attention_bwd_sm100.cu for the algorithms), templated on the head size D (128 or
// 64), and the host launcher.  attention_bwd_sm100.cu instantiates D = 128 in dkv_kernel, dq_kernel and prep_kernel;
// attention_d64_sm100.cu instantiates D = 64 in dkv_d64_kernel, dq_d64_kernel and prep_d64_kernel.
//
// At D = 64 every tile is one 64-wide d chunk (one 128-byte swizzle span), so each TMA operand is one box, S^T / dP^T / S / dP take 4
// k-steps instead of 8, and dV, dK and the deterministic dQ are n = 64 MMAs with half the accumulators.  The single pass's dQ stage
// splits the tile's keys instead of the head dims: warpgroup wg computes all 64 columns of dS K over its own 64 keys and reduce-adds
// them, so every dQ element receives two additions per key tile.
#pragma once
#include <cuda.h>
#include <type_traits>

#include "b200_common.cuh"
#include "b200_mask_tiles.cuh"
#include "b200_ops.h"
#include "b200_philox.cuh"
#include "b200_ptx.cuh"

namespace b200 {
namespace attn_bwd {
using namespace ptx;

constexpr int HD = 128;
constexpr int kThreads = 288;      // dq_kernel: warps 0-7 two MMA warpgroups, warp 8 TMA producer
constexpr int kThreadsDkv = 384;   // dkv_kernel: warpgroup 0 = producer (warp 0) giving its registers to the MMA warpgroups 1 and 2
template <int D> constexpr uint32_t kBigBytes = 128 * D * 2;     // a 128-row tile: D / 64 d chunks [chunk][row][128 B swizzled]
template <int D> constexpr uint32_t kSmallBytes = 64 * D * 2;    // a 64-row tile, same structure
constexpr uint32_t BIG_HALF = 128 * 64 * 2;                      // one d chunk of a 128-row tile
constexpr uint32_t SMALL_HALF = 64 * 64 * 2;                     // one d chunk of a 64-row tile
// dq_kernel: two resident 128-row tiles + two double-buffered 64-row tiles
template <int D> constexpr uint32_t kSmemBytes = 2 * kBigBytes<D> + 4 * kSmallBytes<D> + 1024 + 256;

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
  const float* stats;    // [B,H,2,sq_pad]: lse * log2(e), then delta; rows >= sq are zero
  int sq_pad;            // sq rounded up to the 64-row query tile
  float* dq;             // fp32 [B,Sq,H,D]
  void* dk;              // [B,Sk,Hk,D] with element strides (dkv_sb, dkv_ss, dkv_sh): may be slices of a packed dQKV tensor
  void* dv;
  int64_t dkv_sb, dkv_ss, dkv_sh;
  int64_t dq_sb, dq_ss, dq_sh;   // element strides of the fp32 dQ [B,Sq,H,D] (may be laid out seq-major)
  const int4* colmask;   // [b, mask_heads, sk] hidden row ranges per key column (see AttnArgs::colmask); nullptr: none
  int mask_heads;
};

// resident tile (128 rows) in slot 0 / 1, streamed tiles (64 rows): operand a in slots [0, 2), operand b in slots [2, 4)
template <int D> struct Smem {
  uint32_t base;
  __device__ uint32_t big(int i) const { return base + i * kBigBytes<D>; }
  __device__ uint32_t small(int i) const { return base + 2 * kBigBytes<D> + i * kSmallBytes<D>; }
  __device__ uint32_t bar(int i) const { return base + 2 * kBigBytes<D> + 4 * kSmallBytes<D> + 8u * i; }
};

// dkv_kernel smem (offsets from the 1024-aligned base): resident K, V; a 2-stage ring of {Q, dO, lse2 / delta}; with the dQ stage also
// two dS^T buffers (double-buffered: one warpgroup may write the next tile's dS^T while the other still multiplies the last one) and a
// 64 x 64 fp32 dQ staging tile per MMA warpgroup, the source of the bulk reduce-add.
template <int D> struct DkvSmem {
  static constexpr uint32_t BIG = kBigBytes<D>, SMALL = kSmallBytes<D>;
  static constexpr uint32_t K = 0, V = BIG, Q = 2 * BIG, DO = Q + 2 * SMALL, DS = DO + 2 * SMALL;
  static constexpr uint32_t DS_BYTES = 128 * 64 * 2;          // [key 128][query 64] 16-bit, 128B-swizzled
  static constexpr uint32_t STAGE = DS + 2 * DS_BYTES;
  static constexpr uint32_t STAGE_BYTES = 64 * 64 * 4;         // per warpgroup: two [query 64][32 fp32] 128B-swizzled boxes
  static constexpr uint32_t STATS = STAGE + 2 * STAGE_BYTES;   // per ring stage: lse2[64], delta[64]
  static constexpr uint32_t BARS = STATS + 2 * 512;
  static constexpr uint32_t BYTES = BARS + 64 + 1024;
};
static_assert(DkvSmem<HD>::BYTES <= 227 * 1024, "dkv_kernel shared memory");

// DQ = true: the single-pass backward.  Each query tile's dQ partial dS K (all 128 keys of the tile) is added into the fp32 dQ by a
// TMA bulk reduce-add; dQ must be zero on entry.  DQ = false: dK / dV only (dq_kernel computes dQ).
// DROPOUT (P = dropout::DropoutParams<Params>): with Zs = Z / (1 - p) for the keep mask Z of p.seed_offset, dV += (Zs P)^T dO and
// dS = P (Zs dP - delta) scale (dP = dO V^T is the gradient of the dropped probabilities; delta = rowsum(dO O) on the dropped O).
// SKIP (MASKED only, P = mask_skip::SkipParams<...>): walk only the (query head, 64-row query tile) pairs the column mask does not hide
// from the CTA's key tile (b200_mask_tiles.cuh); the producer publishes each pair beside its stage.
template <typename T, bool MASKED, bool DQ, int D, bool DROPOUT = false, bool SKIP = false, typename P = Params>
__device__ __forceinline__ void dkv_body(const CUtensorMap& map_q, const CUtensorMap& map_k, const CUtensorMap& map_v,
                                         const CUtensorMap& map_do, const CUtensorMap& map_dq, const P p) {
  static_assert(D == HD || D == 64, "head_dim 128 or 64");
  static_assert(!SKIP || MASKED, "tile skipping needs a column mask");
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr int BN = 128, BQ = 64;
  constexpr int kHalves = D / 64;
  using L = DkvSmem<D>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* const base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sK = base + L::K, sV = base + L::V;
  auto sQ = [&](int s) { return base + L::Q + s * L::SMALL; };
  auto sDO = [&](int s) { return base + L::DO + s * L::SMALL; };
  auto stats = [&](int s) { return reinterpret_cast<const float*>(base_ptr + L::STATS + s * 512); };
  const uint32_t kv_full = base + L::BARS;
  auto qdo_full = [&](int s) { return base + L::BARS + 8 * (1 + s); };
  auto qdo_empty = [&](int s) { return base + L::BARS + 8 * (3 + s); };     // 8 warp arrivals
  // SKIP: stage s's pair {query head << 20 | query tile (-1: end of the list), open}: one word, from which the D = 128 dropout kernel
  // recomputes head and m0 where it needs them instead of holding both
  auto slot = [&](int s) { return base + L::BARS + 40 + 8 * s; };
  (void)slot;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kv_head = blockIdx.x, batch = blockIdx.y, n_tile = blockIdx.z;   // key tiles slowest: under the causal mask the long ones start first
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
    if constexpr (DQ) tma_prefetch_desc(&map_dq);
    mbar_init(kv_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(qdo_full(s), 1); mbar_init(qdo_empty(s), 8); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dealloc<24>();
    if constexpr (SKIP) {
      if (warp == 0 && lane == 0) {
        // ================= TMA producer over the pairs the column mask does not hide =================
        // (one lane in 24 registers: the classes of the pairs come precomputed with the tile summary)
        if (total > 0) {   // (the consumers wait for K / V only then)
          mbar_expect_tx(kv_full, 2 * L::BIG);
          tma_load_4d(sK, &map_k, kv_full, 0, n0, kv_head, batch);
          if constexpr (kHalves == 2) tma_load_4d(sK + BIG_HALF, &map_k, kv_full, 64, n0, kv_head, batch);
          tma_load_4d(sV, &map_v, kv_full, 0, n0, kv_head, batch);
          if constexpr (kHalves == 2) tma_load_4d(sV + BIG_HALF, &map_v, kv_full, 64, n0, kv_head, batch);
        }
        int cnt = 0;
        for (int it = 0; it < total; ++it) {
          const int head = kv_head * group + it / tiles_per_head;
          const int mt = m_first + it % tiles_per_head, m0 = mt * BQ;
          const int cls = __ldg(p.classes + ((batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.n_ktiles + n_tile) * num_m + mt);
          if (cls == mask_skip::kHidden) continue;
          const int s = cnt & 1;
          const float* st = p.stats + ((int64_t)batch * p.h + head) * 2 * p.sq_pad + m0;
          mbar_wait(qdo_empty(s), ((cnt >> 1) & 1) ^ 1);
          mask_skip::st_slot(slot(s), head << 20 | mt);
          mask_skip::st_slot(slot(s) + 4, cls == mask_skip::kOpen);
          mbar_expect_tx(qdo_full(s), 2 * L::SMALL + 512);
          tma_load_4d(sQ(s), &map_q, qdo_full(s), 0, m0, head, batch);
          if constexpr (kHalves == 2) tma_load_4d(sQ(s) + SMALL_HALF, &map_q, qdo_full(s), 64, m0, head, batch);
          tma_load_4d(sDO(s), &map_do, qdo_full(s), 0, m0, head, batch);
          if constexpr (kHalves == 2) tma_load_4d(sDO(s) + SMALL_HALF, &map_do, qdo_full(s), 64, m0, head, batch);
          bulk_load(base + L::STATS + s * 512, st, 256, qdo_full(s));
          bulk_load(base + L::STATS + s * 512 + 256, st + p.sq_pad, 256, qdo_full(s));
          ++cnt;
        }
        {   // end of the list: the consumers' loop has no other bound (it would cost the D = 128 dropout kernel a register)
          const int s = cnt & 1;
          mbar_wait(qdo_empty(s), ((cnt >> 1) & 1) ^ 1);
          mask_skip::st_slot(slot(s), -1);
          mbar_arrive(qdo_full(s));
        }
        for (int it = max(0, cnt - 2); it < cnt; ++it) mbar_wait(qdo_empty(it & 1), (it >> 1) & 1);   // the consumers' waits are unbounded
      }
    } else if (warp == 0 && lane == 0 && total > 0) {
      // ================= TMA producer: one box per 64-wide d chunk =================
      mbar_expect_tx(kv_full, 2 * L::BIG);
      tma_load_4d(sK, &map_k, kv_full, 0, n0, kv_head, batch);
      if constexpr (kHalves == 2) tma_load_4d(sK + BIG_HALF, &map_k, kv_full, 64, n0, kv_head, batch);
      tma_load_4d(sV, &map_v, kv_full, 0, n0, kv_head, batch);
      if constexpr (kHalves == 2) tma_load_4d(sV + BIG_HALF, &map_v, kv_full, 64, n0, kv_head, batch);
      for (int it = 0; it < total; ++it) {
        const int s = it & 1;
        const int head = kv_head * group + it / tiles_per_head;
        const int m0 = (m_first + it % tiles_per_head) * BQ;
        const float* st = p.stats + ((int64_t)batch * p.h + head) * 2 * p.sq_pad + m0;
        mbar_wait(qdo_empty(s), ((it >> 1) & 1) ^ 1);
        mbar_expect_tx(qdo_full(s), 2 * L::SMALL + 512);
        tma_load_4d(sQ(s), &map_q, qdo_full(s), 0, m0, head, batch);
        if constexpr (kHalves == 2) tma_load_4d(sQ(s) + SMALL_HALF, &map_q, qdo_full(s), 64, m0, head, batch);
        tma_load_4d(sDO(s), &map_do, qdo_full(s), 0, m0, head, batch);
        if constexpr (kHalves == 2) tma_load_4d(sDO(s) + SMALL_HALF, &map_do, qdo_full(s), 64, m0, head, batch);
        bulk_load(base + L::STATS + s * 512, st, 256, qdo_full(s));
        bulk_load(base + L::STATS + s * 512 + 256, st + p.sq_pad, 256, qdo_full(s));
      }
      for (int it = max(0, total - 2); it < total; ++it) mbar_wait(qdo_empty(it & 1), (it >> 1) & 1);   // the consumers' waits are unbounded
    }
  } else {
    // ================= MMA warpgroups: wg owns keys [64 wg, 64 wg + 64) of the tile; accumulator row = key, column = query =================
    reg_alloc<240>();
    const int wg = (warp >> 2) - 1, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // tile-relative key rows rl and rl + 8
    float dv_acc[D / 2], dk_acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) { dv_acc[i] = 0.f; dk_acc[i] = 0.f; }
    // DROPOUT: this lane's keys n0 + rl (+ 8) have parity kpar; it draws the calls of the queries of parity kpar and trades the bits its
    // partner (lane ^ 4, keys of the other parity) needs for the calls of the other parity (see b200_philox.cuh)
    uint32_t dk0 = 0, dk1 = 0, dkc = 0;
    int64_t doff = 0;
    const int kpar = (lane >> 2) & 1;
    if constexpr (DROPOUT) {
      const uint64_t seed = (uint64_t)__ldg(p.seed_offset);
      doff = __ldg(p.seed_offset + 1);
      dk0 = (uint32_t)seed; dk1 = (uint32_t)(seed >> 32);
      dkc = dropout::key_counter(n0 + rl);
    }
    (void)kpar;
    if (total > 0) mbar_wait_unbounded(kv_full, 0);
    for (int it = 0; SKIP || it < total; ++it) {   // SKIP: it counts the pairs processed, head and m0 come from the producer
      const int s = it & 1;
      int head, m0;
      if constexpr (SKIP) {
        mbar_wait_unbounded(qdo_full(s), (it >> 1) & 1);
        const int w = mask_skip::ld_slot(slot(s));
        if (w < 0) break;
        head = w >> 20; m0 = (w & 0xfffff) * BQ;
      } else {
        head = kv_head * group + it / tiles_per_head;
        m0 = (m_first + it % tiles_per_head) * BQ;
        mbar_wait_unbounded(qdo_full(s), (it >> 1) & 1);
      }
      float st[BQ / 2], dpt[BQ / 2];
      wgmma_fence_regs(st);
      wgmma_fence_regs(dpt);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < kHalves; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss_n64<BF16, 0, 0>(st, make_smem_desc(sK + kb * BIG_HALF + wg * 8192 + k * 32, 16, 1024),
                                   make_smem_desc(sQ(s) + kb * SMALL_HALF + k * 32, 16, 1024), (kb | k) != 0);      // S^T = K Q^T
      wgmma_commit();
#pragma unroll
      for (int kb = 0; kb < kHalves; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss_n64<BF16, 0, 0>(dpt, make_smem_desc(sV + kb * BIG_HALF + wg * 8192 + k * 32, 16, 1024),
                                   make_smem_desc(sDO(s) + kb * SMALL_HALF + k * 32, 16, 1024), (kb | k) != 0);     // dP^T = V dO^T
      wgmma_commit();
      // DROPOUT, while S^T and dP^T are in flight: z0 / z1 hold the calls of the even / odd queries 2 q (+ 1) of column groups
      // 2 cc, 2 cc + 1 at bits 8 cc .., shifted so that the element (query 8 jn + 2 q + e, key rl + 8 h) is bit 8 (jn >> 1) + 4 (jn & 1) + 2 h
      uint32_t z0 = 0, z1 = 0;
      if constexpr (DROPOUT) {
        uint32_t c2, c3, own = 0;
        dropout::plane_counter(doff, batch, p.h, head, c2, c3);
#pragma unroll 1
        for (int cc = 0; cc < BQ / 16; ++cc)   // one call's temporaries live at a time
          own |= dropout::keep_bits(dropout::row_counter(m0 + 16 * cc + 2 * q + kpar), dkc, dk0, dk1, c2, c3, p.keep) << (8 * cc);
        const uint32_t other = __shfl_xor_sync(0xffffffffu, own, 4);
        z0 = (kpar ? other : own) >> kpar;
        z1 = (kpar ? own : other) >> kpar;
      }
      int4 cm[2];
      if constexpr (MASKED) {
        const int4* cmp = p.colmask + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.sk;
        const bool open = SKIP && (mask_skip::ld_slot(slot(s) + 4) & 1);   // SKIP: an open pair tests against an empty mask
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int key = n0 + rl + h * 8;
          cm[h] = key < p.sk && !open ? __ldg(cmp + key) : make_int4(0, 0, 0, 0);
        }
      }
      const float* lse2 = stats(s);        // lse[query] * log2(e)
      const float* dlt = lse2 + BQ;        // delta[query]
      wgmma_wait<1>();
      wgmma_fence_regs(st);
      // P^T = exp2(S^T scale - lse2[query]) in place of S^T, packed as the A fragments of dV += P^T dO (16-query step ks = column groups 2 ks, 2 ks + 1)
      uint32_t pa[BQ / 16][4], dsa[BQ / 16][4];
#pragma unroll
      for (int jn = 0; jn < BQ / 8; ++jn) {
        const float2 l2 = *reinterpret_cast<const float2*>(lse2 + jn * 8 + 2 * q);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int row = m0 + jn * 8 + 2 * q + e;      // query
          const int lim = row >= p.sq ? -1 : p.causal ? min(p.sk - 1, row + p.causal_off) : p.sk - 1;   // last visible key of this query row
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int key = n0 + rl + h * 8;
            float x = ex2(fmaf(st[jn * 4 + h * 2 + e], p.scale_log2, -(e ? l2.y : l2.x)));
            if (key > lim) x = 0.f;
            if constexpr (MASKED) {
              if ((row >= cm[h].x && row < cm[h].y) || (row >= cm[h].z && row < cm[h].w)) x = 0.f;
            }
            st[jn * 4 + h * 2 + e] = x;
          }
        }
        if constexpr (DROPOUT) {   // st keeps the undropped P^T for dS^T; dV takes Zs P^T
          float zp[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int bit = 8 * (jn >> 1) + 4 * (jn & 1) + 2 * (i >> 1);
            zp[i] = (((i & 1) ? z1 : z0) >> bit) & 1u ? st[jn * 4 + i] * p.rscale : 0.f;
          }
          pa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(zp[0], zp[1]);
          pa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(zp[2], zp[3]);
        } else {
          pa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(st[jn * 4 + 0], st[jn * 4 + 1]);
          pa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(st[jn * 4 + 2], st[jn * 4 + 3]);
        }
      }
      wgmma_fence_regs(dv_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BQ / 16; ++ks) {   // B = dO tile read MN-major (N = head dim): 16 query rows = 2048 B per step, d chunks SMALL_HALF apart
        const uint64_t desc = make_smem_desc(sDO(s) + ks * 2048, SMALL_HALF, 1024);
        if constexpr (D == HD) wgmma_rs_n128<BF16, 1>(dv_acc, pa[ks], desc, 1);   // dV += P^T dO
        else wgmma_rs_n64<BF16, 1>(dv_acc, pa[ks], desc, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_regs(dpt);
      // dS^T = P^T (dP^T - delta[query]) scale: A fragments of dK += dS^T Q and, with DQ, the tile's rows of the dS^T buffer
      uint8_t* const ds_buf = base_ptr + L::DS + (it & 1) * L::DS_BYTES;
#pragma unroll
      for (int jn = 0; jn < BQ / 8; ++jn) {
        const float2 dl = *reinterpret_cast<const float2*>(dlt + jn * 8 + 2 * q);
        float ds[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float dp = dpt[jn * 4 + i];
          if constexpr (DROPOUT) {
            const int bit = 8 * (jn >> 1) + 4 * (jn & 1) + 2 * (i >> 1);
            dp = (((i & 1) ? z1 : z0) >> bit) & 1u ? dp * p.rscale : 0.f;
          }
          ds[i] = st[jn * 4 + i] * (dp - ((i & 1) ? dl.y : dl.x)) * p.scale;
        }
        dsa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(ds[0], ds[1]);
        dsa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(ds[2], ds[3]);
        if constexpr (DQ) {        // [key][query] rows of 128 B, 16-byte chunk c of row r stored at chunk c ^ (r % 8)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = rl + h * 8;
            *reinterpret_cast<uint32_t*>(ds_buf + r * 128 + ((jn ^ (r & 7)) << 4) + 4 * q) = dsa[jn >> 1][(jn & 1) * 2 + h];
          }
        }
      }
      wgmma_fence_regs(dk_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BQ / 16; ++ks) {   // B = Q tile read MN-major, as dO above
        const uint64_t desc = make_smem_desc(sQ(s) + ks * 2048, SMALL_HALF, 1024);
        if constexpr (D == HD) wgmma_rs_n128<BF16, 1>(dk_acc, dsa[ks], desc, 1);   // dK += dS^T Q
        else wgmma_rs_n64<BF16, 1>(dk_acc, dsa[ks], desc, 1);
      }
      wgmma_commit();
      if constexpr (DQ) {
        // D = 128: dQ[query, 64 wg .. 64 wg + 63] = dS K over the tile's 128 keys: A = dS^T buffer read M-major (M = query), B = K
        // half wg read N-major (N = head dim); 16 keys = 2048 B per step in both.
        // D = 64: dQ[query, 0 .. 63] = dS K over the warpgroup's own 64 keys (rows 64 wg .. of both operands, 8192 B in).
        fence_proxy_async();
        named_bar_sync(1, 256);         // both warpgroups' dS^T rows are in shared memory
        const uint32_t sDS = base + L::DS + (it & 1) * L::DS_BYTES;
        float dq[HD / 4];
        wgmma_fence_regs(dq);
        wgmma_fence();
        if constexpr (D == HD) {
#pragma unroll
          for (int ks = 0; ks < BN / 16; ++ks)
            wgmma_ss_n64<BF16, 1, 1>(dq, make_smem_desc(sDS + ks * 2048, L::DS_BYTES, 1024),
                                     make_smem_desc(sK + wg * BIG_HALF + ks * 2048, BIG_HALF, 1024), ks != 0);
        } else {
#pragma unroll
          for (int ks = 0; ks < BN / 32; ++ks)
            wgmma_ss_n64<BF16, 1, 1>(dq, make_smem_desc(sDS + wg * 8192 + ks * 2048, L::DS_BYTES, 1024),
                                     make_smem_desc(sK + wg * 8192 + ks * 2048, BIG_HALF, 1024), ks != 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                // dV and dK are done with P^T, dS^T and the Q / dO stage
        wgmma_fence_regs(dv_acc);
        wgmma_fence_regs(dk_acc);
        keep_regs(pa);
        keep_regs(dsa);
        __syncwarp();
        if (lane == 0) mbar_arrive(qdo_empty(s));
        wgmma_wait<0>();
        wgmma_fence_regs(dq);
        // stage the 64 x 64 fp32 partial as two [query][32] boxes (128B-swizzled like the map) and reduce-add it into dQ
        const bool leader = (threadIdx.x & 127) == 0;
        if (leader) bulk_wait_group_read<0>();      // the previous tile's reduce has read the staging tile
        named_bar_sync(2 + wg, 128);
        uint8_t* const stage = base_ptr + L::STAGE + wg * L::STAGE_BYTES;
#pragma unroll
        for (int j = 0; j < HD / 16; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = (warp & 3) * 16 + (lane >> 2) + h * 8;      // query row of the tile
            const int c = 2 * (j & 3) + (q >> 1);                     // 16-byte chunk of the box row
            *reinterpret_cast<float2*>(stage + (j >> 2) * 8192 + r * 128 + ((c ^ (r & 7)) << 4) + (q & 1) * 8) =
                make_float2(dq[j * 4 + h * 2], dq[j * 4 + h * 2 + 1]);
          }
        fence_proxy_async();
        named_bar_sync(2 + wg, 128);
        if (leader) {
          const uint32_t src = base + L::STAGE + wg * L::STAGE_BYTES;
          tma_reduce_add_4d(&map_dq, src, D == HD ? wg * 64 : 0, m0, head, batch);
          tma_reduce_add_4d(&map_dq, src + 8192, D == HD ? wg * 64 + 32 : 32, m0, head, batch);
          bulk_commit_group();
        }
      } else {
        wgmma_wait<0>();
        wgmma_fence_regs(dv_acc);
        wgmma_fence_regs(dk_acc);
        keep_regs(pa);
        keep_regs(dsa);
        __syncwarp();
        if (lane == 0) mbar_arrive(qdo_empty(s));
      }
    }
    if constexpr (DQ) {
      if ((threadIdx.x & 127) == 0) bulk_wait_group<0>();      // the reduces are done reading shared memory before the CTA exits
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
      for (int jn = 0; jn < D / 8; ++jn) {
        *reinterpret_cast<uint32_t*>(dv_row + jn * 8 + 2 * q) = pack2<T>(dv_acc[jn * 4 + h * 2], dv_acc[jn * 4 + h * 2 + 1]);
        *reinterpret_cast<uint32_t*>(dk_row + jn * 8 + 2 * q) = pack2<T>(dk_acc[jn * 4 + h * 2], dk_acc[jn * 4 + h * 2 + 1]);
      }
    }
  }
}

// DROPOUT: as in dkv_body, with the forward's call layout (row = query)
// SKIP: walk only the 64-key tiles the column mask does not hide from the CTA's 128 rows (classified by their 128-key summary tile)
template <typename T, bool MASKED, int D, bool DROPOUT = false, bool SKIP = false, typename P = Params>
__device__ __forceinline__ void dq_body(const CUtensorMap& map_q, const CUtensorMap& map_k, const CUtensorMap& map_v,
                                        const CUtensorMap& map_do, const P p) {
  static_assert(D == HD || D == 64, "head_dim 128 or 64");
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr int BM = 128, BK = 64;
  constexpr int kHalves = D / 64;
  extern __shared__ uint8_t smem_raw[];
  const Smem<D> sm{(smem_u32(smem_raw) + 1023u) & ~1023u};
  const uint32_t sQ = sm.big(0), sDO = sm.big(1);
  auto sK = [&](int s) { return sm.small(s); };
  auto sV = [&](int s) { return sm.small(2 + s); };
  const uint32_t qdo_full = sm.bar(0);
  auto kv_full = [&](int s) { return sm.bar(1 + s); };
  auto kv_empty = [&](int s) { return sm.bar(3 + s); };     // 8 warp arrivals
  auto slot = [&](int s) { return sm.bar(6 + s); };         // SKIP: stage s's key tile, 2 j + open (-1: end of the list)
  (void)slot;

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
    if constexpr (SKIP) {
      if (n_tiles > 0) {
        // ================= TMA producer over the key tiles the column mask does not hide: lane l classifies tile jb + l =================
        const int* tiles = p.tiles + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.n_ktiles * 8;
        if (lane == 0) {
          mbar_expect_tx(qdo_full, 2 * kBigBytes<D>);
          tma_load_4d(sQ, &map_q, qdo_full, 0, m0, head, batch);
          if constexpr (kHalves == 2) tma_load_4d(sQ + BIG_HALF, &map_q, qdo_full, 64, m0, head, batch);
          tma_load_4d(sDO, &map_do, qdo_full, 0, m0, head, batch);
          if constexpr (kHalves == 2) tma_load_4d(sDO + BIG_HALF, &map_do, qdo_full, 64, m0, head, batch);
        }
        int cnt = 0;
        for (int jb = 0; jb < n_tiles; jb += 32) {
          const int cls = jb + lane < n_tiles ? mask_skip::tile_class(tiles + ((jb + lane) * BK / mask_skip::kTileKeys) * 8, m0, m0 + BM)
                                              : mask_skip::kHidden;
          uint32_t vis = __ballot_sync(0xffffffffu, cls != mask_skip::kHidden);
          const uint32_t open = __ballot_sync(0xffffffffu, cls == mask_skip::kOpen);
          while (vis) {
            const int bit = __ffs(vis) - 1;
            vis &= vis - 1;
            if (lane == 0) {
              const int j = jb + bit, s = cnt & 1, n0 = j * BK;
              mbar_wait(kv_empty(s), ((cnt >> 1) & 1) ^ 1);
              mask_skip::st_slot(slot(s), 2 * j + ((open >> bit) & 1));
              mbar_expect_tx(kv_full(s), 2 * kSmallBytes<D>);
              tma_load_4d(sK(s), &map_k, kv_full(s), 0, n0, kv_head, batch);
              if constexpr (kHalves == 2) tma_load_4d(sK(s) + SMALL_HALF, &map_k, kv_full(s), 64, n0, kv_head, batch);
              tma_load_4d(sV(s), &map_v, kv_full(s), 0, n0, kv_head, batch);
              if constexpr (kHalves == 2) tma_load_4d(sV(s) + SMALL_HALF, &map_v, kv_full(s), 64, n0, kv_head, batch);
            }
            ++cnt;
          }
        }
        if (lane == 0 && cnt < n_tiles) {   // the consumers' loop would go on: end it
          const int s = cnt & 1;
          mbar_wait(kv_empty(s), ((cnt >> 1) & 1) ^ 1);
          mask_skip::st_slot(slot(s), -1);
          mbar_arrive(kv_full(s));
        }
      }
    } else if (lane == 0 && n_tiles > 0) {
      // ================= TMA producer: one box per 64-wide d chunk =================
      mbar_expect_tx(qdo_full, 2 * kBigBytes<D>);
      tma_load_4d(sQ, &map_q, qdo_full, 0, m0, head, batch);
      if constexpr (kHalves == 2) tma_load_4d(sQ + BIG_HALF, &map_q, qdo_full, 64, m0, head, batch);
      tma_load_4d(sDO, &map_do, qdo_full, 0, m0, head, batch);
      if constexpr (kHalves == 2) tma_load_4d(sDO + BIG_HALF, &map_do, qdo_full, 64, m0, head, batch);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j & 1, n0 = j * BK;
        mbar_wait(kv_empty(s), ((j >> 1) & 1) ^ 1);
        mbar_expect_tx(kv_full(s), 2 * kSmallBytes<D>);
        tma_load_4d(sK(s), &map_k, kv_full(s), 0, n0, kv_head, batch);
        if constexpr (kHalves == 2) tma_load_4d(sK(s) + SMALL_HALF, &map_k, kv_full(s), 64, n0, kv_head, batch);
        tma_load_4d(sV(s), &map_v, kv_full(s), 0, n0, kv_head, batch);
        if constexpr (kHalves == 2) tma_load_4d(sV(s) + SMALL_HALF, &map_v, kv_full(s), 64, n0, kv_head, batch);
      }
    }
  } else {
    // ================= MMA warpgroups: wg owns query rows [64 wg, 64 wg + 64); accumulator row = query, column = key / head dim =================
    const int wg = warp >> 2, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float dq_acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) dq_acc[i] = 0.f;
    float lse2[2], dl[2];
    int lim[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m0 + rl + h * 8;
      row_ok[h] = row < p.sq;
      const int64_t stat = ((int64_t)batch * p.h + head) * 2 * p.sq_pad + row;
      lse2[h] = row_ok[h] ? p.stats[stat] : 0.f;
      dl[h] = row_ok[h] ? p.stats[stat + p.sq_pad] : 0.f;
      lim[h] = p.causal ? min(p.sk - 1, row + p.causal_off) : p.sk - 1;
    }
    const int4* cmp = MASKED ? p.colmask + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.sk : nullptr;
    (void)cmp;
    uint32_t dk0 = 0, dk1 = 0, dc2 = 0, dc3 = 0, drc = 0;
    if constexpr (DROPOUT) {
      const uint64_t seed = (uint64_t)__ldg(p.seed_offset);
      dk0 = (uint32_t)seed; dk1 = (uint32_t)(seed >> 32);
      dropout::plane_counter(__ldg(p.seed_offset + 1), batch, p.h, head, dc2, dc3);
      drc = dropout::row_counter(m0 + rl);
    }
    // DROPOUT: the keep bits of key tile jt, bit 8 (jn >> 1) + 4 h + 2 (jn & 1) + e as in the forward; tile j + 1's are drawn while the
    // dQ MMAs of tile j are in flight, where S and dP are dead
    auto draw = [&](int jt) {
      uint32_t bits = 0;
      if constexpr (DROPOUT) {
#pragma unroll 1
        for (int kk = 0; kk < BK / 16; ++kk)   // one call's temporaries live at a time
          bits |= dropout::keep_bits(drc, dropout::key_counter(jt * BK + 16 * kk + 2 * q), dk0, dk1, dc2, dc3, p.keep) << (8 * kk);
      }
      return bits;
    };
    uint32_t keep = 0;
    if constexpr (DROPOUT) {
      if (!SKIP && n_tiles > 0) keep = draw(0);
    }
    (void)draw;
    if (n_tiles > 0) mbar_wait(qdo_full, 0);
    for (int j = 0; j < n_tiles; ++j) {   // SKIP: j counts the tiles processed, jt is the one published for stage s
      const int s = j & 1;
      mbar_wait(kv_full(s), (j >> 1) & 1);
      int jt = j;
      bool open = false;   // SKIP: no key of the tile hides a row of the CTA
      if constexpr (SKIP) {
        const int w = mask_skip::ld_slot(slot(s));
        if (w < 0) break;
        jt = w >> 1; open = w & 1;
        if constexpr (DROPOUT) keep = draw(jt);   // before the MMAs: the next tile is not known yet
      }
      const int n0 = jt * BK;
      float sv[BK / 2], dpv[BK / 2];
      wgmma_fence_regs(sv);
      wgmma_fence_regs(dpv);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < kHalves; ++kb)
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
          if constexpr (MASKED) { if (!open && key < p.sk) m = __ldg(cmp + key); }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m0 + rl + h * 8;
            float x = ex2(fmaf(sv[jn * 4 + h * 2 + e], p.scale_log2, -lse2[h]));
            if (!row_ok[h] || key > lim[h]) x = 0.f;
            if constexpr (MASKED) {
              if ((row >= m.x && row < m.y) || (row >= m.z && row < m.w)) x = 0.f;
            }
            float dp = dpv[jn * 4 + h * 2 + e];
            if constexpr (DROPOUT) dp = (keep >> (8 * (jn >> 1) + 4 * h + 2 * (jn & 1) + e)) & 1u ? dp * p.rscale : 0.f;
            ds[h * 2 + e] = x * (dp - dl[h]) * p.scale;
          }
        }
        dsa[jn >> 1][(jn & 1) * 2 + 0] = pack2<T>(ds[0], ds[1]);
        dsa[jn >> 1][(jn & 1) * 2 + 1] = pack2<T>(ds[2], ds[3]);
      }
      wgmma_fence_regs(dq_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BK / 16; ++ks) {     // B = K tile read MN-major (N = head dim): 16 key rows = 2048 B per step
        const uint64_t desc = make_smem_desc(sK(s) + ks * 2048, SMALL_HALF, 1024);
        if constexpr (D == HD) wgmma_rs_n128<BF16, 1>(dq_acc, dsa[ks], desc, 1);   // dQ += dS K
        else wgmma_rs_n64<BF16, 1>(dq_acc, dsa[ks], desc, 1);
      }
      wgmma_commit();
      if constexpr (DROPOUT && !SKIP) {
        if (j + 1 < n_tiles) keep = draw(j + 1);
      }
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
      for (int jn = 0; jn < D / 8; ++jn)
        *reinterpret_cast<float2*>(dst + jn * 8 + 2 * q) = make_float2(dq_acc[jn * 4 + h * 2], dq_acc[jn * 4 + h * 2 + 1]);
    }
  }
}

// One warp per padded query row (b, s < sq_pad, head): stats = {lse * log2(e), delta = sum_d dO * O} (zero for s >= sq); with ZERO_DQ
// also zeroes the row of the fp32 dQ accumulator.  O and dO share the element strides (sb, ss, sh), d contiguous.  A lane takes 4
// elements; at D = 64 lanes 16-31 add zeros, so delta is summed in the order of the head_dim 128 kernel on zero-padded rows.
template <typename T, bool ZERO_DQ, int D>
__device__ __forceinline__ void prep_body(const T* __restrict__ o, const T* __restrict__ d_o, const float* __restrict__ lse,
                                          float* __restrict__ stats, float* __restrict__ dq, int64_t rows, int sq, int sq_pad, int h,
                                          int64_t sb, int64_t ss, int64_t sh, int64_t dq_sb, int64_t dq_ss, int64_t dq_sh) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // row = (b*sq_pad + s)*h + head
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int64_t bs = row / h;
  const int head = (int)(row - bs * h);
  const int64_t bb = bs / sq_pad;
  const int sidx = (int)(bs - bb * sq_pad);
  float* st = stats + (bb * h + head) * 2 * sq_pad + sidx;
  if (sidx >= sq) {
    if (lane == 0) { st[0] = 0.f; st[sq_pad] = 0.f; }
    return;
  }
  const bool active = D == HD || lane < D / 4;
  const int64_t off = bb * sb + (int64_t)sidx * ss + (int64_t)head * sh + lane * 4;
  float acc = 0.f;
  if (active) {
    const uint2 a = *reinterpret_cast<const uint2*>(o + off);
    const uint2 b = *reinterpret_cast<const uint2*>(d_o + off);
    const T* pa = reinterpret_cast<const T*>(&a);
    const T* pb = reinterpret_cast<const T*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) acc += to_f(pa[i]) * to_f(pb[i]);
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o2);
  if (lane == 0) {
    st[0] = lse[(bb * h + head) * sq + sidx] * 1.4426950408889634f;
    st[sq_pad] = acc;
  }
  if constexpr (ZERO_DQ) {
    if (active)
      *reinterpret_cast<float4*>(dq + bb * dq_sb + (int64_t)sidx * dq_ss + (int64_t)head * dq_sh + lane * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ---- kernels: head_dim 128 (attention_bwd_sm100.cu) ----
template <typename T, bool MASKED, bool DQ>
__global__ void __launch_bounds__(kThreadsDkv, 1)
dkv_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
           const __grid_constant__ CUtensorMap map_do, const __grid_constant__ CUtensorMap map_dq, const Params p) {
  dkv_body<T, MASKED, DQ, HD>(map_q, map_k, map_v, map_do, map_dq, p);
}

template <typename T, bool MASKED>
__global__ void __launch_bounds__(kThreads, 1)
dq_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
          const __grid_constant__ CUtensorMap map_do, const Params p) {
  dq_body<T, MASKED, HD>(map_q, map_k, map_v, map_do, p);
}

template <typename T, bool ZERO_DQ>
__global__ void prep_kernel(const T* __restrict__ o, const T* __restrict__ d_o, const float* __restrict__ lse, float* __restrict__ stats,
                            float* __restrict__ dq, int64_t rows, int sq, int sq_pad, int h, int64_t sb, int64_t ss, int64_t sh,
                            int64_t dq_sb, int64_t dq_ss, int64_t dq_sh) {
  prep_body<T, ZERO_DQ, HD>(o, d_o, lse, stats, dq, rows, sq, sq_pad, h, sb, ss, sh, dq_sb, dq_ss, dq_sh);
}

// ---- kernels: head_dim 64 (attention_d64_sm100.cu) ----
template <typename T, bool MASKED, bool DQ>
__global__ void __launch_bounds__(kThreadsDkv, 1)
dkv_d64_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
               const __grid_constant__ CUtensorMap map_do, const __grid_constant__ CUtensorMap map_dq, const Params p) {
  dkv_body<T, MASKED, DQ, 64>(map_q, map_k, map_v, map_do, map_dq, p);
}

template <typename T, bool MASKED>
__global__ void __launch_bounds__(kThreads, 1)
dq_d64_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
              const __grid_constant__ CUtensorMap map_do, const Params p) {
  dq_body<T, MASKED, 64>(map_q, map_k, map_v, map_do, p);
}

template <typename T, bool ZERO_DQ>
__global__ void prep_d64_kernel(const T* __restrict__ o, const T* __restrict__ d_o, const float* __restrict__ lse, float* __restrict__ stats,
                                float* __restrict__ dq, int64_t rows, int sq, int sq_pad, int h, int64_t sb, int64_t ss, int64_t sh,
                                int64_t dq_sb, int64_t dq_ss, int64_t dq_sh) {
  prep_body<T, ZERO_DQ, 64>(o, d_o, lse, stats, dq, rows, sq, sq_pad, h, sb, ss, sh, dq_sb, dq_ss, dq_sh);
}

template <int D, typename T, bool MASKED, bool DQ> constexpr auto dkv_kernel_for() {
  if constexpr (D == HD) return dkv_kernel<T, MASKED, DQ>;
  else return dkv_d64_kernel<T, MASKED, DQ>;
}
template <int D, typename T, bool MASKED> constexpr auto dq_kernel_for() {
  if constexpr (D == HD) return dq_kernel<T, MASKED>;
  else return dq_d64_kernel<T, MASKED>;
}
template <int D, typename T, bool ZERO_DQ> constexpr auto prep_kernel_for() {
  if constexpr (D == HD) return prep_kernel<T, ZERO_DQ>;
  else return prep_d64_kernel<T, ZERO_DQ>;
}

// deterministic: dkv_kernel without the dQ stage, then dq_kernel; otherwise the single pass (dQ zeroed by prep_kernel)
template <int D, typename T, bool MASKED>
void launch(const Params& p, bool deterministic, const CUtensorMap (&mq)[2], const CUtensorMap (&mk)[2], const CUtensorMap (&mv)[2],
            const CUtensorMap (&mdo)[2], const CUtensorMap& mdq, cudaStream_t s) {
  const dim3 grid_kv(p.hk, p.b, (p.sk + 127) / 128), grid_q((p.sq + 127) / 128, p.h, p.b);
  if (deterministic) {
    constexpr auto dkv = dkv_kernel_for<D, T, MASKED, false>();
    constexpr auto dq = dq_kernel_for<D, T, MASKED>();
    set_max_dynamic_smem<dkv>(DkvSmem<D>::BYTES);
    set_max_dynamic_smem<dq>(kSmemBytes<D>);
    dkv<<<grid_kv, kThreadsDkv, DkvSmem<D>::BYTES, s>>>(mq[1], mk[0], mv[0], mdo[1], mdq, p);
    dq<<<grid_q, kThreads, kSmemBytes<D>, s>>>(mq[0], mk[1], mv[1], mdo[0], p);
  } else {
    constexpr auto dkv = dkv_kernel_for<D, T, MASKED, true>();
    set_max_dynamic_smem<dkv>(DkvSmem<D>::BYTES);
    dkv<<<grid_kv, kThreadsDkv, DkvSmem<D>::BYTES, s>>>(mq[1], mk[0], mv[0], mdo[1], mdq, p);
  }
}

// The backward at head size D (the operands checked by attention_bwd): builds the tensor maps, launches the stats kernel and calls
// launch(T(), std::bool_constant<MASKED>(), params, deterministic, maps...) for the main kernels of the operands' type and mask.
template <int D, typename Launch>
int run_with(const AttnBwdArgs& a, cudaStream_t s, Launch&& launch) {
  const AttnArgs& f = a.fwd;
  if (a.dq_strides[0] % 4 || a.dq_strides[1] % 4 || a.dq_strides[2] % 4 || (reinterpret_cast<uintptr_t>(a.dq) & 15)) return 1;   // TMA / float4
  if (a.dkv_strides[0] % 2 || a.dkv_strides[1] % 2 || a.dkv_strides[2] % 2) return 1;
  // every operand as a 128-row box map (the resident tile of dq_kernel) and as a 64-row box map (the streamed tile of dkv_kernel)
  CUtensorMap mq[2], mk[2], mv[2], mdo[2], mdq;
  for (int i = 0; i < 2; ++i) {
    const uint32_t rows = i ? 64 : 128;
    if (!attn::make_map4(&mq[i], f.q, f.d, f.sq, f.h, f.b, f.q_strides[1], f.q_strides[2], f.q_strides[0], rows, f.dtype)) return 2;
    if (!attn::make_map4(&mk[i], f.k, f.d, f.sk, f.hk, f.b, f.k_strides[1], f.k_strides[2], f.k_strides[0], rows, f.dtype)) return 2;
    if (!attn::make_map4(&mv[i], f.v, f.d, f.sk, f.hk, f.b, f.v_strides[1], f.v_strides[2], f.v_strides[0], rows, f.dtype)) return 2;
    if (!attn::make_map4(&mdo[i], a.d_o, f.d, f.sq, f.h, f.b, a.o_strides[1], a.o_strides[2], a.o_strides[0], rows, f.dtype)) return 2;
  }
  // the fp32 dQ accumulator over its own strides, in the reduce boxes of the single pass: 32 d (128 B) x 64 query rows
  if (!attn::make_map4(&mdq, a.dq, f.d, f.sq, f.h, f.b, a.dq_strides[1], a.dq_strides[2], a.dq_strides[0], 64, kF32)) return 2;
  const int sq_pad = attention_bwd_stats_pad(f.sq);
  const int64_t rows = (int64_t)f.b * sq_pad * f.h;
  const int wpb = 8;
  const unsigned blocks = (unsigned)((rows + wpb - 1) / wpb);
  auto prep = [&](auto kern, auto* o) {
    using P = std::remove_const_t<std::remove_pointer_t<decltype(o)>>;
    kern<<<blocks, wpb * 32, 0, s>>>(o, reinterpret_cast<const P*>(a.d_o), f.lse, a.stats, a.dq, rows, f.sq, sq_pad, f.h, a.o_strides[0],
                                     a.o_strides[1], a.o_strides[2], a.dq_strides[0], a.dq_strides[1], a.dq_strides[2]);
  };
  const bool det = a.deterministic;
  if (f.dtype == kBF16) {
    const auto* o = reinterpret_cast<const __nv_bfloat16*>(f.o);
    det ? prep(prep_kernel_for<D, __nv_bfloat16, false>(), o) : prep(prep_kernel_for<D, __nv_bfloat16, true>(), o);
  } else {
    const auto* o = reinterpret_cast<const __half*>(f.o);
    det ? prep(prep_kernel_for<D, __half, false>(), o) : prep(prep_kernel_for<D, __half, true>(), o);
  }
  Params p;
  p.b = f.b; p.sq = f.sq; p.sk = f.sk; p.h = f.h; p.hk = f.hk;
  p.scale = f.scale; p.scale_log2 = f.scale * 1.4426950408889634f;
  p.causal = f.causal; p.causal_off = f.sk - f.sq;
  p.colmask = reinterpret_cast<const int4*>(f.colmask);
  p.mask_heads = f.mask_heads > 0 ? f.mask_heads : 1;
  p.stats = a.stats; p.sq_pad = sq_pad; p.dq = a.dq; p.dk = a.dk; p.dv = a.dv;
  p.dkv_sb = a.dkv_strides[0]; p.dkv_ss = a.dkv_strides[1]; p.dkv_sh = a.dkv_strides[2];
  p.dq_sb = a.dq_strides[0]; p.dq_ss = a.dq_strides[1]; p.dq_sh = a.dq_strides[2];
  if (f.dtype == kBF16) {
    if (p.colmask) launch(__nv_bfloat16(), std::true_type(), p, det, mq, mk, mv, mdo, mdq);
    else launch(__nv_bfloat16(), std::false_type(), p, det, mq, mk, mv, mdo, mdq);
  } else {
    if (p.colmask) launch(__half(), std::true_type(), p, det, mq, mk, mv, mdo, mdq);
    else launch(__half(), std::false_type(), p, det, mq, mk, mv, mdo, mdq);
  }
  return B200_LAUNCH_RESULT();
}

template <int D>
int run(const AttnBwdArgs& a, cudaStream_t s) {
  return run_with<D>(a, s, [&](auto tag_t, auto tag_masked, const Params& p, bool det, const CUtensorMap (&mq)[2], const CUtensorMap (&mk)[2],
                               const CUtensorMap (&mv)[2], const CUtensorMap (&mdo)[2], const CUtensorMap& mdq) {
    launch<D, decltype(tag_t), decltype(tag_masked)::value>(p, det, mq, mk, mv, mdo, mdq, s);
  });
}

}  // namespace attn_bwd
}  // namespace b200
