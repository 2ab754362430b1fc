// Persistent warp-specialised GEMM for sm_90a: TMA (cp.async.bulk.tensor) -> 128B-swizzled smem ring -> wgmma.mma_async
// (bf16 / fp16 operands from shared memory, fp32 accumulators in registers) -> epilogue with fused bias / activation / accumulate,
// staged through swizzled shared memory and written by asynchronous TMA stores.  Hand-written PTX; no CUTLASS.
//
// Parity (behaviour): phi MatmulKernel / fused_gemm_epilogue (paddle/phi/kernels/fusion/gpu/fused_gemm_epilogue_kernel.cu)
// which call cuBLASLt in the reference.
//
// Operand layouts (all four combinations, selected by the wgmma transpose bits, no transposition copies):
//   A: [M,K] row-major (K-major)  or  [K,M] row-major (MN-major, "a_is_km")  -> needed for dW = X^T dY
//   B: [N,K] row-major (K-major, "b_is_nk")  or  [K,N] row-major (MN-major)  -> paddle Linear weight is [in,out]
// Roles (384 threads = 3 warpgroups): warpgroup 0 = producer (warp 0 TMA, warp 1 the copy role of the fused all-gather) and gives its
// registers away; warpgroups 1 and 2 each own 64 rows of the 128 x BN tile, issue the MMAs of a k-block as one commit group, keep one
// group in flight, and hand their accumulators to TMA stores while the producer is already filling the ring for the next tile.
// No kernel here may contain a function call (printf, a __noinline__ function): ptxas then serializes every wgmma of the kernel (C7510).
// Also in this kernel: strided batches, the grouped (MoE expert) modes, the reduce-scatter push epilogue and the fused all-gather.
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace gemm {
using namespace ptx;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 x 2B = 128B = one swizzle atom row
constexpr int MMA_K = 16;
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr uint32_t A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB

template <int BN> struct Cfg {
  static constexpr int kStages = BN == 256 ? 4 : 6;
  static constexpr uint32_t B_STAGE_BYTES = BN * BLOCK_K * 2;
  static constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr uint32_t SMEM_BYTES = kStages * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 232448, "gemm: shared memory budget (227 KB per block)");
};

struct Params {
  int m, n, k, batch;
  void* d;
  const void* bias;
  int64_t ldd, stride_d;
  int in_dtype, out_dtype;
  int has_bias, act, accumulate;
  int tma_store;           // D goes out through the shared staging buffer and TMA stores (map_d); 0 = per-thread global stores
  // grouped GEMM (MoE experts, see GemmArgs::grouped): 1 = rows grouped by expert (256-row block -> expert table), 2 = per-expert weight gradient
  int grouped;
  const int* tile_expert;
  const int* expert_k0;
  const int* expert_kb;
  int rs_world, rs_rows;   // fused reduce-scatter push (see GemmArgs)
  void* rs_dst[8];
  // fused all-gather -> GEMM (see GemmArgs): warp 1 of every CTA pulls the peers' row shards into the local A buffer
  int ag_world, ag_rank, ag_rows, ag_chunks;
  const char* ag_src[8];
  char* ag_dst;
  uint32_t* ag_flags;
  uint32_t* ag_pad[8];
  uint32_t ag_epoch;
};

constexpr int kAgChunkBytes = 16384;
constexpr int kAgReadySlot = 4, kAgDoneSlot = 5, kPadRanks = 8;

__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// bounded spins: a dead peer / protocol bug traps instead of hanging the GPU (no printf: any call in this kernel serializes its wgmma)
__device__ __forceinline__ void spin_sys_ge(const uint32_t* p, uint32_t target) {
  const uint64_t t0 = globaltimer_ns();
  while ((int32_t)(ld_acquire_sys_u32(p) - target) < 0) {
    if (globaltimer_ns() - t0 > 10000000000ull) __trap();
  }
}
__device__ __forceinline__ void spin_gpu_ge(const uint32_t* p, uint32_t target) {
  const uint64_t t0 = globaltimer_ns();
  while (ld_acquire_gpu_u32(p) < target) {
    if (globaltimer_ns() - t0 > 10000000000ull) __trap();
  }
}

// Copy role of the fused all-gather: chunk g of the remote data is handled by warp (g % #CTAs); finished chunks bump the
// counter of their 128-row block, which the TMA producers poll before loading A rows of that block.
__device__ __forceinline__ void ag_copy_role(const Params& p, int lane) {
  const int nwarps = gridDim.x, wid = blockIdx.x;
  const int blocks_per_rank = p.ag_rows / BLOCK_M;
  const int64_t block_bytes = (int64_t)BLOCK_M * p.k * 2;
  const int64_t per_src = (int64_t)blocks_per_rank * p.ag_chunks;
  const int64_t total = (int64_t)(p.ag_world - 1) * per_src;
  uint32_t* my_pad = p.ag_pad[p.ag_rank];
  if (wid == 0 && lane < p.ag_world && lane != p.ag_rank)        // my shard is in place (stream order before this kernel)
    st_release_sys_u32(p.ag_pad[lane] + kAgReadySlot * kPadRanks + p.ag_rank, p.ag_epoch);
  int cur_src = -1;
  for (int64_t g = wid; g < total; g += nwarps) {
    const int pr = (int)(g / per_src) + 1;
    const int src = (p.ag_rank + pr) % p.ag_world;
    const int64_t rem = g - (int64_t)(pr - 1) * per_src;
    const int blk_in = (int)(rem / p.ag_chunks), ch = (int)(rem % p.ag_chunks);
    if (src != cur_src) {
      if (lane == 0) spin_sys_ge(my_pad + kAgReadySlot * kPadRanks + src, p.ag_epoch);
      __syncwarp();
      cur_src = src;
    }
    const uint4* sp = reinterpret_cast<const uint4*>(p.ag_src[src] + blk_in * block_bytes + (int64_t)ch * kAgChunkBytes);
    uint4* dp = reinterpret_cast<uint4*>(p.ag_dst + ((int64_t)src * blocks_per_rank + blk_in) * block_bytes + (int64_t)ch * kAgChunkBytes);
#pragma unroll 1
    for (int it = 0; it < kAgChunkBytes / 16 / 32 / 4; ++it) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = sp[(it * 4 + j) * 32 + lane];     // 4 independent 16 B loads over NVLink in flight
#pragma unroll
      for (int j = 0; j < 4; ++j) dp[(it * 4 + j) * 32 + lane] = v[j];
    }
    __syncwarp();
    if (lane == 0) {
      __threadfence();
      atomicAdd(p.ag_flags + src * blocks_per_rank + blk_in, 1u);
    }
  }
  __syncwarp();
  if (lane == 0) {
    __threadfence();
    const int done_idx = p.ag_world * blocks_per_rank;
    if (atomicAdd(p.ag_flags + done_idx, 1u) == (uint32_t)nwarps - 1) {    // every pull of this rank has completed
      for (int r = 0; r < p.ag_world; ++r)
        if (r != p.ag_rank) st_release_sys_u32(p.ag_pad[r] + kAgDoneSlot * kPadRanks + p.ag_rank, p.ag_epoch);
    }
  }
  if (wid == 0 && lane < p.ag_world && lane != p.ag_rank)        // peers finished reading my shard: it may be reused after exit
    spin_sys_ge(my_pad + kAgDoneSlot * kPadRanks + lane, p.ag_epoch);
}

// two adjacent output columns of one row (what a thread holds per 8-column group of the accumulator fragment)
template <typename TO>
__device__ __forceinline__ void store_pair(TO* __restrict__ dst, float v0, float v1, int valid, bool accumulate) {
  if (valid >= 2 && (reinterpret_cast<uintptr_t>(dst) & (2 * sizeof(TO) - 1)) == 0) {
    struct alignas(2 * sizeof(TO)) Pair { TO a, b; };
    Pair o;
    if (accumulate) {
      const Pair old = *reinterpret_cast<const Pair*>(dst);
      v0 += to_f(old.a);
      v1 += to_f(old.b);
    }
    o.a = from_f<TO>(v0);
    o.b = from_f<TO>(v1);
    *reinterpret_cast<Pair*>(dst) = o;
  } else {
    if (valid >= 1) dst[0] = from_f<TO>(accumulate ? v0 + to_f(dst[0]) : v0);
    if (valid >= 2) dst[1] = from_f<TO>(accumulate ? v1 + to_f(dst[1]) : v1);
  }
}

// Staged epilogue: the consumer warpgroup's 64 x BN half-tile leaves as boxes of 64 rows x 128 bytes (64 16-bit or 32 fp32 columns),
// written 128B-swizzled into one of two 8 KB slots of the warpgroup's staging buffer and stored by TMA. Box c (counted over the
// warpgroup's whole run in `cnt`) uses slot c & 1, so it is written while the store of box c - 1 still reads the other slot.
// Invariant: once the warpgroup has passed the named barrier of box c, slot (c + 1) & 1 is free (the elected thread waited for the
// store of box c - 1 to finish reading it just before that barrier). In accumulate mode the old D box is TMA-loaded into its slot
// first and added in fp32, rounded once, as in store_pair. Two loads are in flight: boxes 0 and 1 of a tile land during the mainloop,
// box c + 2 is loaded into box c's slot as soon as the store of box c has read it. TMA clips the boxes at the tensor bounds, so
// partial tiles need no per-element tests.
constexpr uint32_t kStageSlotBytes = 8192;

template <typename TO, int BN>
__device__ __forceinline__ int epilogue_boxes(const Params& p, int n0) {   // boxes that start right of column n are skipped
  constexpr int CB = 128 / sizeof(TO);
  return min(BN / CB, (p.n - n0 + CB - 1) / CB);
}

// One epilogue box of the warpgroup's half-tile into its staging slot: bias, activation and old D (accumulate mode) in fp32, one rounding.
// PLAIN (no bias, no activation, no accumulate: every forward and dX GEMM of the model) drops those tests from the unrolled code, which
// is what the epilogue's time goes to; the values are computed with the same fp32 operations (acc + 0.f), so the output bits are the same.
template <typename TO, int BN, bool PLAIN>
__device__ __forceinline__ void write_box(const float (&acc)[BN / 2], const Params& p, uint8_t* slot, int b, int n0, int ww, int lane) {
  constexpr int CB = 128 / sizeof(TO);
  struct alignas(2 * sizeof(TO)) Pair { TO a, b; };
  const int rq = lane >> 2;                               // row within the 8-row swizzle atom
#pragma unroll
  for (int jj = 0; jj < CB / 8; ++jj) {
    const int j = b * (CB / 8) + jj;
    const int col = n0 + j * 8 + (lane & 3) * 2;
    const int valid = p.n - col;
    float b0 = 0.f, b1 = 0.f;
    if (!PLAIN && p.has_bias && valid > 0) {
      if (p.in_dtype == kBF16) {
        const __nv_bfloat16* bp = (const __nv_bfloat16*)p.bias + col;
        b0 = __bfloat162float(bp[0]);
        if (valid > 1) b1 = __bfloat162float(bp[1]);
      } else {
        const __half* bp = (const __half*)p.bias + col;
        b0 = __half2float(bp[0]);
        if (valid > 1) b1 = __half2float(bp[1]);
      }
    }
    const uint32_t byte = (jj * 8 + (lane & 3) * 2) * sizeof(TO);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      Pair* dst = reinterpret_cast<Pair*>(slot + (ww * 16 + h * 8 + rq) * 128 + (((byte >> 4) ^ rq) << 4) + (byte & 15));
      float v0 = acc[j * 4 + h * 2] + b0, v1 = acc[j * 4 + h * 2 + 1] + b1;
      if (!PLAIN && p.act == 1) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
      else if (!PLAIN && p.act == 2) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      if (!PLAIN && p.accumulate) {
        const Pair old = *dst;
        v0 += to_f(old.a);
        v1 += to_f(old.b);
      }
      Pair o;
      o.a = from_f<TO>(v0);
      o.b = from_f<TO>(v1);
      *dst = o;
    }
  }
}

template <typename TO, int BN>
__device__ __forceinline__ void epilogue_tma(const float (&acc)[BN / 2], const Params& p, const CUtensorMap* map_d, uint8_t* stg,
                                             uint32_t ld_bar, uint32_t& cnt, int m0, int n0, int zd, int ww, int lane, int bar_id) {
  constexpr int CB = 128 / sizeof(TO);                    // columns per box
  constexpr int NB = BN / CB;                             // boxes per half-tile (BN >= 64)
  const int nbox = epilogue_boxes<TO, BN>(p, n0);
  const bool elected = ww == 0 && lane == 0;
  const bool plain = !p.has_bias && p.act == 0 && !p.accumulate;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    if (b >= nbox) break;
    uint8_t* slot = stg + (cnt & 1) * kStageSlotBytes;
    if (p.accumulate) mbar_wait_unbounded(ld_bar + 8 * (cnt & 1), (cnt >> 1) & 1);
    if (plain) write_box<TO, BN, true>(acc, p, slot, b, n0, ww, lane);
    else write_box<TO, BN, false>(acc, p, slot, b, n0, ww, lane);
    fence_proxy_async();                                  // generic-proxy writes -> the TMA store (async proxy) reads them
    if (elected) bulk_wait_group_read<0>();               // the store of box cnt - 1 is done with the other slot
    named_bar_sync(bar_id, 128);
    if (elected) {
      tma_store_3d(map_d, smem_u32(slot), n0 + b * CB, m0, zd);
      bulk_commit_group();
      if (p.accumulate && b + 2 < nbox) {
        bulk_wait_group_read<0>();                        // the store of box cnt has read the slot
        const uint32_t s = cnt & 1;
        mbar_expect_tx(ld_bar + 8 * s, kStageSlotBytes);
        tma_load_3d(smem_u32(slot), map_d, ld_bar + 8 * s, n0 + (b + 2) * CB, m0, zd);
      }
    }
    ++cnt;
  }
}

template <int BN, bool BF16, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
            const __grid_constant__ CUtensorMap map_d, const Params p) {
  using C = Cfg<BN>;
  constexpr int kStages = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(1024) uint8_t staging[2][2 * kStageSlotBytes];   // per consumer warpgroup (epilogue_tma)
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B needs 1024B alignment
  const uint32_t bar_base = smem_base + kStages * C::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  auto load_bar = [&](int wg) { return bar_base + 8u * (2 * kStages + 2 * wg); };   // two slots per warpgroup (accumulate mode)
  const uint32_t done_bar = bar_base + 8u * (2 * kStages + 4);                        // every consumer warp has finished

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_m = (p.m + BLOCK_M - 1) / BLOCK_M, num_n = (p.n + BN - 1) / BN;
  const int tiles_per_batch = num_m * num_n;
  const int num_tiles = tiles_per_batch * p.batch;
  const int num_kb = (p.k + BLOCK_K - 1) / BLOCK_K;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    if (p.tma_store) tma_prefetch_desc(&map_d);
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    for (int s = 0; s < 4; ++s) mbar_init(load_bar(0) + 8u * s, 1);
    mbar_init(done_bar, kConsumerWarps);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  // tile order: groups of 8 M-tiles sweep N (operand panels stay L2-resident across the wave)
  auto tile_coords = [&](int tile, int& bz, int& mb, int& nb) {
    bz = tile / tiles_per_batch;
    const int t = tile - bz * tiles_per_batch;
    constexpr int GROUP_M = 8;
    const int in_group = GROUP_M * num_n;
    const int g = t / in_group;
    const int first_m = g * GROUP_M;
    const int gsz = min(num_m - first_m, GROUP_M);
    const int r = t - g * in_group;
    mb = first_m + r % gsz;
    nb = r / gsz;
    if (p.ag_world > 1) {   // fused all-gather: start with the row blocks that are already local
      mb += p.ag_rank * (p.ag_rows / BLOCK_M);
      if (mb >= num_m) mb -= num_m;
    }
  };
  // grouped modes: which batch index each operand uses for this tile, the reduction range, and whether the tile exists at all
  auto tile_group = [&](int bz, int mb, int& za, int& zb, int& zd, int& kbeg, int& nkb) -> bool {
    za = zb = zd = bz; kbeg = 0; nkb = num_kb;
    if (p.grouped == 1) {
      const int e = p.tile_expert[mb >> 1];   // the table has one entry per 256 rows
      if (e < 0) return false;               // padding tile beyond the last expert's rows
      za = 0; zb = e; zd = 0;
    } else if (p.grouped == 2) {
      nkb = p.expert_kb[bz];
      if (nkb <= 0) return false;            // expert received no rows: its weight gradient gets nothing added
      kbeg = p.expert_k0[bz];
      za = 0; zb = 0; zd = bz;
    }
    return true;
  };

  if (warp < 4) {
    reg_dealloc<56>();
    if (warp == 0 && lane == 0) {
      // ================= TMA producer =================
      int stage = 0;
      uint32_t phase = 0;
      const uint64_t hint = 0x1000000000000000ull;  // EVICT_NORMAL
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int bz, mb, nb;
        tile_coords(tile, bz, mb, nb);
        int za, zb, zd, kbeg, nkb;
        if (!tile_group(bz, mb, za, zb, zd, kbeg, nkb)) continue;
        const int m0 = mb * BLOCK_M, n0 = nb * BN;
        if (p.ag_world > 1 && mb / (p.ag_rows / BLOCK_M) != p.ag_rank) {   // rows owned by a peer: wait until the copy warps landed them
          spin_gpu_ge(p.ag_flags + mb, (uint32_t)p.ag_chunks);
          asm volatile("fence.proxy.async;" ::: "memory");                 // generic-proxy writes (other SMs) -> TMA (async proxy) reads
        }
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(full_bar(stage), C::STAGE_BYTES);
          const int k0 = kbeg + kb * BLOCK_K;
          if constexpr (!A_MN) {
            tma_load_3d(sa, &map_a, full_bar(stage), k0, m0, za, hint);  // box {64 k, 128 m}
          } else {
#pragma unroll
            for (int i = 0; i < BLOCK_M / 64; ++i)                      // box {64 m, 64 k}
              tma_load_3d(sa + i * 8192, &map_a, full_bar(stage), m0 + i * 64, k0, za, hint);
          }
          if constexpr (!B_MN) {
            tma_load_3d(sb, &map_b, full_bar(stage), k0, n0, zb, hint);  // box {64 k, BN n}
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)                           // box {64 n, 64 k}
              tma_load_3d(sb + i * 8192, &map_b, full_bar(stage), n0 + i * 64, k0, zb, hint);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
      // The consumers wait unbounded (a reachable trap would cap their registers at the launch budget), so the producer waits,
      // bounded, until they have released every stage and finished: a protocol bug traps here instead of hanging the GPU.
      for (int i = 0; i < kStages; ++i) {
        mbar_wait(empty_bar(stage), phase ^ 1);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      mbar_wait(done_bar, 0);
    } else if (warp == 1 && p.ag_world > 1) {
      ag_copy_role(p, lane);
    }
  } else {
    // ================= MMA + epilogue: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =================
    reg_alloc<224>();
    const int wg = (warp >> 2) - 1, ww = warp & 3;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t boxes = 0;                        // staged epilogue boxes issued by this warpgroup (epilogue_tma)
    const bool elected = ww == 0 && lane == 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int bz, mb, nb;
      tile_coords(tile, bz, mb, nb);
      int za, zb, zd, kbeg, nkb;
      if (!tile_group(bz, mb, za, zb, zd, kbeg, nkb)) continue;
      // accumulate mode: old D of the first two epilogue boxes lands during the mainloop, box 0 into slot boxes & 1 (free since the
      // previous tile's stores) and, after the first k-block, box 1 into the other slot once the previous tile's last store has read it
      const int old_boxes = !(p.tma_store && p.accumulate) ? 0 : (p.out_dtype == kF32 ? epilogue_boxes<float, BN>(p, nb * BN)
                                                                                         : epilogue_boxes<uint16_t, BN>(p, nb * BN));
      const int old_cb = p.out_dtype == kF32 ? 32 : 64;
      auto load_old = [&](int b) {
        const uint32_t s = (boxes + b) & 1;
        mbar_expect_tx(load_bar(wg) + 8 * s, kStageSlotBytes);
        tma_load_3d(smem_u32(staging[wg] + s * kStageSlotBytes), &map_d, load_bar(wg) + 8 * s, nb * BN + b * old_cb,
                    mb * BLOCK_M + wg * 64, zd);
      };
      if (old_boxes > 0 && elected) load_old(0);
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait_unbounded(full_bar(stage), phase);
        const uint32_t sa = smem_base + stage * C::STAGE_BYTES + wg * 8192;   // 64 rows (K-major) or one {64 m, 64 k} box (MN-major)
        const uint32_t sb = smem_base + stage * C::STAGE_BYTES + A_STAGE_BYTES;
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
          // K-major: advance 16 elem = 32 B inside the swizzle row; MN-major: advance 16 k-rows = 2048 B
          const uint64_t adesc = A_MN ? make_smem_desc(sa + k * 2048, 8192, 1024) : make_smem_desc(sa + k * 32, 16, 1024);
          const uint64_t bdesc = B_MN ? make_smem_desc(sb + k * 2048, 8192, 1024) : make_smem_desc(sb + k * 32, 16, 1024);
          if constexpr (BN == 256) wgmma_ss_n256<BF16, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb | k) != 0);
          else if constexpr (BN == 128) wgmma_ss_n128<BF16, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb | k) != 0);
          else wgmma_ss_n64<BF16, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb | k) != 0);
        }
        wgmma_commit();
        if (prev >= 0) {                       // the previous k-block's MMAs have retired: its smem slot goes back to the producer
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(empty_bar(prev));
        }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
        if (kb == 0 && old_boxes > 1 && elected) {
          bulk_wait_group_read<0>();
          load_old(1);
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (lane == 0) mbar_arrive(empty_bar(prev));

      if (p.tma_store) {
        const int m0 = mb * BLOCK_M + wg * 64, n0 = nb * BN;
        if (p.out_dtype == kBF16) epilogue_tma<__nv_bfloat16, BN>(acc, p, &map_d, staging[wg], load_bar(wg), boxes, m0, n0, zd, ww, lane, 1 + wg);
        else if (p.out_dtype == kF16) epilogue_tma<__half, BN>(acc, p, &map_d, staging[wg], load_bar(wg), boxes, m0, n0, zd, ww, lane, 1 + wg);
        else epilogue_tma<float, BN>(acc, p, &map_d, staging[wg], load_bar(wg), boxes, m0, n0, zd, ww, lane, 1 + wg);
        continue;
      }
      // ---- register epilogue (reduce-scatter push, or D not 16-byte aligned for a tensor map) from the accumulator fragment:
      // rows r0 and r0 + 8, per 8-column group the columns 2 (lane % 4), + 1 ----
      const int r0 = mb * BLOCK_M + wg * 64 + ww * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = nb * BN + j * 8 + (lane & 3) * 2;
        const int valid = p.n - col;
        if (valid <= 0) continue;
        float b0 = 0.f, b1 = 0.f;
        if (p.has_bias) {
          if (p.in_dtype == kBF16) {
            const __nv_bfloat16* b = (const __nv_bfloat16*)p.bias + col;
            b0 = __bfloat162float(b[0]);
            if (valid > 1) b1 = __bfloat162float(b[1]);
          } else {
            const __half* b = (const __half*)p.bias + col;
            b0 = __half2float(b[0]);
            if (valid > 1) b1 = __half2float(b[1]);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r0 + h * 8;
          float v0 = acc[j * 4 + h * 2] + b0, v1 = acc[j * 4 + h * 2 + 1] + b1;
          if (p.act == 1) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
          else if (p.act == 2) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          if (row < p.m) {
            void* dptr = p.d;
            int64_t off = (int64_t)zd * p.stride_d + (int64_t)row * p.ldd + col;
            if (p.rs_world > 1) {   // fused reduce-scatter: push this row's partial into its owner's staging slot (peer HBM)
              const int owner = row / p.rs_rows;
              dptr = p.rs_dst[owner];
              off = (int64_t)(row - owner * p.rs_rows) * p.ldd + col;
            }
            if (p.out_dtype == kBF16) store_pair((__nv_bfloat16*)dptr + off, v0, v1, valid, p.accumulate);
            else if (p.out_dtype == kF16) store_pair((__half*)dptr + off, v0, v1, valid, p.accumulate);
            else store_pair((float*)dptr + off, v0, v1, valid, p.accumulate);
          }
        }
      }
    }
    if (p.tma_store && elected) bulk_wait_group<0>();   // the staging buffer must outlive the last store's reads
    __syncwarp();
    if (lane == 0) mbar_arrive(done_bar);
  }
}

// ---------------------------------------------------------------------------------------------- host side
struct MapKey {
  const void* ptr; uint64_t inner, rows, batch, ld, bstride; uint32_t box_inner, box_rows; int dtype;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && inner == o.inner && rows == o.rows && batch == o.batch && ld == o.ld && bstride == o.bstride &&
           box_inner == o.box_inner && box_rows == o.box_rows && dtype == o.dtype;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    auto mix = [&](uint64_t v) { h ^= std::hash<uint64_t>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.inner); mix(k.rows); mix(k.batch); mix(k.ld); mix(k.bstride); mix(k.box_inner); mix(k.box_rows); mix((uint64_t)k.dtype);
    return h;
  }
};

// 3-D map {inner (contiguous), rows, batch}; element = 2 bytes (bf16 / fp16) or 4 bytes (kF32: TMA-store maps of fp32 outputs).
bool make_map(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t ld, uint64_t bstride,
              uint32_t box_inner, uint32_t box_rows, int dtype) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  MapKey key{ptr, inner, rows, batch, ld, bstride, box_inner, box_rows, dtype};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return true; }
  }
  const uint64_t es = dtype == kF32 ? 4 : 2;
  const uint64_t dims[3] = {inner, rows, batch};
  const uint64_t strides[2] = {ld * es, (batch > 1 ? bstride : rows * ld) * es};
  const uint32_t box[3] = {box_inner, box_rows, 1};
  const CUtensorMapDataType type = dtype == kBF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                  : (dtype == kF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  if (!encode_tensor_map(out, type, 3, ptr, dims, strides, box, "gemm")) return false;
  std::lock_guard<std::mutex> g(mu);
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, *out);
  return true;
}

template <int BN, bool BF16, bool A_MN, bool B_MN>
static int launch(const GemmArgs& g, cudaStream_t s) {
  using C = Cfg<BN>;
  CUtensorMap ma, mb;
  uint64_t batch = g.batch > 1 ? g.batch : 1;
  uint64_t batch_a = batch, batch_b = batch;
  if (g.grouped == 1) { batch_a = 1; batch_b = g.groups; batch = 1; }             // rows grouped by expert: B = stacked expert weights
  else if (g.grouped == 2) { batch_a = 1; batch_b = 1; batch = g.groups; }        // per-expert weight gradient: D = stacked [E, m, n]
  bool ok;
  if (!A_MN) ok = make_map(&ma, g.a, g.k, g.m, batch_a, g.lda, g.stride_a, BLOCK_K, BLOCK_M, g.dtype);
  else       ok = make_map(&ma, g.a, g.m, g.k, batch_a, g.lda, g.stride_a, 64, BLOCK_K, g.dtype);
  if (!ok) return 2;
  if (!B_MN) ok = make_map(&mb, g.b, g.k, g.n, batch_b, g.ldb, g.stride_b, BLOCK_K, BN, g.dtype);
  else       ok = make_map(&mb, g.b, g.n, g.k, batch_b, g.ldb, g.stride_b, 64, BLOCK_K, g.dtype);
  if (!ok) return 2;
  Params p;
  p.m = g.m; p.n = g.n; p.k = g.k; p.batch = (int)batch;
  p.d = g.d; p.bias = g.bias; p.ldd = g.ldd; p.stride_d = g.stride_d;
  p.in_dtype = g.dtype; p.out_dtype = g.out_dtype;
  p.has_bias = (g.epilogue >= 1 && g.epilogue <= 3 && g.bias) ? 1 : 0;
  p.act = g.epilogue == 2 ? 1 : (g.epilogue == 3 ? 2 : 0);
  p.accumulate = g.epilogue == 4 ? 1 : 0;
  p.grouped = g.grouped; p.tile_expert = g.tile_expert; p.expert_k0 = g.expert_k0; p.expert_kb = g.expert_kb;
  p.rs_world = g.rs_world > 1 ? g.rs_world : 0;
  p.rs_rows = g.rs_rows;
  for (int i = 0; i < 8; ++i) p.rs_dst[i] = g.rs_dst[i];
  if (p.rs_world) p.ldd = g.n;
  // TMA-store epilogue wherever D can be described by a tensor map: local memory, 16-byte aligned base and strides
  CUtensorMap md{};
  const uint64_t es = g.out_dtype == kF32 ? 4 : 2;
  p.tma_store = !p.rs_world && (reinterpret_cast<uintptr_t>(g.d) & 15) == 0 && ((uint64_t)g.ldd * es) % 16 == 0 &&
                (batch == 1 || ((uint64_t)g.stride_d * es) % 16 == 0);
  if (p.tma_store && !make_map(&md, g.d, g.n, g.m, batch, g.ldd, g.stride_d, 128 / es, 64, g.out_dtype)) return 2;
  p.ag_world = 0;
  if (g.ag_world > 1) {
    // preconditions of the fused all-gather (checked by the caller as well): A is K-major with lda == k, whole 256-row blocks per rank
    if (A_MN || g.lda != g.k || g.ag_rows % (2 * BLOCK_M) || g.m != g.ag_world * g.ag_rows || batch != 1 ||
        ((int64_t)BLOCK_M * g.k * 2) % kAgChunkBytes) {
      set_last_error(__FILE__, __LINE__, "gemm: unsupported shape for the fused all-gather");
      return 4;
    }
    p.ag_world = g.ag_world; p.ag_rank = g.ag_rank; p.ag_rows = g.ag_rows;
    p.ag_chunks = (int)(((int64_t)BLOCK_M * g.k * 2) / kAgChunkBytes);
    for (int i = 0; i < 8; ++i) { p.ag_src[i] = (const char*)g.ag_src[i]; p.ag_pad[i] = (uint32_t*)g.ag_pad[i]; }
    p.ag_dst = (char*)const_cast<void*>(g.a);
    p.ag_flags = (uint32_t*)g.ag_flags;
    p.ag_epoch = g.ag_epoch;
  }
  set_max_dynamic_smem<gemm_kernel<BN, BF16, A_MN, B_MN>>(C::SMEM_BYTES);
  const int num_tiles = ((g.m + BLOCK_M - 1) / BLOCK_M) * ((g.n + BN - 1) / BN) * (int)batch;
  // B200_GEMM_RESERVE_SMS=<n>: keep n SMs out of every persistent GEMM grid so that concurrently launched collective kernels are resident
  // unconditionally (docs/race_detection.md, "cross-rank progress"); default 0
  static const int reserve = [] { const char* e = getenv("B200_GEMM_RESERVE_SMS"); const int v = e ? atoi(e) : 0; return v < 0 ? 0 : v; }();
  const int usable = sm_count() - reserve > 0 ? sm_count() - reserve : 1;
  const int grid = num_tiles < usable ? num_tiles : usable;
  gemm_kernel<BN, BF16, A_MN, B_MN><<<grid, kThreads, C::SMEM_BYTES, s>>>(ma, mb, md, p);
  return B200_LAUNCH_RESULT();
}

template <int BN, bool BF16>
static int launch_layout(const GemmArgs& g, cudaStream_t s) {
  if (g.a_is_km) return g.b_is_nk ? launch<BN, BF16, true, false>(g, s) : launch<BN, BF16, true, true>(g, s);
  return g.b_is_nk ? launch<BN, BF16, false, false>(g, s) : launch<BN, BF16, false, true>(g, s);
}

}  // namespace gemm

int gemm_tcgen05_supported(int m, int n, int k, int64_t lda, int64_t ldb, int64_t ldd, int a_is_km, int b_is_nk) {
  if (m <= 0 || n <= 0 || k <= 0) return 0;
  if (lda % 8 || ldb % 8) return 0;            // TMA global strides must be multiples of 16 bytes
  // inner (contiguous) extents must also keep 16-byte granularity for the tensor map
  const int a_inner = a_is_km ? m : k, b_inner = b_is_nk ? k : n;
  if (a_inner % 8 || b_inner % 8) return 0;
  (void)ldd;
  return 1;
}

int gemm_tcgen05(const GemmArgs& g, cudaStream_t s) {
  if (!gemm_tcgen05_supported(g.m, g.n, g.k, g.lda, g.ldb, g.ldd, g.a_is_km, g.b_is_nk)) return 1;
  if ((reinterpret_cast<uintptr_t>(g.a) & 15) || (reinterpret_cast<uintptr_t>(g.b) & 15)) return 1;
  if (g.dtype != kBF16 && g.dtype != kF16) return 1;
  // tile-N choice: widest tile that keeps the last wave reasonably full
  const int sms = sm_count();
  const int groups = g.grouped == 2 ? g.groups : (g.batch > 1 ? g.batch : 1);
  auto waves_eff = [&](int bn) {
    const int64_t tiles = (int64_t)((g.m + 127) / 128) * ((g.n + bn - 1) / bn) * groups;
    const int64_t waves = (tiles + sms - 1) / sms;
    return (double)tiles / (double)(waves * sms);
  };
  int bn = 256;
  if (g.n <= 64) bn = 64;
  else if (g.n <= 128) bn = 128;
  else if (waves_eff(256) < 0.75 && waves_eff(128) > waves_eff(256) + 0.08) bn = 128;
  const bool bf = g.dtype == kBF16;
  if (bn == 256) return bf ? gemm::launch_layout<256, true>(g, s) : gemm::launch_layout<256, false>(g, s);
  if (bn == 128) return bf ? gemm::launch_layout<128, true>(g, s) : gemm::launch_layout<128, false>(g, s);
  return bf ? gemm::launch_layout<64, true>(g, s) : gemm::launch_layout<64, false>(g, s);
}

}  // namespace b200
