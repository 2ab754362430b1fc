// FP8 (E4M3 / E5M2) GEMM for sm_90a: same persistent warp-specialised structure as gemm_sm100.cu (TMA -> 128B-swizzled smem ring ->
// wgmma.mma_async from two consumer warpgroups -> register epilogue), with fp8 MMAs (K = 32 per instruction, 2x the bf16 rate), fp32
// accumulation and a per-tensor dequantisation scale (+ bias / activation) fused in the epilogue.  Both operands are K-major ("TN"
// GEMM): A [M,K], B [N,K], 1 byte per element.
//
// MX variant (`MX = true`, BN = 128): OCP microscaling - one E8M0 (power-of-two) scale per 32 consecutive K elements of every A row
// and B row.  The scale bytes travel as 512-byte blocks (128 rows x 4 k-blocks, byte = (row % 32) * 16 + (row / 32) * 4 + k-block), one
// bulk copy per operand and stage.  Hopper's MMA has no block-scale input, so every 32-wide k-block is multiplied into a scratch
// accumulator and added to the running one as acc += scratch * 2^sfa[row] * 2^sfb[col] in registers: exact (powers of two), one pass,
// and the other warpgroup's MMAs run under this warpgroup's scaling.
//
// Parity (behaviour): fp8_fp8_half_gemm_fused (paddle/phi/kernels/fusion/fp8_gemm/fp8_gemm_with_cublasLt/*) which calls cuBLASLt.
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace gemm8 {
using namespace ptx;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 128;  // 128 x 1B = 128B = one swizzle atom row
constexpr int MMA_K = 32;     // 32 fp8 elements (32 bytes) per MMA along K
constexpr int kStages = 4;
constexpr int kThreads = 384; // producer warpgroup + two MMA warpgroups (64 rows each)
constexpr int kConsumerWarps = 8;
constexpr uint32_t A_STAGE_BYTES = BLOCK_M * BLOCK_K;      // 16 KB

constexpr uint32_t SF_BLOCK_BYTES = 512;   // scale bytes of 128 rows x 128 k (4 blocks of 32)

template <int BN, bool MX = false> struct Cfg {
  static constexpr uint32_t B_STAGE_BYTES = BN * BLOCK_K;
  static constexpr uint32_t SF_BYTES = MX ? 1024u : 0u;          // [SFA 512 | SFB 512] behind the operand tiles
  static constexpr uint32_t SF_TX = MX ? 2 * SF_BLOCK_BYTES : 0u;
  static constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES + SF_BYTES;
  static constexpr uint32_t TX_BYTES = A_STAGE_BYTES + B_STAGE_BYTES + SF_TX;
  static constexpr uint32_t SMEM_BYTES = kStages * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(BN == 128, "one 128-column scale block per stage; scratch + running accumulators of a wider tile would not fit in registers");
  static_assert(SMEM_BYTES <= 232448, "fp8 gemm: shared memory budget");
};

struct Params {
  int m, n, k, batch;
  void* d;
  const void* bias;
  int64_t ldd, stride_d;
  int out_dtype;
  int has_bias, act;
  float scale;
  const float* scale_a;   // optional device scalars (per-tensor dequantisation factors produced by quantize_fp8): no host round trip
  const float* scale_b;
  const uint8_t* sfa;     // MX: E8M0 scale blocks [m / 128][k / 128][512] of A, same for B over n
  const uint8_t* sfb;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float e8m0(uint32_t byte) { return __uint_as_float(byte << 23); }   // 2^(byte - 127)
__device__ __forceinline__ uint32_t ld_shared_u8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

template <typename TO>
__device__ __forceinline__ void store_pair(TO* __restrict__ dst, float v0, float v1, int valid) {
  if (valid >= 2 && (reinterpret_cast<uintptr_t>(dst) & (2 * sizeof(TO) - 1)) == 0) {
    struct alignas(2 * sizeof(TO)) Pair { TO a, b; };
    Pair o;
    o.a = from_f<TO>(v0);
    o.b = from_f<TO>(v1);
    *reinterpret_cast<Pair*>(dst) = o;
  } else {
    if (valid >= 1) dst[0] = from_f<TO>(v0);
    if (valid >= 2) dst[1] = from_f<TO>(v1);
  }
}

template <int BN, bool A5, bool B5, bool MX>
__global__ void __launch_bounds__(kThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const Params p) {
  using C = Cfg<BN, MX>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B needs 1024B alignment
  const uint32_t bar_base = smem_base + kStages * C::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_m = (p.m + BLOCK_M - 1) / BLOCK_M, num_n = (p.n + BN - 1) / BN;
  const int tiles_per_batch = num_m * num_n;
  const int num_tiles = tiles_per_batch * p.batch;
  const int num_kb = (p.k + BLOCK_K - 1) / BLOCK_K;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
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
        const int m0 = mb * BLOCK_M, n0 = nb * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(full_bar(stage), C::TX_BYTES);
          const int k0 = kb * BLOCK_K;
          tma_load_3d(sa, &map_a, full_bar(stage), k0, m0, bz, hint);  // box {128 k bytes, 128 m}
          tma_load_3d(sb, &map_b, full_bar(stage), k0, n0, bz, hint);  // box {128 k bytes, BN n}
          if constexpr (MX) {
            bulk_load(sb + C::B_STAGE_BYTES, p.sfa + ((int64_t)mb * num_kb + kb) * SF_BLOCK_BYTES, SF_BLOCK_BYTES, full_bar(stage));
            bulk_load(sb + C::B_STAGE_BYTES + SF_BLOCK_BYTES, p.sfb + ((int64_t)nb * num_kb + kb) * SF_BLOCK_BYTES, SF_BLOCK_BYTES, full_bar(stage));
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================= MMA + epilogue: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =================
    reg_alloc<224>();
    const int wg = (warp >> 2) - 1, ww = warp & 3;
    const int rl = wg * 64 + ww * 16 + (lane >> 2);     // first of this thread's two tile rows (the other is rl + 8)
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    const float dq = p.scale * (p.scale_a ? *p.scale_a : 1.f) * (p.scale_b ? *p.scale_b : 1.f);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int bz, mb, nb;
      tile_coords(tile, bz, mb, nb);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      if constexpr (!MX) {
        // The tensor core keeps fewer mantissa bits than fp32 while it accumulates fp8 products, which shows after a few thousand k:
        // every 128-wide k-block is summed by the MMA into a scratch fragment and added to the running sum in fp32 registers.
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(full_bar(stage), phase);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES + wg * 8192, sb = smem_base + stage * C::STAGE_BYTES + A_STAGE_BYTES;
          float t[BN / 2];
          wgmma_fence_regs(t);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BLOCK_K / MMA_K; ++k)      // K-major: 32 fp8 elements = 32 B per step inside the swizzle row
            wgmma_f8_n128<A5, B5>(t, make_smem_desc(sa + k * 32, 16, 1024), make_smem_desc(sb + k * 32, 16, 1024), k != 0);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(t);
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(stage));
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += t[i];
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      } else {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(full_bar(stage), phase);
          const uint32_t sa = smem_base + stage * C::STAGE_BYTES + wg * 8192, sb = smem_base + stage * C::STAGE_BYTES + A_STAGE_BYTES;
          const uint32_t sfa = sb + C::B_STAGE_BYTES, sfb = sfa + SF_BLOCK_BYTES;
#pragma unroll 1
          for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
            float t[BN / 2];
            wgmma_fence_regs(t);
            wgmma_fence();
            wgmma_f8_n128<A5, B5>(t, make_smem_desc(sa + k * 32, 16, 1024), make_smem_desc(sb + k * 32, 16, 1024), 0);
            wgmma_commit();
            // this thread's two row scales and, per 8-column group, two column scales of k-block k
            const float ra0 = e8m0(ld_shared_u8(sfa + (rl & 31) * 16 + (rl >> 5) * 4 + k));
            const float ra1 = e8m0(ld_shared_u8(sfa + ((rl + 8) & 31) * 16 + ((rl + 8) >> 5) * 4 + k));
            wgmma_wait<0>();
            wgmma_fence_regs(t);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int c = j * 8 + (lane & 3) * 2;
              const float cb0 = e8m0(ld_shared_u8(sfb + (c & 31) * 16 + (c >> 5) * 4 + k));
              const float cb1 = e8m0(ld_shared_u8(sfb + ((c + 1) & 31) * 16 + ((c + 1) >> 5) * 4 + k));
              acc[j * 4 + 0] = fmaf(t[j * 4 + 0], ra0 * cb0, acc[j * 4 + 0]);
              acc[j * 4 + 1] = fmaf(t[j * 4 + 1], ra0 * cb1, acc[j * 4 + 1]);
              acc[j * 4 + 2] = fmaf(t[j * 4 + 2], ra1 * cb0, acc[j * 4 + 2]);
              acc[j * 4 + 3] = fmaf(t[j * 4 + 3], ra1 * cb1, acc[j * 4 + 3]);
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(empty_bar(stage));
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }

      // ---- epilogue from the accumulator fragment ----
      const int r0 = mb * BLOCK_M + rl;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = nb * BN + j * 8 + (lane & 3) * 2;
        const int valid = p.n - col;
        if (valid <= 0) continue;
        float b0 = 0.f, b1 = 0.f;
        if (p.has_bias) {
          if (p.out_dtype == kBF16) {
            const __nv_bfloat16* b = (const __nv_bfloat16*)p.bias + col;
            b0 = __bfloat162float(b[0]);
            if (valid > 1) b1 = __bfloat162float(b[1]);
          } else if (p.out_dtype == kF16) {
            const __half* b = (const __half*)p.bias + col;
            b0 = __half2float(b[0]);
            if (valid > 1) b1 = __half2float(b[1]);
          } else {
            const float* b = (const float*)p.bias + col;
            b0 = b[0];
            if (valid > 1) b1 = b[1];
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r0 + h * 8;
          float v0 = acc[j * 4 + h * 2] * dq + b0, v1 = acc[j * 4 + h * 2 + 1] * dq + b1;   // per-tensor dequantisation scale (scale_a * scale_b)
          if (p.act == 1) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
          else if (p.act == 2) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          if (row < p.m) {
            const int64_t off = (int64_t)bz * p.stride_d + (int64_t)row * p.ldd + col;
            if (p.out_dtype == kBF16) store_pair((__nv_bfloat16*)p.d + off, v0, v1, valid);
            else if (p.out_dtype == kF16) store_pair((__half*)p.d + off, v0, v1, valid);
            else store_pair((float*)p.d + off, v0, v1, valid);
          }
        }
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
// 3-D byte map {k (contiguous), rows, batch}
static bool make_map8(CUtensorMap* out, const void* ptr, uint64_t k, uint64_t rows, uint64_t batch, uint64_t ld, uint64_t bstride, uint32_t box_rows) {
  bind_primary_context();
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_last_error(__FILE__, __LINE__, "cuTensorMapEncodeTiled unavailable"); return false; }
  cuuint64_t dims[3] = {k, rows, batch};
  cuuint64_t strides[2] = {ld, batch > 1 ? bstride : rows * ld};
  cuuint32_t box[3] = {(cuuint32_t)BLOCK_K, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error(__FILE__, __LINE__, ("cuTensorMapEncodeTiled (fp8) failed: " + std::to_string((int)r)).c_str());
    return false;
  }
  return true;
}
template <int BN, bool A5, bool B5, bool MX>
static int launch(const GemmFp8Args& g, cudaStream_t s) {
  using C = Cfg<BN, MX>;
  CUtensorMap ma, mb;
  const uint64_t batch = g.batch > 1 ? g.batch : 1;
  if (!make_map8(&ma, g.a, g.k, g.m, batch, g.lda, g.stride_a, BLOCK_M)) return 2;
  if (!make_map8(&mb, g.b, g.k, g.n, batch, g.ldb, g.stride_b, BN)) return 2;
  Params p;
  p.m = g.m; p.n = g.n; p.k = g.k; p.batch = (int)batch;
  p.d = g.d; p.bias = g.bias; p.ldd = g.ldd; p.stride_d = g.stride_d;
  p.out_dtype = g.out_dtype;
  p.has_bias = g.bias ? 1 : 0;
  p.act = g.act;
  p.scale = g.scale;
  p.scale_a = g.scale_a_dev; p.scale_b = g.scale_b_dev;
  p.sfa = g.sfa; p.sfb = g.sfb;
  static bool attr_set = false;
  auto kern = gemm_fp8_kernel<BN, A5, B5, MX>;
  if (!attr_set) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  const int num_tiles = ((g.m + BLOCK_M - 1) / BLOCK_M) * ((g.n + BN - 1) / BN) * (int)batch;
  const int grid = num_tiles < sm_count() ? num_tiles : sm_count();
  kern<<<grid, kThreads, C::SMEM_BYTES, s>>>(ma, mb, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

template <int BN, bool MX>
static int launch_types(const GemmFp8Args& g, cudaStream_t s) {
  if (g.a_e5m2) return g.b_e5m2 ? launch<BN, true, true, MX>(g, s) : launch<BN, true, false, MX>(g, s);
  return g.b_e5m2 ? launch<BN, false, true, MX>(g, s) : launch<BN, false, false, MX>(g, s);
}

}  // namespace gemm8

int gemm_fp8_tcgen05(const GemmFp8Args& g, cudaStream_t s) {
  if (g.m <= 0 || g.n <= 0 || g.k <= 0 || g.k % 16 || g.lda % 16 || g.ldb % 16) return 1;   // TMA strides: multiples of 16 bytes
  if ((reinterpret_cast<uintptr_t>(g.a) | reinterpret_cast<uintptr_t>(g.b)) & 15) return 1;
  if (g.sfa || g.sfb) {
    // MX: whole 128 x 128 x 128 scale blocks only
    if (!g.sfa || !g.sfb || g.m % 128 || g.n % 128 || g.k % 128 || g.batch > 1) return 1;
    if ((reinterpret_cast<uintptr_t>(g.sfa) | reinterpret_cast<uintptr_t>(g.sfb)) & 15) return 1;
    return gemm8::launch_types<128, true>(g, s);
  }
  return gemm8::launch_types<128, false>(g, s);
}

}  // namespace b200
