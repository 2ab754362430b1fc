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
#include <cuda.h>
#include <cstdio>
#include <string>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace attn {
using namespace ptx;

constexpr int BM = 128, BN = 128, HD = 128;
constexpr int kThreads = 288;   // warps 0-7: two MMA / softmax warpgroups, warp 8: TMA producer
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

// MASKED: column-wise row-range mask (flashmask / varlen) compiled in; the dense instantiation carries none of its code or registers
template <typename T, bool MASKED>
__global__ void __launch_bounds__(kThreads, 1)
fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
           const __grid_constant__ CUtensorMap map_v, const Params p) {
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
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
  const int m_tile = (int)gridDim.x - 1 - (int)blockIdx.x;   // long (late) rows first under the causal mask
  const int head = blockIdx.y, batch = blockIdx.z;
  const int kv_head = head / (p.h / p.hk);
  const int m0 = m_tile * BM;
  int n_tiles = (p.sk + BN - 1) / BN;
  if (p.causal) {
    const int last_key = min(p.sk - 1, m0 + BM - 1 + p.causal_off);
    n_tiles = last_key < 0 ? 0 : min(n_tiles, last_key / BN + 1);
  }

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(k_full(s), 1); mbar_init(v_full(s), 1); mbar_init(k_empty(s), 8); mbar_init(v_empty(s), 8); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0 && n_tiles > 0) {
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
      const bool edge = (j * BN + BN > p.sk) || (p.causal && j * BN + BN - 1 > m0 + p.causal_off);
      if (edge) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + rl + h * 8;
          const int lim = (p.causal ? min(p.sk - 1, row + p.causal_off) : p.sk - 1) - j * BN;   // last visible key, tile-relative
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
        float m_new = fmaxf(m_i[h], mx * p.scale_log2);     // scale > 0
        if (m_new == -INFINITY) m_new = 0.f;                // fully masked so far: keep exp2 finite
        const float alpha = ex2(m_i[h] - m_new);
        m_i[h] = m_new;
        float sum = 0.f;
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pv = ex2(fmaf(sv[jn * 4 + h * 2 + e], p.scale_log2, -m_new));
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
      const float inv = l > 0.f ? 1.f / l : 0.f;
      const int row = m0 + rl + h * 8;
      if (row < p.sq) {
        T* orow = reinterpret_cast<T*>(p.o) + (int64_t)batch * p.o_sb + (int64_t)row * p.o_ss + (int64_t)head * p.o_sh;
#pragma unroll
        for (int jn = 0; jn < HD / 8; ++jn)
          *reinterpret_cast<uint32_t*>(orow + jn * 8 + 2 * q) = pack2<T>(o_acc[jn * 4 + h * 2] * inv, o_acc[jn * 4 + h * 2 + 1] * inv);
        if (q == 0 && p.lse) p.lse[((int64_t)batch * p.h + head) * p.sq + row] = l > 0.f ? (m_i[h] + log2f(l)) * 0.69314718055994531f : -INFINITY;
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

}  // namespace b200
