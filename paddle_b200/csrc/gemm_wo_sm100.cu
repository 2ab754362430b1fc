// Weight-only quantised GEMM for sm_90a: out[M,N] = x[M,K] (bf16 / fp16) @ dequant(Wq[N,K] int8 | int4) * scale[N] (+ bias), M <= 64.
//
// The int8 / int4 weights never exist as 16-bit values in HBM or in shared memory: TMA streams raw [128 channels x 128 B] boxes into a
// ring, the two MMA warpgroups expand them IN REGISTERS straight into the A-operand fragment layout of wgmma (A from registers, B =
// the activation tile in shared memory).  The problem is computed transposed (D^T[N, M] = W[N, K] x^T) so that the weight tile is the
// 64-row A operand of each warpgroup even when M is a handful of decode tokens, the per-channel scale is a per-thread scalar in the
// epilogue (accumulator row = output channel), and the token tile (MMA N = 16 / 64) only costs what the batch needs.  Narrow layers
// are split along K over a thread-block CLUSTER whose CTAs reduce their partial tiles through DSMEM - no workspace, no atomics, no
// second kernel.
//
// Parity: paddle/phi/kernels/gpu/weight_only_linear_kernel.cu:27, python/paddle/nn/quant/quantized_linear.py:183.
#include <cuda.h>
#include <cstdio>
#include <string>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace gemm {
bool make_map(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows, uint64_t batch, uint64_t ld, uint64_t bstride,
              uint32_t box_inner, uint32_t box_rows, int dtype);
}
namespace wo {
using namespace ptx;

constexpr int BLOCK_N = 128;     // output channels per CTA: 64 per MMA warpgroup
constexpr int BLOCK_K = 64;
constexpr int kThreads = 288;    // warps 0-7: two MMA warpgroups (dequantise + wgmma + epilogue), warp 8: TMA producer
constexpr uint32_t W_BYTES = BLOCK_N * 128;   // 16 KB raw box

struct Params {
  int m, n, k;                 // tokens, output channels, reduction
  int kb_per_split;            // 64-wide k-blocks handled by one blockIdx.y
  const float* scale;          // [n] per-channel dequantisation factors
  const void* bias;            // [n] in the activation dtype or nullptr
  void* out;                   // [m, n] activation dtype (splits == 1)
  int splits;                  // blockIdx.y extent = cluster size: the CTAs of one output tile
};

template <bool BF16> __device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (BF16) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  } else {
    const __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  }
}
__device__ __forceinline__ uint32_t ld_shared_u16(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t ld_shared_u8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// two consecutive k of one channel -> one packed 16-bit pair in the activation dtype (|value| <= 128: exact in bf16 and fp16)
template <bool INT4, bool BF16> __device__ __forceinline__ uint32_t dequant_pair(uint32_t raw) {
  if constexpr (INT4) return pack2<BF16>((float)((int)((raw & 0xFu) ^ 8u) - 8), (float)((int)(((raw >> 4) & 0xFu) ^ 8u) - 8));   // low nibble = even k
  else return pack2<BF16>((float)(int8_t)(raw & 0xFFu), (float)(int8_t)((raw >> 8) & 0xFFu));
}
__device__ __forceinline__ void keep_regs(uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// NTOK: token tile (MMA N).  INT4: two weights per byte (low nibble = even k).
//
// Data path of one 64-wide k-block:  TMA raw box (128 channels x 128 B, shared by 2 int8 / 4 int4 k-blocks) + the activation tiles of
// those k-blocks in one ring stage -> every MMA thread reads exactly the bytes of its own A-fragment elements (rows lane / 4 and + 8 of
// its warp's 16 channels, k = 2 (lane % 4) .. + 1 and + 8 of each 16-wide step), converts them and issues wgmma with A in registers ->
// D^T[64 channels, NTOK tokens] += A x_tile^T.  The dequantised weights never touch shared memory.
template <int NTOK, int WST, bool INT4, bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
wo_gemm_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, const Params p) {
  constexpr int KB_PER_W = INT4 ? 4 : 2;                        // k-blocks covered by one raw box
  constexpr uint32_t X_BYTES = NTOK * BLOCK_K * 2;
  constexpr uint32_t STAGE_BYTES = W_BYTES + KB_PER_W * X_BYTES;
  static_assert(NTOK * 512 <= WST * STAGE_BYTES, "weight-only gemm: the split-K partial tile is staged in the ring");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bars = base + WST * STAGE_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (WST + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BLOCK_N;
  const int tok0 = blockIdx.z * NTOK;
  const int num_kb_total = (p.k + BLOCK_K - 1) / BLOCK_K;
  const int kb0 = blockIdx.y * p.kb_per_split;
  const int num_kb = max(0, min(p.kb_per_split, num_kb_total - kb0));
  const int num_box = (num_kb + KB_PER_W - 1) / KB_PER_W;    // kb0 is a multiple of KB_PER_W (launcher), so boxes start on 128-byte columns

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&map_w);
    tma_prefetch_desc(&map_x);
    for (int s = 0; s < WST; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // ================= TMA producer: one raw weight box and the activation tiles of its k-blocks per stage =================
      for (int j = 0; j < num_box; ++j) {
        const int st = j % WST;
        const int nvalid = min(KB_PER_W, num_kb - j * KB_PER_W);
        mbar_wait(empty(st), ((j / WST) & 1) ^ 1);
        mbar_expect_tx(full(st), W_BYTES + nvalid * X_BYTES);
        const uint32_t sw = base + st * STAGE_BYTES;
        tma_load_2d(sw, &map_w, full(st), (kb0 + j * KB_PER_W) * (INT4 ? BLOCK_K / 2 : BLOCK_K), n0);
        for (int sub = 0; sub < nvalid; ++sub)
          tma_load_3d(sw + W_BYTES + sub * X_BYTES, &map_x, full(st), (kb0 + j * KB_PER_W + sub) * BLOCK_K, tok0, 0);
      }
    }
  } else {
    // ================= MMA warpgroups: dequantise into the A fragment, D^T[64 channels, NTOK tokens] += A x_tile^T =================
    const int wg = warp >> 2, q = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // channel rows r0 and r0 + 8 of the tile ((r0 + 8) & 7 == r0 & 7)
    float acc[NTOK / 2];
#pragma unroll
    for (int i = 0; i < NTOK / 2; ++i) acc[i] = 0.f;
    for (int j = 0; j < num_box; ++j) {
      const int st = j % WST;
      const int nvalid = min(KB_PER_W, num_kb - j * KB_PER_W);
      mbar_wait(full(st), (j / WST) & 1);
      const uint32_t sw = base + st * STAGE_BYTES;
      const uint32_t row0 = sw + r0 * 128, row1 = row0 + 8 * 128;   // 128 rows x 128 B, SWIZZLE_128B: 16-byte piece c of row r sits at piece c ^ (r & 7)
      const uint32_t sx = r0 & 7;
#pragma unroll
      for (int sub = 0; sub < KB_PER_W; ++sub) {
        if (sub < nvalid) {
          uint32_t a[4][4];
#pragma unroll
          for (int s = 0; s < 4; ++s) {       // 16-wide k-step s of this k-block
            if constexpr (!INT4) {            // piece = 16 k = 16 bytes
              const uint32_t off = (((uint32_t)(sub * 4 + s) ^ sx) << 4) + 2 * q;
              a[s][0] = dequant_pair<false, BF16>(ld_shared_u16(row0 + off));
              a[s][1] = dequant_pair<false, BF16>(ld_shared_u16(row1 + off));
              a[s][2] = dequant_pair<false, BF16>(ld_shared_u16(row0 + off + 8));
              a[s][3] = dequant_pair<false, BF16>(ld_shared_u16(row1 + off + 8));
            } else {                          // piece = 32 k = 16 bytes: step s is its half s & 1, byte c = (k = 2c, k = 2c + 1)
              const uint32_t off = (((uint32_t)(sub * 2 + (s >> 1)) ^ sx) << 4) + (s & 1) * 8 + q;
              a[s][0] = dequant_pair<true, BF16>(ld_shared_u8(row0 + off));
              a[s][1] = dequant_pair<true, BF16>(ld_shared_u8(row1 + off));
              a[s][2] = dequant_pair<true, BF16>(ld_shared_u8(row0 + off + 4));
              a[s][3] = dequant_pair<true, BF16>(ld_shared_u8(row1 + off + 4));
            }
          }
          const uint32_t xs = sw + W_BYTES + sub * X_BYTES;
          wgmma_fence_regs(acc);
          wgmma_fence();
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            const uint64_t bdesc = make_smem_desc(xs + s * 32, 16, 1024);
            if constexpr (NTOK == 16) wgmma_rs_n16<BF16, 0>(acc, a[s], bdesc, 1);
            else wgmma_rs_n64<BF16, 0>(acc, a[s], bdesc, 1);
          }
          wgmma_commit();
          wgmma_wait<0>();                    // the fragment registers are read asynchronously: they stay untouched until the MMAs retire
          wgmma_fence_regs(acc);
#pragma unroll
          for (int s = 0; s < 4; ++s) keep_regs(a[s]);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(st));
    }
    // ---- epilogue: accumulator row = output channel, column = token ----
    if (p.splits > 1) {
      // split-K inside a cluster: park the partial tile [token][channel] in this CTA's shared memory (the ring is idle once BOTH
      // warpgroups have consumed their last box); the cluster reduces it below through DSMEM
      named_bar_sync(1, 256);
#pragma unroll
      for (int jn = 0; jn < NTOK / 8; ++jn)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int tok = jn * 8 + 2 * q + (e & 1), chl = r0 + (e >> 1) * 8;
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + (uint32_t)((tok * BLOCK_N + chl) * 4)), "f"(acc[jn * 4 + e]) : "memory");
        }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ch = n0 + r0 + h * 8;
        if (ch >= p.n) continue;
        const float sc = p.scale[ch];
        float bv = 0.f;
        if (p.bias) bv = BF16 ? __bfloat162float(((const __nv_bfloat16*)p.bias)[ch]) : __half2float(((const __half*)p.bias)[ch]);
#pragma unroll
        for (int jn = 0; jn < NTOK / 8; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int tok = tok0 + jn * 8 + 2 * q + e;
            if (tok >= p.m) continue;
            const float y = acc[jn * 4 + h * 2 + e] * sc + bv;
            if constexpr (BF16) ((__nv_bfloat16*)p.out)[(int64_t)tok * p.n + ch] = __float2bfloat16_rn(y);
            else ((__half*)p.out)[(int64_t)tok * p.n + ch] = __float2half_rn(y);
          }
      }
    }
  }
  if (p.splits > 1) {
    // ---- cluster reduction: the p.splits CTAs of a cluster hold the partial tiles of ONE output tile; CTA r sums 32-channel chunks
    // r, r + splits, ... over all ranks (ld.shared::cluster) and writes the scaled result.  No workspace, no atomics, no second kernel.
    cluster_sync();
    if (warp >= 4 && warp < 8) {
      uint32_t rank;
      asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
      const int tok_n = min(NTOK, p.m - tok0);
      for (int c = (int)rank * 4 + (warp - 4); c < tok_n * 4; c += p.splits * 4) {
        const int tok = c >> 2, chl = (c & 3) * 32 + lane, ch = n0 + chl;
        float acc = 0.f;
        const uint32_t local = base + (uint32_t)((tok * BLOCK_N + chl) * 4);
        for (int qq = 0; qq < p.splits; ++qq) {
          uint32_t remote;
          float v;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(qq));
          asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
          acc += v;
        }
        if (ch < p.n) {
          float y = acc * p.scale[ch];
          if (p.bias) y += BF16 ? __bfloat162float(((const __nv_bfloat16*)p.bias)[ch]) : __half2float(((const __half*)p.bias)[ch]);
          if constexpr (BF16) ((__nv_bfloat16*)p.out)[(int64_t)(tok0 + tok) * p.n + ch] = __float2bfloat16_rn(y);
          else ((__half*)p.out)[(int64_t)(tok0 + tok) * p.n + ch] = __float2half_rn(y);
        }
      }
    }
    cluster_sync();                                        // nobody leaves while a peer may still read its partial tile
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
  }
  return fn;
}
// raw weights as bytes: [n rows, row_bytes], box {128 bytes, 128 rows}, SWIZZLE_128B
static bool make_w_map(CUtensorMap* out, const void* w, int n, int row_bytes) {
  bind_primary_context();
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_last_error(__FILE__, __LINE__, "cuTensorMapEncodeTiled unavailable"); return false; }
  cuuint64_t dims[2] = {(cuuint64_t)row_bytes, (cuuint64_t)n};
  cuuint64_t strides[1] = {(cuuint64_t)row_bytes};
  cuuint32_t box[2] = {128u, (cuuint32_t)BLOCK_N};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error(__FILE__, __LINE__, ("weight-only gemm: cuTensorMapEncodeTiled failed: " + std::to_string((int)r)).c_str()); return false; }
  return true;
}

template <int NTOK, int WST, bool INT4, bool BF16>
static int launch(const WoGemmArgs& g, const CUtensorMap& mw, cudaStream_t s) {
  constexpr int KB_PER_W = INT4 ? 4 : 2;
  constexpr uint32_t SMEM = WST * (W_BYTES + KB_PER_W * NTOK * BLOCK_K * 2) + 1024 + 256;
  static_assert(SMEM <= 232448, "weight-only gemm: shared memory budget");
  static_assert(8 * 2 * WST <= 256, "weight-only gemm: barrier area");
  constexpr int kMaxSplits = 8;                 // portable cluster size
  CUtensorMap mx;
  if (!gemm::make_map(&mx, g.x, g.k, g.m, 1, g.k, 0, BLOCK_K, NTOK, g.bf16 ? kBF16 : kF16)) return 2;
  auto kern = wo_gemm_kernel<NTOK, WST, INT4, BF16>;
  static bool attr_set = false;
  static int wave_ctas[kMaxSplits + 1];         // CTAs the device holds at once when they come in clusters of `splits`
  if (!attr_set) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    for (int c = 1; c <= kMaxSplits; ++c) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(1, c, 1); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = SMEM;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = c; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      int n_clusters = 0;
      if (cudaOccupancyMaxActiveClusters(&n_clusters, kern, &cfg) != cudaSuccess) { cudaGetLastError(); n_clusters = 0; }
      wave_ctas[c] = n_clusters * c;
    }
    if (wave_ctas[1] <= 0) wave_ctas[1] = sm_count();
    attr_set = true;
  }
  Params p;
  p.m = g.m; p.n = g.n; p.k = g.k;
  const int num_kb = (g.k + BLOCK_K - 1) / BLOCK_K;
  const int n_tiles = (g.n + BLOCK_N - 1) / BLOCK_N, t_tiles = (g.m + NTOK - 1) / NTOK;
  // Split-K (a cluster of `splits` CTAs per output tile) when the output tiles alone leave SMs idle or the last wave ragged.  Cost in
  // k-block units: waves x (k-blocks per CTA + fixed prologue / epilogue) + the cluster reduction.
  const int ctas = n_tiles * t_tiles;
  int splits = 1, kb_per = (num_kb + 3) / 4 * 4;
  long best = -1;
  for (int c = 1; c <= kMaxSplits; ++c) {
    if (wave_ctas[c] <= 0) continue;
    const int per = ((num_kb + c - 1) / c + 3) / 4 * 4;           // raw boxes span up to 4 k-blocks: split boundaries stay on box boundaries
    if (c > 1 && (c - 1) * per >= num_kb) continue;               // every rank of the cluster gets work
    const long waves = ((long)ctas * c + wave_ctas[c] - 1) / wave_ctas[c];
    const long cost = waves * (per + 24) + (c > 1 ? 6 : 0);
    if (best < 0 || cost < best) { best = cost; splits = c; kb_per = per; }
  }
  p.splits = splits;
  p.kb_per_split = kb_per;
  p.scale = g.scale; p.bias = g.bias; p.out = g.out;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_tiles, splits, t_tiles); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = SMEM; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = splits; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, mw, mx, p);
  if (e != cudaSuccess) { cudaGetLastError(); set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

template <bool INT4, bool BF16>
static int dispatch_tok(const WoGemmArgs& g, const CUtensorMap& mw, cudaStream_t s) {
  if (g.m <= 16) return launch<16, 8, INT4, BF16>(g, mw, s);      // decode: 128 KB of raw weights in flight
  return launch<64, 4, INT4, BF16>(g, mw, s);
}

}  // namespace wo

int gemm_weight_only(const WoGemmArgs& g, cudaStream_t s) {
  using namespace wo;
  if (g.k % 64 || g.n % 8 || g.m <= 0 || g.m > 64) return 1;      // larger batches: dequantise once + the bf16 GEMM (nn/quant.py)
  if ((reinterpret_cast<uintptr_t>(g.x) | reinterpret_cast<uintptr_t>(g.w) | reinterpret_cast<uintptr_t>(g.out)) & 15) return 1;
  CUtensorMap mw;
  const int row_bytes = g.int4 ? g.k / 2 : g.k;
  if (!make_w_map(&mw, g.w, g.n, row_bytes)) return 2;
  if (g.int4) return g.bf16 ? dispatch_tok<true, true>(g, mw, s) : dispatch_tok<true, false>(g, mw, s);
  return g.bf16 ? dispatch_tok<false, true>(g, mw, s) : dispatch_tok<false, false>(g, mw, s);
}

}  // namespace b200
