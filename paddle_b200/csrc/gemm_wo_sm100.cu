// Weight-only quantised GEMM for sm_90a: out[M,N] = x[M,K] (bf16 / fp16) @ dequant(Wq[N,K] int8 | int4) (+ bias), M <= 64, with per-channel
// scales scale[N] or group-wise scales scale[K / G, N] (G = 64 or 128 consecutive k of one channel share a scale).
//
// The int8 / int4 weights never exist as 16-bit values in HBM or in shared memory: TMA streams raw [128 channels x 128 B] boxes into a
// ring, the two MMA warpgroups expand them IN REGISTERS straight into the A-operand fragment layout of wgmma (A from registers, B =
// the activation tile in shared memory).  The problem is computed transposed (D^T[N, M] = W[N, K] x^T) so that the weight tile is the
// 64-row A operand of each warpgroup even when M is a handful of decode tokens, the per-channel scale is a per-thread scalar in the
// epilogue (accumulator row = output channel), and the token tile (MMA N = 16 / 64) only costs what the batch needs.  Narrow layers
// are split along K over a thread-block CLUSTER whose CTAs reduce their partial tiles through DSMEM - no workspace, no atomics, no
// second kernel.
//
// Group-wise scales: each group's k-blocks accumulate into a separate group accumulator (the group's first wgmma has scale-d = 0); once
// they retire, the thread folds acc += acc_g * s[g][channel] in fp32 (two scales per thread: rows r0 and r0 + 8).  The epilogue and the
// split-K reduction then add only the bias.  A second kernel expands the quantised weight to 16-bit / fp32 in one pass for the batches
// that run the dense GEMM instead.
//
// Parity: paddle/phi/kernels/gpu/weight_only_linear_kernel.cu:27, python/paddle/nn/quant/quantized_linear.py:183.
#include <cuda.h>
#include <cstdio>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_ptx.cuh"

namespace b200 {
namespace wo {
using namespace ptx;

constexpr int BLOCK_N = 128;     // output channels per CTA: 64 per MMA warpgroup
constexpr int BLOCK_K = 64;
constexpr int kThreads = 288;    // warps 0-7: two MMA warpgroups (dequantise + wgmma + epilogue), warp 8: TMA producer
constexpr uint32_t W_BYTES = BLOCK_N * 128;   // 16 KB raw box

struct Params {
  int m, n, k;                 // tokens (experts: rows of xp), output channels, reduction
  int kb_per_split;            // 64-wide k-blocks handled by one blockIdx.y
  const float* scale;          // [n] per-channel or [k / GS, n] group-wise dequantisation factors (experts: [E, ...])
  const void* bias;            // [n] in the activation dtype or nullptr (experts: [E, n])
  void* out;                   // [m, n] activation dtype (splits == 1)
  int splits;                  // blockIdx.y extent = cluster size: the CTAs of one output tile
  const int* offsets;          // experts: [E + 1] first row of every expert
  const int* work;             // experts: [0] item count, then (expert, first row) pairs
};

// two consecutive k of one channel -> one packed 16-bit pair in the activation dtype (|value| <= 128: exact in bf16 and fp16)
template <bool INT4, bool BF16> __device__ __forceinline__ uint32_t dequant_pair(uint32_t raw) {
  using T = std::conditional_t<BF16, __nv_bfloat16, __half>;
  if constexpr (INT4) return pack2<T>((float)((int)((raw & 0xFu) ^ 8u) - 8), (float)((int)(((raw >> 4) & 0xFu) ^ 8u) - 8));   // low nibble = even k
  else return pack2<T>((float)(int8_t)(raw & 0xFFu), (float)(int8_t)((raw >> 8) & 0xFFu));
}
__device__ __forceinline__ void keep_regs(uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// NTOK: token tile (MMA N).  INT4: two weights per byte (low nibble = even k).  GS: scale group size in k (0: per-channel scales).
//
// Data path of one 64-wide k-block:  TMA raw box (128 channels x 128 B, shared by 2 int8 / 4 int4 k-blocks) + the activation tiles of
// those k-blocks in one ring stage -> every MMA thread reads exactly the bytes of its own A-fragment elements (rows lane / 4 and + 8 of
// its warp's 16 channels, k = 2 (lane % 4) .. + 1 and + 8 of each 16-wide step), converts them and issues wgmma with A in registers ->
// D^T[64 channels, NTOK tokens] += A x_tile^T.  The dequantised weights never touch shared memory.
//
// EXPERTS (MoE): out[R, N] = xp[R, K] @ dequant(Wq[e])^T (+ bias[e]) where e owns the row: xp holds the routed slots grouped by expert
// without padding (rows offsets[e] .. offsets[e + 1]) and the weights are stacked [E, N, K].  Each blockIdx.z takes one item of a
// device-built work list of (expert, first row) pairs, one per NTOK-row tile of an expert (moe_wo_plan); the grid's z extent is a static
// bound and CTAs past the real item count exit before anything else.  A cluster's CTAs share blockIdx.z, so they exit together or all
// reach cluster_sync.  Only selected experts' weights, scales and bias are ever read.  Rows of a tile past its expert's last row hold
// other experts' rows or TMA zero fill: they are computed (every token is its own accumulator column) and masked by the epilogue and the
// split-K reduction.
template <int NTOK, int WST, bool INT4, bool BF16, int GS, bool EXPERTS>
__global__ void __launch_bounds__(kThreads, 1)
wo_gemm_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, const Params p) {
  if constexpr (EXPERTS) {
    if ((int)blockIdx.z >= __ldg(p.work)) return;           // uniform over the cluster: every rank has the same blockIdx.z
  }
  constexpr int KB_PER_W = INT4 ? 4 : 2;                        // k-blocks covered by one raw box
  constexpr int KB_PER_G = GS ? GS / BLOCK_K : 1;              // k-blocks per scale group
  constexpr int G_PER_W = GS ? KB_PER_W / KB_PER_G : 1;         // scale groups per raw box
  static_assert(GS == 0 || (GS % BLOCK_K == 0 && KB_PER_W % KB_PER_G == 0), "weight-only gemm: a raw box holds whole scale groups");
  constexpr uint32_t X_BYTES = NTOK * BLOCK_K * 2;
  constexpr uint32_t STAGE_BYTES = W_BYTES + KB_PER_W * X_BYTES;
  static_assert(NTOK * 512 <= WST * STAGE_BYTES, "weight-only gemm: the split-K partial tile is staged in the ring");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bars = base + WST * STAGE_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (WST + s); };

  const int expert = EXPERTS ? __ldg(p.work + 1 + 2 * blockIdx.z) : 0;
  const int tok0 = EXPERTS ? __ldg(p.work + 2 + 2 * blockIdx.z) : blockIdx.z * NTOK;    // first row of this tile in x / out
  const int row_end = EXPERTS ? __ldg(p.offsets + expert + 1) : p.m;                    // rows [tok0, row_end) of the tile are written
  const float* scale = EXPERTS ? p.scale + (int64_t)expert * (GS ? p.k / GS : 1) * p.n : p.scale;
  // written so that both kinds compile to the instructions pinned by tests/golden/wo_gemm_sass.json
  const void* bias = !EXPERTS ? p.bias : (p.bias ? (const void*)((const uint16_t*)p.bias + (int64_t)expert * p.n) : nullptr);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BLOCK_N;
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
        const int kx = (kb0 + j * KB_PER_W) * (INT4 ? BLOCK_K / 2 : BLOCK_K);
        if constexpr (EXPERTS) tma_load_3d(sw, &map_w, full(st), kx, n0, expert);
        else tma_load_2d(sw, &map_w, full(st), kx, n0);
        for (int sub = 0; sub < nvalid; ++sub)
          tma_load_3d(sw + W_BYTES + sub * X_BYTES, &map_x, full(st), (kb0 + j * KB_PER_W + sub) * BLOCK_K, tok0, 0);
      }
    }
  } else {
    // ================= MMA warpgroups: dequantise into the A fragment, D^T[64 channels, NTOK tokens] += A x_tile^T =================
    const int wg = warp >> 2, q = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // channel rows r0 and r0 + 8 of the tile ((r0 + 8) & 7 == r0 & 7)
    float acc[NTOK / 2], acc_g[NTOK / 2];                      // acc_g: the current scale group (group-wise scales only)
#pragma unroll
    for (int i = 0; i < NTOK / 2; ++i) acc[i] = acc_g[i] = 0.f;
    for (int j = 0; j < num_box; ++j) {
      const int st = j % WST;
      const int nvalid = min(KB_PER_W, num_kb - j * KB_PER_W);
      float gsc[G_PER_W][2];                                     // this box's group scales of rows r0 and r0 + 8
      if constexpr (GS > 0) {
        // boxes start on multiples of 4 k-blocks (256 k), so they hold whole groups; read the scales before the wait to hide the loads
        const int g0 = (kb0 + j * KB_PER_W) / KB_PER_G;
#pragma unroll
        for (int gi = 0; gi < G_PER_W; ++gi)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int g = g0 + gi, ch = n0 + r0 + h * 8;
            gsc[gi][h] = (g * GS < p.k && ch < p.n) ? __ldg(scale + (int64_t)g * p.n + ch) : 0.f;
          }
      }
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
          if constexpr (GS == 0) {
            wgmma_fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 4; ++s) {
              const uint64_t bdesc = make_smem_desc(xs + s * 32, 16, 1024);
              if constexpr (NTOK == 16) wgmma_rs_n16<BF16, 0>(acc, a[s], bdesc, 1);
              else wgmma_rs_n64<BF16, 0>(acc, a[s], bdesc, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();                  // the fragment registers are read asynchronously: they stay untouched until the MMAs retire
            wgmma_fence_regs(acc);
#pragma unroll
            for (int s = 0; s < 4; ++s) keep_regs(a[s]);
          } else {
            // the group's first k-block overwrites acc_g (scale-d = 0); its last one folds acc_g into acc with the group's scales
            wgmma_fence_regs(acc_g);
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 4; ++s) {
              const uint64_t bdesc = make_smem_desc(xs + s * 32, 16, 1024);
              const uint32_t accumulate = (s == 0 && sub % KB_PER_G == 0) ? 0u : 1u;
              if constexpr (NTOK == 16) wgmma_rs_n16<BF16, 0>(acc_g, a[s], bdesc, accumulate);
              else wgmma_rs_n64<BF16, 0>(acc_g, a[s], bdesc, accumulate);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc_g);
#pragma unroll
            for (int s = 0; s < 4; ++s) keep_regs(a[s]);
            if (sub % KB_PER_G == KB_PER_G - 1) {   // nvalid is a multiple of KB_PER_G: a group never straddles boxes or splits
#pragma unroll
              for (int i = 0; i < NTOK / 2; ++i) acc[i] = fmaf(acc_g[i], gsc[sub / KB_PER_G][(i >> 1) & 1], acc[i]);
            }
          }
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
        const float sc = GS ? 1.f : scale[ch];              // group-wise scales are already folded into acc
        float bv = 0.f;
        if (bias) bv = BF16 ? __bfloat162float(((const __nv_bfloat16*)bias)[ch]) : __half2float(((const __half*)bias)[ch]);
#pragma unroll
        for (int jn = 0; jn < NTOK / 8; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int tok = tok0 + jn * 8 + 2 * q + e;
            if (tok >= row_end) continue;
            const float y = GS ? acc[jn * 4 + h * 2 + e] + bv : acc[jn * 4 + h * 2 + e] * sc + bv;
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
      const int tok_n = min(NTOK, row_end - tok0);
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
          float y = GS ? acc : acc * scale[ch];
          if (bias) y += BF16 ? __bfloat162float(((const __nv_bfloat16*)bias)[ch]) : __half2float(((const __half*)bias)[ch]);
          if constexpr (BF16) ((__nv_bfloat16*)p.out)[(int64_t)(tok0 + tok) * p.n + ch] = __float2bfloat16_rn(y);
          else ((__half*)p.out)[(int64_t)(tok0 + tok) * p.n + ch] = __float2half_rn(y);
        }
      }
    }
    cluster_sync();                                        // nobody leaves while a peer may still read its partial tile
  }
}

// raw weights as bytes: [n rows, row_bytes], box {128 bytes, 128 rows}, SWIZZLE_128B.  experts > 0: stacked [experts, n rows, row_bytes],
// box {128 bytes, 128 rows, 1 expert}: the same shared-memory layout, and a partial channel tile is zero filled instead of reading the
// next expert's rows
static bool make_w_map(CUtensorMap* out, const void* w, int experts, int n, int row_bytes) {
  const uint64_t dims[3] = {(uint64_t)row_bytes, (uint64_t)n, (uint64_t)experts};
  const uint64_t strides[2] = {(uint64_t)row_bytes, (uint64_t)row_bytes * n};
  const uint32_t box[3] = {128u, (uint32_t)BLOCK_N, 1u};
  return encode_tensor_map(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, experts ? 3 : 2, w, dims, strides, box,
                           experts ? "weight-only expert gemm" : "weight-only gemm");
}

constexpr int kMaxSplits = 8;                   // portable cluster size

// Split-K (a cluster of `splits` CTAs per output tile) when the output tiles alone leave SMs idle or the last wave ragged.  Cost in
// k-block units: waves x (k-blocks per CTA + fixed prologue / epilogue) + the cluster reduction.  wave_ctas[c]: CTAs the device holds at
// once when they come in clusters of c.
static void choose_splits(const int* wave_ctas, int num_kb, int ctas, int* splits, int* kb_per) {
  *splits = 1; *kb_per = (num_kb + 3) / 4 * 4;
  long best = -1;
  for (int c = 1; c <= kMaxSplits; ++c) {
    if (wave_ctas[c] <= 0) continue;
    const int per = ((num_kb + c - 1) / c + 3) / 4 * 4;           // raw boxes span up to 4 k-blocks: split boundaries stay on box boundaries
    if (c > 1 && (c - 1) * per >= num_kb) continue;               // every rank of the cluster gets work
    const long waves = ((long)ctas * c + wave_ctas[c] - 1) / wave_ctas[c];
    const long cost = waves * (per + 24) + (c > 1 ? 6 : 0);
    if (best < 0 || cost < best) { best = cost; *splits = c; *kb_per = per; }
  }
}

// Once per kernel: the dynamic shared memory attribute and wave_ctas[c] for cluster sizes 1 .. kMaxSplits.
template <typename Kern>
static void init_kernel(Kern kern, uint32_t smem, int* wave_ctas) {
  B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  for (int c = 1; c <= kMaxSplits; ++c) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1, c, 1); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = c; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n_clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&n_clusters, kern, &cfg) != cudaSuccess) { cudaGetLastError(); n_clusters = 0; }
    wave_ctas[c] = n_clusters * c;
  }
  if (wave_ctas[1] <= 0) wave_ctas[1] = sm_count();
}

template <typename Kern, typename P>
static int launch_cluster(Kern kern, dim3 grid, uint32_t smem, cudaStream_t s, const CUtensorMap& mw, const CUtensorMap& mx, const P& p) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = grid.y; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, mw, mx, p);
  if (e != cudaSuccess) { cudaGetLastError(); set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

template <int NTOK, int WST, bool INT4>
constexpr uint32_t smem_bytes() { return WST * (W_BYTES + (INT4 ? 4 : 2) * NTOK * BLOCK_K * 2) + 1024 + 256; }

// grid z: the token tiles of g.m rows, or for experts the static work-item bound (g.m / NTOK + min(E, g.m)); the split choice is costed
// on it
template <int NTOK, int WST, bool INT4, bool BF16, int GS, bool EXPERTS>
static int launch(const WoGemmArgs& g, const CUtensorMap& mw, cudaStream_t s) {
  constexpr uint32_t SMEM = smem_bytes<NTOK, WST, INT4>();
  static_assert(SMEM <= 232448, "weight-only gemm: shared memory budget");
  static_assert(8 * 2 * WST <= 256, "weight-only gemm: barrier area");
  CUtensorMap mx;
  if (!gemm::make_map(&mx, g.x, g.k, g.m, 1, g.k, 0, BLOCK_K, NTOK, g.bf16 ? kBF16 : kF16)) return 2;
  auto kern = wo_gemm_kernel<NTOK, WST, INT4, BF16, GS, EXPERTS>;
  static bool attr_set = false;
  static int wave_ctas[kMaxSplits + 1];
  if (!attr_set) { init_kernel(kern, SMEM, wave_ctas); attr_set = true; }
  const int num_kb = (g.k + BLOCK_K - 1) / BLOCK_K;
  const int n_tiles = (g.n + BLOCK_N - 1) / BLOCK_N, items = EXPERTS ? wo_expert_items(g.m, g.experts, NTOK) : (g.m + NTOK - 1) / NTOK;
  if (EXPERTS && items > 65535) { set_last_error(__FILE__, __LINE__, "weight-only expert gemm: too many token tiles"); return 1; }
  int splits, kb_per;
  choose_splits(wave_ctas, num_kb, n_tiles * items, &splits, &kb_per);
  if constexpr (GS > 0) {                                         // the kernel folds whole groups: no split may cut one
    if ((kb_per * BLOCK_K) % GS) { set_last_error(__FILE__, __LINE__, "weight-only gemm: split boundary inside a scale group"); return 3; }
  }
  Params p;
  p.m = g.m; p.n = g.n; p.k = g.k;
  p.kb_per_split = kb_per; p.splits = splits;
  p.scale = g.scale; p.bias = g.bias; p.out = g.out;
  p.offsets = g.offsets; p.work = g.work;
  return launch_cluster(kern, dim3(n_tiles, splits, items), SMEM, s, mw, mx, p);
}

template <bool INT4, bool BF16, int GS, bool EXPERTS>
static int dispatch_tok(const WoGemmArgs& g, const CUtensorMap& mw, cudaStream_t s) {
  if (wo_expert_ntok(g.m) == 16) return launch<16, 8, INT4, BF16, GS, EXPERTS>(g, mw, s);  // decode: 128 KB of raw weights in flight
  return launch<64, 4, INT4, BF16, GS, EXPERTS>(g, mw, s);
}
template <bool INT4, bool BF16, bool EXPERTS>
static int dispatch_group(const WoGemmArgs& g, const CUtensorMap& mw, cudaStream_t s) {
  if (g.group_size == 64) return dispatch_tok<INT4, BF16, 64, EXPERTS>(g, mw, s);
  if (g.group_size == 128) return dispatch_tok<INT4, BF16, 128, EXPERTS>(g, mw, s);
  return dispatch_tok<INT4, BF16, 0, EXPERTS>(g, mw, s);
}
template <bool EXPERTS>
static int dispatch_format(const WoGemmArgs& g, const CUtensorMap& mw, cudaStream_t s) {
  if (g.int4) return g.bf16 ? dispatch_group<true, true, EXPERTS>(g, mw, s) : dispatch_group<true, false, EXPERTS>(g, mw, s);
  return g.bf16 ? dispatch_group<false, true, EXPERTS>(g, mw, s) : dispatch_group<false, false, EXPERTS>(g, mw, s);
}

// One-pass dequantisation for the batches that run the dense GEMM: each CTA reads a [64 channels x 64 k] tile of the quantised weight once
// (along k), turns it around in shared memory and writes [64 k x 64 channels] of out once (along n).  out = float(q) * scale, rounded once
// to OutT: the same value as nn/quant.py's torch expression.  blockIdx.z = expert of a stacked weight [E, n, k] -> [E, k, n].
template <bool INT4, typename OutT>
__global__ void __launch_bounds__(256)
wo_dequant_kernel(const int8_t* __restrict__ w, const float* __restrict__ scale, OutT* __restrict__ out, int n, int k, int group_size) {
  __shared__ float tile[64][65];                             // [k][channel], q as float (exact)
  const int k0 = blockIdx.x * 64, n0 = blockIdx.y * 64, t = threadIdx.x;
  w += (int64_t)blockIdx.z * n * (INT4 ? k / 2 : k);
  scale += (int64_t)blockIdx.z * n * (group_size > 0 ? k / group_size : 1);
  out += (int64_t)blockIdx.z * k * n;
  if constexpr (!INT4) {
    for (int i = t; i < 64 * 64; i += 256) {
      const int nl = i >> 6, kl = i & 63, ch = n0 + nl, kk = k0 + kl;
      tile[kl][nl] = (ch < n && kk < k) ? (float)w[(int64_t)ch * k + kk] : 0.f;
    }
  } else {
    for (int i = t; i < 64 * 32; i += 256) {                 // byte c of a row holds k = 2c (low nibble) and 2c + 1
      const int nl = i >> 5, bl = i & 31, ch = n0 + nl, kk = k0 + 2 * bl;
      const uint32_t raw = (ch < n && kk < k) ? (uint32_t)(uint8_t)w[(int64_t)ch * (k / 2) + kk / 2] : 0u;
      tile[2 * bl][nl] = (float)((int)((raw & 0xFu) ^ 8u) - 8);
      tile[2 * bl + 1][nl] = (float)((int)(((raw >> 4) & 0xFu) ^ 8u) - 8);
    }
  }
  __syncthreads();
  for (int i = t; i < 64 * 64; i += 256) {
    const int kl = i >> 6, nl = i & 63, ch = n0 + nl, kk = k0 + kl;
    if (ch >= n || kk >= k) continue;
    const float v = __fmul_rn(tile[kl][nl], scale[group_size > 0 ? (int64_t)(kk / group_size) * n + ch : ch]);
    OutT* o = out + (int64_t)kk * n + ch;
    if constexpr (std::is_same<OutT, float>::value) *o = v;
    else if constexpr (std::is_same<OutT, __nv_bfloat16>::value) *o = __float2bfloat16_rn(v);
    else *o = __float2half_rn(v);
  }
}

template <bool INT4, typename OutT>
static int launch_dequant(const void* w, const float* scale, void* out, int n, int k, int group_size, int experts, cudaStream_t s) {
  const dim3 grid((k + 63) / 64, (n + 63) / 64, experts);
  wo_dequant_kernel<INT4, OutT><<<grid, 256, 0, s>>>((const int8_t*)w, scale, (OutT*)out, n, k, group_size);
  return B200_LAUNCH_RESULT();
}
template <bool INT4>
static int dispatch_dequant(const void* w, const float* scale, void* out, int n, int k, int group_size, int out_dtype, int experts, cudaStream_t s) {
  if (out_dtype == kBF16) return launch_dequant<INT4, __nv_bfloat16>(w, scale, out, n, k, group_size, experts, s);
  if (out_dtype == kF16) return launch_dequant<INT4, __half>(w, scale, out, n, k, group_size, experts, s);
  if (out_dtype == kF32) return launch_dequant<INT4, float>(w, scale, out, n, k, group_size, experts, s);
  return 1;
}

}  // namespace wo

int weight_dequantize(const void* w, const float* scale, void* out, int n, int k, int int4, int group_size, int out_dtype, cudaStream_t s,
                      int experts) {
  using namespace wo;
  if (n <= 0 || k <= 0 || experts <= 0 || experts > 65535 || (int4 && k % 2) || (group_size > 0 && k % group_size) || (n + 63) / 64 > 65535) return 1;
  return int4 ? dispatch_dequant<true>(w, scale, out, n, k, group_size, out_dtype, experts, s)
              : dispatch_dequant<false>(w, scale, out, n, k, group_size, out_dtype, experts, s);
}

int gemm_weight_only(const WoGemmArgs& g, cudaStream_t s) {
  using namespace wo;
  const bool experts = g.work != nullptr;
  // dense batches above 64 rows: dequantise once + the bf16 GEMM (nn/quant.py)
  if (g.k % 64 || g.n % 8 || g.m <= 0 || (experts ? g.experts <= 0 : g.m > 64)) return 1;
  if (g.group_size > 0 && ((g.group_size != 64 && g.group_size != 128) || g.k % g.group_size)) return 1;
  if ((reinterpret_cast<uintptr_t>(g.x) | reinterpret_cast<uintptr_t>(g.w) | reinterpret_cast<uintptr_t>(g.out)) & 15) return 1;
  CUtensorMap mw;
  if (!make_w_map(&mw, g.w, experts ? g.experts : 0, g.n, g.int4 ? g.k / 2 : g.k)) return 2;
  return experts ? dispatch_format<true>(g, mw, s) : dispatch_format<false>(g, mw, s);
}

}  // namespace b200
