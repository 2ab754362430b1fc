// Bodies of the flash-attention forward kernel and of the paged prefill's work-list kernel (see attention_sm100.cu for the algorithms).
// attention_sm100.cu instantiates them in fwd_kernel and paged_work_kernel, and the sliding-window (WINDOW) paged versions in
// fwd_window_kernel and paged_work_window_kernel.
//
// Sliding window W (WINDOW): the query at absolute position i sees key j iff i - W < j <= i.  Keys below the lowest bound of a CTA's
// rows are never loaded and their block-table entries never read, so blocks wholly below the window may hold anything.
#pragma once
#include <cuda.h>
#include <cmath>
#include <type_traits>

#include "b200_common.cuh"
#include "b200_kv8.cuh"
#include "b200_mask_tiles.cuh"
#include "b200_ops.h"
#include "b200_philox.cuh"
#include "b200_ptx.cuh"

namespace b200 {
namespace dropout {

// A dropout kernel's parameters: the dropout-free ones plus the rate and generator state of AttnDropoutArgs.
template <typename P>
DropoutParams<P> with_dropout(const P& base, const AttnDropoutArgs& d) {
  DropoutParams<P> p{};
  static_cast<P&>(p) = base;
  p.keep = (uint32_t)std::lrint((1.0 - d.p) * 65536.0);
  p.rscale = (float)(1.0 / (1.0 - d.p));
  p.seed_offset = d.seed_offset;
  p.seed_ptr = d.seed_ptr; p.offset_ptr = d.offset_ptr; p.offset_add = d.offset_add;
  p.seed = d.seed; p.offset = d.offset;
  return p;
}

}  // namespace dropout

namespace attn {
using namespace ptx;

constexpr int BM = 128, BN = 128, HD = 128;
constexpr int kThreads = 288;   // warps 0-7: two MMA / softmax warpgroups, warp 8: TMA producer
constexpr int kThreadsQ8 = 384; // 8-bit paged caches: warps 8-11 convert K / V (warp 8 lane 0 also loads Q)
constexpr uint32_t TILE_BYTES = 128 * 128 * 2;   // 32 KB: every operand tile (Q, K, V) at head_dim 128
constexpr uint32_t HALF_BYTES = 128 * 64 * 2;    // one 64-wide K-block of a tile
// Q, 2x K, 2x V tiles of 128 rows x D
template <int D> constexpr uint32_t kSmemBytes = 5 * (128 * D * 2) + 1024 /*align*/ + 256 /*barriers*/;
constexpr uint32_t kDropoutSmemBytes = 128 + kThreads * 8;   // DROPOUT: one 64-bit keep mask per thread past the barriers' 128 bytes
constexpr uint32_t SMEM_BYTES = kSmemBytes<HD>;

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

// MASKED, PAGED, KV, D: see fwd_kernel in attention_sm100.cu.
// WINDOW (PAGED only, P = WindowParams<...>): sliding window p.window, see fwd_body's key range below
// DROPOUT (dense only, P = dropout::DropoutParams<Params>): attention dropout, see attention_dropout_sm100.cu
// SKIP (MASKED dense only, P = mask_skip::SkipParams<...>): walk only the key tiles the column mask does not hide, see b200_mask_tiles.cuh
template <typename T, bool MASKED, bool PAGED, typename KV, int D, bool WINDOW, bool DROPOUT = false, bool SKIP = false, typename P>
__device__ __forceinline__ void fwd_body(const CUtensorMap& map_q, const CUtensorMap& map_k, const CUtensorMap& map_v, const P p) {
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr bool Q8 = !std::is_same<KV, T>::value;
  static_assert(!Q8 || (PAGED && !MASKED), "8-bit caches are paged only");
  static_assert(D == HD || (D == 64 && !Q8), "head_dim 64 reads 16-bit K / V only");
  static_assert(!WINDOW || (PAGED && !MASKED), "sliding windows are paged only");
  static_assert(!DROPOUT || !PAGED, "dropout is dense (training) only");
  static_assert(!SKIP || (MASKED && !PAGED), "tile skipping is for the dense column-masked kernels");
  constexpr int kHalves = D / 64;                            // 64-wide d chunks (128-byte swizzle spans) of a row
  constexpr uint32_t kTile = BM * D * 2;                     // one Q, K or V tile
  constexpr uint32_t kVBlock = kHalves * 8192;               // one 64-key block of a V tile (its d chunks 8192 B apart)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  auto sK = [&](int s) { return base + (1 + s) * kTile; };
  auto sV = [&](int s) { return base + (3 + s) * kTile; };
  const uint32_t bars = base + 5 * kTile;
  const uint32_t q_full = bars;
  auto k_full = [&](int s) { return bars + 8u * (1 + s); };
  auto v_full = [&](int s) { return bars + 8u * (3 + s); };
  auto k_empty = [&](int s) { return bars + 8u * (5 + s); };    // 8 warp arrivals
  auto v_empty = [&](int s) { return bars + 8u * (7 + s); };
  // SKIP: stage s's key tile, 2 j + open (-1: end of the list), published before k_full(s); the next tile (-1: none), published before
  // v_full(s), so it stays valid until the consumers release v_empty(s); the first tile (-1: none), published before q_full
  auto k_slot = [&](int s) { return bars + 80u + 4u * s; };
  auto v_slot = [&](int s) { return bars + 88u + 4u * s; };
  const uint32_t first_slot = bars + 96u;

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
  // WINDOW: row i sees keys (i + causal_off - window, i + causal_off]; lo is the lowest key any row of the tile sees and j0 its key tile.
  // The tiles below j0 are skipped, keys below lo are masked and zeroed in V, and their block-table entries are never read.
  int lo = 0, j0 = 0;
  if constexpr (WINDOW) {
    lo = max(0, m0 + causal_off - p.window + 1);
    j0 = lo / BN;
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
        for (int j = j0; j < n_tiles; ++j) {
          const int s = (j - j0) & 1;
          const uint32_t ph = (((j - j0) >> 1) & 1) ^ 1;
          uint4 kr[8], vr[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {   // both tiles' loads in flight before the first wait
            const int key = j * BN + i * 16 + r0;
            kr[i] = vr[i] = make_uint4(0, 0, 0, 0);
            if (key < sk && (!WINDOW || key >= lo)) {
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
          mbar_expect_tx(q_full, kTile);
          tma_load_4d(sQ, &map_q, q_full, 0, q0 + m0, head, 0);
          if constexpr (kHalves == 2) tma_load_4d(sQ + HALF_BYTES, &map_q, q_full, 64, q0 + m0, head, 0);
        }
        for (int j = j0; j < n_tiles; ++j) {
          const int s = (j - j0) & 1, key = j * BN + c * R;
          const uint32_t ph = (((j - j0) >> 1) & 1) ^ 1;
          // keys past the sequence come from a valid block (masked in S, zeroed in V) so every tile carries the same bytes; so do keys
          // below the window, from the block of lo
          const int blk = lane < kHalves * C ? (key < sk ? __ldg(bt + (WINDOW ? max(key, lo) : key) / bsz) : last_blk) : 0;
          const int row = key % bsz;
          mbar_wait(k_empty(s), ph);
          if (lane == 0) mbar_expect_tx(k_full(s), kTile);
          __syncwarp();
          if (lane < kHalves * C) tma_load_4d(sK(s) + half * HALF_BYTES + c * R * 128, &map_k, k_full(s), half * 64, row, kv_head, blk);
          mbar_wait(v_empty(s), ph);
          if (lane == 0) mbar_expect_tx(v_full(s), kTile);
          __syncwarp();
          if (lane < kHalves * C)
            tma_load_4d(sV(s) + (c * R / 64) * kVBlock + half * 8192 + (c * R % 64) * 128, &map_v, v_full(s), half * 64, row, kv_head, blk);
        }
      }
    } else if constexpr (SKIP) {
      if (n_tiles > 0) {
        // ================= TMA producer over the key tiles the column mask does not hide (b200_mask_tiles.cuh) =================
        // lane l classifies key tile jb + l; lane 0 loads a visible tile once the next one is known, which goes to v_slot for the
        // dropout kernels' bits, and loads Q once the first one is known, which goes to first_slot
        const int* tiles = p.tiles + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.n_ktiles * 8;
        int cnt = 0, pend = -1;   // pend: 2 j + open of the visible tile waiting for its successor
        auto issue = [&](int next) {
          if (lane == 0) {
            if (cnt == 0) {
              mask_skip::st_slot(first_slot, pend >> 1);
              mbar_expect_tx(q_full, kTile);
              tma_load_4d(sQ, &map_q, q_full, 0, m0, head, batch);
              if constexpr (kHalves == 2) tma_load_4d(sQ + HALF_BYTES, &map_q, q_full, 64, m0, head, batch);
            }
            const int s = cnt & 1, n0 = (pend >> 1) * BN;
            const uint32_t ph = ((cnt >> 1) & 1) ^ 1;
            mbar_wait(k_empty(s), ph);
            mask_skip::st_slot(k_slot(s), pend);
            mbar_expect_tx(k_full(s), kTile);
            tma_load_4d(sK(s), &map_k, k_full(s), 0, n0, kv_head, batch);
            if constexpr (kHalves == 2) tma_load_4d(sK(s) + HALF_BYTES, &map_k, k_full(s), 64, n0, kv_head, batch);
            mbar_wait(v_empty(s), ph);
            mask_skip::st_slot(v_slot(s), next);
            mbar_expect_tx(v_full(s), kTile);
#pragma unroll
            for (int kb = 0; kb < 2; ++kb)
#pragma unroll
              for (int i = 0; i < kHalves; ++i)
                tma_load_4d(sV(s) + kb * kVBlock + i * 8192, &map_v, v_full(s), i * 64, n0 + kb * 64, kv_head, batch);
          }
          ++cnt;
        };
        for (int jb = 0; jb < n_tiles; jb += 32) {
          const int cls = jb + lane < n_tiles ? mask_skip::tile_class(tiles + (jb + lane) * 8, m0, m0 + BM) : mask_skip::kHidden;
          uint32_t vis = __ballot_sync(0xffffffffu, cls != mask_skip::kHidden);
          const uint32_t open = __ballot_sync(0xffffffffu, cls == mask_skip::kOpen);
          while (vis) {
            const int bit = __ffs(vis) - 1;
            vis &= vis - 1;
            if (pend >= 0) issue(jb + bit);
            pend = 2 * (jb + bit) + ((open >> bit) & 1);
          }
        }
        if (pend >= 0) issue(-1);
        if (lane == 0 && cnt == 0) {   // nothing visible: the consumers still wait for Q
          mask_skip::st_slot(first_slot, -1);
          mbar_arrive(q_full);
        }
        if (lane == 0 && cnt < n_tiles) {   // the consumers' loop would go on: end it
          const int s = cnt & 1;
          mbar_wait(k_empty(s), ((cnt >> 1) & 1) ^ 1);
          mask_skip::st_slot(k_slot(s), -1);
          mbar_arrive(k_full(s));
        }
      }
    } else if (lane == 0 && n_tiles > 0) {
      // ================= TMA producer =================
      // one box per 64-wide d chunk: two per Q / K tile and four per V tile at D = 128, one and two at D = 64
      mbar_expect_tx(q_full, kTile);
      tma_load_4d(sQ, &map_q, q_full, 0, m0, head, batch);
      if constexpr (kHalves == 2) tma_load_4d(sQ + HALF_BYTES, &map_q, q_full, 64, m0, head, batch);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j & 1, n0 = j * BN;
        const uint32_t ph = ((j >> 1) & 1) ^ 1;
        mbar_wait(k_empty(s), ph);
        mbar_expect_tx(k_full(s), kTile);
        tma_load_4d(sK(s), &map_k, k_full(s), 0, n0, kv_head, batch);               // box {64 d, 128 keys}: K-major B operand
        if constexpr (kHalves == 2) tma_load_4d(sK(s) + HALF_BYTES, &map_k, k_full(s), 64, n0, kv_head, batch);
        mbar_wait(v_empty(s), ph);
        mbar_expect_tx(v_full(s), kTile);
#pragma unroll
        for (int kb = 0; kb < 2; ++kb)                                              // box {64 d, 64 keys}: MN-major B operand
#pragma unroll
          for (int i = 0; i < kHalves; ++i)
            tma_load_4d(sV(s) + kb * kVBlock + i * 8192, &map_v, v_full(s), i * 64, n0 + kb * 64, kv_head, batch);
      }
    }
  } else {
    // ================= MMA + softmax + epilogue: warpgroup wg owns query rows [64 wg, 64 wg + 64) =================
    const int wg = warp >> 2, q = lane & 3;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: rl and rl + 8
    float scale_log2 = p.scale_log2;
    if constexpr (Q8) scale_log2 *= __ldg(p.k_dq + kv_head);  // S is computed on the quantized K
    float o_acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o_acc[i] = 0.f;
    float m_i[2] = {-INFINITY, -INFINITY}, l_i[2] = {0.f, 0.f};   // l_i: this thread's share of the row sum (reduced over the quad at the end)
    // DROPOUT: the keep bits of key tile jt (see b200_philox.cuh); rows rl and rl + 8 share every call, and call kk covers key column
    // groups 2 kk, 2 kk + 1: bit 8 kk + 4 h + 2 (jn & 1) + e.  Tile j + 1's bits are drawn while the P V MMAs of tile j are in flight,
    // where S is dead, and the key and counter words are rebuilt on each draw: held across the loop (or drawn under the S MMAs) they
    // would make the D = 128 kernel spill.
    auto draw = [&](int jt) {
      uint64_t bits = 0;
      if constexpr (DROPOUT) {
        const uint64_t seed = p.seed_ptr ? (uint64_t)__ldg(p.seed_ptr) : p.seed;
        const int64_t offset = p.seed_ptr ? __ldg(p.offset_ptr) + p.offset_add : (int64_t)p.offset;
        uint32_t c2, c3;
        dropout::plane_counter(offset, batch, p.h, head, c2, c3);
        const uint32_t rc = dropout::row_counter(m0 + rl);
        uint32_t lo = 0, hi = 0;   // word h: the bits of row rl + 8 h, call kk at bits 4 kk + 2 (jn & 1) + e
#pragma unroll 1
        for (int kk = 0; kk < BN / 16; ++kk) {   // one call's temporaries live at a time
          const uint32_t b = dropout::keep_bits(rc, dropout::key_counter(jt * BN + 16 * kk + 2 * q), (uint32_t)seed, (uint32_t)(seed >> 32), c2, c3,
                                                p.keep);
          lo |= (b & 15u) << (4 * kk);
          hi |= (b >> 4) << (4 * kk);
        }
        bits = ((uint64_t)hi << 32) | lo;
      }
      return bits;
    };
    // the bits wait in shared memory past the barriers (kDropoutSmemBytes more), not in registers, while S and O fill the register file
    uint64_t* const keep_slot = reinterpret_cast<uint64_t*>(smem_raw + (bars + 128 - smem_u32(smem_raw))) + threadIdx.x;
    (void)keep_slot;
    (void)k_slot; (void)v_slot; (void)first_slot;
    if constexpr (DROPOUT) {
      if ((blockIdx.x | blockIdx.y | blockIdx.z | threadIdx.x) == 0) {   // the pair this launch used, for the backward
        p.seed_offset[0] = p.seed_ptr ? __ldg(p.seed_ptr) : (int64_t)p.seed;
        p.seed_offset[1] = p.seed_ptr ? __ldg(p.offset_ptr) + p.offset_add : (int64_t)p.offset;
      }
      if (!SKIP && j0 < n_tiles) *keep_slot = draw(j0);
    }
    (void)draw;
    if (n_tiles > 0) mbar_wait(q_full, 0);
    if constexpr (SKIP && DROPOUT) {
      const int first = n_tiles > 0 ? mask_skip::ld_slot(first_slot) : -1;
      if (first >= 0) *keep_slot = draw(first);
    }
    for (int j = j0; j < n_tiles; ++j) {   // SKIP: j counts the tiles processed, jt is the one published for stage s
      const int s = (j - j0) & 1, ph = ((j - j0) >> 1) & 1;
      float sv[BN / 2];
      mbar_wait(k_full(s), ph);
      if constexpr (SKIP) {
        if (mask_skip::ld_slot(k_slot(s)) < 0) break;
      }
      // SKIP: the tile's index and class are read from k_slot(s) where they are used, not held in registers; the slot stays valid until
      // k_empty(s) is released, after the masks
      auto tile = [&] {
        if constexpr (SKIP) return mask_skip::ld_slot(k_slot(s)) >> 1;
        else return j;
      };
      wgmma_fence_regs(sv);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < kHalves; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss_n128<BF16, 0, 0>(sv, make_smem_desc(sQ + kb * HALF_BYTES + wg * 8192 + k * 32, 16, 1024),
                                    make_smem_desc(sK(s) + kb * HALF_BYTES + k * 32, 16, 1024), (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sv);
      __syncwarp();
      if (!SKIP && lane == 0) mbar_arrive(k_empty(s));
      // ---- masks (raw logits; the softmax scale is folded into the exp2 FFMA) ----
      const int jt = tile();
      const bool edge = PAGED ? (jt * BN + BN > sk) || (jt * BN + BN - 1 > m0 + causal_off)
                              : (jt * BN + BN > p.sk) || (p.causal && jt * BN + BN - 1 > m0 + p.causal_off);
      if (edge) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + rl + h * 8;
          const int lim = (p.causal ? min(sk - 1, row + causal_off) : sk - 1) - jt * BN;   // last visible key, tile-relative
#pragma unroll
          for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (jn * 8 + 2 * q + e > lim) sv[jn * 4 + h * 2 + e] = -INFINITY;
        }
      }
      if constexpr (WINDOW) {     // the window's left edge: only the tiles below the last row's first visible key
        if (jt * BN < m0 + BM + causal_off - p.window) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int first = m0 + rl + h * 8 + causal_off - p.window + 1 - jt * BN;   // this row's first visible key, tile-relative
#pragma unroll
            for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (jn * 8 + 2 * q + e < first) sv[jn * 4 + h * 2 + e] = -INFINITY;
          }
        }
      }
      // flashmask / varlen: key column j hides the query rows [lt_start, lt_end) and [ut_start, ut_end) (SKIP: tested unless the tile is open)
      if (MASKED && !(SKIP && (mask_skip::ld_slot(k_slot(s)) & 1))) {
        const int4* cm = p.colmask + ((int64_t)batch * p.mask_heads + (p.mask_heads > 1 ? head : 0)) * p.sk;
        const int k0 = tile() * BN;
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = k0 + jn * 8 + 2 * q + e;
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
      if constexpr (SKIP) {
        __syncwarp();
        if (lane == 0) mbar_arrive(k_empty(s));
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
        for (int jn = 0; jn < D / 8; ++jn) { o_acc[jn * 4 + h * 2] *= alpha; o_acc[jn * 4 + h * 2 + 1] *= alpha; }
        if constexpr (DROPOUT) {   // after the row sum: l and lse stay those of the undropped softmax
          const uint32_t keep = reinterpret_cast<const uint32_t*>(keep_slot)[h];   // bits of row h in word h (see draw)
#pragma unroll
          for (int jn = 0; jn < BN / 8; ++jn)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (!((keep >> (4 * (jn >> 1) + 2 * (jn & 1) + e)) & 1u)) sv[jn * 4 + h * 2 + e] = 0.f;
            }
        }
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
      if constexpr (WINDOW && !Q8) {   // V rows below the window hold another block's rows (possibly NaN): zero them as past the sequence
        if (j == j0 && lo > j * BN) {
          const int tid = threadIdx.x & 127;
          constexpr int kRowShift = D == 128 ? 4 : 3;
          for (int e = tid; e < (lo - j * BN) << kRowShift; e += 128) {
            const int r = e >> kRowShift;
            st_shared_zero16(sV(s) + (r >> 6) * kVBlock + ((e >> 3) & (kHalves - 1)) * 8192 + (r & 63) * 128 + (e & 7) * 16);
          }
          fence_proxy_async();
          named_bar_sync(1 + wg, 128);
        }
      }
      if constexpr (PAGED && !Q8) {   // (the converter writes zeros past the sequence)
        if (j * BN + BN > sk) {   // V rows past the sequence hold stale cache contents (possibly NaN) and P = 0 does not cancel NaN: zero them
          const int tid = threadIdx.x & 127;
          constexpr int kRowShift = D == 128 ? 4 : 3;           // log2 of the 16-byte chunks of a key row
          for (int e = (sk - j * BN) * (1 << kRowShift) + tid; e < BN << kRowShift; e += 128) {   // key row e >> kRowShift, d-half (e / 8) & 1
            const int r = e >> kRowShift;
            st_shared_zero16(sV(s) + (r >> 6) * kVBlock + ((e >> 3) & (kHalves - 1)) * 8192 + (r & 63) * 128 + (e & 7) * 16);
          }
          fence_proxy_async();                    // generic-proxy stores before this warpgroup's wgmma reads them
          named_bar_sync(1 + wg, 128);
        }
      }
      wgmma_fence_regs(o_acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < BN / 16; ++ks) {   // V tile MN-major: 64-key block ks / 4, 16 key rows = 2048 B per step, 64-wide d chunks 8192 B apart
        const uint64_t vdesc = make_smem_desc(sV(s) + (ks >> 2) * kVBlock + (ks & 3) * 2048, 8192, 1024);
        if constexpr (D == 128) wgmma_rs_n128<BF16, 1>(o_acc, pa[ks], vdesc, 1);
        else wgmma_rs_n64<BF16, 1>(o_acc, pa[ks], vdesc, 1);
      }
      wgmma_commit();
      if constexpr (DROPOUT && SKIP) {
        const int jn = mask_skip::ld_slot(v_slot(s));
        if (jn >= 0) *keep_slot = draw(jn);
      } else if constexpr (DROPOUT) {
        if (j + 1 < n_tiles) *keep_slot = draw(j + 1);
      }
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
      if constexpr (DROPOUT) inv *= p.rscale;             // 1 / (1 - p): kept entries of P enter P V unscaled
      const int row = m0 + rl + h * 8;
      if (row < nrows) {
        T* orow = reinterpret_cast<T*>(p.o) + (PAGED ? 0 : (int64_t)batch * p.o_sb) + (int64_t)(q0 + row) * p.o_ss + (int64_t)head * p.o_sh;
#pragma unroll
        for (int jn = 0; jn < D / 8; ++jn)
          *reinterpret_cast<uint32_t*>(orow + jn * 8 + 2 * q) = pack2<T>(o_acc[jn * 4 + h * 2] * inv, o_acc[jn * 4 + h * 2 + 1] * inv);
        if (q == 0 && p.lse) p.lse[((int64_t)(PAGED ? 0 : batch) * p.h + head) * p.sq + q0 + row] = l > 0.f ? (m_i[h] + log2f(l)) * 0.69314718055994531f : -INFINITY;
      }
    }
  }
}

// MASKED: column-wise row-range mask (flashmask / varlen) compiled in; the dense instantiation carries none of its code or registers
// PAGED: queries = new tokens of each sequence, K / V read through the block table (see attention_sm100.cu); always causal, never MASKED
// KV: the cache element type; kv8::I8 / kv8::E4M3 (PAGED only) select the converter warpgroup and QuantPagedParams
// D: the head size, 128 or 64 (64: 16-bit K / V).  attention_sm100.cu instantiates D = 128 and the paged D = 64 kernels,
// attention_d64_sm100.cu the dense D = 64 ones.
template <typename T, bool MASKED, bool PAGED = false, typename KV = T, int D = HD>
__global__ void __launch_bounds__(std::is_same<KV, T>::value ? kThreads : kThreadsQ8, 1)
fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
           const std::conditional_t<PAGED, std::conditional_t<std::is_same<KV, T>::value, PagedParams, QuantPagedParams>, Params> p) {
  fwd_body<T, MASKED, PAGED, KV, D, false>(map_q, map_k, map_v, p);
}

// The dense forward at head size D over the strided [B,S,H,D] views of AttnArgs (checked by attention_fwd_supported): builds the
// tensor maps and parameters and calls launch(T(), std::bool_constant<MASKED>(), maps, params, grid, smem) for the operands' type and mask.
template <int D, typename Launch>
int fwd_dense_with(const AttnArgs& a, cudaStream_t s, Launch&& launch) {
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
  const dim3 grid((a.sq + BM - 1) / BM, a.h, a.b);
  constexpr uint32_t smem = kSmemBytes<D>;
  if (a.dtype == kBF16 && !p.colmask) launch(__nv_bfloat16(), std::false_type(), mq, mk, mv, p, grid, smem);
  else if (a.dtype == kBF16) launch(__nv_bfloat16(), std::true_type(), mq, mk, mv, p, grid, smem);
  else if (!p.colmask) launch(__half(), std::false_type(), mq, mk, mv, p, grid, smem);
  else launch(__half(), std::true_type(), mq, mk, mv, p, grid, smem);
  return B200_LAUNCH_RESULT();
}

template <int D>
int fwd_dense(const AttnArgs& a, cudaStream_t s) {
  return fwd_dense_with<D>(a, s, [&](auto tag_t, auto tag_masked, const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                     const Params& p, dim3 grid, uint32_t smem) {
    using T = decltype(tag_t);
    constexpr bool MASKED = decltype(tag_masked)::value;
    set_max_dynamic_smem<fwd_kernel<T, MASKED, false, T, D>>(smem);
    fwd_kernel<T, MASKED, false, T, D><<<grid, kThreads, smem, s>>>(mq, mk, mv, p);
  });
}

// A paged instantiation's parameters with a sliding window: key j is visible to query i iff i - window < j <= i (window >= 1).
template <typename P> struct WindowParams : P {
  int window;
};

// Work list of the paged kernel: one (sequence, 128-row query tile) per slot, sorted by key tiles (heaviest first, ties in sequence
// order) so a long prefix starts early instead of running alone at the end; slots past the list get sequence -1.  One CTA; the
// O(tiles^2) ranking is a few hundred thousand compares at the largest batches, well under the attention it schedules.
// scratch: int32 [slots] key-tile counts followed by [b + 1] tile offsets.
// WINDOW: a tile counts only the key tiles from the one holding its first row's lowest visible key (m0 + past - window + 1).
template <bool WINDOW>
__device__ __forceinline__ void paged_work(const int* __restrict__ n_q, const int* __restrict__ past, int b, int slots, int* scratch, int2* work,
                                           int window) {
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
    if constexpr (WINDOW) keys[w] -= max(0, m0 + past[sq] - window + 1) / BN;
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

}  // namespace b200
