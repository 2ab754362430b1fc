// Single-token decode attention against a contiguous KV cache (serving path of FusedMultiTransformer /
// masked_multihead_attention).  HBM-bound: every cached key / value row is read exactly once with 16-byte loads.
//
// Parity (behaviour): masked_multihead_attention (paddle/phi/kernels/fusion/gpu/masked_multihead_attention_kernel.cu).
//
// Layout: q [B, H, D]; k_cache / v_cache [B, Hkv, S_max, D] (the two halves of paddle's cache_kv [2, B, H, S_max, D]);
// lens[b] = number of valid cached positions (the new token already written).  Grid = (splits, H, B): every CTA owns a
// contiguous range of positions; thread t handles positions t, t+128, ... with a private online softmax (m, l, acc[D]);
// the CTA combines its threads through shared memory and writes one partial (m, l, acc) per split; a second tiny kernel
// merges the splits.  D = 128, fp16 / bf16.
//
// Paged caches (block_multihead_attention, paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu): with `block_tables`
// [B, max_blocks] the caches are [num_blocks, Hkv, block_size, D] and position p of sequence b lives in block block_tables[b, p / block_size]
// at row p % block_size - one table lookup per cached row, the rest of the kernel is unchanged.
//
// Paged int8 / fp8 e4m3 caches (decode_split_q8_kernel): the same walk over 8-bit rows, dequantized with per-KV-head scales.
#include <cuda.h>
#include <cstdio>
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_kv8.cuh"
#include "include/b200_ops.h"

namespace b200 {
namespace decode {

constexpr int D = 128, kThreads = 128;

// Combine the CTA's per-thread online-softmax partials (m, l, acc) and write this split's partial (m, l, acc * v_scale).
__device__ __forceinline__ void split_epilogue(float m, float l, const float (&acc)[D], float* red, float (*sacc)[D + 1], float* __restrict__ part_acc,
                                               float* __restrict__ part_ml, int h, int splits, float v_scale) {
  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  // CTA-wide maximum, then every thread rescales its partial to it
  red[tid] = m;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (tid < o) red[tid] = fmaxf(red[tid], red[tid + o]);
    __syncthreads();
  }
  const float mg = red[0];
  __syncthreads();
  const float f = (m == -INFINITY) ? 0.f : exp2f(m - mg);
  l *= f;
  red[tid] = l;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (tid < o) red[tid] += red[tid + o];
    __syncthreads();
  }
  const float lg = red[0];
  // sum the 128 per-thread accumulators: 4 rounds of 32 threads' vectors through shared memory, thread t owns output dim t
  float out = 0.f;
  for (int r = 0; r < kThreads / 32; ++r) {
    __syncthreads();
    if ((tid >> 5) == r) {
#pragma unroll
      for (int i = 0; i < D; ++i) sacc[tid & 31][i] = acc[i] * f;
    }
    __syncthreads();
#pragma unroll 8
    for (int j = 0; j < 32; ++j) out += sacc[j][tid];
  }
  const int64_t pi = ((int64_t)b * h + head) * splits + split;
  part_acc[pi * D + tid] = out * v_scale;
  if (tid == 0) { part_ml[pi * 2] = mg; part_ml[pi * 2 + 1] = lg; }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) decode_split_kernel(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
                                                                const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                float* __restrict__ part_ml, int h, int hkv, int smax, int splits, float scale_log2,
                                                                const int* __restrict__ block_tables, int max_blocks, int block_size) {
  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (h / hkv);
  const int len = block_tables ? min(lens[b], max_blocks * block_size) : min(lens[b], smax);
  const int per = (len + splits - 1) / splits;
  const int p0 = split * per, p1 = min(len, p0 + per);
  __shared__ float sq[D];
  __shared__ float red[kThreads];
  __shared__ float sacc[32][D + 1];           // one slice of the cross-thread reduction at a time
  const int tid = threadIdx.x;
  sq[tid] = to_f(q[((int64_t)b * h + head) * D + tid]) * scale_log2;
  __syncthreads();
  const T* kbase = kc + ((int64_t)b * hkv + kvh) * (int64_t)smax * D;
  const T* vbase = vc + ((int64_t)b * hkv + kvh) * (int64_t)smax * D;
  const int* bt = block_tables ? block_tables + (int64_t)b * max_blocks : nullptr;
  // element offset of cached position `pos` of this (sequence, kv head)
  auto row_off = [&](int pos) -> int64_t {
    if (!bt) return (int64_t)pos * D;
    const int blk = bt[pos / block_size];
    return (((int64_t)blk * hkv + kvh) * block_size + pos % block_size) * D;
  };
  if (bt) { kbase = kc; vbase = vc; }
  float m = -INFINITY, l = 0.f;
  float acc[D];
#pragma unroll
  for (int i = 0; i < D; ++i) acc[i] = 0.f;
  for (int pos = p0 + tid; pos < p1; pos += kThreads) {
    const int64_t roff = row_off(pos);
    const Vec16<T>* kr = reinterpret_cast<const Vec16<T>*>(kbase + roff);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      const Vec16<T> kv = ld16(reinterpret_cast<const T*>(kr + c));
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(to_f(kv.v[e]), sq[c * 8 + e], s);
    }
    const float m_new = fmaxf(m, s);
    const float alpha = exp2f(m - m_new), pv = exp2f(s - m_new);
    l = l * alpha + pv;
    const Vec16<T>* vr = reinterpret_cast<const Vec16<T>*>(vbase + roff);
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      const Vec16<T> vv = ld16(reinterpret_cast<const T*>(vr + c));
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[c * 8 + e] = fmaf(acc[c * 8 + e], alpha, pv * to_f(vv.v[e]));
    }
    m = m_new;
  }
  split_epilogue(m, l, acc, red, sacc, part_acc, part_ml, h, splits, 1.f);
}

// Paged 8-bit caches (KV = kv8::I8 / kv8::E4M3): one 16-byte load carries 16 elements.  The K dequant scale is folded into sq, the V
// dequant scale is applied once to the split's partial output; with power-of-two scales the result is bit-identical to
// decode_split_kernel on a 16-bit cache holding the dequantized values.
template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) decode_split_q8_kernel(const T* __restrict__ q, const uint8_t* __restrict__ kc, const uint8_t* __restrict__ vc,
                                                                   const int* __restrict__ lens, float* __restrict__ part_acc,
                                                                   float* __restrict__ part_ml, int h, int hkv, int splits, float scale_log2,
                                                                   const float* __restrict__ k_dq, const float* __restrict__ v_dq,
                                                                   const int* __restrict__ block_tables, int max_blocks, int block_size) {
  const int split = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (h / hkv);
  const int len = min(lens[b], max_blocks * block_size);
  const int per = (len + splits - 1) / splits;
  const int p0 = split * per, p1 = min(len, p0 + per);
  __shared__ float sq[D];
  __shared__ float red[kThreads];
  __shared__ float sacc[32][D + 1];
  const int tid = threadIdx.x;
  sq[tid] = to_f(q[((int64_t)b * h + head) * D + tid]) * scale_log2 * __ldg(k_dq + kvh);
  __syncthreads();
  const int* bt = block_tables + (int64_t)b * max_blocks;
  float m = -INFINITY, l = 0.f;
  float acc[D];
#pragma unroll
  for (int i = 0; i < D; ++i) acc[i] = 0.f;
  for (int pos = p0 + tid; pos < p1; pos += kThreads) {
    const int64_t roff = (((int64_t)bt[pos / block_size] * hkv + kvh) * block_size + pos % block_size) * D;
    const uint4* kr = reinterpret_cast<const uint4*>(kc + roff);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < D / 16; ++c) {
      float kf[16];
      kv8::to_float16<KV>(kr[c], kf);
#pragma unroll
      for (int e = 0; e < 16; e += 4) {   // re-read q from shared memory every row: 128 q registers on top of acc would spill
        float4 qv;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(qv.x), "=f"(qv.y), "=f"(qv.z), "=f"(qv.w)
                     : "r"((uint32_t)__cvta_generic_to_shared(sq + c * 16 + e)));
        s = fmaf(kf[e], qv.x, s);
        s = fmaf(kf[e + 1], qv.y, s);
        s = fmaf(kf[e + 2], qv.z, s);
        s = fmaf(kf[e + 3], qv.w, s);
      }
    }
    const float m_new = fmaxf(m, s);
    const float alpha = exp2f(m - m_new), pv = exp2f(s - m_new);
    l = l * alpha + pv;
    const uint4* vr = reinterpret_cast<const uint4*>(vc + roff);
#pragma unroll
    for (int c = 0; c < D / 16; ++c) {
      float vf[16];
      kv8::to_float16<KV>(vr[c], vf);
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[c * 16 + e] = fmaf(acc[c * 16 + e], alpha, pv * vf[e]);
    }
    m = m_new;
  }
  split_epilogue(m, l, acc, red, sacc, part_acc, part_ml, h, splits, __ldg(v_dq + kvh));
}

template <typename T>
__global__ void __launch_bounds__(D) decode_merge_kernel(const float* __restrict__ part_acc, const float* __restrict__ part_ml, T* __restrict__ out,
                                                         int splits) {
  const int64_t bh = blockIdx.x;
  const int tid = threadIdx.x;
  float mg = -INFINITY;
  for (int s = 0; s < splits; ++s) mg = fmaxf(mg, part_ml[(bh * splits + s) * 2]);
  float l = 0.f, o = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float ms = part_ml[(bh * splits + s) * 2];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - mg);
    l += part_ml[(bh * splits + s) * 2 + 1] * f;
    o += part_acc[(bh * splits + s) * D + tid] * f;
  }
  out[bh * D + tid] = from_f<T>(l > 0.f ? o / l : 0.f);
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
namespace decode_multi {

constexpr int D = 128, BN = 64, kRows = 64, kThreads = 128, kStages = 3;
constexpr int kTile16 = BN * D * 2, kTile8 = BN * D;   // one K or V tile of 64 keys: 16 KB in 16 bits, 8 KB in 8 bits

struct Params {
  const void* q; const void* k_cache; const void* v_cache;
  void* out; float* part_acc; float* part_ml;
  const int* block_tables; const int* cu_q; const int* n_q; const int* past;
  const float* k_dq; const float* v_dq;
  int64_t q_st, q_sh, o_st;   // element strides: q (token, head), out (token; heads are D apart)
  int h, hkv, splits, max_blocks, block_size;
  float scale_log2;
};

// shared memory: Q tile [64][128] 16-bit | K, V 16-bit tiles (kStages, or 1 for 8-bit caches) | 8-bit caches: raw K, V tiles (kStages).
// Two tiles stay in flight while one is computed; two CTAs fit on an SM.
template <bool Q8> struct Smem {
  static constexpr int kKV = kRows * D * 2;
  static constexpr int kRaw = kKV + (Q8 ? 1 : kStages) * 2 * kTile16;
  static constexpr int kBytes = kRaw + (Q8 ? kStages * 2 * kTile8 : 0);
};

// byte offset of 16-byte chunk c (0..15) of row `row` in a [rows][128] 16-bit tile; the XOR spreads 8 consecutive rows over all banks
__device__ __forceinline__ uint32_t swz(int row, int c) { return (uint32_t)(row * (D * 2) + ((c ^ (row & 7)) << 4)); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {   // !valid: zero-fill, nothing is read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

template <typename T> __device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void mma16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
  const __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

// KV = T: 16-bit caches; KV = kv8::I8 / kv8::E4M3: 8-bit caches with fp32 [Hkv] dequant scales
template <typename T, typename KV>
__global__ void __launch_bounds__(kThreads) multi_split_kernel(const Params p) {
  constexpr bool Q8 = !std::is_same<T, KV>::value;
  using S = Smem<Q8>;
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int nq = p.n_q[b], g_size = p.h / p.hkv, nrows = nq * g_size;
  if (nq <= 0 || nrows > kRows) return;                      // skipped, or past the row limit (multi_merge_kernel writes NaN)
  const int past = p.past[b];
  const int len = min(past + nq, p.max_blocks * p.block_size);
  const int ntiles = (len + BN - 1) / BN, per = (ntiles + p.splits - 1) / p.splits;
  const int t0 = split * per, t1 = min(ntiles, t0 + per);
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int* bt = p.block_tables + (int64_t)b * p.max_blocks;
  const int cu = p.cu_q[b];

  // Q tile: rows past nrows are zero
#pragma unroll
  for (int i = 0; i < kRows * D / 8 / kThreads; ++i) {
    const int row = i * (kThreads / 16) + (tid >> 4), c = tid & 15;
    const bool ok = row < nrows;
    const T* src = reinterpret_cast<const T*>(p.q);
    if (ok) src += (int64_t)(cu + row / g_size) * p.q_st + (int64_t)(kvh * g_size + row % g_size) * p.q_sh + c * 8;
    cp_async16(sbase + swz(row, c), src, ok);
  }
  // cached K / V rows of key tile `tile` into stage `st`; keys at or past len are zero-filled
  auto load_kv = [&](int tile, int st) {
    constexpr int kEl = Q8 ? 16 : 8;                         // elements per 16-byte chunk
    constexpr int kChunks = D / kEl;
#pragma unroll
    for (int i = 0; i < BN * kChunks / kThreads; ++i) {
      const int row = i * (kThreads / kChunks) + tid / kChunks, c = tid % kChunks;
      const int pos = tile * BN + row;
      const bool ok = pos < len;
      int64_t off = 0;
      if (ok) off = (((int64_t)bt[pos / p.block_size] * p.hkv + kvh) * p.block_size + pos % p.block_size) * D + c * kEl;
      if constexpr (Q8) {
        const uint32_t dst = sbase + S::kRaw + st * 2 * kTile8 + row * D + c * 16;
        cp_async16(dst, reinterpret_cast<const uint8_t*>(p.k_cache) + off, ok);
        cp_async16(dst + kTile8, reinterpret_cast<const uint8_t*>(p.v_cache) + off, ok);
      } else {
        const uint32_t dst = sbase + S::kKV + st * 2 * kTile16 + swz(row, c);
        cp_async16(dst, reinterpret_cast<const T*>(p.k_cache) + off, ok);
        cp_async16(dst + kTile16, reinterpret_cast<const T*>(p.v_cache) + off, ok);
      }
    }
  };
  if (t0 < t1) load_kv(t0, 0);
  cp_async_commit();
  if (t0 + 1 < t1) load_kv(t0 + 1, 1);
  cp_async_commit();

  float qk_scale = p.scale_log2, v_scale = 1.f;
  if constexpr (Q8) { qk_scale *= __ldg(p.k_dq + kvh); v_scale = __ldg(p.v_dq + kvh); }
  const bool active = warp * 16 < nrows;
  const int r_lo = warp * 16 + (lane >> 2);                  // this lane's two rows: r_lo and r_lo + 8
  int limit[2];                                              // keys < limit are visible to the row
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) limit[hh] = min(len, past + (r_lo + hh * 8) / g_size + 1);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float acc[D / 8][4];
#pragma unroll
  for (int n = 0; n < D / 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  uint32_t qf[D / 16][4];

  for (int t = t0; t < t1; ++t) {
    const int st = (t - t0) % kStages;
    cp_async_wait<1>();                                      // tile t has landed (only tile t + 1 may still be in flight)
    __syncthreads();                                         // ... for every thread, and nobody still reads the stage refilled next
    if (t + 2 < t1) load_kv(t + 2, (st + 2) % kStages);
    cp_async_commit();
    if (t == t0 && active) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) ldsm_x4(qf[kk], sbase + swz(warp * 16 + (lane & 15), kk * 2 + (lane >> 4)));
    }
    uint32_t kv16 = sbase + S::kKV + st * 2 * kTile16;
    if constexpr (Q8) {                                      // raw 8-bit tiles -> the 16-bit tiles, exactly
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
        *reinterpret_cast<uint4*>(dst + swz(row, 2 * c)) = make_uint4(w[0], w[1], w[2], w[3]);
        *reinterpret_cast<uint4*>(dst + swz(row, 2 * c + 1)) = make_uint4(w[4], w[5], w[6], w[7]);
      }
      __syncthreads();
    }
    if (active) {
      // S = Q K^T: 16 rows x 64 keys per warp
      float s[BN / 8][4];
#pragma unroll
      for (int n = 0; n < BN / 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
        for (int np = 0; np < BN / 16; ++np) {
          uint32_t bf[4];
          ldsm_x4(bf, kv16 + swz(np * 16 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1)));
          mma16816<T>(s[2 * np], qf[kk], bf[0], bf[1]);
          mma16816<T>(s[2 * np + 1], qf[kk], bf[2], bf[3]);
        }
      }
      // mask, online softmax (log2 domain); a row's 64 scores are spread over the 4 lanes of a quad
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int n = 0; n < BN / 8; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = t * BN + n * 8 + 2 * (lane & 3) + e;
            float& v = s[n][hh * 2 + e];
            v = key < limit[hh] ? v * qk_scale : -INFINITY;
            mx = fmaxf(mx, v);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[hh], mx);
        const float base = m_new == -INFINITY ? 0.f : m_new;   // a row with no visible key yet keeps p = 0 (never exp2(-inf + inf))
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
      // O += P V: P's accumulator fragments are the A fragments of the next MMA
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        const uint32_t pa[4] = {pack2<T>(s[2 * kk][0], s[2 * kk][1]), pack2<T>(s[2 * kk][2], s[2 * kk][3]),
                                pack2<T>(s[2 * kk + 1][0], s[2 * kk + 1][1]), pack2<T>(s[2 * kk + 1][2], s[2 * kk + 1][3])};
#pragma unroll
        for (int np = 0; np < D / 16; ++np) {
          uint32_t bf[4];
          ldsm_x4_t(bf, kv16 + kTile16 + swz(kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), np * 2 + (lane >> 4)));
          mma16816<T>(acc[2 * np], pa, bf[0], bf[1]);
          mma16816<T>(acc[2 * np + 1], pa, bf[2], bf[3]);
        }
      }
    }
  }
  cp_async_wait<0>();
  if (!active) return;
  // this split's partial for the warp's rows (an empty split writes m = -inf, l = 0, acc = 0)
  const int64_t pbase = (((int64_t)b * p.hkv + kvh) * p.splits + split) * kRows;
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

// grid (64 rows, Hkv, B), D threads: combines the splits of one query row, as decode_merge_kernel does, and writes it in place.  A
// sequence over the row limit gets NaN rows rather than a silently partial result.
template <typename T>
__global__ void __launch_bounds__(D) multi_merge_kernel(const Params p) {
  const int r = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int nq = p.n_q[b], g_size = p.h / p.hkv, nrows = nq * g_size;
  if (nq <= 0) return;
  T* out = reinterpret_cast<T*>(p.out);
  const int64_t cu = p.cu_q[b];
  if (nrows > kRows) {
    for (int rr = r; rr < nrows; rr += kRows)
      out[(cu + rr / g_size) * p.o_st + (int64_t)(kvh * g_size + rr % g_size) * D + tid] = from_f<T>(__int_as_float(0x7fc00000));
    return;
  }
  if (r >= nrows) return;
  const int64_t pb = ((int64_t)b * p.hkv + kvh) * p.splits * kRows + r;
  float mg = -INFINITY;
  for (int s = 0; s < p.splits; ++s) mg = fmaxf(mg, p.part_ml[(pb + (int64_t)s * kRows) * 2]);
  float l = 0.f, o = 0.f;
  for (int s = 0; s < p.splits; ++s) {
    const int64_t i = pb + (int64_t)s * kRows;
    const float ms = p.part_ml[i * 2];
    const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - mg);
    l += p.part_ml[i * 2 + 1] * f;
    o += p.part_acc[i * D + tid] * f;
  }
  out[(cu + r / g_size) * p.o_st + (int64_t)(kvh * g_size + r % g_size) * D + tid] = from_f<T>(l > 0.f ? o / l : 0.f);
}

}  // namespace decode_multi

int decode_attention_splits(int b, int h, int smax) {
  // enough CTAs to fill the machine, at least 256 positions per split
  int splits = (2 * sm_count() + b * h - 1) / (b * h);
  const int max_by_len = (smax + 255) / 256;
  if (splits > max_by_len) splits = max_by_len;
  return splits < 1 ? 1 : (splits > 64 ? 64 : splits);
}

int decode_attention(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml, int b,
                     int h, int hkv, int smax, int d, int splits, float scale, int dtype, cudaStream_t s, const int* block_tables, int max_blocks,
                     int block_size) {
  using namespace decode;
  if (d != D || h % hkv || (dtype != kBF16 && dtype != kF16)) return 1;
  if (block_tables && (max_blocks <= 0 || block_size <= 0)) return 1;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  if (dtype == kBF16) {
    decode_split_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>((const __nv_bfloat16*)q, (const __nv_bfloat16*)k_cache, (const __nv_bfloat16*)v_cache, lens,
                                                                   part_acc, part_ml, h, hkv, smax, splits, sl2, block_tables, max_blocks, block_size);
    decode_merge_kernel<__nv_bfloat16><<<b * h, D, 0, s>>>(part_acc, part_ml, (__nv_bfloat16*)out, splits);
  } else {
    decode_split_kernel<__half><<<grid, kThreads, 0, s>>>((const __half*)q, (const __half*)k_cache, (const __half*)v_cache, lens, part_acc, part_ml, h, hkv,
                                                           smax, splits, sl2, block_tables, max_blocks, block_size);
    decode_merge_kernel<__half><<<b * h, D, 0, s>>>(part_acc, part_ml, (__half*)out, splits);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

int decode_attention_paged_q8(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml,
                              int b, int h, int hkv, int d, int splits, float scale, int dtype, int kv_dtype, const float* k_dq, const float* v_dq,
                              const int* block_tables, int max_blocks, int block_size, cudaStream_t s) {
  using namespace decode;
  if (d != D || h % hkv || (dtype != kBF16 && dtype != kF16) || (kv_dtype != kI8 && kv_dtype != kE4M3)) return 1;
  if (!block_tables || !k_dq || !v_dq || max_blocks <= 0 || block_size <= 0) return 1;
  dim3 grid(splits, h, b);
  const float sl2 = scale * 1.4426950408889634f;
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    decode_split_q8_kernel<T, decltype(tag_kv)><<<grid, kThreads, 0, s>>>((const T*)q, (const uint8_t*)k_cache, (const uint8_t*)v_cache, lens,
                                                                          part_acc, part_ml, h, hkv, splits, sl2, k_dq, v_dq, block_tables,
                                                                          max_blocks, block_size);
    decode_merge_kernel<T><<<b * h, D, 0, s>>>(part_acc, part_ml, (T*)out, splits);
  };
  if (dtype == kBF16) {
    if (kv_dtype == kI8) launch(__nv_bfloat16(), kv8::I8()); else launch(__nv_bfloat16(), kv8::E4M3());
  } else {
    if (kv_dtype == kI8) launch(__half(), kv8::I8()); else launch(__half(), kv8::E4M3());
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

int decode_attention_paged_multi(const PagedMultiArgs& a, cudaStream_t s) {
  using namespace decode_multi;
  if (a.d != D || a.hkv <= 0 || a.h % a.hkv || a.h / a.hkv > kRows || (a.dtype != kBF16 && a.dtype != kF16)) return 1;
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
  const dim3 grid(a.splits, a.hkv, a.b), mgrid(kRows, a.hkv, a.b);
  auto launch = [&](auto tag_t, auto tag_kv) {
    using T = decltype(tag_t);
    using KV = decltype(tag_kv);
    constexpr int smem = Smem<!std::is_same<T, KV>::value>::kBytes;
    static bool attr = false;   // one flag per instantiation
    if (!attr) { B200_CUDA_CHECK(cudaFuncSetAttribute(multi_split_kernel<T, KV>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); attr = true; }
    multi_split_kernel<T, KV><<<grid, kThreads, smem, s>>>(p);
    multi_merge_kernel<T><<<mgrid, D, 0, s>>>(p);
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
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_last_error(__FILE__, __LINE__, cudaGetErrorString(e)); return 3; }
  return 0;
}

}  // namespace b200
