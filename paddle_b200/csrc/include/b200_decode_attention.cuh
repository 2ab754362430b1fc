// Bodies of the paged decode, verify and shared-prefix attention kernels (see decode_attention.cu for the algorithms).  Each body is a
// __device__ __forceinline__ template with a compile-time WINDOW flag, instantiated by the kernels of decode_attention.cu.
//
// Sliding window W (WINDOW = true): the query at absolute position i sees key j iff i - W < j <= i (W keys including itself), the mask
// of models trained with a local window (Mistral, Phi-3) and a way to bound a sequence's KV memory.  Only the key range and the left
// edge of the mask change:
// - decode: a split covers positions [max(0, len - W), len), so a call touches min(len, W) rows per query;
// - verify: the splits cover the key tiles from the one holding past - W + 1, and row r of token j masks keys below past + j - W + 1.
// Keys below the lowest bound of a CTA's rows are never loaded and their block-table entries never read, so blocks wholly below the
// window may hold NaN or belong to another sequence.
#pragma once
#include <cuda.h>
#include <type_traits>

#include "b200_common.cuh"
#include "b200_kv8.cuh"
#include "b200_ops.h"

namespace b200 {
namespace decode {

constexpr int kThreads = 128;

// Combine the CTA's per-thread online-softmax partials (m, l, acc) and write this split's partial (m, l, acc * v_scale).
template <int D>
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
  // sum the 128 per-thread accumulators: 4 rounds of 32 threads' vectors through shared memory, thread t < D owns output dim t
  float out = 0.f;
  for (int r = 0; r < kThreads / 32; ++r) {
    __syncthreads();
    if ((tid >> 5) == r) {
#pragma unroll
      for (int i = 0; i < D; ++i) sacc[tid & 31][i] = acc[i] * f;
    }
    __syncthreads();
    if (D < kThreads && tid >= D) continue;
#pragma unroll 8
    for (int j = 0; j < 32; ++j) out += sacc[j][tid];
  }
  const int64_t pi = ((int64_t)b * h + head) * splits + split;
  if (D == kThreads || tid < D) part_acc[pi * D + tid] = out * v_scale;
  if (tid == 0) { part_ml[pi * 2] = mg; part_ml[pi * 2 + 1] = lg; }
}

// The positions [p0, p1) of this split: the last `window` of the len cached ones with WINDOW, all of them otherwise
template <bool WINDOW>
__device__ __forceinline__ void split_range(int len, int splits, int window, int& p0, int& p1) {
  if constexpr (WINDOW) {
    const int lo = max(0, len - window);
    const int per = (len - lo + splits - 1) / splits;
    p0 = lo + (int)blockIdx.x * per;
    p1 = min(len, p0 + per);
  } else {
    const int per = (len + splits - 1) / splits;
    p0 = (int)blockIdx.x * per;
    p1 = min(len, p0 + per);
  }
}

template <typename T, int D, bool WINDOW>
__device__ __forceinline__ void decode_split(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc, const int* __restrict__ lens,
                                             float* __restrict__ part_acc, float* __restrict__ part_ml, int h, int hkv, int smax, int splits,
                                             float scale_log2, const int* __restrict__ block_tables, int max_blocks, int block_size, int window) {
  const int head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (h / hkv);
  const int len = block_tables ? min(lens[b], max_blocks * block_size) : min(lens[b], smax);
  int p0, p1;
  split_range<WINDOW>(len, splits, window, p0, p1);
  __shared__ float sq[D];
  __shared__ float red[kThreads];
  __shared__ float sacc[32][D + 1];           // one slice of the cross-thread reduction at a time
  const int tid = threadIdx.x;
  if (D == kThreads || tid < D) sq[tid] = to_f(q[((int64_t)b * h + head) * D + tid]) * scale_log2;
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
      if constexpr (WINDOW) {   // q re-read from shared memory every row, as in decode_split_q8 (the same FMAs): 128 q registers would spill
#pragma unroll
        for (int e = 0; e < 8; e += 4) {
          float4 qv;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(qv.x), "=f"(qv.y), "=f"(qv.z), "=f"(qv.w)
                       : "r"((uint32_t)__cvta_generic_to_shared(sq + c * 8 + e)));
          s = fmaf(to_f(kv.v[e]), qv.x, s);
          s = fmaf(to_f(kv.v[e + 1]), qv.y, s);
          s = fmaf(to_f(kv.v[e + 2]), qv.z, s);
          s = fmaf(to_f(kv.v[e + 3]), qv.w, s);
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) s = fmaf(to_f(kv.v[e]), sq[c * 8 + e], s);
      }
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
  split_epilogue<D>(m, l, acc, red, sacc, part_acc, part_ml, h, splits, 1.f);
}

// Paged 8-bit caches (KV = kv8::I8 / kv8::E4M3): one 16-byte load carries 16 elements.  The K dequant scale is folded into sq, the V
// dequant scale is applied once to the split's partial output; with power-of-two scales the result is bit-identical to
// decode_split on a 16-bit cache holding the dequantized values.
template <typename T, typename KV, bool WINDOW>
__device__ __forceinline__ void decode_split_q8(const T* __restrict__ q, const uint8_t* __restrict__ kc, const uint8_t* __restrict__ vc,
                                                const int* __restrict__ lens, float* __restrict__ part_acc, float* __restrict__ part_ml, int h, int hkv,
                                                int splits, float scale_log2, const float* __restrict__ k_dq, const float* __restrict__ v_dq,
                                                const int* __restrict__ block_tables, int max_blocks, int block_size, int window) {
  constexpr int D = 128;
  const int head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (h / hkv);
  const int len = min(lens[b], max_blocks * block_size);
  int p0, p1;
  split_range<WINDOW>(len, splits, window, p0, p1);
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
  split_epilogue<D>(m, l, acc, red, sacc, part_acc, part_ml, h, splits, __ldg(v_dq + kvh));
}

template <typename T, int D>
__device__ __forceinline__ void decode_merge(const float* __restrict__ part_acc, const float* __restrict__ part_ml, T* __restrict__ out, int splits) {
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

namespace decode_multi {

constexpr int BN = 64, kRows = 64, kThreads = 128, kStages = 3;
// one K or V tile of 64 keys: 16 KB in 16 bits, 8 KB in 8 bits at D = 128
template <int D> constexpr int kTile16 = BN * D * 2;
template <int D> constexpr int kTile8 = BN * D;

struct Params {
  const void* q; const void* k_cache; const void* v_cache;
  void* out; float* part_acc; float* part_ml;   // part_acc: [B, Hkv, splits, 64 rows, D]
  const int* block_tables; const int* cu_q; const int* n_q; const int* past;
  const float* k_dq; const float* v_dq;
  int64_t q_st, q_sh, o_st;   // element strides: q (token, head), out (token; heads are D apart)
  int h, hkv, splits, max_blocks, block_size;
  float scale_log2;
  int window;                 // > 0: sliding window (read by the WINDOW kernels only)
};

// shared memory: Q tile [64][D] 16-bit | K, V 16-bit tiles (kStages, or 1 for 8-bit caches) | 8-bit caches: raw K, V tiles (kStages).
// Two tiles stay in flight while one is computed; two CTAs fit on an SM at D = 128.
template <bool Q8, int D> struct Smem {
  static constexpr int kKV = kRows * D * 2;
  static constexpr int kRaw = kKV + (Q8 ? 1 : kStages) * 2 * kTile16<D>;
  static constexpr int kBytes = kRaw + (Q8 ? kStages * 2 * kTile8<D> : 0);
};

// byte offset of 16-byte chunk c (0 .. D / 8 - 1) of row `row` in a [rows][D] 16-bit tile; the XOR spreads 8 consecutive rows over all banks
template <int D>
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

// The split kernel's body for head size D, inlined into the verify kernels (multi_split_kernel) and, with SHARED, into the
// shared-prefix kernel (decode_shared::shared_split_kernel, P = decode_shared::Params).  KV = T: 16-bit caches; KV = kv8::I8 /
// kv8::E4M3: 8-bit caches with fp32 [Hkv] dequant scales (D = 128 only).  The two kinds differ only in
// - the key range [lo, hi): verify rows see the keys of their own sequence below past + n_q, in absolute 64-key tiles; a shared task
//   sees the keys [lo, hi) of its task, in tiles from lo;
// - where Q row r comes from: token r / G of the sequence, or member r / G of the group;
// - the mask: bottom-right causal per token (and, with WINDOW, the window's left edge), or none below hi;
// - where the partials go: the split's 64 rows of the sequence, or the task's rows (an empty task split writes an empty partial).
// WINDOW: the splits cover the key tiles from the one holding past - window + 1 (the first token's lowest key); keys below it are
// zero-filled without reading their table entries, and row r of token j also masks the keys below past + j - window + 1.
template <typename T, typename KV, int D, bool WINDOW = false, bool SHARED = false, typename P>
__device__ __forceinline__ void multi_split(const P& p, int window = 0) {
  constexpr bool Q8 = !std::is_same<T, KV>::value;
  static_assert(D == 128 || (D == 64 && !Q8), "head_dim 128, or 64 on 16-bit caches");
  static_assert(!SHARED || (D == 128 && !WINDOW), "shared-prefix decode is head_dim 128 and unwindowed");
  constexpr int kTile16 = decode_multi::kTile16<D>, kTile8 = decode_multi::kTile8<D>;
  using S = Smem<Q8, D>;
  constexpr int kQShift = D == 128 ? 4 : 3;                  // log2 of the 16-byte chunks of a Q row
  extern __shared__ __align__(128) uint8_t smem[];
  // The prologue of each kind, in the order its kernel has always computed it (the order of the loads shapes ptxas's schedule).
  // keys at or past hi are never loaded: verify rows' len, or the end of a shared task's keys.  lo: a shared task's first key, or with
  // WINDOW the lowest key any verify row sees
  int split, kvh, b = 0, g_size, nrows, t0, t1, hi, lo = 0, past = 0, cu = 0, m0 = 0, tid, warp, lane;
  int64_t pbase = 0;
  uint32_t sbase;
  const int* bt;
  if constexpr (SHARED) {
    const int* task = p.tasks + (int64_t)blockIdx.x * kSharedTaskInts;
    kvh = blockIdx.y;
    const int tb = task[0];
    m0 = task[1];
    const int cnt = task[2];
    lo = task[3];
    split = task[5];
    const int splits = task[6];
    g_size = p.h / p.hkv;
    nrows = cnt * g_size;
    const int cap = p.max_blocks * p.block_size, len_tb = p.lens[tb];
    // prefix: keys below prefix_len, never past the reference member's cached ones (a bad group is NaN-ed by the merge); suffix: up to len
    hi = task[4] >= 0 ? min(min(task[4], len_tb - 1), cap) : min(len_tb, cap);
    const int ntiles = hi > lo ? (hi - lo + BN - 1) / BN : 0, per = (ntiles + splits - 1) / splits;
    t0 = split * per;
    t1 = min(ntiles, t0 + per);
    pbase = (int64_t)kvh * p.rows + task[7];
    tid = threadIdx.x; warp = tid >> 5; lane = tid & 31;
    if (t0 >= t1) {                                          // no keys: an empty partial (the merge skips it)
      for (int r = tid; r < nrows; r += kThreads) { p.part_ml[(pbase + r) * 2] = -INFINITY; p.part_ml[(pbase + r) * 2 + 1] = 0.f; }
      return;
    }
    sbase = (uint32_t)__cvta_generic_to_shared(smem);
    bt = p.block_tables + (int64_t)tb * p.max_blocks;
  } else {
    split = blockIdx.x;
    kvh = blockIdx.y;
    b = blockIdx.z;
    const int nq = p.n_q[b];
    g_size = p.h / p.hkv;
    nrows = nq * g_size;
    if (nq <= 0 || nrows > kRows) return;                    // skipped, or past the row limit (multi_merge_kernel writes NaN)
    past = p.past[b];
    hi = min(past + nq, p.max_blocks * p.block_size);
    if constexpr (WINDOW) {
      lo = max(0, past - window + 1);
      const int first = lo / BN, ntiles = (hi + BN - 1) / BN, per = (ntiles - first + p.splits - 1) / p.splits;
      t0 = first + split * per;
      t1 = min(ntiles, t0 + per);
    } else {
      const int ntiles = (hi + BN - 1) / BN, per = (ntiles + p.splits - 1) / p.splits;
      t0 = split * per;
      t1 = min(ntiles, t0 + per);
    }
    sbase = (uint32_t)__cvta_generic_to_shared(smem);
    tid = threadIdx.x; warp = tid >> 5; lane = tid & 31;
    bt = p.block_tables + (int64_t)b * p.max_blocks;
    cu = p.cu_q[b];
  }
  const int key0 = SHARED ? lo : 0;                          // the first key of tile 0

  // Q tile: rows past nrows are zero
#pragma unroll
  for (int i = 0; i < kRows * D / 8 / kThreads; ++i) {
    const int row = i * (kThreads >> kQShift) + (tid >> kQShift), c = tid & ((1 << kQShift) - 1);
    const bool ok = row < nrows;
    const T* src = reinterpret_cast<const T*>(p.q);
    if (ok) {
      int token;
      if constexpr (SHARED) token = p.cu_q[p.group_seqs[m0 + row / g_size]];
      else token = cu + row / g_size;
      src += (int64_t)token * p.q_st + (int64_t)(kvh * g_size + row % g_size) * p.q_sh + c * 8;
    }
    cp_async16(sbase + swz<D>(row, c), src, ok);
  }
  // cached K / V rows of key tile `tile` into stage `st`; keys at or past hi (and below lo with WINDOW) are zero-filled
  auto load_kv = [&](int tile, int st) {
    constexpr int kEl = Q8 ? 16 : 8;                         // elements per 16-byte chunk
    constexpr int kChunks = D / kEl;
#pragma unroll
    for (int i = 0; i < BN * kChunks / kThreads; ++i) {
      const int row = i * (kThreads / kChunks) + tid / kChunks, c = tid % kChunks;
      const int pos = key0 + tile * BN + row;
      const bool ok = WINDOW ? pos < hi && pos >= lo : pos < hi;
      int64_t off = 0;
      if (ok) off = (((int64_t)bt[pos / p.block_size] * p.hkv + kvh) * p.block_size + pos % p.block_size) * D + c * kEl;
      if constexpr (Q8) {
        const uint32_t dst = sbase + S::kRaw + st * 2 * kTile8 + row * D + c * 16;
        cp_async16(dst, reinterpret_cast<const uint8_t*>(p.k_cache) + off, ok);
        cp_async16(dst + kTile8, reinterpret_cast<const uint8_t*>(p.v_cache) + off, ok);
      } else {
        const uint32_t dst = sbase + S::kKV + st * 2 * kTile16 + swz<D>(row, c);
        cp_async16(dst, reinterpret_cast<const T*>(p.k_cache) + off, ok);
        cp_async16(dst + kTile16, reinterpret_cast<const T*>(p.v_cache) + off, ok);
      }
    }
  };
  if (SHARED || t0 < t1) load_kv(t0, 0);                     // (a shared task with no tile has returned)
  cp_async_commit();
  if (t0 + 1 < t1) load_kv(t0 + 1, 1);
  cp_async_commit();

  float qk_scale = p.scale_log2, v_scale = 1.f;
  if constexpr (Q8) { qk_scale *= __ldg(p.k_dq + kvh); v_scale = __ldg(p.v_dq + kvh); }
  const bool active = warp * 16 < nrows;
  const int r_lo = warp * 16 + (lane >> 2);                  // this lane's two rows: r_lo and r_lo + 8
  int limit[2];                                              // verify: keys < limit are visible to the row
  if constexpr (!SHARED) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) limit[hh] = min(hi, past + (r_lo + hh * 8) / g_size + 1);
  }
  int lower[2] = {0, 0};                                     // ... and keys >= lower (WINDOW)
  if constexpr (WINDOW) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) lower[hh] = past + (r_lo + hh * 8) / g_size - window + 1;
  }
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
      for (int kk = 0; kk < D / 16; ++kk) ldsm_x4(qf[kk], sbase + swz<D>(warp * 16 + (lane & 15), kk * 2 + (lane >> 4)));
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
        *reinterpret_cast<uint4*>(dst + swz<D>(row, 2 * c)) = make_uint4(w[0], w[1], w[2], w[3]);
        *reinterpret_cast<uint4*>(dst + swz<D>(row, 2 * c + 1)) = make_uint4(w[4], w[5], w[6], w[7]);
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
          ldsm_x4(bf, kv16 + swz<D>(np * 16 + (lane & 7) + ((lane >> 4) << 3), kk * 2 + ((lane >> 3) & 1)));
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
            const int key = key0 + t * BN + n * 8 + 2 * (lane & 3) + e;
            float& v = s[n][hh * 2 + e];
            const bool visible = SHARED ? key < hi : key < limit[hh] && (!WINDOW || key >= lower[hh]);   // SHARED: every key below hi
            v = visible ? v * qk_scale : -INFINITY;
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
          ldsm_x4_t(bf, kv16 + kTile16 + swz<D>(kk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3), np * 2 + (lane >> 4)));
          mma16816<T>(acc[2 * np], pa, bf[0], bf[1]);
          mma16816<T>(acc[2 * np + 1], pa, bf[2], bf[3]);
        }
      }
    }
  }
  cp_async_wait<0>();
  if (!active) return;
  // this split's partial for the warp's rows (an empty verify split writes m = -inf, l = 0, acc = 0)
  if constexpr (!SHARED) pbase = (((int64_t)b * p.hkv + kvh) * p.splits + split) * kRows;
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

// grid (64 rows, Hkv, B), D threads: combines the splits of one query row, as decode_merge does, and writes it in place.  A
// sequence over the row limit gets NaN rows rather than a silently partial result.
template <typename T, int D>
__device__ __forceinline__ void multi_merge(const Params& p) {
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
}  // namespace b200
