// Token sampling for sm_90a: one launch picks the next token of every row of a [rows, vocab] logits (or probability) matrix.
//
// One CTA samples one row, reading it in place with any row stride.  Per-row parameters are device arrays (no host read, no workspace:
// the launch can be captured in a CUDA graph).  The rules are defined by value, never by sort order:
//   greedy (temperature <= 0)  argmax, lowest index among equal values
//   top_k (0 = off)            keep every token whose value is >= the k-th largest value (ties kept)
//   top_p (1 = off)            with w_i = exp(logit_i / T - max) (probabilities: w_i = p_i) over the top-k set and Z = sum w, keep token i
//                              when the mass of the strictly larger tokens is <= top_p * Z
//   draw                       exponential race: argmax over kept tokens of s_i - log(-log u_i), s_i = logit_i / T (probabilities: log p_i)
//   threshold (optional)       non-truncated: tokens below it (but the top-1) leave the race; truncated: a winner below it (but the top-1)
//                              falls back to the smallest kept token >= threshold, or to the top-1 when there is none
// u_i depends only on (seed, offset, i): Philox4x32-10, key (seed lo, seed hi), counter (i >> 2, 0, offset lo, offset hi), word i & 3,
// u = ((w >> 8) + 0.5) * 2^-24.  kernels/sampling.py:sample_ref computes the same stream with int64 torch ops.
//
// No sort: the top-k and top-p cutoffs are found by radix select on an order-preserving 32-bit key of the value (11-bit digits, 2048-bin
// shared-memory histograms of counts, or of mass for top-p; the key's low bits that are zero for every value of the input type are
// skipped: fp32 has 32 significant key bits (three digits), fp16 19 and bf16 16 (two digits)).  Each digit
// re-reads the row, which stays in L2 (a 152064-token fp32 row is 594 KB: more than shared memory).  Passes per row: 1 (greedy),
// 1 + 2-3 (top_k), 1 + 2-3 (top_p), the race; top_k's first digit rides on the argmax pass.
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"
#include "include/b200_philox.cuh"

namespace b200 {
namespace {

constexpr int kThreads = 1024;
constexpr int kDigit = 11;
constexpr int kBins = 1 << kDigit;
constexpr int kMaxTop = 1024;          // return_top: at most this many sorted candidates per row

struct SampleSmem {
  int cnt[kBins];
  float mass[kBins];
  union { int i[kThreads]; float f[kThreads]; } scan;
  unsigned long long red[32];
  int bin, low_bin;
  int above_i;
  float above_f, total_f;
  uint32_t top_key[kMaxTop];
  int top_idx[kMaxTop];
  int warp_cnt[32];
};

__device__ __forceinline__ uint4 philox_quad(int64_t seed, int64_t offset, uint32_t quad) {
  return philox4x32_10(make_uint4(quad, 0u, (uint32_t)offset, (uint32_t)((uint64_t)offset >> 32)), (uint32_t)seed,
                       (uint32_t)((uint64_t)seed >> 32));
}

__device__ __forceinline__ uint32_t word_of(const uint4& w, int j) { return j == 0 ? w.x : j == 1 ? w.y : j == 2 ? w.z : w.w; }

// (0, 1), exact in fp32: 2^24 evenly spaced points
__device__ __forceinline__ float uniform_of(uint32_t w) { return ((float)(w >> 8) + 0.5f) * 5.9604644775390625e-8f; }

// order-preserving key: a < b (as floats, -0 == +0) <=> key(a) < key(b)
__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t b = __float_as_uint(v == 0.f ? 0.f : v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// four consecutive values starting at token 4q (-inf past the end); 8 / 16-byte loads when the row is aligned
template <typename T>
__device__ __forceinline__ void load_quad(const T* __restrict__ x, int q, int V, bool vec, float v[4]) {
  const int i0 = q * 4;
  if (vec && i0 + 4 <= V) {
    if constexpr (sizeof(T) == 4) {
      const float4 f = __ldg(reinterpret_cast<const float4*>(x + i0));
      v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(x + i0));
      const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = to_f(h[j]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = i0 + j < V ? to_f(x[i0 + j]) : -INFINITY;
  }
}

// f(token index, value, key) for every token of the row
template <typename T, typename F>
__device__ __forceinline__ void for_each_token(const T* __restrict__ x, int V, bool vec, F&& f) {
  const int nq = (V + 3) >> 2;
  for (int q = threadIdx.x; q < nq; q += kThreads) {
    float v[4];
    load_quad(x, q, V, vec, v);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (q * 4 + j < V) f(q * 4 + j, v[j], order_key(v[j]));
  }
}

__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, SampleSmem& sm) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xffffffffu, v, o); v = y > v ? y : v; }
  if (lane == 0) sm.red[wid] = v;
  __syncthreads();
  v = sm.red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long y = __shfl_xor_sync(0xffffffffu, v, o); v = y > v ? y : v; }
  __syncthreads();
  return v;
}

// Scans the histogram h[0, nbins) from the top bin down, starting from `base` (what lies above it).  The chosen bin is the first whose
// running total crosses `target` (counts: >= target; mass: > target; with scale >= 0 the target is scale * the histogram's total).  If no
// bin crosses (fp32 rounding in a later mass digit), the lowest non-empty bin is chosen, which keeps the whole bucket.  Leaves sm.bin and
// sm.above_* = base + the total of the bins above the chosen one, and sm.total_f; every thread must call it.
template <typename V, bool STRICT>
__device__ void find_bin(SampleSmem& sm, const V* h, int nbins, V base, V target, float scale) {
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int per = nbins > kThreads ? nbins / kThreads : 1;          // 2 or 1
  V loc[2] = {V(0), V(0)};
  V sum = V(0);
  for (int j = 0; j < per; ++j) {
    const int d = t * per + j;
    loc[j] = d < nbins ? h[nbins - 1 - d] : V(0);
    sum += loc[j];
  }
  V incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const V y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  V* ws = reinterpret_cast<V*>(sm.red);
  if (lane == 31) ws[wid] = incl;
  if (t == 0) { sm.bin = -1; sm.low_bin = 0x7FFFFFFF; }
  __syncthreads();
  if (wid == 0) {
    V w = ws[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const V y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    ws[32 + lane] = w;
  }
  __syncthreads();
  V* cum = reinterpret_cast<V*>(sm.scan.i);
  cum[t] = (wid ? ws[32 + wid - 1] : V(0)) + incl;                   // the running total after this thread's bins
  __syncthreads();
  const V total = cum[kThreads - 1];
  if (scale >= 0.f) target = (V)(scale * (float)total);
  // A thread crosses when its bins take the running total (base + cum) across the target; start and end come from the same array as
  // its neighbours', so some thread crosses whenever the whole histogram does.  Of several (a non-monotone fp32 scan), the top bin wins.
  auto crosses = [&](V s) { return STRICT ? s > target : s >= target; };
  const V start = base + (t ? cum[t - 1] : V(0));
  if (crosses(base + cum[t]) && !crosses(start)) {
    int mine = -1;
    V acc = start;
    for (int j = 0; j < per && t * per + j < nbins; ++j) {
      if (loc[j] > V(0)) mine = nbins - 1 - (t * per + j);        // no bin crosses on its own: the thread's lowest non-empty one
      acc += loc[j];
      if (crosses(acc)) break;
    }
    atomicMax(&sm.bin, mine);
  }
  for (int j = 0; j < per; ++j)                                       // the fallback: lowest non-empty bin
    if (t * per + j < nbins && loc[j] > V(0)) atomicMin(&sm.low_bin, nbins - 1 - (t * per + j));
  __syncthreads();
  if (sm.bin < 0) {                                                   // nothing crosses: keep the whole bucket
    __syncthreads();
    if (t == 0) sm.bin = sm.low_bin == 0x7FFFFFFF ? 0 : sm.low_bin;
    __syncthreads();
  }
  const int b = sm.bin;
  const int d = nbins - 1 - b;
  if (d / per == t && d < nbins) {                                    // the owner of the chosen bin reports what lies above it
    V a2 = base + (t ? cum[t - 1] : V(0));
    for (int j = 0; j < d - t * per; ++j) a2 += loc[j];
    if constexpr (std::is_same<V, float>::value) sm.above_f = a2;
    else sm.above_i = a2;
  }
  if (t == 0) sm.total_f = (float)total;
  __syncthreads();
}

// The key's lowest bit that can be set for a value of type T: the selects stop there, so their cutoffs are exact keys.  fp16 -> fp32
// keeps 10 mantissa bits (the low 13 key bits are zero), bf16 -> fp32 keeps 7 (low 16 zero).
template <typename T>
__device__ constexpr int key_low_bit() { return std::is_same<T, __half>::value ? 13 : std::is_same<T, __nv_bfloat16>::value ? 16 : 0; }

// The key whose bits above `low` are `prefix`: the skipped bits are 0 for a non-negative value and 1 for a negative one (key = ~bits).
__device__ __forceinline__ uint32_t full_key(uint32_t prefix, int low) {
  const uint32_t k = prefix << low;
  return (k & 0x80000000u) ? k : k | ((1u << low) - 1u);
}

__device__ __forceinline__ bool prefix_match(uint32_t key, int hi, uint32_t prefix) { return hi >= 32 || (key >> hi) == prefix; }

// Smallest key among the K largest (K <= V): radix select on counts.  With first_done, sm.cnt already holds the first digit's histogram.
template <typename T>
__device__ uint32_t kth_key(SampleSmem& sm, const T* __restrict__ x, int V, bool vec, int K, bool first_done) {
  constexpr int LOW = key_low_bit<T>();
  uint32_t prefix = 0;
  int need = K;
  for (int hi = 32; hi > LOW;) {
    const int bits = min(kDigit, hi - LOW), shift = hi - bits;
    if (!(first_done && hi == 32)) {
      for (int i = threadIdx.x; i < (1 << bits); i += kThreads) sm.cnt[i] = 0;
      __syncthreads();
      for_each_token(x, V, vec, [&](int, float, uint32_t key) {
        if (prefix_match(key, hi, prefix)) atomicAdd(&sm.cnt[(key >> shift) & ((1u << bits) - 1)], 1);
      });
      __syncthreads();
    }
    find_bin<int, false>(sm, sm.cnt, 1 << bits, 0, need, -1.f);
    need -= sm.above_i;
    prefix = (prefix << bits) | (uint32_t)sm.bin;
    hi = shift;
  }
  return full_key(prefix, LOW);
}

template <typename T, bool PROB>
__global__ void __launch_bounds__(kThreads, 1) sample_kernel(const SampleArgs a) {
  __shared__ SampleSmem sm;
  constexpr int LOW = key_low_bit<T>();
  const int row = blockIdx.x, t = threadIdx.x, V = a.vocab;
  const T* __restrict__ x = reinterpret_cast<const T*>(a.x) + (int64_t)row * a.stride;
  const bool vec = (reinterpret_cast<uintptr_t>(x) & (4 * sizeof(T) - 1)) == 0;
  const float temp = a.temperature[row], top_p = a.top_p[row];
  const int top_k = a.top_k[row];
  const bool greedy = !(temp > 0.f);
  const bool k_on = !greedy && top_k > 0 && top_k < V;
  const bool p_on = !greedy && top_p < 1.f;

  // pass 1: argmax (highest key, then lowest index) and top_k's first digit
  if (k_on)
    for (int i = t; i < kBins; i += kThreads) sm.cnt[i] = 0;
  __syncthreads();
  unsigned long long best = 0;
  for_each_token(x, V, vec, [&](int i, float, uint32_t key) {
    const unsigned long long pk = ((unsigned long long)key << 32) | (0xFFFFFFFFu - (uint32_t)i);
    best = pk > best ? pk : best;
    if (k_on) atomicAdd(&sm.cnt[key >> (32 - kDigit)], 1);
  });
  __syncthreads();
  best = block_max_u64(best, sm);
  const int top1 = (int)(0xFFFFFFFFu - (uint32_t)best);
  int id = top1;

  if (!greedy) {
    uint32_t cut = k_on ? kth_key(sm, x, V, vec, top_k, true) : 0u;
    const float vmax = to_f(x[top1]);
    const float smax = PROB ? 0.f : vmax / temp;
    auto weight = [&](float v) { return PROB ? v : expf(v / temp - smax); };
    if (p_on) {                                                      // radix select on mass over the top-k set
      const uint32_t kc = cut;
      uint32_t prefix = 0;
      float above = 0.f, target = 0.f;
      for (int hi = 32; hi > LOW;) {
        const int bits = min(kDigit, hi - LOW), shift = hi - bits;
        for (int i = t; i < (1 << bits); i += kThreads) sm.mass[i] = 0.f;
        __syncthreads();
        for_each_token(x, V, vec, [&](int, float v, uint32_t key) {
          if (key >= kc && prefix_match(key, hi, prefix)) atomicAdd(&sm.mass[(key >> shift) & ((1u << bits) - 1)], weight(v));
        });
        __syncthreads();
        find_bin<float, true>(sm, sm.mass, 1 << bits, above, target, hi == 32 ? top_p : -1.f);
        if (hi == 32) target = top_p * sm.total_f;
        above = sm.above_f;
        prefix = (prefix << bits) | (uint32_t)sm.bin;
        hi = shift;
      }
      cut = max(cut, full_key(prefix, LOW));
    }

    // the race, and the truncated-threshold fallback (smallest kept token >= threshold, lowest index)
    const bool thr_on = a.threshold != nullptr;
    const float thr = thr_on ? a.threshold[row] : 0.f;
    const bool thr_race = thr_on && !a.truncated, thr_fall = thr_on && a.truncated;
    unsigned long long win = 0, low = ~0ull;
    const int nq = (V + 3) >> 2;
    for (int q = t; q < nq; q += kThreads) {
      float v[4];
      load_quad(x, q, V, vec, v);
      bool in[4], any = false;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = q * 4 + j;
        const uint32_t key = order_key(v[j]);
        in[j] = i < V && key >= cut;
        if (in[j] && thr_fall && v[j] >= thr) {
          const unsigned long long pk = ((unsigned long long)key << 32) | (uint32_t)i;
          low = pk < low ? pk : low;
        }
        in[j] = in[j] && (!thr_race || v[j] >= thr || i == top1);
        any |= in[j];
      }
      if (!any) continue;
      const uint4 w = philox_quad(a.seed[row], a.offset[row], (uint32_t)q);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!in[j]) continue;
        const float s = PROB ? logf(v[j]) : v[j] / temp;
        const float r = s - logf(-logf(uniform_of(word_of(w, j))));
        const unsigned long long pk = ((unsigned long long)order_key(r) << 32) | (0xFFFFFFFFu - (uint32_t)(q * 4 + j));
        win = pk > win ? pk : win;
      }
    }
    win = block_max_u64(win, sm);
    low = ~block_max_u64(~low, sm);
    id = win ? (int)(0xFFFFFFFFu - (uint32_t)win) : top1;
    if (thr_fall && id != top1 && to_f(x[id]) < thr) id = low != ~0ull ? (int)(uint32_t)low : top1;
  }
  if (t == 0) {
    a.ids[row] = id;
    reinterpret_cast<T*>(a.vals)[row] = x[id];
  }

  // return_top: the k_out largest values, descending, ties by lowest index
  if (a.k_out > 0) {
    const int k = min(a.k_out, V);
    const uint32_t kt = kth_key(sm, x, V, vec, k, false);
    if (t == 0) sm.above_i = 0;
    __syncthreads();
    for_each_token(x, V, vec, [&](int i, float, uint32_t key) {
      if (key > kt) {
        const int slot = atomicAdd(&sm.above_i, 1);                 // < k: kt is the exact k-th largest key
        if (slot < k) {
          sm.top_key[slot] = key;
          sm.top_idx[slot] = i;
        }
      }
    });
    __syncthreads();
    int filled = sm.above_i;                                          // < k
    const int lane = t & 31, wid = t >> 5;
    for (int c = 0; c * kThreads < V && filled < k; ++c) {            // ties at the k-th value, in index order
      const int i = c * kThreads + t;
      const bool eq = i < V && order_key(to_f(x[i])) == kt;
      const unsigned m = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) sm.warp_cnt[wid] = __popc(m);
      __syncthreads();
      int pos = filled + __popc(m & ((1u << lane) - 1));
      int tot = 0;
      for (int w2 = 0; w2 < 32; ++w2) {
        if (w2 < wid) pos += sm.warp_cnt[w2];
        tot += sm.warp_cnt[w2];
      }
      if (eq && pos < k) { sm.top_key[pos] = kt; sm.top_idx[pos] = i; }
      filled += tot;
      __syncthreads();
    }
    if (t < k) {
      const uint32_t mk = sm.top_key[t];
      const int mi = sm.top_idx[t];
      int rank = 0;
      for (int j = 0; j < k; ++j) rank += sm.top_key[j] > mk || (sm.top_key[j] == mk && sm.top_idx[j] < mi);
      reinterpret_cast<T*>(a.top_vals)[(int64_t)row * a.k_out + rank] = x[mi];
      a.top_ids[(int64_t)row * a.k_out + rank] = mi;
    }
  }
}

__global__ void uniforms_kernel(int64_t seed, int64_t offset, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = uniform_of(word_of(philox_quad(seed, offset, (uint32_t)(i >> 2)), i & 3));
}

}  // namespace

int sample_tokens(const SampleArgs& a, cudaStream_t s) {
  if (a.rows <= 0) return 0;
  if (a.vocab <= 0 || a.rows > 0x7FFFFFFF || a.k_out < 0 || a.k_out > kMaxTop) return 1;
  B200_DISPATCH_DTYPE(a.dtype, T, {
    if (a.is_prob) sample_kernel<T, true><<<(unsigned)a.rows, kThreads, 0, s>>>(a);
    else sample_kernel<T, false><<<(unsigned)a.rows, kThreads, 0, s>>>(a);
  });
  B200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int sample_max_top() { return kMaxTop; }

void sampling_uniforms(int64_t seed, int64_t offset, int n, float* out, cudaStream_t s) {
  if (n <= 0) return;
  uniforms_kernel<<<(n + 255) / 256, 256, 0, s>>>(seed, offset, n, out);
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
