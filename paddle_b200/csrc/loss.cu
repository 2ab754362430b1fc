// Fused softmax + cross-entropy (single device and vocab-parallel pieces) for sm_90a.
// Parity (behaviour): paddle/phi/kernels/gpu/cross_entropy_kernel.cu, c_softmax_with_cross_entropy_kernel.cu.
// One CTA per row, one streaming pass (online softmax), fp32 math; backward is one read + one write and may run
// in place over the logits buffer.
#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

static constexpr int kCEThreads = 512;

__device__ __forceinline__ void online_combine(float& m, float& s, float m2, float s2) {
  // A part whose max is -inf holds no mass.  Skip it: for a vector of masked (-inf) logits, s2 = exp(-inf - -inf) = NaN,
  // and NaN * exp(-inf - m) would turn a finite running sum into NaN.
  if (m2 == -INFINITY) return;
  const float nm = fmaxf(m, m2);
  if (nm == -INFINITY) { s = 0.f; m = nm; return; }
  s = s * __expf(m - nm) + s2 * __expf(m2 - nm);
  m = nm;
}

// block-wide (max, sumexp) reduction
__device__ __forceinline__ void block_online(float& m, float& s, float* sm_m, float* sm_s) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    online_combine(m, s, m2, s2);
  }
  if (lane == 0) { sm_m[wid] = m; sm_s[wid] = s; }
  __syncthreads();
  m = lane < nw ? sm_m[lane] : -INFINITY;
  s = lane < nw ? sm_s[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    online_combine(m, s, m2, s2);
  }
  __syncthreads();
}

template <typename T>
__device__ __forceinline__ void row_online(const T* __restrict__ xr, int vocab, float& m, float& s) {
  constexpr int N = Vec16<T>::N;
  constexpr int U = 4;  // 4 independent 16B loads in flight per thread
  m = -INFINITY; s = 0.f;
  const int nvec = ((vocab * (int)sizeof(T)) % 16 == 0) ? vocab / N : 0;  // rows stay 16B-aligned only then
  for (int v0 = threadIdx.x; v0 < nvec; v0 += blockDim.x * U) {
    Vec16<T> xv[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int v = v0 + k * blockDim.x;
      if (v < nvec) xv[k] = ld16_stream(xr + v * N);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int v = v0 + k * blockDim.x;
      if (v < nvec) {
        float lm = -INFINITY;
#pragma unroll
        for (int j = 0; j < N; ++j) lm = fmaxf(lm, to_f(xv[k].v[j]));
        float ls = 0.f;
#pragma unroll
        for (int j = 0; j < N; ++j) ls += __expf(to_f(xv[k].v[j]) - lm);
        online_combine(m, s, lm, ls);
      }
    }
  }
  for (int c = nvec * N + threadIdx.x; c < vocab; c += blockDim.x) online_combine(m, s, to_f(xr[c]), 1.f);
}

template <typename T>
__global__ void __launch_bounds__(kCEThreads) softmax_ce_fwd_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels,
                                                                     float* __restrict__ loss, float* __restrict__ lse_out,
                                                                     int vocab, int64_t ignore_index) {
  __shared__ float sm_m[32], sm_s[32];
  const int64_t row = blockIdx.x;
  const T* xr = logits + row * vocab;
  float m, s;
  row_online(xr, vocab, m, s);
  block_online(m, s, sm_m, sm_s);
  if (threadIdx.x == 0) {
    const float lse = m + __logf(s);
    lse_out[row] = lse;
    const int64_t lab = labels[row];
    loss[row] = (lab == ignore_index || lab < 0 || lab >= vocab) ? 0.f : lse - to_f(xr[lab]);
  }
}

template <typename T>
__global__ void __launch_bounds__(kCEThreads) softmax_ce_bwd_kernel(const T* logits, const int64_t* __restrict__ labels,
                                                                     const float* __restrict__ lse, const float* __restrict__ dloss,
                                                                     T* dlogits, int vocab, int64_t ignore_index) {
  constexpr int N = Vec16<T>::N;
  const int64_t row = blockIdx.x;
  const T* xr = logits + row * vocab;
  T* gr = dlogits + row * vocab;
  const int64_t lab = labels[row];
  const bool ignored = (lab == ignore_index || lab < 0 || lab >= vocab);
  const float g = ignored ? 0.f : dloss[row];
  const float l = lse[row];
  const int nvec = ((vocab * (int)sizeof(T)) % 16 == 0) ? vocab / N : 0;  // rows stay 16B-aligned only then
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    Vec16<T> xv = ld16(xr + v * N), o;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      float p = __expf(to_f(xv.v[j]) - l);
      if (v * N + j == lab) p -= 1.f;
      o.v[j] = from_f<T>(p * g);
    }
    st16(gr + v * N, o);
  }
  for (int c = nvec * N + threadIdx.x; c < vocab; c += blockDim.x) {
    float p = __expf(to_f(xr[c]) - l);
    if (c == lab) p -= 1.f;
    gr[c] = from_f<T>(p * g);
  }
}

void softmax_ce_fwd(const void* logits, const int64_t* labels, float* loss, float* lse, int64_t rows, int vocab,
                    int64_t ignore_index, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (softmax_ce_fwd_kernel<T><<<(unsigned)rows, kCEThreads, 0, s>>>((const T*)logits, labels, loss, lse, vocab, ignore_index)));
  B200_CUDA_CHECK(cudaGetLastError());
}

void softmax_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* dloss, void* dlogits,
                    int64_t rows, int vocab, int64_t ignore_index, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (softmax_ce_bwd_kernel<T><<<(unsigned)rows, kCEThreads, 0, s>>>((const T*)logits, labels, lse, dloss, (T*)dlogits, vocab, ignore_index)));
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ vocab parallel
template <typename T>
__global__ void __launch_bounds__(kCEThreads) vp_max_kernel(const T* __restrict__ logits, float* __restrict__ row_max, int vocab) {
  __shared__ float red[33];
  constexpr int N = Vec16<T>::N;
  const T* xr = logits + (int64_t)blockIdx.x * vocab;
  float m = -INFINITY;
  const int nvec = ((vocab * (int)sizeof(T)) % 16 == 0) ? vocab / N : 0;  // rows stay 16B-aligned only then
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    Vec16<T> xv = ld16(xr + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) m = fmaxf(m, to_f(xv.v[j]));
  }
  for (int c = nvec * N + threadIdx.x; c < vocab; c += blockDim.x) m = fmaxf(m, to_f(xr[c]));
  m = block_max(m, red);
  if (threadIdx.x == 0) row_max[blockIdx.x] = m;
}

template <typename T>
__global__ void __launch_bounds__(kCEThreads) vp_sumexp_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels,
                                                                const float* __restrict__ row_max, float* __restrict__ sumexp,
                                                                float* __restrict__ target_logit, int vocab, int64_t vocab_start) {
  __shared__ float red[33];
  constexpr int N = Vec16<T>::N;
  const int64_t row = blockIdx.x;
  const T* xr = logits + row * vocab;
  const float m = row_max[row];
  float s = 0.f;
  const int nvec = ((vocab * (int)sizeof(T)) % 16 == 0) ? vocab / N : 0;  // rows stay 16B-aligned only then
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    Vec16<T> xv = ld16(xr + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) s += __expf(to_f(xv.v[j]) - m);
  }
  for (int c = nvec * N + threadIdx.x; c < vocab; c += blockDim.x) s += __expf(to_f(xr[c]) - m);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    sumexp[row] = s;
    const int64_t lab = labels[row] - vocab_start;
    target_logit[row] = (lab >= 0 && lab < vocab) ? to_f(xr[lab]) : 0.f;
  }
}

template <typename T>
__global__ void __launch_bounds__(kCEThreads) vp_bwd_kernel(const T* logits, const int64_t* __restrict__ labels,
                                                             const float* __restrict__ row_max, const float* __restrict__ sumexp,
                                                             const float* __restrict__ dloss, T* dlogits, int vocab,
                                                             int64_t vocab_start, int64_t ignore_index) {
  constexpr int N = Vec16<T>::N;
  const int64_t row = blockIdx.x;
  const T* xr = logits + row * vocab;
  T* gr = dlogits + row * vocab;
  const int64_t glab = labels[row];
  const int64_t lab = glab - vocab_start;
  const float g = (glab == ignore_index) ? 0.f : dloss[row];
  const float m = row_max[row], inv = 1.f / sumexp[row];
  const int nvec = ((vocab * (int)sizeof(T)) % 16 == 0) ? vocab / N : 0;  // rows stay 16B-aligned only then
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    Vec16<T> xv = ld16(xr + v * N), o;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      float p = __expf(to_f(xv.v[j]) - m) * inv;
      if (v * N + j == lab) p -= 1.f;
      o.v[j] = from_f<T>(p * g);
    }
    st16(gr + v * N, o);
  }
  for (int c = nvec * N + threadIdx.x; c < vocab; c += blockDim.x) {
    float p = __expf(to_f(xr[c]) - m) * inv;
    if (c == lab) p -= 1.f;
    gr[c] = from_f<T>(p * g);
  }
}

void vocab_parallel_ce_stats(const void* logits, const int64_t* labels, float* row_max, int64_t rows, int vocab,
                             int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (vp_max_kernel<T><<<(unsigned)rows, kCEThreads, 0, s>>>((const T*)logits, row_max, vocab)));
  B200_CUDA_CHECK(cudaGetLastError());
}

void vocab_parallel_ce_sumexp(const void* logits, const int64_t* labels, const float* row_max, float* sumexp,
                              float* target_logit, int64_t rows, int vocab, int64_t vocab_start, int dtype,
                              cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (vp_sumexp_kernel<T><<<(unsigned)rows, kCEThreads, 0, s>>>((const T*)logits, labels, row_max, sumexp, target_logit, vocab, vocab_start)));
  B200_CUDA_CHECK(cudaGetLastError());
}

void vocab_parallel_ce_bwd(const void* logits, const int64_t* labels, const float* row_max, const float* sumexp,
                           const float* dloss, void* dlogits, int64_t rows, int vocab, int64_t vocab_start,
                           int64_t ignore_index, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (vp_bwd_kernel<T><<<(unsigned)rows, kCEThreads, 0, s>>>((const T*)logits, labels, row_max, sumexp, dloss, (T*)dlogits, vocab, vocab_start, ignore_index)));
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
