// Fused bias + dropout + residual-add and bias + activation for sm_90a (HBM-bound: one pass, 16-byte vectors, Philox per vector).
//
// Parity (behaviour): python/paddle/incubate/nn/functional/fused_dropout_add.py (paddle/phi/kernels/fusion/gpu/fused_dropout_add_kernel.cu),
// fused_bias_dropout_residual_layer_norm (the elementwise half; the LayerNorm half is csrc/norm.cu), fused_bias_act
// (paddle/phi/kernels/fusion/gpu/fused_bias_act_kernel.cu).
//   out = dropout(x + bias) * scale + y           mask (1 byte / element) kept for the backward
//   dx  = dout * mask * scale                     (dy = dout, dbias = column sum of dx: done by the caller)
//   out = act(x + bias)                           act: gelu / relu / silu, and the gated forms swiglu / geglu (out has cols / 2 columns)
#include <curand_kernel.h>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

static inline int ew_grid(int64_t work_items, int threads) {
  const int64_t blocks = (work_items + threads - 1) / threads;
  const int64_t cap = (int64_t)sm_count() * 8;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// one Philox stream per 16-byte vector: (seed, subsequence = vector index, offset) -> up to 8 uniforms
template <typename T>
__global__ void __launch_bounds__(256)
bias_dropout_add_kernel(const T* __restrict__ x, const T* __restrict__ bias, const T* __restrict__ y, T* __restrict__ out, uint8_t* __restrict__ mask, int64_t nvec,
                        int cols, float p, float scale, uint64_t seed, uint64_t offset) {
  constexpr int N = Vec16<T>::N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)i, offset, &st);
    float r[8];
    const float4 r0 = curand_uniform4(&st);
    r[0] = r0.x; r[1] = r0.y; r[2] = r0.z; r[3] = r0.w;
    if (N > 4) {
      const float4 r1 = curand_uniform4(&st);
      r[4] = r1.x; r[5] = r1.y; r[6] = r1.z; r[7] = r1.w;
    }
    const Vec16<T> vx = ld16_stream(x + i * N);
    Vec16<T> o;
    uint8_t m[N];
    Vec16<T> vb, vy;
    if (bias) vb = ld16(bias + (i * N) % cols);
    if (y) vy = ld16_stream(y + i * N);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      float v = to_f(vx.v[j]);
      if (bias) v += to_f(vb.v[j]);
      const bool keep = r[j] >= p;              // curand_uniform is in (0, 1]: p = 0 keeps everything
      m[j] = keep ? 1 : 0;
      v = keep ? v * scale : 0.f;
      if (y) v += to_f(vy.v[j]);
      o.v[j] = from_f<T>(v);
    }
    st16_stream(out + i * N, o);
    if (N == 8) *reinterpret_cast<uint2*>(mask + i * N) = *reinterpret_cast<const uint2*>(m);
    else *reinterpret_cast<uint32_t*>(mask + i * N) = *reinterpret_cast<const uint32_t*>(m);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) dropout_bwd_kernel(const T* __restrict__ dout, const uint8_t* __restrict__ mask, T* __restrict__ dx, int64_t nvec, float scale) {
  constexpr int N = Vec16<T>::N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const Vec16<T> g = ld16_stream(dout + i * N);
    uint8_t m[N];
    if (N == 8) *reinterpret_cast<uint2*>(m) = *reinterpret_cast<const uint2*>(mask + i * N);
    else *reinterpret_cast<uint32_t*>(m) = *reinterpret_cast<const uint32_t*>(mask + i * N);
    Vec16<T> o;
#pragma unroll
    for (int j = 0; j < N; ++j) o.v[j] = from_f<T>(m[j] ? to_f(g.v[j]) * scale : 0.f);
    st16_stream(dx + i * N, o);
  }
}

void bias_dropout_add_fwd(const void* x, const void* bias, const void* y, void* out, uint8_t* mask, int64_t n, int cols, float p, int upscale, uint64_t seed,
                          uint64_t offset, int dtype, cudaStream_t s) {
  if (n == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    if (n % N || cols % N) { set_last_error(__FILE__, __LINE__, "bias_dropout_add: element count and row width must be multiples of the 16B vector"); return; }
    const float scale = upscale ? (p < 1.f ? 1.f / (1.f - p) : 0.f) : 1.f;
    bias_dropout_add_kernel<T><<<ew_grid(n / N, 256), 256, 0, s>>>((const T*)x, (const T*)bias, (const T*)y, (T*)out, mask, n / N, cols, p, scale, seed, offset);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

void dropout_bwd(const void* dout, const uint8_t* mask, void* dx, int64_t n, float p, int upscale, int dtype, cudaStream_t s) {
  if (n == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    if (n % N) { set_last_error(__FILE__, __LINE__, "dropout_bwd: element count must be a multiple of the 16B vector"); return; }
    const float scale = upscale ? (p < 1.f ? 1.f / (1.f - p) : 0.f) : 1.f;
    dropout_bwd_kernel<T><<<ew_grid(n / N, 256), 256, 0, s>>>((const T*)dout, mask, (T*)dx, n / N, scale);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ bias + activation
__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case 0: return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));                 // gelu (erf)
    case 1: return fmaxf(v, 0.f);                                                      // relu
    default: return v / (1.f + __expf(-v));                                            // silu / swish
  }
}

// gated = 0: out[r, c] = act(x[r, c] + bias[c]);  gated = 1: out[r, c] = act(x[r, c] + b[c]) * (x[r, half + c] + b[half + c]), half = cols / 2
template <typename T>
__global__ void __launch_bounds__(256) bias_act_kernel(const T* __restrict__ x, const T* __restrict__ bias, T* __restrict__ out, int64_t rows, int cols, int act, int gated) {
  constexpr int N = Vec16<T>::N;
  const int ocols = gated ? cols / 2 : cols;
  const int64_t nvec = rows * (ocols / N);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (ocols / N);
    const int c = (int)(i % (ocols / N)) * N;
    const Vec16<T> a = ld16_stream(x + r * cols + c);
    Vec16<T> ba, g, bg, o;
    if (bias) ba = ld16(bias + c);
    if (gated) {
      g = ld16_stream(x + r * cols + ocols + c);
      if (bias) bg = ld16(bias + ocols + c);
    }
#pragma unroll
    for (int j = 0; j < N; ++j) {
      float v = to_f(a.v[j]) + (bias ? to_f(ba.v[j]) : 0.f);
      v = act_apply(v, act);
      if (gated) v *= to_f(g.v[j]) + (bias ? to_f(bg.v[j]) : 0.f);
      o.v[j] = from_f<T>(v);
    }
    st16_stream(out + r * ocols + c, o);
  }
}

void bias_act_fwd(const void* x, const void* bias, void* out, int64_t rows, int cols, int act, int gated, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    const int ocols = gated ? cols / 2 : cols;
    if (ocols % N || (gated && cols % 2)) { set_last_error(__FILE__, __LINE__, "bias_act: row width must be a multiple of the 16B vector"); return; }
    bias_act_kernel<T><<<ew_grid(rows * (ocols / N), 256), 256, 0, s>>>((const T*)x, (const T*)bias, (T*)out, rows, cols, act, gated);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
