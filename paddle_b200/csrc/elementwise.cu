// SwiGLU, rotary embedding, residual add for sm_90a (HBM-bound: 16-byte vector access, streaming hints).
// Parity (behaviour): python/paddle/incubate/nn/functional/swiglu.py, fused_rotary_position_embedding.py
// (paddle/phi/kernels/fusion/gpu/fused_rope_kernel.cu).
#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

__device__ __forceinline__ float sigmoidf_fast(float x) { return 1.f / (1.f + __expf(-x)); }

// rows x cols outputs; gate/up row stride = ld (== cols, or 2*cols when packed)
template <typename T>
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const T* __restrict__ gate, const T* __restrict__ up,
                                                          T* __restrict__ out, int64_t rows, int cols, int64_t ld) {
  constexpr int N = Vec16<T>::N;
  constexpr int U = 4;  // independent 16B loads in flight per thread and tensor
  const int vec_per_row = cols / N;
  const int64_t total = rows * vec_per_row;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < total; i0 += stride * U) {
    Vec16<T> g[U], u[U];
    int64_t oidx[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t i = i0 + k * stride;
      if (i < total) {
        const int64_t r = i / vec_per_row;
        const int c = (int)(i - r * vec_per_row) * N;
        g[k] = ld16_stream(gate + r * ld + c);
        u[k] = ld16_stream(up + r * ld + c);
        oidx[k] = r * cols + c;
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (i0 + k * stride < total) {
        Vec16<T> o;
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float x = to_f(g[k].v[j]);
          o.v[j] = from_f<T>(x * sigmoidf_fast(x) * to_f(u[k].v[j]));
        }
        st16_stream(out + oidx[k], o);
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const T* __restrict__ dout, const T* __restrict__ gate,
                                                          const T* __restrict__ up, T* __restrict__ dgate,
                                                          T* __restrict__ dup, int64_t rows, int cols, int64_t ld) {
  constexpr int N = Vec16<T>::N;
  constexpr int U = 2;
  const int vec_per_row = cols / N;
  const int64_t total = rows * vec_per_row;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i0 < total; i0 += stride * U) {
    Vec16<T> g[U], u[U], d[U];
    int64_t gi[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t i = i0 + k * stride;
      if (i < total) {
        const int64_t r = i / vec_per_row;
        const int c = (int)(i - r * vec_per_row) * N;
        gi[k] = r * ld + c;
        g[k] = ld16_stream(gate + gi[k]);
        u[k] = ld16_stream(up + gi[k]);
        d[k] = ld16_stream(dout + r * cols + c);
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (i0 + k * stride < total) {
        Vec16<T> og, ou;
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float x = to_f(g[k].v[j]), y = to_f(u[k].v[j]), dy = to_f(d[k].v[j]);
          const float sg = sigmoidf_fast(x);
          og.v[j] = from_f<T>(dy * y * sg * (1.f + x * (1.f - sg)));
          ou.v[j] = from_f<T>(dy * x * sg);
        }
        st16_stream(dgate + gi[k], og);
        st16_stream(dup + gi[k], ou);
      }
    }
  }
}

static inline int ew_grid(int64_t work_items, int threads) {
  int64_t blocks = (work_items + threads - 1) / threads;
  const int64_t cap = (int64_t)sm_count() * 16;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

void swiglu_fwd(const void* gate, const void* up, void* out, int64_t rows, int cols, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    if (cols % N) { set_last_error(__FILE__, __LINE__, "swiglu: cols must be a multiple of the 16B vector"); return; }
    const T* g = (const T*)gate;
    const T* u = up ? (const T*)up : g + cols;
    const int64_t ld = up ? cols : 2 * (int64_t)cols;
    swiglu_fwd_kernel<T><<<ew_grid((rows * (cols / N) + 3) / 4, 256), 256, 0, s>>>(g, u, (T*)out, rows, cols, ld);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

void swiglu_bwd(const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows, int cols,
                int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    if (cols % N) { set_last_error(__FILE__, __LINE__, "swiglu: cols must be a multiple of the 16B vector"); return; }
    const T* g = (const T*)gate;
    const T* u = up ? (const T*)up : g + cols;
    T* dg = (T*)dgate;
    T* du = up ? (T*)dup : dg + cols;
    const int64_t ld = up ? cols : 2 * (int64_t)cols;
    swiglu_bwd_kernel<T><<<ew_grid((rows * (cols / N) + 1) / 2, 256), 256, 0, s>>>((const T*)dout, g, u, dg, du, rows, cols, ld);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ rotary
// x: [tokens, heads, dim]. neox: pairs are (i, i + dim/2); else interleaved (2i, 2i+1).
// One thread handles one 16-byte vector of the first half and its partner vector (neox) or one vector (interleaved).
template <typename T, bool kNeox>
__global__ void __launch_bounds__(256) rope_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                    const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                    const int64_t* __restrict__ pos_ids, int64_t tokens, int seq,
                                                    int heads, int dim, float sign, int64_t row_stride) {
  constexpr int N = Vec16<T>::N;
  const int half = dim / 2;
  const int vec_per_head = kNeox ? half / N : dim / N;
  const int64_t total = tokens * heads * vec_per_head;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % vec_per_head);
    const int64_t th = i / vec_per_head;
    const int64_t tok = th / heads;
    const int64_t pos = pos_ids ? pos_ids[tok] : (tok % seq);
    const int head = (int)(th - tok * heads);
    const T* xp = x + tok * row_stride + (int64_t)head * dim;
    T* yp = y + tok * row_stride + (int64_t)head * dim;
    if constexpr (kNeox) {
      const int c = v * N;
      Vec16<T> a = ld16_stream(xp + c), b = ld16_stream(xp + half + c), oa, ob;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float cs = cos_t[pos * half + c + j], sn = sign * sin_t[pos * half + c + j];
        const float fa = to_f(a.v[j]), fb = to_f(b.v[j]);
        oa.v[j] = from_f<T>(fa * cs - fb * sn);
        ob.v[j] = from_f<T>(fb * cs + fa * sn);
      }
      st16_stream(yp + c, oa);
      st16_stream(yp + half + c, ob);
    } else {
      const int c = v * N;
      Vec16<T> a = ld16_stream(xp + c), o;
#pragma unroll
      for (int j = 0; j < N; j += 2) {
        const int p = (c + j) >> 1;
        const float cs = cos_t[pos * half + p], sn = sign * sin_t[pos * half + p];
        const float f0 = to_f(a.v[j]), f1 = to_f(a.v[j + 1]);
        o.v[j] = from_f<T>(f0 * cs - f1 * sn);
        o.v[j + 1] = from_f<T>(f1 * cs + f0 * sn);
      }
      st16_stream(yp + c, o);
    }
  }
}

void rope_apply(const void* x, void* y, const float* cos_t, const float* sin_t, const int64_t* pos_ids, int64_t tokens,
                int seq, int heads, int dim, int neox, int backward, int dtype, int64_t row_stride, cudaStream_t s) {
  if (tokens == 0) return;
  const float sign = backward ? -1.f : 1.f;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    if ((dim / 2) % N) { set_last_error(__FILE__, __LINE__, "rope: head_dim/2 must be a multiple of the 16B vector"); return; }
    if (neox) {
      const int64_t items = tokens * heads * ((dim / 2) / N);
      rope_kernel<T, true><<<ew_grid(items, 256), 256, 0, s>>>((const T*)x, (T*)y, cos_t, sin_t, pos_ids, tokens, seq, heads, dim, sign, row_stride > 0 ? row_stride : (int64_t)heads * dim);
    } else {
      const int64_t items = tokens * heads * (dim / N);
      rope_kernel<T, false><<<ew_grid(items, 256), 256, 0, s>>>((const T*)x, (T*)y, cos_t, sin_t, pos_ids, tokens, seq, heads, dim, sign, row_stride > 0 ? row_stride : (int64_t)heads * dim);
    }
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

template <typename T>
__global__ void __launch_bounds__(256) add_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, int64_t nvec) {
  constexpr int N = Vec16<T>::N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    Vec16<T> va = ld16_stream(a + i * N), vb = ld16_stream(b + i * N), o;
#pragma unroll
    for (int j = 0; j < N; ++j) o.v[j] = from_f<T>(to_f(va.v[j]) + to_f(vb.v[j]));
    st16_stream(y + i * N, o);
  }
}

void add_fwd(const void* a, const void* b, void* y, int64_t n, int dtype, cudaStream_t s) {
  if (n == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, {
    constexpr int N = Vec16<T>::N;
    if (n % N) { set_last_error(__FILE__, __LINE__, "add: n must be a multiple of the 16B vector"); return; }
    add_kernel<T><<<ew_grid(n / N, 256), 256, 0, s>>>((const T*)a, (const T*)b, (T*)y, n / N);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
