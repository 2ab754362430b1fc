// Fused RMSNorm / LayerNorm forward+backward for sm_90a.
// Parity (behaviour): paddle/phi/kernels/fusion/gpu/fused_layernorm_kernel.cu, fused_rms_norm (reference).
// Design: one CTA per row, row cached in registers (16-byte vectors, block size sized to the row so no lane idles),
// fp32 statistics; the backward is a persistent grid that keeps per-CTA dW/dB partial sums in registers across rows,
// software-pipelined two rows deep, and writes them once (two-stage reduction, no atomics).
// HBM-bound: forward moves 2 x row bytes, backward 3 x row bytes.
#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

static constexpr int kMaxVPT = 8;      // vectors per thread cached in registers
static constexpr int kMaxThreads = 512;

// pick (threads, vpt) with threads*vpt >= nvec, threads a multiple of 32 in [64, 512], minimal padding waste
// (register budget: the forward may run 512 threads for vpt<=2; the backward and wide rows are capped at 256 threads)
static inline void pick_shape(int nvec, int& threads, int& vpt, bool bwd) {
  for (vpt = 1; vpt <= kMaxVPT; vpt *= 2) {
    const int cap = (!bwd && vpt <= 2) ? 512 : 256;
    threads = ((nvec + vpt - 1) / vpt + 31) / 32 * 32;
    if (threads <= cap) break;
  }
  if (threads < 64) threads = 64;
}

template <typename T, int VPT, bool kResidual, bool kLayerNorm>
__global__ void __launch_bounds__(VPT <= 2 ? 512 : 256)
norm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ residual, const T* __restrict__ w,
                const T* __restrict__ b, T* __restrict__ y, T* __restrict__ res_out, float* __restrict__ mean_out,
                float* __restrict__ rstd_out, int cols, float eps) {
  constexpr int N = Vec16<T>::N;
  __shared__ float red[33];
  const int64_t row = blockIdx.x;
  const T* xr = x + row * cols;
  const int nvec = cols / N;
  const int nt = blockDim.x;
  Vec16<T> xv[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * nt;
    if (v < nvec) xv[i] = ld16_stream(xr + v * N);
  }
  if constexpr (kResidual) {
    Vec16<T> rv[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * nt;
      if (v < nvec) rv[i] = ld16_stream(residual + row * cols + v * N);
    }
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * nt;
      if (v < nvec) {
#pragma unroll
        for (int j = 0; j < N; ++j) xv[i].v[j] = from_f<T>(to_f(xv[i].v[j]) + to_f(rv[i].v[j]));
        st16(res_out + row * cols + v * N, xv[i]);
      }
    }
  }
  float sum = 0.f, sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * nt;
    if (v < nvec) {
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float f = to_f(xv[i].v[j]);
        sum += f;
        sq += f * f;
      }
    }
  }
  float mean = 0.f, rstd;
  if constexpr (kLayerNorm) {
    mean = block_sum(sum, red) / cols;
    float var = 0.f;  // second pass over registers: numerically stable variance
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * nt;
      if (v < nvec) {
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float d = to_f(xv[i].v[j]) - mean;
          var += d * d;
        }
      }
    }
    rstd = rsqrtf(block_sum(var, red) / cols + eps);
  } else {
    rstd = rsqrtf(block_sum(sq, red) / cols + eps);
  }
  if (threadIdx.x == 0) {
    if (rstd_out) rstd_out[row] = rstd;
    if (kLayerNorm && mean_out) mean_out[row] = mean;
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * nt;
    if (v < nvec) {
      Vec16<T> o, wv, bv;
      if (w) wv = ld16(w + v * N);
      if (b) bv = ld16(b + v * N);
#pragma unroll
      for (int j = 0; j < N; ++j) {
        float f = (to_f(xv[i].v[j]) - mean) * rstd;
        if (w) f *= to_f(wv.v[j]);
        if (b) f += to_f(bv.v[j]);
        o.v[j] = from_f<T>(f);
      }
      st16_stream(y + row * cols + v * N, o);
    }
  }
}

template <typename T, bool kLayerNorm>
static void launch_norm_fwd(const void* x, const void* residual, const void* w, const void* b, void* y, void* res_out,
                            float* mean, float* rstd, int64_t rows, int cols, float eps, cudaStream_t s) {
  constexpr int N = Vec16<T>::N;
  if (cols % N != 0 || cols > 256 * kMaxVPT * N) {
    set_last_error(__FILE__, __LINE__, "norm: cols must be a multiple of the 16B vector and <= 512*8 vectors");
    return;
  }
  int threads, vpt;
  pick_shape(cols / N, threads, vpt, false);
  dim3 grid((unsigned)rows), block(threads);
#define LAUNCH(V)                                                                                                   \
  if (residual)                                                                                                     \
    norm_fwd_kernel<T, V, true, kLayerNorm><<<grid, block, 0, s>>>((const T*)x, (const T*)residual, (const T*)w,   \
                                                                   (const T*)b, (T*)y, (T*)res_out, mean, rstd, cols, eps); \
  else                                                                                                              \
    norm_fwd_kernel<T, V, false, kLayerNorm><<<grid, block, 0, s>>>((const T*)x, nullptr, (const T*)w, (const T*)b, \
                                                                    (T*)y, nullptr, mean, rstd, cols, eps);
  if (vpt == 1) { LAUNCH(1) } else if (vpt == 2) { LAUNCH(2) } else if (vpt == 4) { LAUNCH(4) } else { LAUNCH(8) }
#undef LAUNCH
  B200_CUDA_CHECK(cudaGetLastError());
}

void rms_norm_fwd(const void* x, const void* residual, const void* w, const void* b, void* y, void* res_out,
                  float* rstd, int64_t rows, int cols, float eps, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (launch_norm_fwd<T, false>(x, residual, w, b, y, res_out, nullptr, rstd, rows, cols, eps, s)));
}

void layer_norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int64_t rows,
                    int cols, float eps, int dtype, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (launch_norm_fwd<T, true>(x, nullptr, w, b, y, nullptr, mean, rstd, rows, cols, eps, s)));
}

// ------------------------------------------------------------------------------------------------ backward
// Persistent: CTA c handles rows c, c+G, ...; dW/dB partials for the thread's own columns live in registers.
// The loads of row i+G are issued before the reductions of row i complete (register double buffer).
template <typename T, int VPT, bool kLayerNorm>
__global__ void __launch_bounds__(256)
norm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ w,
                const float* __restrict__ mean_in, const float* __restrict__ rstd_in, T* __restrict__ dx,
                float* __restrict__ dw_partial, float* __restrict__ db_partial, int64_t rows, int cols) {
  constexpr int N = Vec16<T>::N;
  __shared__ float red[33];
  const int nvec = cols / N;
  const int nt = blockDim.x;
  float dw_acc[VPT][N];
  float db_acc[kLayerNorm ? VPT : 1][kLayerNorm ? N : 1];
  float wf[VPT][N];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * nt;
    Vec16<T> wv;
    if (v < nvec && w) wv = ld16(w + v * N);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      dw_acc[i][j] = 0.f;
      if constexpr (kLayerNorm) db_acc[i][j] = 0.f;
      wf[i][j] = (v < nvec && w) ? to_f(wv.v[j]) : 1.f;
    }
  }
  Vec16<T> xn[VPT], gn[VPT];  // next row (prefetch)
  int64_t row = blockIdx.x;
  if (row < rows) {
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * nt;
      if (v < nvec) {
        xn[i] = ld16_stream(x + row * cols + v * N);
        gn[i] = ld16_stream(dy + row * cols + v * N);
      }
    }
  }
  for (; row < rows; row += gridDim.x) {
    Vec16<T> xv[VPT], gv[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) { xv[i] = xn[i]; gv[i] = gn[i]; }
    const int64_t nrow = row + gridDim.x;
    if (nrow < rows) {
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int v = threadIdx.x + i * nt;
        if (v < nvec) {
          xn[i] = ld16_stream(x + nrow * cols + v * N);
          gn[i] = ld16_stream(dy + nrow * cols + v * N);
        }
      }
    }
    const float rstd = rstd_in[row];
    const float mean = kLayerNorm ? mean_in[row] : 0.f;
    float s1 = 0.f, s2 = 0.f;  // s1 = sum(dy*w), s2 = sum(dy*w*xhat)
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * nt;
      if (v < nvec) {
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float xh = (to_f(xv[i].v[j]) - mean) * rstd;
          const float g = to_f(gv[i].v[j]);
          const float gw = g * wf[i][j];
          s1 += gw;
          s2 += gw * xh;
          dw_acc[i][j] += g * xh;
          if constexpr (kLayerNorm) db_acc[i][j] += g;
        }
      }
    }
    s2 = block_sum(s2, red) / cols;
    if constexpr (kLayerNorm) s1 = block_sum(s1, red) / cols; else s1 = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * nt;
      if (v < nvec) {
        Vec16<T> o;
#pragma unroll
        for (int j = 0; j < N; ++j) {
          const float xh = (to_f(xv[i].v[j]) - mean) * rstd;
          const float gw = to_f(gv[i].v[j]) * wf[i][j];
          o.v[j] = from_f<T>((gw - s1 - xh * s2) * rstd);
        }
        st16_stream(dx + row * cols + v * N, o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * nt;
    if (v < nvec) {
      if (dw_partial) {
        float4* d = reinterpret_cast<float4*>(dw_partial + (int64_t)blockIdx.x * cols + v * N);
#pragma unroll
        for (int q = 0; q < N / 4; ++q) d[q] = make_float4(dw_acc[i][4 * q], dw_acc[i][4 * q + 1], dw_acc[i][4 * q + 2], dw_acc[i][4 * q + 3]);
      }
      if constexpr (kLayerNorm) {
        if (db_partial) {
          float4* d = reinterpret_cast<float4*>(db_partial + (int64_t)blockIdx.x * cols + v * N);
#pragma unroll
          for (int q = 0; q < N / 4; ++q) d[q] = make_float4(db_acc[i][4 * q], db_acc[i][4 * q + 1], db_acc[i][4 * q + 2], db_acc[i][4 * q + 3]);
        }
      }
    }
  }
}

int norm_bwd_num_partials(int64_t rows) {
  const int64_t g = (int64_t)sm_count() * 4;
  return (int)(rows < g ? rows : g);
}

template <typename T, bool kLayerNorm>
static void launch_norm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx,
                            float* dwp, float* dbp, int64_t rows, int cols, int n_partial, cudaStream_t s) {
  constexpr int N = Vec16<T>::N;
  if (cols % N != 0 || cols > 256 * kMaxVPT * N) {
    set_last_error(__FILE__, __LINE__, "norm bwd: unsupported cols");
    return;
  }
  int threads, vpt;
  pick_shape(cols / N, threads, vpt, true);
  dim3 grid((unsigned)n_partial), block(threads);
#define LAUNCH(V)                                                                                              \
  norm_bwd_kernel<T, V, kLayerNorm><<<grid, block, 0, s>>>((const T*)dy, (const T*)x, (const T*)w, mean, rstd, \
                                                           (T*)dx, dwp, dbp, rows, cols);
  if (vpt == 1) { LAUNCH(1) } else if (vpt == 2) { LAUNCH(2) } else if (vpt == 4) { LAUNCH(4) } else { LAUNCH(8) }
#undef LAUNCH
  B200_CUDA_CHECK(cudaGetLastError());
}

void rms_norm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx, float* dw_partial,
                  float* db_partial, int64_t rows, int cols, int dtype, int n_partial, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (launch_norm_bwd<T, false>(dy, x, w, nullptr, rstd, dx, dw_partial, db_partial, rows, cols, n_partial, s)));
}

void layer_norm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx,
                    float* dw_partial, float* db_partial, int64_t rows, int cols, int dtype, int n_partial,
                    cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (launch_norm_bwd<T, true>(dy, x, w, mean, rstd, dx, dw_partial, db_partial, rows, cols, n_partial, s)));
}

// out[c] = sum_p partial[p][c]; 2-D grid: x over columns (coalesced), y splits the partial rows, smem tree over y.
template <typename T>
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ partial, T* __restrict__ out, int n_partial, int cols) {
  __shared__ float sm[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;  // blockDim = (32, 8)
  float acc = 0.f;
  if (c < cols)
    for (int p = threadIdx.y; p < n_partial; p += 8) acc += partial[(int64_t)p * cols + c];
  sm[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sm[k][threadIdx.x];
    out[c] = from_f<T>(t);
  }
}

void reduce_partials(const float* partial, void* out, int n_partial, int cols, int dtype, cudaStream_t s) {
  dim3 block(32, 8), grid((cols + 31) / 32);
  B200_DISPATCH_DTYPE(dtype, T, (reduce_partials_kernel<T><<<grid, block, 0, s>>>(partial, (T*)out, n_partial, cols)));
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
