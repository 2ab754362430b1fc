// Fused per-tensor fp8 quantisation for the O2-fp8 training recipe: one reduction kernel for the absolute maximum and one cast kernel
// that writes the fp8 tensor AND its transpose (the backward GEMMs need K-major operands of both x and x^T) plus the
// dequantisation factor, everything on the device (no float() read-backs, no .t().contiguous() copies).
// Parity (role): paddle/phi/kernels/fusion/fp8_gemm + the quantisation ops around fp8_fp8_half_gemm_fused.
#include <cuda_fp8.h>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

template <typename T>
__global__ void __launch_bounds__(512) fp8_amax_kernel(const T* __restrict__ x, int64_t n, float* __restrict__ amax) {
  __shared__ float red[33];
  constexpr int N = Vec16<T>::N;
  float m = 0.f;
  const int64_t nvec = n / N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const Vec16<T> v = ld16_stream(x + i * N);
#pragma unroll
    for (int j = 0; j < N; ++j) m = fmaxf(m, fabsf(to_f(v.v[j])));
  }
  for (int64_t i = nvec * N + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(to_f(x[i])));
  m = block_max(m, red);
  if (threadIdx.x == 0 && m > 0.f) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));   // non-negative floats order like ints
}

void fp8_amax(const void* x, int64_t n, int dtype, float* amax, cudaStream_t s) {
  if (n == 0) return;
  int64_t blocks = (n / 8 + 511) / 512;
  const int64_t cap = (int64_t)sm_count() * 4;
  const int grid = (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
  B200_DISPATCH_DTYPE(dtype, T, (fp8_amax_kernel<T><<<grid, 512, 0, s>>>((const T*)x, n, amax)));
  B200_CUDA_CHECK(cudaGetLastError());
}

template <bool E5M2>
__device__ __forceinline__ uint8_t to_fp8(float v) {
  return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, E5M2 ? __NV_E5M2 : __NV_E4M3);
}

// 64 x 64 tile per CTA (256 threads): 16-byte loads, 8-byte row-major stores, transposed 16-byte stores through shared memory
template <typename T, bool E5M2>
__global__ void __launch_bounds__(256) fp8_cast_kernel(const T* __restrict__ x, int64_t M, int64_t K, const float* __restrict__ amax,
                                                        uint8_t* __restrict__ q, uint8_t* __restrict__ qT, float* __restrict__ inv_scale) {
  __shared__ uint8_t tile[64][64 + 16];
  const float fmax = E5M2 ? 57344.f : 448.f;
  const float am = fmaxf(*amax, 1e-12f);
  const float scale = fmax / am;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *inv_scale = am / fmax;
  const int64_t r0 = (int64_t)blockIdx.y * 64, c0 = (int64_t)blockIdx.x * 64;
  constexpr int N = Vec16<T>::N;                 // 8 for 16-bit inputs, 4 for fp32
  constexpr int VPR = 64 / N;                    // vectors per tile row
  for (int v = threadIdx.x; v < 64 * VPR; v += 256) {
    const int r = v / VPR, c = (v % VPR) * N;
    const Vec16<T> in = ld16(x + (r0 + r) * K + c0 + c);
    uint8_t o[N];
#pragma unroll
    for (int j = 0; j < N; ++j) o[j] = to_fp8<E5M2>(to_f(in.v[j]) * scale);
    if constexpr (N == 8) {
      *reinterpret_cast<uint2*>(q + (r0 + r) * K + c0 + c) = *reinterpret_cast<const uint2*>(o);
      *reinterpret_cast<uint2*>(&tile[r][c]) = *reinterpret_cast<const uint2*>(o);
    } else {
      *reinterpret_cast<uint32_t*>(q + (r0 + r) * K + c0 + c) = *reinterpret_cast<const uint32_t*>(o);
      *reinterpret_cast<uint32_t*>(&tile[r][c]) = *reinterpret_cast<const uint32_t*>(o);
    }
  }
  if (qT == nullptr) return;
  __syncthreads();
  {   // qT[c0 + kk][r0 + m .. m + 16): 64 rows of 64 bytes = 256 x 16-byte stores
    const int kk = threadIdx.x >> 2, m = (threadIdx.x & 3) * 16;
    uint8_t o[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j] = tile[m + j][kk];
    *reinterpret_cast<uint4*>(qT + (c0 + kk) * M + r0 + m) = *reinterpret_cast<const uint4*>(o);
  }
}

void fp8_cast_transpose(const void* x, int64_t m, int64_t k, int dtype, const float* amax, int e5m2, void* q, void* qT, float* inv_scale, cudaStream_t s) {
  if (m == 0 || k == 0) return;
  if (m % 64 || k % 64) { set_last_error(__FILE__, __LINE__, "fp8_cast_transpose: M and K must be multiples of 64"); return; }
  dim3 grid((unsigned)(k / 64), (unsigned)(m / 64));
  B200_DISPATCH_DTYPE(dtype, T, {
    if (e5m2) fp8_cast_kernel<T, true><<<grid, 256, 0, s>>>((const T*)x, m, k, amax, (uint8_t*)q, (uint8_t*)qT, inv_scale);
    else fp8_cast_kernel<T, false><<<grid, 256, 0, s>>>((const T*)x, m, k, amax, (uint8_t*)q, (uint8_t*)qT, inv_scale);
  });
  B200_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------- MX (block-scaled) quantisation
// One thread = one block of 32 consecutive k of one row: amax, power-of-two scale (rounded UP so that nothing saturates: 2^e >=
// amax / 448), 32 e4m3 bytes, one E8M0 byte.  Neighbouring threads take neighbouring blocks of the same row: 64-byte loads coalesce.
__device__ __forceinline__ int64_t mx_sf_offset(int64_t row, int64_t kb32, int64_t k_tiles) {
  const int64_t mt = row >> 7, r = row & 127;
  return ((mt * k_tiles + (kb32 >> 2)) << 9) + (r & 31) * 16 + (r >> 5) * 4 + (kb32 & 3);
}

template <typename T>
__global__ void mx_quantize_kernel(const T* __restrict__ x, int64_t rows, int64_t K, uint8_t* __restrict__ q, uint8_t* __restrict__ sf) {
  const int64_t nblk = K >> 5;
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= rows * nblk) return;
  const int64_t row = idx / nblk, kb = idx - row * nblk;
  const T* src = x + row * K + kb * 32;
  float v[32];
  if constexpr (sizeof(T) == 2) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const Vec16<T> t = ld16(src + i * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i * 8 + j] = to_f(t.v[j]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = to_f(src[i]);
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) amax = fmaxf(amax, fabsf(v[i]));
  int e = -127;
  if (amax > 0.f && isfinite(amax)) {
    int ex;
    const float m = frexpf(amax * (1.f / 448.f), &ex);      // amax / 448 = m 2^ex, m in [0.5, 1): ceil(log2) = ex, or ex - 1 when m == 0.5
    e = (m == 0.5f) ? ex - 1 : ex;
    e = max(-127, min(127, e));
  }
  const float inv = exp2f((float)-e);                          // exact power of two
  uint8_t o[32];
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const __nv_fp8x2_storage_t pr = __nv_cvt_float2_to_fp8x2(make_float2(v[i] * inv, v[i + 1] * inv), __NV_SATFINITE, __NV_E4M3);
    o[i] = (uint8_t)(pr & 0xFF);
    o[i + 1] = (uint8_t)(pr >> 8);
  }
  uint4* dst = reinterpret_cast<uint4*>(q + row * K + kb * 32);
  dst[0] = *reinterpret_cast<const uint4*>(o);
  dst[1] = *reinterpret_cast<const uint4*>(o + 16);
  sf[mx_sf_offset(row, kb, K >> 7)] = (uint8_t)(e + 127);
}

int mx_quantize(const void* x, int64_t rows, int64_t k, int dtype, void* q, uint8_t* sf, cudaStream_t s) {
  if (rows <= 0 || k <= 0 || rows % 128 || k % 128) return 1;
  const int64_t total = rows * (k / 32);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  B200_DISPATCH_DTYPE(dtype, T, { mx_quantize_kernel<T><<<blocks, 256, 0, s>>>((const T*)x, rows, k, (uint8_t*)q, sf); });
  return B200_LAUNCH_RESULT();
}

__global__ void mx_dequantize_kernel(const uint8_t* __restrict__ q, const uint8_t* __restrict__ sf, int64_t rows, int64_t K, float* __restrict__ out) {
  const int64_t nblk = K >> 5;
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= rows * nblk) return;
  const int64_t row = idx / nblk, kb = idx - row * nblk;
  const float sc = exp2f((float)((int)sf[mx_sf_offset(row, kb, K >> 7)] - 127));
  const uint8_t* src = q + row * K + kb * 32;
  float* dst = out + row * K + kb * 32;
#pragma unroll 8
  for (int i = 0; i < 32; ++i) {
    const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)src[i], __NV_E4M3);
    dst[i] = __half2float(*reinterpret_cast<const __half*>(&h)) * sc;
  }
}

int mx_dequantize(const void* q, const uint8_t* sf, int64_t rows, int64_t k, float* out, cudaStream_t s) {
  if (rows <= 0 || k <= 0 || rows % 128 || k % 128) return 1;
  const int64_t total = rows * (k / 32);
  mx_dequantize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const uint8_t*)q, sf, rows, k, out);
  return B200_LAUNCH_RESULT();
}

// ------------------------------------------------------------------------------------------------ per-token int8
// One block per row, two passes over it (the second is served from L1 / L2).  The expression is the torch one of nn/quant.py
// (llm_int8_linear), in fp32 with IEEE division and round-half-even, so both give the same bits.
template <typename T>
__global__ void __launch_bounds__(128) quantize_rows_s8_kernel(const T* __restrict__ x, const uint8_t* __restrict__ mask, int64_t k,
                                                               int8_t* __restrict__ q, float* __restrict__ row_scale) {
  __shared__ float red[33];
  constexpr int N = Vec16<T>::N;
  const T* xr = x + blockIdx.x * k;
  int8_t* qr = q + blockIdx.x * k;
  float m = 0.f;
  for (int64_t c = threadIdx.x * N; c < k; c += blockDim.x * N) {
    const Vec16<T> v = ld16(xr + c);
#pragma unroll
    for (int j = 0; j < N; ++j)
      if (!mask || !mask[c + j]) m = fmaxf(m, fabsf(to_f(v.v[j])));
  }
  m = block_max(m, red);
  const float sc = __fdiv_rn(fmaxf(m, 1e-8f), 127.f);
  if (threadIdx.x == 0) row_scale[blockIdx.x] = sc;
  for (int64_t c = threadIdx.x * N; c < k; c += blockDim.x * N) {
    const Vec16<T> v = ld16(xr + c);
    alignas(8) int8_t o[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float t = mask && mask[c + j] ? 0.f : rintf(__fdiv_rn(to_f(v.v[j]), sc));
      o[j] = (int8_t)fminf(fmaxf(t, -128.f), 127.f);
    }
    if constexpr (N == 8) *reinterpret_cast<uint2*>(qr + c) = *reinterpret_cast<const uint2*>(o);
    else *reinterpret_cast<uint32_t*>(qr + c) = *reinterpret_cast<const uint32_t*>(o);
  }
}

void quantize_rows_s8(const void* x, const uint8_t* mask, int64_t rows, int64_t k, int dtype, int8_t* q, float* row_scale, cudaStream_t s) {
  if (rows == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (quantize_rows_s8_kernel<T><<<(unsigned)rows, 128, 0, s>>>((const T*)x, mask, k, q, row_scale)));
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
