// Fused optimizer kernels for sm_90a: AdamW (multi-precision), SGD-momentum, LAMB, grad-norm, unscale.
// Parity (behaviour): paddle/phi/kernels/gpu/adamw_kernel.cu, fused_adam_kernel.cu, lamb_kernel.cu, amp_kernel.cu
// (check_finite_and_unscale / update_loss_scaling), clip_by_global_norm.
// Design: parameters live in flat arenas, so one launch covers one (dtype, hyper-parameter) group; clip coefficient,
// loss-scale and found-inf are read from device memory -> no host synchronisation anywhere in the step.
#include <type_traits>

#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

// ---- split master weights ------------------------------------------------------------------------------------------
// fp32 master = bf16 parameter (round-to-nearest of the master, the value the forward uses) + a signed 16-bit residual of the
// low mantissa bits: bits(master) = (bits(bf16) << 16) + residual.  4 bytes per parameter instead of 6 (bf16 copy + fp32 master):
// 26 GB less for a 13B model, which buys larger micro-batches instead of activation recompute.
// The only inexact case is a round-to-even tie whose residual is +0x8000 (stored as 0x7fff: one fp32 ulp).
__device__ __forceinline__ float split_master_join(__nv_bfloat16 w, int16_t lo) {
  const uint32_t hi = (uint32_t)__bfloat16_as_ushort(w) << 16;
  return __uint_as_float(hi + (uint32_t)(int32_t)lo);
}
__device__ __forceinline__ void split_master_split(float f, __nv_bfloat16& w, int16_t& lo) {
  w = __float2bfloat16_rn(f);
  int32_t d = (int32_t)(__float_as_uint(f) - ((uint32_t)__bfloat16_as_ushort(w) << 16));
  d = d > 32767 ? 32767 : (d < -32768 ? -32768 : d);
  if (f != f) d = 0;
  lo = (int16_t)d;
}

template <typename TP, typename TG, typename TS>
__global__ void __launch_bounds__(256) adamw_kernel(TP* __restrict__ p, const TG* __restrict__ g, float* __restrict__ master,
                                                     TS* __restrict__ m, TS* __restrict__ v, int64_t n, AdamWArgs a) {
  if (a.found_inf && *a.found_inf != 0.f) return;
  float gscale = a.inv_scale ? *a.inv_scale : 1.f;
  if (a.grad_sq_norm && a.max_norm > 0.f) {
    const float norm = sqrtf(*a.grad_sq_norm) * gscale;
    if (norm > a.max_norm) gscale *= a.max_norm / (norm + 1e-6f);
  }
  const float lr = a.dyn ? a.dyn[0] * a.lr : a.lr;
  const float step_size = lr / (a.dyn ? a.dyn[1] : a.bias_c1);
  const float inv_c2 = rsqrtf(a.dyn ? a.dyn[2] : a.bias_c2);
  const float decay = 1.f - lr * a.weight_decay;
  constexpr int U = 4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; base < n; base += stride * U) {
    float pf[U], gf[U], mf[U], vf[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * stride;
      if (i < n) {
        pf[u] = master ? master[i] : to_f(p[i]);
        gf[u] = to_f(g[i]) * gscale;
        mf[u] = to_f(m[i]);
        vf[u] = to_f(v[i]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * stride;
      if (i < n) {
        const float mm = a.beta1 * mf[u] + (1.f - a.beta1) * gf[u];
        const float vv = a.beta2 * vf[u] + (1.f - a.beta2) * gf[u] * gf[u];
        const float denom = sqrtf(vv) * inv_c2 + a.eps;
        const float np = pf[u] * decay - step_size * (mm / denom);
        m[i] = from_f<TS>(mm);
        v[i] = from_f<TS>(vv);
        if (master) master[i] = np;
        p[i] = from_f<TP>(np);
      }
    }
  }
}

// ---- vectorised variant: 8 elements per thread-iteration, every tensor accessed with 16-byte transactions ----------
template <typename T> __device__ __forceinline__ void load8(const T* p, float (&o)[8]) {
  if constexpr (sizeof(T) == 4) {
    const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  } else {
    Vec16<T> v = ld16(p);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = to_f(v.v[j]);
  }
}
template <typename T> __device__ __forceinline__ void store8(T* p, const float (&o)[8]) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(o[4], o[5], o[6], o[7]);
  } else {
    Vec16<T> v;
#pragma unroll
    for (int j = 0; j < 8; ++j) v.v[j] = from_f<T>(o[j]);
    st16(p, v);
  }
}

template <typename TP, typename TG, typename TS>
__global__ void __launch_bounds__(256) adamw_vec_kernel(TP* __restrict__ p, const TG* __restrict__ g, float* __restrict__ master,
                                                         TS* __restrict__ m, TS* __restrict__ v, int64_t n, AdamWArgs a,
                                                         int16_t* __restrict__ lo = nullptr) {
  if (a.found_inf && *a.found_inf != 0.f) return;
  float gscale = a.inv_scale ? *a.inv_scale : 1.f;
  if (a.grad_sq_norm && a.max_norm > 0.f) {
    const float norm = sqrtf(*a.grad_sq_norm) * gscale;
    if (norm > a.max_norm) gscale *= a.max_norm / (norm + 1e-6f);
  }
  const float lr = a.dyn ? a.dyn[0] * a.lr : a.lr;
  const float step_size = lr / (a.dyn ? a.dyn[1] : a.bias_c1);
  const float inv_c2 = rsqrtf(a.dyn ? a.dyn[2] : a.bias_c2);
  const float decay = 1.f - lr * a.weight_decay;
  const float omb1 = 1.f - a.beta1, omb2 = 1.f - a.beta2;
  const int64_t npack = n / 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npack; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = i * 8;
    float pf[8], gf[8], mf[8], vf[8];
    load8(g + e, gf);
    load8(m + e, mf);
    load8(v + e, vf);
    if constexpr (std::is_same<TP, __nv_bfloat16>::value) {
      if (lo) {
        const Vec16<__nv_bfloat16> w = ld16(p + e);
        const Vec16<int16_t> r = ld16(lo + e);
#pragma unroll
        for (int j = 0; j < 8; ++j) pf[j] = split_master_join(w.v[j], r.v[j]);
      } else if (master) load8(master + e, pf); else load8(p + e, pf);
    } else {
      if (master) load8(master + e, pf); else load8(p + e, pf);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gg = gf[j] * gscale;
      mf[j] = a.beta1 * mf[j] + omb1 * gg;
      vf[j] = a.beta2 * vf[j] + omb2 * gg * gg;
      pf[j] = pf[j] * decay - step_size * (mf[j] / (sqrtf(vf[j]) * inv_c2 + a.eps));
    }
    store8(m + e, mf);
    store8(v + e, vf);
    if constexpr (std::is_same<TP, __nv_bfloat16>::value) {
      if (lo) {
        Vec16<__nv_bfloat16> w;
        Vec16<int16_t> r;
#pragma unroll
        for (int j = 0; j < 8; ++j) split_master_split(pf[j], w.v[j], r.v[j]);
        st16(p + e, w);
        st16(lo + e, r);
        continue;
      }
    }
    if (master) store8(master + e, pf);
    store8(p + e, pf);
  }
  // scalar tail
  if (blockIdx.x == 0) {
    for (int64_t i = npack * 8 + threadIdx.x; i < n; i += blockDim.x) {
      float pf = master ? master[i] : to_f(p[i]);
      if constexpr (std::is_same<TP, __nv_bfloat16>::value) {
        if (lo) pf = split_master_join(p[i], lo[i]);
      }
      const float gg = to_f(g[i]) * gscale;
      const float mm = a.beta1 * to_f(m[i]) + omb1 * gg;
      const float vv = a.beta2 * to_f(v[i]) + omb2 * gg * gg;
      pf = pf * decay - step_size * (mm / (sqrtf(vv) * inv_c2 + a.eps));
      m[i] = from_f<TS>(mm);
      v[i] = from_f<TS>(vv);
      if constexpr (std::is_same<TP, __nv_bfloat16>::value) {
        if (lo) { split_master_split(pf, p[i], lo[i]); continue; }
      }
      if (master) master[i] = pf;
      p[i] = from_f<TP>(pf);
    }
  }
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static inline int opt_grid(int64_t n, int threads, int unroll) {
  int64_t blocks = (n + (int64_t)threads * unroll - 1) / ((int64_t)threads * unroll);
  const int64_t cap = (int64_t)sm_count() * 8;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

template <typename TP, typename TG>
static void adamw_dispatch_state(void* p, const void* g, float* master, void* m, void* v, int64_t n, int state_dtype,
                                 const AdamWArgs& a, cudaStream_t s, int16_t* lo = nullptr) {
  const bool vec = aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v) && (!master || aligned16(master)) && (!lo || aligned16(lo)) && n >= 8;
  if (lo) {   // split master weights: bf16 parameters only, vectorised kernel only (arena slabs are 256-byte aligned)
    if (!std::is_same<TP, __nv_bfloat16>::value || !vec) { set_last_error(__FILE__, __LINE__, "adamw: split master weights need 16-byte aligned bf16 parameters"); return; }
    const int grid = opt_grid(n, 256, 8 * 2);
    if (state_dtype == kF32) adamw_vec_kernel<TP, TG, float><<<grid, 256, 0, s>>>((TP*)p, (const TG*)g, nullptr, (float*)m, (float*)v, n, a, lo);
    else if (state_dtype == kBF16) adamw_vec_kernel<TP, TG, __nv_bfloat16><<<grid, 256, 0, s>>>((TP*)p, (const TG*)g, nullptr, (__nv_bfloat16*)m, (__nv_bfloat16*)v, n, a, lo);
    else set_last_error(__FILE__, __LINE__, "adamw: optimizer state must be fp32 or bf16");
    return;
  }
  const int grid = vec ? opt_grid(n, 256, 8 * 2) : opt_grid(n, 256, 4);
  if (state_dtype == kF32) {
    if (vec) adamw_vec_kernel<TP, TG, float><<<grid, 256, 0, s>>>((TP*)p, (const TG*)g, master, (float*)m, (float*)v, n, a);
    else adamw_kernel<TP, TG, float><<<grid, 256, 0, s>>>((TP*)p, (const TG*)g, master, (float*)m, (float*)v, n, a);
  } else if (state_dtype == kBF16) {
    if (vec) adamw_vec_kernel<TP, TG, __nv_bfloat16><<<grid, 256, 0, s>>>((TP*)p, (const TG*)g, master, (__nv_bfloat16*)m, (__nv_bfloat16*)v, n, a);
    else adamw_kernel<TP, TG, __nv_bfloat16><<<grid, 256, 0, s>>>((TP*)p, (const TG*)g, master, (__nv_bfloat16*)m, (__nv_bfloat16*)v, n, a);
  }
  else
    set_last_error(__FILE__, __LINE__, "adamw: optimizer state must be fp32 or bf16");
}

void adamw_step(void* p, const void* g, float* master, void* m, void* v, int64_t n, int p_dtype, int g_dtype,
                int state_dtype, const AdamWArgs& a, cudaStream_t s, int16_t* master_lo) {
  if (n == 0) return;
  if (master_lo && p_dtype != kBF16) { set_last_error(__FILE__, __LINE__, "adamw: split master weights need bf16 parameters"); return; }
  if (p_dtype == kF32 && g_dtype == kF32) adamw_dispatch_state<float, float>(p, g, master, m, v, n, state_dtype, a, s);
  else if (p_dtype == kBF16 && g_dtype == kBF16) adamw_dispatch_state<__nv_bfloat16, __nv_bfloat16>(p, g, master, m, v, n, state_dtype, a, s, master_lo);
  else if (p_dtype == kBF16 && g_dtype == kF32) adamw_dispatch_state<__nv_bfloat16, float>(p, g, master, m, v, n, state_dtype, a, s, master_lo);
  else if (p_dtype == kF16 && g_dtype == kF16) adamw_dispatch_state<__half, __half>(p, g, master, m, v, n, state_dtype, a, s);
  else if (p_dtype == kF16 && g_dtype == kF32) adamw_dispatch_state<__half, float>(p, g, master, m, v, n, state_dtype, a, s);
  else set_last_error(__FILE__, __LINE__, "adamw: unsupported param/grad dtype combination");
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ grad norm
template <typename T>
__global__ void __launch_bounds__(512) grad_sq_norm_kernel(const T* __restrict__ g, int64_t n, float* __restrict__ out,
                                                            float* __restrict__ found_inf) {
  __shared__ float red[33];
  constexpr int N = Vec16<T>::N;
  float acc = 0.f;
  const int64_t nvec = n / N;
  const bool aligned = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  if (aligned) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
      Vec16<T> v = ld16_stream(g + i * N);
#pragma unroll
      for (int j = 0; j < N; ++j) { const float f = to_f(v.v[j]); acc += f * f; }
    }
    for (int64_t i = nvec * N + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
      const float f = to_f(g[i]); acc += f * f;
    }
  } else {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
      const float f = to_f(g[i]); acc += f * f;
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) {
    atomicAdd(out, acc);  // one atomic per CTA (<= 8*SMs)
    if (found_inf && !isfinite(acc)) *found_inf = 1.f;
  }
}

void grad_sq_norm(const void* g, int64_t n, int dtype, float* out, float* found_inf, cudaStream_t s) {
  if (n == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (grad_sq_norm_kernel<T><<<opt_grid(n, 512, 8), 512, 0, s>>>((const T*)g, n, out, found_inf)));
  B200_CUDA_CHECK(cudaGetLastError());
}

template <typename T>
__global__ void __launch_bounds__(256) scale_kernel(T* __restrict__ g, int64_t n, const float* __restrict__ scale_dev, float scale_host) {
  const float sc = (scale_dev ? *scale_dev : 1.f) * scale_host;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    g[i] = from_f<T>(to_f(g[i]) * sc);
}

void scale_inplace(void* g, int64_t n, int dtype, const float* scale_dev, float scale_host, cudaStream_t s) {
  if (n == 0) return;
  B200_DISPATCH_DTYPE(dtype, T, (scale_kernel<T><<<opt_grid(n, 256, 4), 256, 0, s>>>((T*)g, n, scale_dev, scale_host)));
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ SGD momentum
template <typename TP, typename TG>
__global__ void __launch_bounds__(256) sgd_kernel(TP* __restrict__ p, const TG* __restrict__ g, float* __restrict__ master,
                                                   float* __restrict__ mom, int64_t n, float lr, float momentum, float wd, int nesterov) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pf = master ? master[i] : to_f(p[i]);
    float gf = to_f(g[i]) + wd * pf;
    if (mom) {
      const float mv = momentum * mom[i] + gf;
      mom[i] = mv;
      gf = nesterov ? gf + momentum * mv : mv;
    }
    pf -= lr * gf;
    if (master) master[i] = pf;
    p[i] = from_f<TP>(pf);
  }
}

void sgd_momentum_step(void* p, const void* g, float* master, void* mom, int64_t n, int p_dtype, int g_dtype, float lr,
                       float momentum, float weight_decay, int nesterov, cudaStream_t s) {
  if (n == 0) return;
  const int grid = opt_grid(n, 256, 4);
  if (p_dtype == kF32 && g_dtype == kF32) sgd_kernel<float, float><<<grid, 256, 0, s>>>((float*)p, (const float*)g, master, (float*)mom, n, lr, momentum, weight_decay, nesterov);
  else if (p_dtype == kBF16 && g_dtype == kBF16) sgd_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, 256, 0, s>>>((__nv_bfloat16*)p, (const __nv_bfloat16*)g, master, (float*)mom, n, lr, momentum, weight_decay, nesterov);
  else if (p_dtype == kF16 && g_dtype == kF16) sgd_kernel<__half, __half><<<grid, 256, 0, s>>>((__half*)p, (const __half*)g, master, (float*)mom, n, lr, momentum, weight_decay, nesterov);
  else set_last_error(__FILE__, __LINE__, "sgd: unsupported dtype combination");
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ LAMB (two stage)
template <typename TP, typename TG>
__global__ void __launch_bounds__(256) lamb1_kernel(const TP* __restrict__ p, const TG* __restrict__ g, const float* __restrict__ master,
                                                     float* __restrict__ m, float* __restrict__ v, float* __restrict__ update, int64_t n,
                                                     float beta1, float beta2, float eps, float wd, float c1, float c2,
                                                     float* __restrict__ p_sq, float* __restrict__ u_sq) {
  __shared__ float red[33];
  float ps = 0.f, us = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float pf = master ? master[i] : to_f(p[i]);
    const float gf = to_f(g[i]);
    const float mm = beta1 * m[i] + (1.f - beta1) * gf;
    const float vv = beta2 * v[i] + (1.f - beta2) * gf * gf;
    m[i] = mm; v[i] = vv;
    const float u = (mm / c1) / (sqrtf(vv / c2) + eps) + wd * pf;
    update[i] = u;
    ps += pf * pf; us += u * u;
  }
  ps = block_sum(ps, red);
  us = block_sum(us, red);
  if (threadIdx.x == 0) { atomicAdd(p_sq, ps); atomicAdd(u_sq, us); }
}

template <typename TP>
__global__ void __launch_bounds__(256) lamb2_kernel(TP* __restrict__ p, float* __restrict__ master, const float* __restrict__ update,
                                                     int64_t n, float lr, const float* __restrict__ p_sq, const float* __restrict__ u_sq) {
  const float pn = sqrtf(*p_sq), un = sqrtf(*u_sq);
  const float trust = (pn > 0.f && un > 0.f) ? pn / un : 1.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pf = master ? master[i] : to_f(p[i]);
    pf -= lr * trust * update[i];
    if (master) master[i] = pf;
    p[i] = from_f<TP>(pf);
  }
}

void lamb_stage1(const void* p, const void* g, const float* master, void* m, void* v, float* update, int64_t n,
                 int p_dtype, int g_dtype, float beta1, float beta2, float eps, float weight_decay, float bias_c1,
                 float bias_c2, float* p_sq, float* u_sq, cudaStream_t s) {
  if (n == 0) return;
  const int grid = opt_grid(n, 256, 4);
  if (p_dtype == kF32 && g_dtype == kF32) lamb1_kernel<float, float><<<grid, 256, 0, s>>>((const float*)p, (const float*)g, master, (float*)m, (float*)v, update, n, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, p_sq, u_sq);
  else if (p_dtype == kBF16 && g_dtype == kBF16) lamb1_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)p, (const __nv_bfloat16*)g, master, (float*)m, (float*)v, update, n, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, p_sq, u_sq);
  else if (p_dtype == kF16 && g_dtype == kF16) lamb1_kernel<__half, __half><<<grid, 256, 0, s>>>((const __half*)p, (const __half*)g, master, (float*)m, (float*)v, update, n, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, p_sq, u_sq);
  else set_last_error(__FILE__, __LINE__, "lamb: unsupported dtype combination");
  B200_CUDA_CHECK(cudaGetLastError());
}

void lamb_stage2(void* p, float* master, const float* update, int64_t n, int p_dtype, float lr, const float* p_sq,
                 const float* u_sq, cudaStream_t s) {
  if (n == 0) return;
  const int grid = opt_grid(n, 256, 4);
  B200_DISPATCH_DTYPE(p_dtype, T, (lamb2_kernel<T><<<grid, 256, 0, s>>>((T*)p, master, update, n, lr, p_sq, u_sq)));
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
