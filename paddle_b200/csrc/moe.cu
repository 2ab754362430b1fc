// Mixture-of-experts routing on the device (no host round trips): the reference's gate utility kernels
// (paddle/phi/kernels/gpu/number_count_kernel.cu, assign_pos_kernel.cu, limit_by_capacity_kernel.cu,
// prune_gate_by_capacity_kernel.cu:33) plus the planning / gather / combine kernels of the grouped-GEMM expert path
// (csrc/gemm_sm100_2cta.cu, GemmArgs::grouped): token slots are laid out grouped by expert in 256-row aligned segments, so every
// 256-row block of the grouped GEMM belongs to exactly one expert and the tile scheduler only reads a small device table.
#include "include/b200_common.cuh"
#include "include/b200_ops.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------ reference gate utilities
__global__ void number_count_kernel(const int64_t* __restrict__ idx, int64_t n, int64_t* __restrict__ counts, int upper) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = idx[i];
    if (e >= 0 && e < upper) atomicAdd(reinterpret_cast<unsigned long long*>(counts + e), 1ull);
  }
}

// pos[--cursor[e]] = i  (cursor starts as the inclusive cumulative count, like the reference's atomicAdd(cum_count + e, -1))
__global__ void assign_pos_kernel(const int64_t* __restrict__ idx, int64_t n, int64_t* __restrict__ cursor, int64_t* __restrict__ pos) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = idx[i];
    if (e >= 0) {
      const long long p = (long long)atomicAdd(reinterpret_cast<unsigned long long*>(cursor + e), (unsigned long long)(-1ll)) - 1;
      pos[p] = i;
    }
  }
}

// out[w][e] = min(expert_count[w][e], what is left of capacity[e] after workers 0..w-1); one thread per expert walks the workers in order
__global__ void limit_by_capacity_kernel(const int64_t* __restrict__ ec, const int64_t* __restrict__ cap, int64_t* __restrict__ out,
                                         int n_expert, int n_worker) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_expert) return;
  int64_t left = cap[e];
  for (int w = 0; w < n_worker; ++w) {
    const int64_t want = ec[(int64_t)w * n_expert + e];
    const int64_t take = want < left ? want : left;
    out[(int64_t)w * n_expert + e] = take;
    left -= take;
  }
}

// a token keeps its expert while the expert still has room (remaining[e] is consumed), otherwise it is dropped (-1)
__global__ void prune_gate_kernel(const int64_t* __restrict__ idx, int64_t n, long long* __restrict__ remaining, int64_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = idx[i];
    int64_t r = e;
    if (e >= 0) {
      const long long before = atomicAdd(reinterpret_cast<unsigned long long*>(remaining + e), (unsigned long long)(-1ll));
      if (before <= 0) r = -1;
    }
    out[i] = r;
  }
}

void moe_number_count(const int64_t* idx, int64_t n, int64_t* counts, int upper, cudaStream_t s) {
  if (n == 0) return;
  const int grid = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  number_count_kernel<<<grid, 256, 0, s>>>(idx, n, counts, upper);
  B200_CUDA_CHECK(cudaGetLastError());
}
void moe_assign_pos(const int64_t* idx, int64_t n, int64_t* cursor, int64_t* pos, cudaStream_t s) {
  if (n == 0) return;
  const int grid = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  assign_pos_kernel<<<grid, 256, 0, s>>>(idx, n, cursor, pos);
  B200_CUDA_CHECK(cudaGetLastError());
}
void moe_limit_by_capacity(const int64_t* ec, const int64_t* cap, int64_t* out, int n_expert, int n_worker, cudaStream_t s) {
  limit_by_capacity_kernel<<<(n_expert + 127) / 128, 128, 0, s>>>(ec, cap, out, n_expert, n_worker);
  B200_CUDA_CHECK(cudaGetLastError());
}
void moe_prune_gate(const int64_t* idx, int64_t n, int64_t* remaining, int64_t* out, cudaStream_t s) {
  if (n == 0) return;
  const int grid = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  prune_gate_kernel<<<grid, 256, 0, s>>>(idx, n, reinterpret_cast<long long*>(remaining), out);
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ grouped-path planning
// plan[0..E)        cursor (running fill of every expert's segment, starts at the padded segment start)
// One block: counts -> 256-row aligned segment starts -> tile table and per-expert reduction ranges for the weight gradients.
__global__ void moe_plan_kernel(const int64_t* __restrict__ counts, int n_expert, int n_tiles, int* __restrict__ seg_start,
                                int* __restrict__ cursor, int* __restrict__ tile_expert, int* __restrict__ k0, int* __restrict__ kb) {
  __shared__ int s_start[1025];
  if (threadIdx.x == 0) {
    int off = 0;
    for (int e = 0; e < n_expert; ++e) {
      s_start[e] = off;
      const int c = (int)counts[e];
      off += (c + 255) / 256 * 256;
    }
    s_start[n_expert] = off;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n_expert; e += blockDim.x) {
    seg_start[e] = s_start[e];
    cursor[e] = s_start[e];
    k0[e] = s_start[e];
    kb[e] = (s_start[e + 1] - s_start[e]) / 64;
  }
  if (threadIdx.x == 0) seg_start[n_expert] = s_start[n_expert];
  for (int t = threadIdx.x; t < n_tiles; t += blockDim.x) {
    const int row = t * 256;
    int e = -1;
    if (row < s_start[n_expert]) {
      int lo = 0, hi = n_expert - 1;               // last expert whose segment starts at or before `row` and is not empty there
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_start[mid] <= row) lo = mid; else hi = mid - 1;
      }
      e = lo;
    }
    tile_expert[t] = e;
  }
}

// dest[i] = row of slot i in the grouped layout (-1: dropped slot)
__global__ void moe_dest_kernel(const int64_t* __restrict__ idx, int64_t n, int* __restrict__ cursor, int* __restrict__ dest) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = idx[i];
    dest[i] = e >= 0 ? atomicAdd(cursor + e, 1) : -1;
  }
}

void moe_plan(const int64_t* counts, int n_expert, int n_tiles, int* seg_start, int* cursor, int* tile_expert, int* k0, int* kb,
              cudaStream_t s) {
  if (n_expert > 1024) { set_last_error(__FILE__, __LINE__, "moe_plan: at most 1024 experts per rank"); return; }
  moe_plan_kernel<<<1, 256, 0, s>>>(counts, n_expert, n_tiles, seg_start, cursor, tile_expert, k0, kb);
  B200_CUDA_CHECK(cudaGetLastError());
}
void moe_dest(const int64_t* idx, int64_t n, int* cursor, int* dest, cudaStream_t s) {
  if (n == 0) return;
  const int grid = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  moe_dest_kernel<<<grid, 256, 0, s>>>(idx, n, cursor, dest);
  B200_CUDA_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ row movement
// dst[dest[i]] = scale[i] * src[i / topk]   (one warp per slot, 16-byte vectors)
template <typename T>
__global__ void __launch_bounds__(256) rows_scatter_kernel(const T* __restrict__ src, const int* __restrict__ dest, const float* __restrict__ scale,
                                                            int64_t n_slots, int topk, int d, T* __restrict__ dst) {
  constexpr int N = Vec16<T>::N;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i < n_slots; i += warps) {
    const int r = dest[i];
    if (r < 0) continue;
    const float sc = scale ? scale[i] : 1.f;
    const T* s = src + (i / topk) * (int64_t)d;
    T* o = dst + (int64_t)r * d;
    for (int c = lane * N; c < d; c += 32 * N) {
      Vec16<T> v = ld16(s + c);
      if (scale) {
#pragma unroll
        for (int j = 0; j < N; ++j) v.v[j] = from_f<T>(to_f(v.v[j]) * sc);
      }
      st16(o + c, v);
    }
  }
}

// out[t] = sum_k w[t*topk+k] * src[dest[t*topk+k]]   (fixed k order: deterministic)
template <typename T>
__global__ void __launch_bounds__(256) rows_combine_kernel(const T* __restrict__ src, const int* __restrict__ dest, const float* __restrict__ w,
                                                            int64_t n_tok, int topk, int d, T* __restrict__ out) {
  constexpr int N = Vec16<T>::N;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t t = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); t < n_tok; t += warps) {
    for (int c = lane * N; c < d; c += 32 * N) {
      float acc[N];
#pragma unroll
      for (int j = 0; j < N; ++j) acc[j] = 0.f;
      for (int k = 0; k < topk; ++k) {
        const int r = dest[t * topk + k];
        if (r < 0) continue;
        const float wk = w ? w[t * topk + k] : 1.f;
        const Vec16<T> v = ld16(src + (int64_t)r * d + c);
#pragma unroll
        for (int j = 0; j < N; ++j) acc[j] += wk * to_f(v.v[j]);
      }
      Vec16<T> o;
#pragma unroll
      for (int j = 0; j < N; ++j) o.v[j] = from_f<T>(acc[j]);
      st16(out + t * (int64_t)d + c, o);
    }
  }
}

// dw[i] = <src[dest[i]], g[i / topk]>   (gradient of the combine weights)
template <typename T>
__global__ void __launch_bounds__(256) rows_dot_kernel(const T* __restrict__ src, const int* __restrict__ dest, const T* __restrict__ g,
                                                        int64_t n_slots, int topk, int d, float* __restrict__ dw) {
  constexpr int N = Vec16<T>::N;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i < n_slots; i += warps) {
    const int r = dest[i];
    float acc = 0.f;
    if (r >= 0) {
      const T* a = src + (int64_t)r * d;
      const T* b = g + (i / topk) * (int64_t)d;
      for (int c = lane * N; c < d; c += 32 * N) {
        const Vec16<T> x = ld16(a + c), y = ld16(b + c);
#pragma unroll
        for (int j = 0; j < N; ++j) acc += to_f(x.v[j]) * to_f(y.v[j]);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) dw[i] = acc;
  }
}

static int row_grid(int64_t rows) {
  const int64_t blocks = (rows + 7) / 8;
  const int64_t cap = (int64_t)sm_count() * 8;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

void moe_rows_scatter(const void* src, const int* dest, const float* scale, int64_t n_slots, int topk, int d, void* dst, int dtype, cudaStream_t s) {
  if (n_slots == 0) return;
  if (d % 8) { set_last_error(__FILE__, __LINE__, "moe rows: feature dim must be a multiple of 8"); return; }
  B200_DISPATCH_DTYPE(dtype, T, (rows_scatter_kernel<T><<<row_grid(n_slots), 256, 0, s>>>((const T*)src, dest, scale, n_slots, topk, d, (T*)dst)));
  B200_CUDA_CHECK(cudaGetLastError());
}
void moe_rows_combine(const void* src, const int* dest, const float* w, int64_t n_tok, int topk, int d, void* out, int dtype, cudaStream_t s) {
  if (n_tok == 0) return;
  if (d % 8) { set_last_error(__FILE__, __LINE__, "moe rows: feature dim must be a multiple of 8"); return; }
  B200_DISPATCH_DTYPE(dtype, T, (rows_combine_kernel<T><<<row_grid(n_tok), 256, 0, s>>>((const T*)src, dest, w, n_tok, topk, d, (T*)out)));
  B200_CUDA_CHECK(cudaGetLastError());
}
void moe_rows_dot(const void* src, const int* dest, const void* g, int64_t n_slots, int topk, int d, float* dw, int dtype, cudaStream_t s) {
  if (n_slots == 0) return;
  if (d % 8) { set_last_error(__FILE__, __LINE__, "moe rows: feature dim must be a multiple of 8"); return; }
  B200_DISPATCH_DTYPE(dtype, T, (rows_dot_kernel<T><<<row_grid(n_slots), 256, 0, s>>>((const T*)src, dest, (const T*)g, n_slots, topk, d, dw)));
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace b200
