// Attention dropout for training on the sm_90a flash-attention kernels (head_dim 128 and 64, bf16/fp16, dense or column-masked): the
// forward, the single-pass dK/dV + dQ backward and the deterministic dK/dV + dQ pair, instantiated from the bodies in
// include/b200_attention_fwd.cuh and include/b200_attention_bwd.cuh with DROPOUT = true.  They live in their own object so that the
// dropout-free objects keep exactly their kernels.
//
// Mask: Z[b, h, i, j] = (Philox draw < round((1 - p) 2^16)), one Philox4x32-10 call per 8 elements laid out so the forward / dQ tiles
// (row = query) and the transposed dK / dV tiles (row = key) evaluate it without wasted draws (include/b200_philox.cuh).  Each kernel
// regenerates the bits of its own tile while the tile's first MMAs are in flight; nothing is stored.
//
// Forward: P is dropped after its row sum is accumulated (l and lse are those of the undropped softmax), the dropped entries are zeroed
// before P is packed into the A fragments of P V, and 1 / (1 - p) is folded into the epilogue's 1 / l, so kept entries see exactly the
// rounding of the p = 0 kernel.  Backward, with Zs = Z / (1 - p): dV += (Zs P)^T dO, dS = P (Zs dP - delta) scale; delta = rowsum(dO O)
// on the dropped O, so the stats kernel is the dropout-free one.
//
// Seed and offset: the forward resolves them on the device from the generator state (a captured CUDA graph reads the graph's seed and
// offset slots at replay, so every replay draws a fresh mask) or from a fixed pair, and writes the pair it used to seed_offset, which is
// the backward's only source.
#include <cuda.h>
#include <cmath>

#include "include/b200_attention_bwd.cuh"
#include "include/b200_attention_fwd.cuh"
#include "include/b200_ops.h"
#include "include/b200_philox.cuh"

namespace b200 {
using dropout::with_dropout;

namespace attn {

template <typename T, bool MASKED, int D>
__global__ void __launch_bounds__(kThreads, 1)
fwd_dropout_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                   const dropout::DropoutParams<Params> p) {
  fwd_body<T, MASKED, false, T, D, false, true>(map_q, map_k, map_v, p);
}

template <int D>
int fwd_dense_dropout(const AttnArgs& a, const AttnDropoutArgs& d, cudaStream_t s) {
  return fwd_dense_with<D>(a, s, [&](auto tag_t, auto tag_masked, const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                     const Params& base, dim3 grid, uint32_t smem) {
    using T = decltype(tag_t);
    constexpr bool MASKED = decltype(tag_masked)::value;
    const uint32_t bytes = smem + kDropoutSmemBytes;
    set_max_dynamic_smem<fwd_dropout_kernel<T, MASKED, D>>(bytes);
    fwd_dropout_kernel<T, MASKED, D><<<grid, kThreads, bytes, s>>>(mq, mk, mv, with_dropout(base, d));
  });
}

}  // namespace attn

namespace attn_bwd {

template <typename T, bool MASKED, bool DQ, int D>
__global__ void __launch_bounds__(kThreadsDkv, 1)
dkv_dropout_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                   const __grid_constant__ CUtensorMap map_do, const __grid_constant__ CUtensorMap map_dq, const dropout::DropoutParams<Params> p) {
  dkv_body<T, MASKED, DQ, D, true>(map_q, map_k, map_v, map_do, map_dq, p);
}

template <typename T, bool MASKED, int D>
__global__ void __launch_bounds__(kThreads, 1)
dq_dropout_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                  const __grid_constant__ CUtensorMap map_do, const dropout::DropoutParams<Params> p) {
  dq_body<T, MASKED, D, true>(map_q, map_k, map_v, map_do, p);
}

// as launch() in b200_attention_bwd.cuh, on the dropout kernels
template <int D>
int run_dropout(const AttnBwdArgs& a, const AttnDropoutArgs& d, cudaStream_t s) {
  return run_with<D>(a, s, [&](auto tag_t, auto tag_masked, const Params& base, bool det, const CUtensorMap (&mq)[2], const CUtensorMap (&mk)[2],
                               const CUtensorMap (&mv)[2], const CUtensorMap (&mdo)[2], const CUtensorMap& mdq) {
    using T = decltype(tag_t);
    constexpr bool MASKED = decltype(tag_masked)::value;
    const auto p = with_dropout(base, d);
    const dim3 grid_kv(p.hk, p.b, (p.sk + 127) / 128), grid_q((p.sq + 127) / 128, p.h, p.b);
    if (det) {
      set_max_dynamic_smem<dkv_dropout_kernel<T, MASKED, false, D>>(DkvSmem<D>::BYTES);
      set_max_dynamic_smem<dq_dropout_kernel<T, MASKED, D>>(kSmemBytes<D>);
      dkv_dropout_kernel<T, MASKED, false, D><<<grid_kv, kThreadsDkv, DkvSmem<D>::BYTES, s>>>(mq[1], mk[0], mv[0], mdo[1], mdq, p);
      dq_dropout_kernel<T, MASKED, D><<<grid_q, kThreads, kSmemBytes<D>, s>>>(mq[0], mk[1], mv[1], mdo[0], p);
    } else {
      set_max_dynamic_smem<dkv_dropout_kernel<T, MASKED, true, D>>(DkvSmem<D>::BYTES);
      dkv_dropout_kernel<T, MASKED, true, D><<<grid_kv, kThreadsDkv, DkvSmem<D>::BYTES, s>>>(mq[1], mk[0], mv[0], mdo[1], mdq, p);
    }
  });
}

}  // namespace attn_bwd

int attention_fwd_dropout(const AttnArgs& a, const AttnDropoutArgs& d, cudaStream_t s) {
  if (!attention_fwd_supported(a) || !(d.p > 0.0 && d.p < 1.0) || !d.seed_offset) return 1;
  if (a.colmask && a.mask_tiles) return attention_fwd_flashmask(a, &d, s);
  return a.d == 64 ? attn::fwd_dense_dropout<64>(a, d, s) : attn::fwd_dense_dropout<attn::HD>(a, d, s);
}

int attention_bwd_dropout(const AttnBwdArgs& a, const AttnDropoutArgs& d, cudaStream_t s) {
  if (!attention_fwd_supported(a.fwd) || !(d.p > 0.0 && d.p < 1.0) || !d.seed_offset) return 1;
  if (a.fwd.colmask && a.fwd.mask_tiles) return attention_bwd_flashmask(a, &d, s);
  return a.fwd.d == 64 ? attn_bwd::run_dropout<64>(a, d, s) : attn_bwd::run_dropout<attn_bwd::HD>(a, d, s);
}

}  // namespace b200
