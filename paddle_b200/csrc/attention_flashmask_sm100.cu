// Column-masked flash attention that skips what the mask hides (flashmask, packed variable-length batches, packed documents, sliding
// windows; head_dim 128 and 64, bf16/fp16, with and without dropout), instantiated from the bodies in include/b200_attention_fwd.cuh and
// include/b200_attention_bwd.cuh with SKIP = true.  They live in their own object so that the other objects keep exactly their kernels;
// the MASKED kernels there, which test every element of every tile up to the causal limit, stay reachable for comparison
// (B200_ATTN_MASK_SKIP=0 in kernels/attention.py).
//
// Every launch first builds the tile summary of the column mask (mask_tiles_kernel, include/b200_mask_tiles.cuh) into scratch the caller
// allocates, then runs the main kernels over it.  Per CTA, the producer warp streams only the tiles the mask does not wholly hide,
// publishing each one's index and class beside its stage:
//   forward: the 128-key tiles of a 128-row query tile, classified 32 at a time against the summary;
//   dK / dV (+ dQ): the (query head, 64-row query tile) pairs of a 128-key tile, whose classes the backward's summary kernel writes too
//     (the producer runs in 24 registers);
//   deterministic dQ: the 64-key tiles of a 128-row query tile (classified by the 128-key summary tile holding them).
// Tiles the mask leaves open skip the per-element mask test; the causal and Sk edge tests stay.  Hidden tiles contribute nothing, so
// the results are those of the MASKED kernels except where a wholly hidden tile came first in a row's walk: there the MASKED forward's
// running max restarts from 0 instead of -inf, which changes roundings, not values.  For documents packed on 128-row boundaries the
// kernels walk exactly the tiles, in the same order, that a causal call on each document alone walks, and give the same bits.
//
// The dropout mask is a pure function of (batch, head, query, key), so skipping tiles does not change it.
#include <cuda.h>
#include <type_traits>

#include "include/b200_attention_bwd.cuh"
#include "include/b200_attention_fwd.cuh"
#include "include/b200_mask_tiles.cuh"
#include "include/b200_ops.h"
#include "include/b200_philox.cuh"

namespace b200 {
namespace mask_skip {

__global__ void __launch_bounds__(256) mask_tiles_kernel(const int4* __restrict__ colmask, int* __restrict__ tiles, int8_t* __restrict__ classes,
                                                         int64_t n, int sk, int n_ktiles, int num_m) {
  mask_tiles_body(colmask, tiles, classes, n, sk, n_ktiles, num_m);
}

int n_ktiles(int sk) { return (sk + kTileKeys - 1) / kTileKeys; }
int64_t n_summaries(const AttnArgs& a) { return (int64_t)a.b * (a.mask_heads > 0 ? a.mask_heads : 1) * n_ktiles(a.sk); }
int8_t* classes_of(const AttnArgs& a) { return reinterpret_cast<int8_t*>(a.mask_tiles + n_summaries(a) * 8); }

// with_classes: also the dK / dV kernel's classes of the 64-row query tiles
void build_tiles(const AttnArgs& a, bool with_classes, cudaStream_t s) {
  const int64_t n = n_summaries(a);
  const int num_m = (a.sq + kClassRows - 1) / kClassRows;
  if (n > 0)
    mask_tiles_kernel<<<(unsigned)((n + 7) / 8), 256, 0, s>>>(reinterpret_cast<const int4*>(a.colmask), a.mask_tiles,
                                                               with_classes ? classes_of(a) : nullptr, n, a.sk, n_ktiles(a.sk), num_m);
}

template <typename P>
SkipParams<P> with_tiles(const P& base, const AttnArgs& a) {
  SkipParams<P> p{};
  static_cast<P&>(p) = base;
  p.tiles = a.mask_tiles;
  p.classes = classes_of(a);
  p.n_ktiles = n_ktiles(a.sk);
  return p;
}

}  // namespace mask_skip

namespace attn {

template <bool DROPOUT> using FwdSkipParams = mask_skip::SkipParams<std::conditional_t<DROPOUT, dropout::DropoutParams<Params>, Params>>;

template <typename T, int D, bool DROPOUT>
__global__ void __launch_bounds__(kThreads, 1)
fwd_skip_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                const FwdSkipParams<DROPOUT> p) {
  fwd_body<T, true, false, T, D, false, DROPOUT, true>(map_q, map_k, map_v, p);
}

template <int D, bool DROPOUT>
int fwd_skip(const AttnArgs& a, const AttnDropoutArgs* d, cudaStream_t s) {
  mask_skip::build_tiles(a, false, s);
  return fwd_dense_with<D>(a, s, [&](auto tag_t, auto tag_masked, const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                                     const Params& base, dim3 grid, uint32_t smem) {
    using T = decltype(tag_t);
    if constexpr (decltype(tag_masked)::value) {
      constexpr auto kern = fwd_skip_kernel<T, D, DROPOUT>;
      const uint32_t bytes = smem + (DROPOUT ? kDropoutSmemBytes : 0);
      set_max_dynamic_smem<kern>(bytes);
      if constexpr (DROPOUT) kern<<<grid, kThreads, bytes, s>>>(mq, mk, mv, mask_skip::with_tiles(dropout::with_dropout(base, *d), a));
      else kern<<<grid, kThreads, bytes, s>>>(mq, mk, mv, mask_skip::with_tiles(base, a));
    }
  });
}

}  // namespace attn

namespace attn_bwd {

template <bool DROPOUT> using SkipParams = mask_skip::SkipParams<std::conditional_t<DROPOUT, dropout::DropoutParams<Params>, Params>>;

template <typename T, bool DQ, int D, bool DROPOUT>
__global__ void __launch_bounds__(kThreadsDkv, 1)
dkv_skip_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                const __grid_constant__ CUtensorMap map_do, const __grid_constant__ CUtensorMap map_dq, const SkipParams<DROPOUT> p) {
  dkv_body<T, true, DQ, D, DROPOUT, true>(map_q, map_k, map_v, map_do, map_dq, p);
}

template <typename T, int D, bool DROPOUT>
__global__ void __launch_bounds__(kThreads, 1)
dq_skip_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
               const __grid_constant__ CUtensorMap map_do, const SkipParams<DROPOUT> p) {
  dq_body<T, true, D, DROPOUT, true>(map_q, map_k, map_v, map_do, p);
}

// as launch() in b200_attention_bwd.cuh, on the tile-skipping kernels
template <int D, bool DROPOUT>
int run_skip(const AttnBwdArgs& a, const AttnDropoutArgs* d, cudaStream_t s) {
  mask_skip::build_tiles(a.fwd, true, s);
  return run_with<D>(a, s, [&](auto tag_t, auto tag_masked, const Params& base, bool det, const CUtensorMap (&mq)[2], const CUtensorMap (&mk)[2],
                               const CUtensorMap (&mv)[2], const CUtensorMap (&mdo)[2], const CUtensorMap& mdq) {
    using T = decltype(tag_t);
    if constexpr (decltype(tag_masked)::value) {
      SkipParams<DROPOUT> p;
      if constexpr (DROPOUT) p = mask_skip::with_tiles(dropout::with_dropout(base, *d), a.fwd);
      else p = mask_skip::with_tiles(base, a.fwd);
      const dim3 grid_kv(p.hk, p.b, (p.sk + 127) / 128), grid_q((p.sq + 127) / 128, p.h, p.b);
      if (det) {
        constexpr auto dkv = dkv_skip_kernel<T, false, D, DROPOUT>;
        constexpr auto dq = dq_skip_kernel<T, D, DROPOUT>;
        set_max_dynamic_smem<dkv>(DkvSmem<D>::BYTES);
        set_max_dynamic_smem<dq>(kSmemBytes<D>);
        dkv<<<grid_kv, kThreadsDkv, DkvSmem<D>::BYTES, s>>>(mq[1], mk[0], mv[0], mdo[1], mdq, p);
        dq<<<grid_q, kThreads, kSmemBytes<D>, s>>>(mq[0], mk[1], mv[1], mdo[0], p);
      } else {
        constexpr auto dkv = dkv_skip_kernel<T, true, D, DROPOUT>;
        set_max_dynamic_smem<dkv>(DkvSmem<D>::BYTES);
        dkv<<<grid_kv, kThreadsDkv, DkvSmem<D>::BYTES, s>>>(mq[1], mk[0], mv[0], mdo[1], mdq, p);
      }
    }
  });
}

}  // namespace attn_bwd

int attention_mask_tiles_ints(int b, int mask_heads, int sq, int sk) {
  const int64_t n = (int64_t)b * mask_heads * mask_skip::n_ktiles(sk);
  return (int)(n * 8 + (n * ((sq + mask_skip::kClassRows - 1) / mask_skip::kClassRows) + 3) / 4);
}

int attention_fwd_flashmask(const AttnArgs& a, const AttnDropoutArgs* d, cudaStream_t s) {
  if (!attention_fwd_supported(a) || !a.colmask || !a.mask_tiles) return 1;
  if (a.d == 64) return d ? attn::fwd_skip<64, true>(a, d, s) : attn::fwd_skip<64, false>(a, d, s);
  return d ? attn::fwd_skip<attn::HD, true>(a, d, s) : attn::fwd_skip<attn::HD, false>(a, d, s);
}

int attention_bwd_flashmask(const AttnBwdArgs& a, const AttnDropoutArgs* d, cudaStream_t s) {
  if (!attention_fwd_supported(a.fwd) || !a.fwd.colmask || !a.fwd.mask_tiles) return 1;
  if (a.fwd.d == 64) return d ? attn_bwd::run_skip<64, true>(a, d, s) : attn_bwd::run_skip<64, false>(a, d, s);
  return d ? attn_bwd::run_skip<attn_bwd::HD, true>(a, d, s) : attn_bwd::run_skip<attn_bwd::HD, false>(a, d, s);
}

}  // namespace b200
