// Flash-attention backward for sm_90a (head_dim 128, and 64 in attention_d64_sm100.cu; bf16/fp16), wgmma + TMA.
//
//   prep_kernel: delta[row] = dO . O, lse pre-scaled by log2(e), both per query row into a padded stats buffer the main kernel stages
//     per tile with bulk copies; in single-pass mode it also zeroes the fp32 dQ accumulator.
//   dkv_kernel: one CTA owns a 128-key K/V tile of one (batch, kv head) - 64 keys per MMA warpgroup - and walks the 64-row query tiles
//     that can see it (and, under GQA, every query head of the group).  It computes the TRANSPOSED tiles S^T = K Q^T and dP^T = V dO^T
//     (accumulator row = key), so that P^T and dS^T, packed to 16 bits, are already the register A fragments of dV += P^T dO and
//     dK += dS^T Q; the dV / dK accumulators stay in registers across the whole loop.  S^T and dP^T are committed as separate groups
//     (the exp of P^T overlaps the dP^T MMAs) and dV is issued before dS^T is formed.
//     With the dQ stage (the default, single-pass backward: 5 GEMMs, one main launch) dS^T also goes to shared memory, each warpgroup
//     computes dQ = dS K for 64 of the 128 head dims over all 128 keys of the tile and adds it into the fp32 dQ with a TMA bulk
//     reduce-add.  The additions land in arrival order, so dQ is reproducible only to rounding.
//   dq_kernel (deterministic mode, FLAGS_cudnn_deterministic, after dkv_kernel without the dQ stage): one CTA owns 128 query rows of
//     one (batch, head) - 64 per warpgroup - and walks the 64-key tiles it can see: S = Q K^T, dP = dO V^T (accumulator row = query),
//     dS packed in registers is the A fragment of dQ += dS K.  Every dQ element is written once, by one thread, in a fixed order: the
//     result is bitwise reproducible, at the price of recomputing S and dP (7 GEMMs for 5).
// The K and Q tiles are consumed K-major (S) and MN-major (dQ, dK) from one copy by choice of descriptor.
//
// The kernel bodies and the launcher live in include/b200_attention_bwd.cuh.
//
// Parity (behaviour): flash_attn_grad (paddle/phi/kernels/gpu/flash_attn_grad_kernel.cu -> flash-attention library).
#include <cuda.h>

#include "include/b200_attention_bwd.cuh"
#include "include/b200_ops.h"

namespace b200 {

int attention_bwd_stats_pad(int sq) { return (sq + 63) / 64 * 64; }

int attention_bwd(const AttnBwdArgs& a, cudaStream_t s) {
  if (!attention_fwd_supported(a.fwd)) return 1;
  if (a.fwd.colmask && a.fwd.mask_tiles) return attention_bwd_flashmask(a, nullptr, s);
  return a.fwd.d == 64 ? attention_bwd_d64(a, s) : attn_bwd::run<attn_bwd::HD>(a, s);
}

}  // namespace b200
