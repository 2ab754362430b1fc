// Flash attention for training at head_dim 64 (bf16/fp16, sm_90a): the dense and column-masked forward and the backward (single pass,
// and the deterministic dK/dV + dQ pair), instantiated from the head_dim 128 kernels' bodies (include/b200_attention_fwd.cuh,
// include/b200_attention_bwd.cuh) with D = 64.  attention_fwd / attention_bwd call these launchers when d == 64; they keep the tiling
// of the 128-wide kernels (128 query rows x 128 keys in the forward, 128 keys x 64 query rows in dK / dV), so every operand tile is one
// 64-wide d chunk and each TMA load one box.  The kernels live in their own object so that the head_dim 128 objects keep their kernels.
#include <cuda.h>

#include "include/b200_attention_bwd.cuh"
#include "include/b200_attention_fwd.cuh"
#include "include/b200_ops.h"

namespace b200 {

int attention_fwd_d64(const AttnArgs& a, cudaStream_t s) { return attn::fwd_dense<64>(a, s); }

int attention_bwd_d64(const AttnBwdArgs& a, cudaStream_t s) { return attn_bwd::run<64>(a, s); }

}  // namespace b200
