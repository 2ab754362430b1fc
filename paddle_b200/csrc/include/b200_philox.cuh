// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), shared by the token sampler (sampling.cu) and
// the attention dropout mask (attention_dropout_sm100.cu).  kernels/sampling.py:philox4x32_10 is its torch twin.
//
// ---- The attention dropout mask ----
// Element (batch b, head h, query i, key j) of a call with seed s and generator offset o is kept iff its 16-bit draw is below
// keep = round((1 - p) * 2^16): the keep rate is keep / 2^16, within 2^-17 of 1 - p.  The draw comes from one Philox call that serves
// eight elements, two rows by four keys:
//   rows {i0, i0 + 8} x keys {j0, j0 + 1, j0 + 8, j0 + 9},   i0 = 16 (i >> 4) + (i & 7),  j0 = 16 (j >> 4) + 2 ((j & 7) >> 1)
//   key   (s lo, s hi)
//   counter (kc, rc, (o + b H + h) lo, (o + b H + h) hi),    rc = 8 (i >> 4) + (i & 7),  kc = 4 (j >> 4) + ((j & 7) >> 1)
//   draw  = 16-bit half (j & 1) of output word 2 ((i >> 3) & 1) + ((j >> 3) & 1)
// so a call's eight elements are exactly eight halves of its four words (no two share bits), and the (b, h) planes of one call take
// the B H consecutive generator offsets o .. o + B H - 1 (a launch reserves that many; the next one starts past them).
// kernels/attention.py:dropout_keep_mask evaluates the same definition with torch ops.
//
// The shape fits all three kernels' register fragments (a thread of an m64 accumulator holds rows {r, r + 8} and column pairs
// {2c, 2c + 1} + 8 n):
//   forward and deterministic dQ (row = query): a thread's rows and its keys at column groups 2n, 2n + 1 are exactly one call.
//     Cost: one call per 8 elements, 8 calls per 128-key forward tile and 4 per 64-key dQ tile per thread.
//   dK / dV (row = key, transposed): a thread holds keys {k, k + 8} and queries {2c, 2c + 1} + 8 n; the lane holding keys
//     {k + 1, k + 9} is lane ^ 4.  The lane with even k computes the call of its even query i0 = 2c, its partner the call of the odd
//     query 2c + 1, and each hands the other its call's 8 keep bits with one shuffle.  Cost: one call per 8 elements, 4 calls and one
//     shuffle per 64-query tile per thread.
#pragma once
#include <cstdint>

namespace b200 {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

namespace dropout {

// The row and key halves of a call's counter (see above); the caller passes i0 with i0 & 8 == 0 and j0 with j0 & 9 == 0.
__device__ __forceinline__ uint32_t row_counter(int i) { return (uint32_t)(((i >> 4) << 3) | (i & 7)); }
__device__ __forceinline__ uint32_t key_counter(int j) { return (uint32_t)(((j >> 4) << 2) | ((j & 7) >> 1)); }

// Keep bits of one call: bit 4 rh + 2 jh + je for the element at row i0 + 8 rh, key j0 + 8 jh + je.
__device__ __forceinline__ uint32_t keep_bits(uint32_t rc, uint32_t kc, uint32_t k0, uint32_t k1, uint32_t c2, uint32_t c3, uint32_t keep) {
  const uint4 w = philox4x32_10(make_uint4(kc, rc, c2, c3), k0, k1);
  const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
  uint32_t bits = 0;
#pragma unroll
  for (int d = 0; d < 4; ++d) {   // word d = 2 rh + jh, its low half je = 0
    bits |= (uint32_t)((ws[d] & 0xFFFFu) < keep) << (2 * d);
    bits |= (uint32_t)((ws[d] >> 16) < keep) << (2 * d + 1);
  }
  return bits;
}

// A dense attention kernel's parameters with dropout (the forward's attn::Params or the backward's attn_bwd::Params).
template <typename P> struct DropoutParams : P {
  uint32_t keep;           // an element is kept iff its 16-bit draw < keep = round((1 - p) 2^16)
  float rscale;            // 1 / (1 - p)
  int64_t* seed_offset;    // int64 [2] (seed, offset): written by the forward, the only source of the backward's mask
  // forward only: the generator state, resolved on the device as at::cuda::philox::unpack does, so a captured graph draws a fresh
  // mask on every replay: seed_ptr != nullptr: seed = *seed_ptr, offset = *offset_ptr + offset_add; otherwise (seed, offset).
  const int64_t* seed_ptr;
  const int64_t* offset_ptr;
  int64_t offset_add;
  uint64_t seed, offset;
};

// The per-(batch, head) counter words of a call: o + b H + h as two 32-bit halves.
__device__ __forceinline__ void plane_counter(int64_t offset, int batch, int h, int head, uint32_t& c2, uint32_t& c3) {
  const uint64_t o = (uint64_t)offset + (uint64_t)batch * (uint64_t)h + (uint64_t)head;
  c2 = (uint32_t)o;
  c3 = (uint32_t)(o >> 32);
}

}  // namespace dropout
}  // namespace b200
