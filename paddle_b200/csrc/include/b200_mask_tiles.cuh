// Tile skipping for the column-masked flash-attention kernels (attention_flashmask_sm100.cu).
//
// Tile summary: per (batch, mask head, 128-key tile), int32 [8] = the extremes of the column mask's bounds over the tile's keys below
// Sk: {max lts, min lte, max uts, min ute} (the hidden test) then {min lts, max lte, min uts, max ute} (the open test).  mask_tiles_kernel builds it on the device at
// the start of every masked launch, so nothing is read on the host.
//
// Tile class of the query rows [r0, r1) against a key tile, from its summary:
//   hidden  (kHidden):  every key hides every row: (max lts <= r0 and min lte >= r1) or (max uts <= r0 and min ute >= r1);
//   open    (kOpen):    no key hides any row: (min lts >= r1 or max lte <= r0) and (min uts >= r1 or max ute <= r0);
//   partial (kPartial): otherwise.
// Hidden tiles are neither loaded nor multiplied; open tiles skip the per-element mask test.  kernels.attention.colmask_tile_classes
// is the torch twin.
//
// Work lists: the producer warp classifies 32 tiles at a time (one per lane, then a ballot), loads only the visible ones and publishes
// each one's index and class in a shared-memory slot beside its stage, written before the stage's full barrier is armed.  When the
// list ends before the consumers' loop bound, it publishes -1 on the next stage with a plain arrive; the consumers stop there.
#pragma once
#include <climits>
#include <cstdint>

namespace b200 {
namespace mask_skip {

constexpr int kHidden = 0, kPartial = 1, kOpen = 2;
constexpr int kTileKeys = 128;   // keys per summary tile

// The parameters of a tile-skipping kernel: P plus the tile summary int32 [b, mask_heads, n_ktiles, 8] and, for the dK / dV kernel,
// the classes int8 [b, mask_heads, n_ktiles, ceil(sq / 64)] of its 64-row query tiles (its producer has no registers to classify).
template <typename P> struct SkipParams : P {
  const int* tiles;
  const int8_t* classes;
  int n_ktiles;
};

constexpr int kClassRows = 64;

__device__ __forceinline__ int tile_class(const int* t, int r0, int r1) {
  const int4 h = __ldg(reinterpret_cast<const int4*>(t));
  if ((h.x <= r0 && h.y >= r1) || (h.z <= r0 && h.w >= r1)) return kHidden;
  const int4 o = __ldg(reinterpret_cast<const int4*>(t) + 1);
  if ((o.x >= r1 || o.y <= r0) && (o.z >= r1 || o.w <= r0)) return kOpen;
  return kPartial;
}

__device__ __forceinline__ void st_slot(uint32_t addr, int v) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ int ld_slot(uint32_t addr) {
  int v;
  asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// One warp per summary tile: colmask int4 [rows = b * mask_heads, sk] -> tiles int32 [rows, n_ktiles, 8] and, unless classes is
// nullptr, the classes int8 [rows, n_ktiles, num_m] of the 64-row query tiles against it.
__device__ __forceinline__ void mask_tiles_body(const int4* __restrict__ colmask, int* __restrict__ tiles, int8_t* __restrict__ classes,
                                                int64_t n, int sk, int n_ktiles, int num_m) {
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= n) return;
  const int lane = threadIdx.x & 31;
  const int64_t row = w / n_ktiles;
  const int t = (int)(w - row * n_ktiles);
  int v[8] = {INT_MIN, INT_MAX, INT_MIN, INT_MAX, INT_MAX, INT_MIN, INT_MAX, INT_MIN};   // v[c]: max / min of bound c, v[4 + c]: min / max
#pragma unroll
  for (int i = 0; i < kTileKeys / 32; ++i) {
    const int key = t * kTileKeys + i * 32 + lane;
    if (key < sk) {
      const int4 m = __ldg(colmask + row * sk + key);
      const int b[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        v[c] = c & 1 ? min(v[c], b[c]) : max(v[c], b[c]);
        v[4 + c] = c & 1 ? max(v[4 + c], b[c]) : min(v[4 + c], b[c]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    v[c] = c & 1 ? __reduce_min_sync(0xffffffffu, v[c]) : __reduce_max_sync(0xffffffffu, v[c]);
    v[4 + c] = c & 1 ? __reduce_max_sync(0xffffffffu, v[4 + c]) : __reduce_min_sync(0xffffffffu, v[4 + c]);
  }
  int out = v[0];
#pragma unroll
  for (int c = 1; c < 8; ++c) out = lane == c ? v[c] : out;   // no dynamically indexed (local-memory) array
  if (lane < 8) tiles[w * 8 + lane] = out;
  if (classes) {
    for (int mt = lane; mt < num_m; mt += 32) {
      const int r0 = mt * kClassRows, r1 = r0 + kClassRows;
      int cls = kPartial;
      if ((v[0] <= r0 && v[1] >= r1) || (v[2] <= r0 && v[3] >= r1)) cls = kHidden;
      else if ((v[4] >= r1 || v[5] <= r0) && (v[6] >= r1 || v[7] <= r0)) cls = kOpen;
      classes[w * num_m + mt] = (int8_t)cls;
    }
  }
}

}  // namespace mask_skip
}  // namespace b200
