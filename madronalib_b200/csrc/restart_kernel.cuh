// restart_kernel.cuh -- the lane-selective reset of every stateful bank (mlb_*_reset, DESIGN.md "Restart").
//
// A bank describes its per-lane state as regions.  Region r covers, for lane (or instrument) l,
//   rows k = 0 .. rows-1 of lane_words consecutive 32-bit words at dst + k * row_pitch + l * lane_pitch,
// which is an SoA word array [W][N] (rows W, row_pitch N, lane_pitch 1, lane_words 1; 64-bit words: lane_pitch 2,
// lane_words 2) or a per-lane segment (a delay ring of `stride` floats: rows 1, lane_pitch = lane_words = stride).
// Each word is set from the template `src` (same layout as dst: a bank's start state) or, without one, to `fill`.
//
// One launch resets every listed lane of a bank: one warp per (lane, region) work item, float4 stores wherever the
// region's words are 16-byte aligned (the delay rings and 64-float rows always are).
#pragma once
#include "ops.cuh"

namespace mlb
{
constexpr int kResetWarps = 8;  // work items per 256-thread CTA

struct ResetRegion
{
  uint32_t* dst;
  const uint32_t* src;  // template of the same layout, or null: `fill`
  uint32_t fill;
  int rows;
  int lane_words;
  long long row_pitch, lane_pitch;  // in words
};

__global__ void __launch_bounds__(32 * kResetWarps)
    reset_lanes_kernel(const ResetRegion* __restrict__ regions, int n_regions, const int32_t* __restrict__ lanes,
                       long long n_items)
{
  const long long item = (long long)blockIdx.x * kResetWarps + (threadIdx.x >> 5);
  if (item >= n_items) return;  // the whole warp
  const int lane = threadIdx.x & 31;
  const ResetRegion r = regions[item % n_regions];
  const long long base = (long long)lanes[item / n_regions] * r.lane_pitch;
  const bool vec = (r.lane_words & 3) == 0 && (r.row_pitch & 3) == 0 && (base & 3) == 0 &&
                   ((reinterpret_cast<uintptr_t>(r.dst) | reinterpret_cast<uintptr_t>(r.src)) & 15) == 0;
  for (int k = 0; k < r.rows; ++k)
  {
    const long long at = base + k * r.row_pitch;
    uint32_t* d = r.dst + at;
    const uint32_t* s = r.src ? r.src + at : nullptr;
    if (vec)
    {
      uint4* d4 = reinterpret_cast<uint4*>(d);
      const uint4* s4 = reinterpret_cast<const uint4*>(s);
      const uint4 f4 = make_uint4(r.fill, r.fill, r.fill, r.fill);
      for (int i = lane; i < (r.lane_words >> 2); i += 32) d4[i] = s4 ? s4[i] : f4;
    }
    else
      for (int i = lane; i < r.lane_words; i += 32) d[i] = s ? s[i] : r.fill;
  }
}
}  // namespace mlb
