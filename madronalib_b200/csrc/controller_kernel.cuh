// controller_kernel.cuh -- K11: the smoothed MIDI controllers of EventsToSignals (source/app/MLEventsToSignals.h:
// 170-180, .cpp:264-285 and 431-435) for G instruments x C requested controllers.
//
// Per vector, every SmoothedController first takes the vector's writes of its inputValue (the last one wins), then
// runs output = LinearGlide(inputValue) (source/DSP/MLDSPGens.h:433-515).  The glide is K7's: glide_plan (scalars
// only), glide_lane / glide_of / glide_sample (the row with the warp across the 64 samples), so there is one
// LinearGlide in the library.  Scalar state is SoA [CS_COUNT][C][G]; the mCurrVec rows [C][G][64] are read and written only
// while their glide moves (an idle row equals its target in every sample: K7's rule).
//
// One warp per (controller, 32 instruments): lane l owns instrument g0 + l, scans that instrument's (usually empty)
// change range of the vector and plans its glide; the warp then walks the 32 rows with the lanes across the samples
// (ctrl_walk), so that every row store is one coalesced 256-byte warp store and idle rows are written as constants
// without reading anything.  With a voice map the finished row is stored once per voice of its instrument.
#pragma once
#include "voice_kernel.cuh"

namespace mlb
{
constexpr int kCtrlWarps = 8;  // warps per 256-thread CTA
enum CtrlState { CS_INPUT = 0, CS_TARGET, CS_REM, CS_STEP, CS_COUNT };

struct CtrlArgs
{
  const int32_t* offsets;                // [T][G + 1] into changes
  const mlb_controller_change* changes;  // event order
  const int32_t* ctrl;                   // [C] controller numbers
  uint32_t* state;                       // [CS_COUNT][C][G]
  float* rows;                           // [C][G][64] LinearGlide::mCurrVec
  float* out;                            // [T][n_planes][N][64]
  const int32_t* vmap_off;               // voice map or null: the voices of instrument g are
  const int32_t* vmap_voice;             //   vmap_voice[vmap_off[g] .. vmap_off[g + 1]); g = G: the unmapped voices
  int G, C, N, T, plane0, n_planes, n_gblk;
  float per_f, dy;                       // LinearGlide: vectors per glide, 1 / that
};

// The warp's 32 planned glides, row by row with the lanes across the samples: a moving row advances in delay memory
// (two 128-byte lines), an idle one is its target and reads nothing.  Instrument rows: row j goes to plane row
// g0 + j; with a voice map, once to each voice of instrument g0 + j.
MLB_DEV void ctrl_walk(const GlideLane& mine, float* grow_base, float* plane, const CtrlArgs& a, int g0, int lane)
{
#pragma unroll 1
  for (int j = 0; j < 32 && g0 + j < a.G; ++j)
  {
    const GlideLane l = glide_of(mine, j);
    float* row = grow_base + (size_t)(g0 + j) * MLB_BLOCK + lane;
    const float r0 = l.mode == 2 ? row[0] : 0.f, r1 = l.mode == 2 ? row[32] : 0.f;
    const float y0 = glide_sample(l, r0, lane), y1 = glide_sample(l, r1, lane + 32);
    if (l.mode >= 1) row[0] = y0, row[32] = y1;
    if (a.vmap_off == nullptr)
    {
      float* dst = plane + (size_t)(g0 + j) * MLB_BLOCK + lane;
      __stcs(dst, y0);
      __stcs(dst + 32, y1);
      continue;
    }
    const int k1 = __ldg(a.vmap_off + g0 + j + 1);
    for (int k = __ldg(a.vmap_off + g0 + j); k < k1; ++k)
    {
      float* dst = plane + (size_t)__ldg(a.vmap_voice + k) * MLB_BLOCK + lane;
      __stcs(dst, y0);
      __stcs(dst + 32, y1);
    }
  }
}

__global__ void __launch_bounds__(32 * kCtrlWarps) controller_bank_kernel(CtrlArgs a)
{
  const int w = blockIdx.x * kCtrlWarps + (threadIdx.x >> 5);
  if (w >= a.C * a.n_gblk) return;
  const int lane = threadIdx.x & 31;
  const int c = w / a.n_gblk, gb = w % a.n_gblk, g0 = gb * 32, g = g0 + lane;
  const bool mine_ok = g < a.G;
  const size_t CG = (size_t)a.C * a.G, s = (size_t)c * a.G + g;
  const int number = __ldg(a.ctrl + c);
  uint32_t in = 0u, st0 = 0u, st1 = 0u, st2 = 0xFFFFFFFFu;  // step, target, vectorsRemaining (idle for a spare lane)
  if (mine_ok)
  {
    in = a.state[CS_INPUT * CG + s];
    st0 = a.state[CS_STEP * CG + s];
    st1 = a.state[CS_TARGET * CG + s];
    st2 = a.state[CS_REM * CG + s];
  }
  float* const grow_base = a.rows + (size_t)c * a.G * MLB_BLOCK;
  const uint2* ch = reinterpret_cast<const uint2*>(a.changes);
  for (int t = 0; t < a.T; ++t)
  {
    GlideLane mine;
    mine.mode = -1, mine.a = 0.f, mine.b = 0.f;
    if (mine_ok)
    {
      // the vector's writes of this controller (processControllerEvent clamps the number to 128, .cpp:743-744)
      const int32_t* off = a.offsets + (size_t)t * (a.G + 1) + g;
      const int i1 = __ldg(off + 1);
      for (int i = __ldg(off); i < i1; ++i)
      {
        const uint2 e = __ldg(ch + i);
        if (min((int)(e.x & 0xFFFFu), 128) == number) in = e.y;
      }
      const GlidePlanned p = glide_plan(st0, st1, st2, u2f(in), a.per_f, a.dy, grow_base + (size_t)g * MLB_BLOCK);
      st0 = p.s0, st1 = p.s1, st2 = p.s2;
      mine = glide_lane(p.g);
    }
    float* const plane = a.out + ((size_t)t * a.n_planes + a.plane0 + c) * a.N * MLB_BLOCK;
    ctrl_walk(mine, grow_base, plane, a, g0, lane);
    if (a.vmap_off != nullptr)
    {
      // the voices of no instrument get +0, shared out over the controller's warps
      const int u1 = __ldg(a.vmap_off + a.G + 1);
      for (int k = __ldg(a.vmap_off + a.G) + gb; k < u1; k += a.n_gblk)
      {
        float* dst = plane + (size_t)__ldg(a.vmap_voice + k) * MLB_BLOCK + lane;
        __stcs(dst, 0.f);
        __stcs(dst + 32, 0.f);
      }
    }
    __syncwarp();  // rows written across lanes are read by their own lane (glide_plan) in the next vector
  }
  if (mine_ok)
  {
    a.state[CS_INPUT * CG + s] = in;
    a.state[CS_STEP * CG + s] = st0;
    a.state[CS_TARGET * CG + s] = st1;
    a.state[CS_REM * CG + s] = st2;
  }
}

}  // namespace mlb
