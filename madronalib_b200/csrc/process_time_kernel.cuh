// process_time_kernel.cuh -- K13: AudioContext::ProcessTime (source/app/MLAudioContext.h:23-56, .cpp:16-101), the
// host-transport-locked quarter-note phasor that AudioContext::getBeatPhase() returns, for G instruments.
//
// Per block, each clock applies its transport updates in order (setTimeAndRate, .cpp:16-78), then runs processVector
// (.cpp:88-101): 64 steps of omega_ += dpdt_ (a float += double, i.e. the double sum rounded to float) with the
// float wrap omega_ -= 1.f.  The recurrence is serial, so one thread owns one instrument, with its state in
// registers.  Every operation is the _rn intrinsic of the reference's binary32 / binary64 operation, so nothing can be
// contracted into an FMA.
//
// One warp per 32 instruments: lane l computes instrument g0 + l's row into shared memory, then the warp stores the
// 32 rows with the lanes across the samples, so that every row store is one coalesced 256-byte warp store (the
// layout of controller_kernel.cuh).  With a voice map the row is stored once per voice of its instrument.
#pragma once
#include "voice_kernel.cuh"

namespace mlb
{
constexpr int kPtWarps = 1;  // warps per CTA: a bank of a few thousand instruments spreads its stores over every SM

struct PtArgs
{
  const int32_t* offsets;        // [T][G + 1] into tr
  const mlb_transport* tr;       // in order
  uint64_t* state;               // [MLB_PT_WORDS][G]
  float* out;                    // [T][n_planes][N][64]
  const int32_t* vmap_off;       // voice map or null: the voices of instrument g are
  const int32_t* vmap_voice;     //   vmap_voice[vmap_off[g] .. vmap_off[g + 1]); g = G: the unmapped voices
  int G, N, T, plane0, n_planes, n_gblk;
};

struct PtClock
{
  float omega;
  double dpdt, ppq1, phase1, bpm, sr;
  bool playing1, active1;
  unsigned long long since_prev, since_start;
};

// ProcessTime::setTimeAndRate (.cpp:16-78)
MLB_DEV void pt_set_time(PtClock& c, const mlb_transport& u)
{
  const double ppq = u.ppq_pos, bpm = u.bpm;
  if (isnan(ppq) || isinf(ppq) || isnan(bpm) || isinf(bpm)) return;
  c.sr = u.sample_rate;
  c.bpm = bpm;
  const bool playing = u.is_playing != 0;
  const bool active = (c.ppq1 != ppq) && playing;
  const bool just_started = playing && !c.playing1;
  double phase = 0.;
  if (active)
  {
    phase = ppq > 0. ? __dsub_rn(ppq, floor(ppq)) : ppq;
    c.omega = __double2float_rn(phase);
    if (just_started)
    {
      c.since_start = 0;
      c.omega = 0.f;
      const double minutes_per_sample = __ddiv_rn(__ddiv_rn(1., c.sr), 60.);  // (1. / sampleRate) / 60.
      c.dpdt = __dmul_rn(bpm, minutes_per_sample);
    }
    else
    {
      double d = __dsub_rn(phase, c.phase1);
      if (d < 0.) d = __dadd_rn(d, 1.);
      const double r = __ddiv_rn(d, __ull2double_rn(c.since_prev));
      c.dpdt = r < 0. ? 0. : (r > 1. ? 1. : r);  // ml::clamp: a NaN passes through
    }
  }
  else
  {
    c.omega = -1.f;
    c.dpdt = 0.;
  }
  c.ppq1 = ppq;
  c.phase1 = phase;
  c.active1 = active;
  c.playing1 = playing;
  c.since_prev = 0;
}

__global__ void __launch_bounds__(32 * kPtWarps) process_time_kernel(PtArgs a)
{
  __shared__ float rows[kPtWarps][32][MLB_BLOCK + 1];  // +1: the lanes' column writes fall in distinct banks
  const int wl = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gb = blockIdx.x * kPtWarps + wl, g0 = gb * 32, g = g0 + lane;
  if (gb >= a.n_gblk) return;
  const bool mine = g < a.G;
  const size_t G = (size_t)a.G;
  PtClock c = {};
  if (mine)
  {
    const uint64_t* s = a.state + g;
    c.omega = __uint_as_float((uint32_t)s[MLB_PT_OMEGA * G]);
    c.dpdt = __longlong_as_double((long long)s[MLB_PT_DPDT * G]);
    c.ppq1 = __longlong_as_double((long long)s[MLB_PT_PPQ_POS1 * G]);
    c.phase1 = __longlong_as_double((long long)s[MLB_PT_PPQ_PHASE1 * G]);
    c.playing1 = s[MLB_PT_PLAYING1 * G] != 0;
    c.active1 = s[MLB_PT_ACTIVE1 * G] != 0;
    c.since_prev = s[MLB_PT_SAMPLES_PREV * G];
    c.since_start = s[MLB_PT_SAMPLES_START * G];
    c.bpm = __longlong_as_double((long long)s[MLB_PT_BPM * G]);
    c.sr = __longlong_as_double((long long)s[MLB_PT_SAMPLE_RATE * G]);
  }
  float(*const my)[MLB_BLOCK + 1] = rows[wl];
  for (int t = 0; t < a.T; ++t)
  {
    if (mine)
    {
      const int32_t* off = a.offsets + (size_t)t * (a.G + 1) + g;
      const int i1 = __ldg(off + 1);
      for (int i = __ldg(off); i < i1; ++i) pt_set_time(c, a.tr[i]);
      // ProcessTime::processVector (.cpp:88-101)
      float w = c.omega;
#pragma unroll 8
      for (int n = 0; n < MLB_BLOCK; ++n)
      {
        my[lane][n] = w;
        w = __double2float_rn(__dadd_rn((double)w, c.dpdt));
        if (w > 1.f) w = __fsub_rn(w, 1.f);
      }
      c.omega = w;
      c.since_prev += MLB_BLOCK;
      c.since_start += MLB_BLOCK;
    }
    __syncwarp();
    float* const plane = a.out + ((size_t)t * a.n_planes + a.plane0) * a.N * MLB_BLOCK;
#pragma unroll 1
    for (int j = 0; j < 32 && g0 + j < a.G; ++j)
    {
      const float y0 = my[j][lane], y1 = my[j][lane + 32];
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
    if (a.vmap_off != nullptr)
    {
      // the voices of no instrument get +0, shared out over the warps
      const int u1 = __ldg(a.vmap_off + a.G + 1);
      for (int k = __ldg(a.vmap_off + a.G) + gb; k < u1; k += a.n_gblk)
      {
        float* dst = plane + (size_t)__ldg(a.vmap_voice + k) * MLB_BLOCK + lane;
        __stcs(dst, 0.f);
        __stcs(dst + 32, 0.f);
      }
    }
    __syncwarp();  // the rows are rewritten by their own lanes in the next block
  }
  if (mine)
  {
    uint64_t* s = a.state + g;
    s[MLB_PT_OMEGA * G] = __float_as_uint(c.omega);
    s[MLB_PT_DPDT * G] = (uint64_t)__double_as_longlong(c.dpdt);
    s[MLB_PT_PPQ_POS1 * G] = (uint64_t)__double_as_longlong(c.ppq1);
    s[MLB_PT_PPQ_PHASE1 * G] = (uint64_t)__double_as_longlong(c.phase1);
    s[MLB_PT_PLAYING1 * G] = c.playing1 ? 1u : 0u;
    s[MLB_PT_ACTIVE1 * G] = c.active1 ? 1u : 0u;
    s[MLB_PT_SAMPLES_PREV * G] = c.since_prev;
    s[MLB_PT_SAMPLES_START * G] = c.since_start;
    s[MLB_PT_BPM * G] = (uint64_t)__double_as_longlong(c.bpm);
    s[MLB_PT_SAMPLE_RATE * G] = (uint64_t)__double_as_longlong(c.sr);
  }
}

}  // namespace mlb
