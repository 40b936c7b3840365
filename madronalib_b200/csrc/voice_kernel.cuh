// voice_kernel.cuh -- K7: EventsToSignals::Voice for V voices (SURVEY 8f row 3).
// Reference: source/app/MLEventsToSignals.cpp:47-263 (E below), MLEventsToSignals.h:99-168,
// glides source/DSP/MLDSPGens.h:433-590 (G).  One lane = one Voice; a launch runs n_blocks vectors:
// beginProcess (drift), the vector's note events (sample-accurate gate / pitch glide / age), the
// instantaneous controller values, endProcess (vector-accurate LinearGlides, bend and drift added to
// pitch).  Input: one 72-byte mlb_voice_events record per voice and vector; output: up to 8 rows.
// Scalar state is SoA [word][V]; the six LinearGlide::mCurrVec rows are only touched while a glide
// is moving (an idle LinearGlide's row equals its target in every lane of the row).
#pragma once
#include "functors.cuh"

namespace mlb
{
enum VoiceGlide { VG_BEND = 0, VG_MOD, VG_X, VG_Y, VG_Z, VG_DRIFT, VG_PRESSURE, VG_COUNT };
enum VoiceState
{
  VS_PG_CURR = 0, VS_PG_STEP, VS_PG_TARGET, VS_PG_REM, VS_PG_PER, VS_PG_DY,  // pitchGlide (G:517-590)
  VS_GL = 6,                       // 6 x {step, target, vectorsRemaining, spare}
  VS_VEL = VS_GL + 4 * VG_COUNT,   // currentVelocity, currentPitch, bend, mod, x, y, z
  VS_PITCH, VS_BEND, VS_MOD, VS_X, VS_Y, VS_Z, VS_PRESSURE,
  VS_AGE, VS_AGE_STEP, VS_SEED, VS_DRIFT_COUNTER, VS_NEXT_DRIFT, VS_CUR_DRIFT,
  VS_COUNT
};
enum VoiceCoef { VC_GLIDE_SAMPLES = 0, VC_DRIFT_AMOUNT, VC_BEND_RANGE, VC_VOICE_ROW, VC_COUNT };

struct VoiceArgs
{
  const mlb_voice_events* ev;  // [T][V]
  float* out;                  // [T][P][V][64], rows in planes 0..7
  size_t out_block;            // floats per block of out: P * V * 64 (P = 8, or more when controller planes follow)
  uint32_t* state;             // [VS_COUNT][V]
  const float* coef;           // [VC_COUNT][V]
  float* grows;                // [VG_COUNT][V][64]  LinearGlide::mCurrVec
  int V, T;
  unsigned row_mask;
  float sr;                    // Voice::sr (a double in the reference, set from this value)
  float gl_per, gl_dy;         // LinearGlide coefficients of bend/mod/x/y/z (sr * kGlideTimeSeconds)
  float dr_per, dr_dy;         // ... of pitchDriftGlide (sr * kDriftTimeSeconds)
  float pc_per, pc_dy;         // ... of the channel-pressure SmoothedController (int(sr * kControllerGlideTimeSeconds))
  int midi;                    // MLB_VOICES_MIDI: z row += smoothed channel pressure (processVector, E:432-447)
};

struct VoiceRegs
{
  uint32_t pg[4];
  float pg_per_f, pg_dy;
  float vel, pitch;
  uint32_t age, age_step;
  int next_frame;
};

// SampleAccurateLinearGlide::setGlideTimeInSamples, G:527-532
MLB_DEV void voice_set_glide_time(VoiceRegs& r, float t)
{
  int n = cvt_trunc(t);
  if (n < 1) n = 1;
  r.pg_per_f = __int2float_rn(n);
  r.pg_dy = __fdiv_rn(1.0f, __int2float_rn(n));
}
// one output frame, E:134-140: gate, glided pitch, age -> seconds (samplesToSeconds, E:12-18)
// Row tiles in shared memory: 32 rows x 64 floats per warp, 8 KB, unpadded, swizzled by 16-byte groups:
// frames 4g..4g+3 of row j sit in group g ^ (j & 7) of the row.  A lane reads and writes its own row with
// 128-bit accesses (each quarter-warp touches 8 different groups), and the warp stores one row with two full
// 128-byte lines from 32 different banks.  8 KB instead of a padded 32 x 65 tile is what lets 14 warps
// (2 CTAs of 7) live on an SM instead of 12.  14 warps x 16 KB = 224 KB is the most an SM holds; even so, on the 132
// SMs of an H100 SXM (1 848 warp slots) the 2 048 warps of a 65 536-voice bank take 1.11 waves, and 6 warps per CTA
// (12 per SM, 1.29 waves) measured faster there (DESIGN.md section 7): the default, 7 stays the most MLB_VOICE_WARPS allows.
constexpr int kVoiceTileFloats = 32 * MLB_BLOCK;
constexpr int kVoiceWarpsPerCta = 7;       // gate + pitch tiles: 7 x 16 KB = 112 KB per CTA, two CTAs per SM
constexpr int kVoiceWarpsPerCtaDefault = 6;
constexpr int kVoiceWarpsPerCtaTime = 4;   // + elapsed-time tile: 4 x 24 KB

// frame t of this lane's row (scalar access: the retrigger path, which can revisit frames); sw = (lane & 7) << 2
MLB_DEV int voice_word(int t, int sw) { return t ^ sw; }

// samplesToSeconds (E:12-18) is an FP64 divide: only in the kernel instance that writes the elapsed-time row
MLB_DEV void voice_tick(VoiceRegs& r, float sr, bool want_time, float& p, float& tm)
{
  const float co[2] = {r.pg_per_f, r.pg_dy};
  p = sample_glide_tick<true>(r.pitch, r.pg, co);
  r.age += r.age_step;
  if (want_time) tm = __double2float_rn(__ddiv_rn((double)r.age, (double)sr));
}
// the warp's 32 rows of one output plane: tile row j -> plane[(v0 + j)][0..63], two 128-B lines per row
__device__ __noinline__ void voice_store_tile(const float* tile, float* plane, int v0, int V, int lane)
{
  __syncwarp();
#pragma unroll 4
  for (int j = 0; j < 32; ++j)
  {
    if (v0 + j >= V) break;
    float* dst = plane + (size_t)(v0 + j) * MLB_BLOCK;
    const float* row = tile + j * MLB_BLOCK + ((((lane >> 2) ^ (j & 7)) << 2) | (lane & 3));
    __stcs(dst + lane, row[0]);
    __stcs(dst + 32 + lane, row[32]);
  }
  __syncwarp();
}

// LinearGlide::operator()(float), G:459-505.  The row mCurrVec lives in delay memory and is touched only
// while the glide moves: an idle glide's row equals DSPVector(target) (landing writes the target into
// every element, construction and setValue leave zeros with target zero).
struct GlidePlan
{
  int mode;  // -1 idle, 0 land on target, 1 start, 2 continue
  float step, target, cv;
};
// st: step, target, vectorsRemaining -> updated in place.  Out of line: seven calls per vector, and the kernel's
// instruction footprint is what its warps stall on (one copy instead of seven).
struct GlidePlanned
{
  GlidePlan g;
  uint32_t s0, s1, s2;
};
__device__ __noinline__ GlidePlanned glide_plan(uint32_t s0, uint32_t s1, uint32_t s2, float f, float per_f, float dy,
                                                 const float* row)
{
  GlidePlanned o;
  GlidePlan& g = o.g;
  g.step = u2f(s0), g.target = u2f(s1);
  g.cv = 0.f;
  const int rem_prev = (int32_t)s2;
  int remaining = rem_prev;
  const int per = cvt_trunc(per_f);
  if (f != g.target)
  {
    g.target = f;
    remaining = per;
  }
  if (remaining < 0)
    g.mode = -1;
  else if (remaining == 0)
  {
    g.mode = 0;
    g.step = 0.f;
    remaining--;
  }
  else if (remaining == per)
  {
    g.mode = 1;
    // currentValue = mCurrVec[63]; an idle row is its (previous) target
    g.cv = rem_prev < 0 ? u2f(s1) : row[MLB_BLOCK - 1];
    g.step = __fmul_rn(__fsub_rn(g.target, g.cv), dy);
    remaining--;
  }
  else
  {
    g.mode = 2;
    remaining--;
  }
  o.s0 = f2u(g.step), o.s1 = f2u(g.target), o.s2 = (uint32_t)remaining;
  return o;
}
// ---- the glides of a vector, run TRANSPOSED: the warp walks its 32 voices, lane = sample index ----
// A lane plans its own voice's glides (glide_plan above, scalars only); the 64-sample rows are then produced
// row by row with the warp across the samples, so that
//   * the mode of a row is warp-uniform (no divergence between idle / starting / moving glides),
//   * a moving glide's row in delay memory is read and written as two full 128-byte lines (a lane walking
//     its own 256-byte row touched 32 sectors per load and fetched each twice), and idle rows cost no memory,
//   * the loads of several rows are in flight together (four rows per step, predicated),
//   * the finished sample goes straight to the output plane (the kPitch row picks up bend and drift on the
//     way out of its tile; the glide-only rows never see shared memory).
// What a lane offers to the others: mode, a = step (moving / starting) or target (idle), b = start value.
struct GlideLane
{
  int mode;  // <= 0 idle, 1 start, 2 continue
  float a, b;
};
MLB_DEV GlideLane glide_lane(const GlidePlan& g)
{
  GlideLane l;
  l.mode = g.mode;
  l.a = g.mode >= 1 ? g.step : g.target;
  l.b = g.cv;
  return l;
}
MLB_DEV GlideLane glide_of(const GlideLane& mine, int j)  // voice j's plan, to every lane
{
  GlideLane l;
  l.mode = __shfl_sync(0xffffffffu, mine.mode, j);
  l.a = __shfl_sync(0xffffffffu, mine.a, j);
  l.b = __shfl_sync(0xffffffffu, mine.b, j);
  return l;
}
// sample n of the row: idle -> target; start -> cv + ramp[n] * step; continue -> row[n] + step  (G:459-505)
MLB_DEV float glide_sample(const GlideLane& l, float r, int n)
{
  const float y2 = __fadd_rn(r, l.a);
  const float y1 = __fadd_rn(l.b, __fmul_rn(unity_ramp(n), l.a));
  return l.mode == 2 ? y2 : (l.mode == 1 ? y1 : l.a);
}
// Advance one glide whose row nobody wants: only the voices whose glide moves are visited, four at a time.
__device__ __noinline__ void glide_advance(int m_mode, float m_a, float m_b, float* grow_base, int v0, int V, int lane)
{
  GlideLane mine;
  mine.mode = m_mode, mine.a = m_a, mine.b = m_b;
  unsigned act = __ballot_sync(0xffffffffu, mine.mode >= 1 && v0 + lane < V);
  while (act)
  {
    int jj[4];
    bool ok[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
      ok[k] = act != 0u;
      jj[k] = ok[k] ? __ffs(act) - 1 : 0;
      act &= act - (ok[k] ? 1u : 0u);
    }
    GlideLane l[4];
    float r0[4], r1[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) l[k] = glide_of(mine, jj[k]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
      const float* row = grow_base + (size_t)(v0 + jj[k]) * MLB_BLOCK + lane;
      const bool ld = ok[k] && l[k].mode == 2;
      r0[k] = ld ? row[0] : 0.f;
      r1[k] = ld ? row[32] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
      if (!ok[k]) continue;
      float* row = grow_base + (size_t)(v0 + jj[k]) * MLB_BLOCK + lane;
      row[0] = glide_sample(l[k], r0[k], lane);
      row[32] = glide_sample(l[k], r1[k], lane + 32);
    }
  }
}
// One glide-only output row (kZ / kX / kY / kMod) for the warp's 32 voices: sample -> plane, moving rows updated
// in delay memory.  With `extra`, a second glide (the MIDI channel-pressure glide, added to kZ) runs alongside.
__device__ __noinline__ void glide_row_out(int m_mode, float m_a, float m_b, float* grow_base, bool extra, int x_mode,
                                           float x_a, float x_b, float* extra_base, float* plane, int v0, int V, int lane)
{
  GlideLane mine, xmine;
  mine.mode = m_mode, mine.a = m_a, mine.b = m_b;
  xmine.mode = x_mode, xmine.a = x_a, xmine.b = x_b;
  unsigned moving = __ballot_sync(0xffffffffu, mine.mode >= 1);
  if (extra) moving |= __ballot_sync(0xffffffffu, xmine.mode >= 1);
#pragma unroll 1
  for (int j0 = 0; j0 < 32; j0 += 4)
  {
    if (v0 + j0 >= V) break;
    if (((moving >> j0) & 0xFu) == 0u)  // four idle voices: their rows are their targets, nothing in delay memory
    {
#pragma unroll
      for (int k = 0; k < 4; ++k)
      {
        if (v0 + j0 + k >= V) break;
        float y = __shfl_sync(0xffffffffu, mine.a, j0 + k);
        if (extra) y = __fadd_rn(y, __shfl_sync(0xffffffffu, xmine.a, j0 + k));
        const size_t off = (size_t)(v0 + j0 + k) * MLB_BLOCK + lane;
        __stcs(plane + off, y);
        __stcs(plane + off + 32, y);
      }
      continue;
    }
    GlideLane l[4], e[4];
    float r0[4], r1[4], s0[4], s1[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
      l[k] = glide_of(mine, j0 + k);
      if (extra) e[k] = glide_of(xmine, j0 + k);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
      const bool ok = v0 + j0 + k < V;
      const float* row = grow_base + (size_t)(v0 + j0 + k) * MLB_BLOCK + lane;
      const bool ld = ok && l[k].mode == 2;
      r0[k] = ld ? row[0] : 0.f;
      r1[k] = ld ? row[32] : 0.f;
      s0[k] = s1[k] = 0.f;
      if (extra)
      {
        const float* xrow = extra_base + (size_t)(v0 + j0 + k) * MLB_BLOCK + lane;
        const bool lx = ok && e[k].mode == 2;
        s0[k] = lx ? xrow[0] : 0.f;
        s1[k] = lx ? xrow[32] : 0.f;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
    {
      if (v0 + j0 + k >= V) break;
      const size_t off = (size_t)(v0 + j0 + k) * MLB_BLOCK + lane;
      float y0 = glide_sample(l[k], r0[k], lane), y1 = glide_sample(l[k], r1[k], lane + 32);
      if (l[k].mode >= 1) grow_base[off] = y0, grow_base[off + 32] = y1;
      if (extra)
      {
        const float x0 = glide_sample(e[k], s0[k], lane), x1 = glide_sample(e[k], s1[k], lane + 32);
        if (e[k].mode >= 1) extra_base[off] = x0, extra_base[off + 32] = x1;
        y0 = __fadd_rn(y0, x0), y1 = __fadd_rn(y1, x1);
      }
      __stcs(plane + off, y0);
      __stcs(plane + off + 32, y1);
    }
  }
}

// Two instances: TIME = false (gate + pitch tiles, 7 warps per CTA, at most 128 registers so that two CTAs share an SM)
// and TIME = true (a third tile for the elapsed-time row and the FP64 divide per frame; 4 warps per CTA, free to use
// more registers).
template <bool TIME>
__global__ void __launch_bounds__(32 * (TIME ? kVoiceWarpsPerCtaTime : kVoiceWarpsPerCta), 2) voice_bank_kernel(const VoiceArgs a)
{
  extern __shared__ __align__(16) float voice_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v_raw = blockIdx.x * blockDim.x + threadIdx.x;
  const int v0 = v_raw - lane;
  if (v0 >= a.V) return;                      // whole warp out of range
  const bool live = v_raw < a.V;
  const int v = live ? v_raw : a.V - 1;       // dead lanes shadow the last voice, their stores are masked
  const size_t V = (size_t)a.V;
  constexpr bool want_time = TIME;  // == (a.row_mask & 128) != 0, the host picks the instance
  const int n_tiles = want_time ? 3 : 2;  // gate, pitch (+ elapsed time)
  float* const tiles = voice_smem + (size_t)warp * n_tiles * kVoiceTileFloats;
  float* const gate = tiles + lane * MLB_BLOCK;  // this lane's row, groups swizzled by l7
  float* const pitch = gate + kVoiceTileFloats;
  float* const tm = pitch + kVoiceTileFloats;
  const int l7 = lane & 7, sw = l7 << 2;
  float4* const gate4 = reinterpret_cast<float4*>(gate);
  float4* const pitch4 = reinterpret_cast<float4*>(pitch);
  float4* const tm4 = reinterpret_cast<float4*>(tm);
  uint32_t st[VS_COUNT];  // the glide words [VS_GL, VS_VEL) are not kept here (see glide_plan below)
#pragma unroll
  for (int i = 0; i < VS_COUNT; ++i)
    if (i < VS_GL || i >= VS_VEL) st[i] = a.state[(size_t)i * V + v];
  const float glide_samples = a.coef[(size_t)VC_GLIDE_SAMPLES * V + v];  // (float)pitchGlideTimeInSamples
  const float drift_amount = a.coef[(size_t)VC_DRIFT_AMOUNT * V + v];
  const float bend_range = a.coef[(size_t)VC_BEND_RANGE * V + v];
  const float voice_row = a.coef[(size_t)VC_VOICE_ROW * V + v];

  VoiceRegs r;
#pragma unroll
  for (int i = 0; i < 4; ++i) r.pg[i] = st[VS_PG_CURR + i];
  r.pg_per_f = u2f(st[VS_PG_PER]), r.pg_dy = u2f(st[VS_PG_DY]);
  r.vel = u2f(st[VS_VEL]), r.pitch = u2f(st[VS_PITCH]);
  r.age = st[VS_AGE], r.age_step = st[VS_AGE_STEP];
  float cur[5] = {u2f(st[VS_BEND]), u2f(st[VS_MOD]), u2f(st[VS_X]), u2f(st[VS_Y]), u2f(st[VS_Z])};
  float cur_pressure = u2f(st[VS_PRESSURE]);
  uint32_t seed = st[VS_SEED];
  int drift_counter = (int)st[VS_DRIFT_COUNTER], next_drift = (int)st[VS_NEXT_DRIFT];
  float cur_drift = u2f(st[VS_CUR_DRIFT]);


  for (int t = 0; t < a.T; ++t)
  {
    // ---- beginProcess, E:90-124 ----
    r.next_frame = 0;
    drift_counter += MLB_BLOCK;
    if (drift_counter >= next_drift)
    {
      const float d = noise_tick(seed);  // RandomScalarSource::getFloat == NoiseGen's LCG step
      const float next_mul = __fadd_rn(1.0f, fabsf(noise_tick(seed)));
      cur_drift = d;
      drift_counter = 0;
      next_drift = __double2int_rz(__dmul_rn(__dmul_rn((double)a.sr, (double)next_mul), 8.0));
    }
    // ---- the vector's note events (E:126-220) and the tail fill of endProcess (E:224-236) ----
    // The reference runs, per event, [pre-actions; frames up to the event; post-actions], then fills the
    // rest of the vector.  Here every lane emits ONE frame per iteration of a warp-uniform loop and
    // steps its own event cursor in between, so lanes with different event times do not serialise.
    const uint32_t* rec = reinterpret_cast<const uint32_t*>(a.ev + ((size_t)t * V + v));
    if (t + 1 < a.T)  // the next vector's record (72 B, streamed from DRAM once): have it in L2 by then
    {
      const char* nx = reinterpret_cast<const char*>(a.ev + ((size_t)(t + 1) * V + v));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(nx));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(nx + 64));
    }
    const uint32_t head = rec[0], times = rec[1], types = rec[2], flags = rec[3];
    const int n_events = min((int)(head & 0xFFu), MLB_VOICE_MAX_EVENTS);
    const unsigned set_mask = (head >> 8) & 0xFFu;
    // Decode the (at most 4) note events once.  ev_d = frame before which the event takes effect
    // (retrigger: its gate-0 frame is ev_d - 1), ev_kind = 0 ignored / 1 on / 2 retrigger / 3 off.
    int ev_d[MLB_VOICE_MAX_EVENTS], ev_kind[MLB_VOICE_MAX_EVENTS];
    bool monotone = true;
    {
      int nf = 0;  // nextFrameToProcess as the reference would see it
#pragma unroll
      for (int k = 0; k < MLB_VOICE_MAX_EVENTS; ++k)
      {
        int dest = (int)((times >> (8 * k)) & 0xFFu);
        dest = dest > MLB_BLOCK ? MLB_BLOCK : dest;
        const int type = (int)((types >> (8 * k)) & 0xFFu);
        int kind = type == MLB_EV_NOTE_ON ? 1 : type == MLB_EV_NOTE_RETRIG ? 2 : type == MLB_EV_NOTE_OFF ? 3 : 0;
        if (k >= n_events) kind = 0;
        if (kind == 2 && dest == 0) dest = 1;
        const int bound = kind == 2 ? dest - 1 : dest;
        if (kind != 0)
        {
          if (bound < nf) monotone = false;  // the reference would step back (e.g. a pedal-release note-off at frame 0)
          nf = dest;
        }
        ev_d[k] = dest, ev_kind[k] = kind;
      }
    }
    if (__all_sync(0xffffffffu, monotone))
    {
      // Fast path: frames 0..63 are each emitted once, in order.  Event k's pre-actions (age reset, glide
      // time) apply as soon as event k-1 is done, its post-actions (new pitch / velocity) before frame ev_d[k].
      int k = 0;
      // the current event's frame and kind are kept in scalars (cur_d = 1000 when there is none), so that the
      // 64-iteration frame loop below never indexes the decoded event arrays
      int cur_d = 1000, cur_kind = 0;
      auto advance = [&]()  // make the next non-ignored event current and apply its pre-actions
      {
        while (k < MLB_VOICE_MAX_EVENTS && ev_kind[k] == 0) ++k;
        cur_d = 1000, cur_kind = 0;
        if (k < MLB_VOICE_MAX_EVENTS)
        {
          cur_d = ev_d[k], cur_kind = ev_kind[k];
          const unsigned fl = (flags >> (8 * k)) & 0xFFu;
          if (cur_kind != 3)
          {
            if (fl & MLB_EVF_RESET) r.age = 0;
            r.age_step = 1;
          }
          if (cur_kind == 1) voice_set_glide_time(r, (fl & MLB_EVF_GLIDE) ? glide_samples : 0.f);
        }
      };
      auto complete = [&]()  // post-actions of the current event, then move on
      {
        if (cur_kind == 3)
          r.vel = 0.f;
        else
          r.pitch = u2f(rec[4 + k]), r.vel = u2f(rec[8 + k]);
        ++k;
        advance();
      };
      advance();
#pragma unroll 1
      for (int q = 0; q < MLB_BLOCK / 4; ++q)
      {
        // nothing of the current event falls into frames 4q .. 4q+3 (a retrigger's gate-0 frame is cur_d - 1):
        // four plain frames, one 128-bit store per row
        if (cur_d > 4 * q + 3 + (cur_kind == 2 ? 1 : 0))
        {
          float p[4], tmv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int i = 0; i < 4; ++i) voice_tick(r, a.sr, want_time, p[i], tmv[i]);
          gate4[q ^ l7] = make_float4(r.vel, r.vel, r.vel, r.vel);
          pitch4[q ^ l7] = make_float4(p[0], p[1], p[2], p[3]);
          if (want_time) tm4[q ^ l7] = make_float4(tmv[0], tmv[1], tmv[2], tmv[3]);
        }
        else
        {
#pragma unroll 1
          for (int f = 4 * q; f < 4 * q + 4; ++f)
          {
            while (cur_d <= f) complete();
            const bool retrig_frame = cur_kind == 2 && cur_d - 1 == f;
            float pv, tv = 0.f;
            const float gv = retrig_frame ? 0.f : r.vel;
            voice_tick(r, a.sr, want_time, pv, tv);
            const int x = voice_word(f, sw);
            gate[x] = gv, pitch[x] = pv;
            if (want_time) tm[x] = tv;
          }
        }
      }
      while (k < MLB_VOICE_MAX_EVENTS) complete();  // events at frame 64: only their value changes remain
      r.next_frame = MLB_BLOCK;
    }
    else
    {
      int k = 0;
      bool pre_applied = false, retrig_frame_done = false;
      bool active = true;
      while (active)
      {
        int emit_at = -1;
        float emit_gate = 0.f;
        while (k < n_events)
        {
          int dest = (int)((times >> (8 * k)) & 0xFFu);
          dest = dest > MLB_BLOCK ? MLB_BLOCK : dest;
          const int type = (int)((types >> (8 * k)) & 0xFFu);
          const unsigned fl = (flags >> (8 * k)) & 0xFFu;
          const bool is_on = type == MLB_EV_NOTE_ON, is_rt = type == MLB_EV_NOTE_RETRIG, is_off = type == MLB_EV_NOTE_OFF;
          if (!(is_on || is_rt || is_off))
          {
            ++k;  // kNoteSustain & co: writeNoteEvent does nothing
            continue;
          }
          if (!pre_applied)
          {
            if (is_on || is_rt)
            {
              if (fl & MLB_EVF_RESET) r.age = 0;
              r.age_step = 1;
            }
            if (is_on) voice_set_glide_time(r, (fl & MLB_EVF_GLIDE) ? glide_samples : 0.f);
            pre_applied = true;
          }
          if (is_rt && dest == 0) dest = 1;
          const int bound = is_rt ? dest - 1 : dest;  // writeOutputFrames(bound)
          if (r.next_frame < bound)
          {
            emit_at = r.next_frame++;
            emit_gate = r.vel;
            break;
          }
          r.next_frame = bound;  // writeOutputFrames always ends with nextFrameToProcess = endFrame
          if (is_rt && !retrig_frame_done)
          {
            retrig_frame_done = true;  // the retrigger frame: gate 0 at dest - 1 (E:183-189)
            emit_at = dest - 1;
            emit_gate = 0.f;
            break;
          }
          // post-actions
          if (is_off)
            r.vel = 0.f;
          else
          {
            r.pitch = u2f(rec[4 + k]);
            r.vel = u2f(rec[8 + k]);
          }
          if (is_rt) r.next_frame = dest;
          ++k;
          pre_applied = false, retrig_frame_done = false;
        }
        if (emit_at < 0)
        {
          if (r.next_frame < MLB_BLOCK)
          {
            emit_at = r.next_frame++;
            emit_gate = r.vel;
          }
          else
            active = false;
        }
        if (emit_at >= 0)
        {
          float pv, tv = 0.f;
          voice_tick(r, a.sr, want_time, pv, tv);
          const int x = voice_word(emit_at, sw);
          gate[x] = emit_gate, pitch[x] = pv;
          if (want_time) tm[x] = tv;
        }
      }
    }
    if (set_mask & MLB_SET_BEND) cur[0] = u2f(rec[12]);
    if (set_mask & MLB_SET_MOD) cur[1] = u2f(rec[13]);
    if (set_mask & MLB_SET_X) cur[2] = u2f(rec[14]);
    if (set_mask & MLB_SET_Y) cur[3] = u2f(rec[15]);
    if (set_mask & MLB_SET_Z) cur[4] = u2f(rec[16]);
    if (set_mask & MLB_SET_PRESSURE) cur_pressure = u2f(rec[17]);
    // ---- endProcess, E:222-262 ----
    if (r.vel == 0.f) cur[4] = 0.f;
    GlidePlan gp[VG_COUNT];
#pragma unroll
    for (int i = 0; i < VG_COUNT; ++i)
    {
      if (i == VG_PRESSURE && !a.midi)
      {
        gp[i].mode = -1, gp[i].step = gp[i].target = gp[i].cv = 0.f;
        continue;
      }
      // {step, target, vectorsRemaining} live in the state array between vectors (coalesced [word][V] lines),
      // not in registers across the frame loop
      uint32_t* const gw = a.state + (size_t)(VS_GL + 4 * i) * V + v;
      const GlidePlanned o =
          glide_plan(gw[0], gw[V], gw[2 * V], i == VG_DRIFT ? cur_drift : (i == VG_PRESSURE ? cur_pressure : cur[i]),
                     i == VG_DRIFT ? a.dr_per : (i == VG_PRESSURE ? a.pc_per : a.gl_per),
                     i == VG_DRIFT ? a.dr_dy : (i == VG_PRESSURE ? a.pc_dy : a.gl_dy),
                     a.grows + ((size_t)i * V + v) * MLB_BLOCK);
      gp[i] = o.g;
      if (live) gw[0] = o.s0, gw[V] = o.s1, gw[2 * V] = o.s2;
    }
    float* const planes = a.out + (size_t)t * a.out_block;
    const size_t plane_floats = V * MLB_BLOCK;
    GlideLane gl[VG_COUNT];
#pragma unroll
    for (int i = 0; i < VG_COUNT; ++i) gl[i] = glide_lane(gp[i]);
    __syncwarp();  // the tiles are complete
    // ---- kPitch: the tile row + bendGlide * pitchBend * (1/12) + driftSig * driftAmount * kDriftScale (E:255-261),
    //      straight to the plane; the bend and drift glides advance whether or not the row is wanted ----
    {
      const bool want_pitch = (a.row_mask & 1u) != 0;
      const float* tp = tiles + kVoiceTileFloats;
      float* const gb = a.grows + (size_t)VG_BEND * V * MLB_BLOCK;
      float* const gd = a.grows + (size_t)VG_DRIFT * V * MLB_BLOCK;
#pragma unroll 1
      for (int j0 = 0; j0 < 32; j0 += 4)
      {
        if (v0 + j0 >= a.V) break;
        GlideLane lb[4], ld[4];
        float rng[4], amt[4], b0[4], b1[4], d0[4], d1[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
        {
          lb[k] = glide_of(gl[VG_BEND], j0 + k);
          ld[k] = glide_of(gl[VG_DRIFT], j0 + k);
          rng[k] = __shfl_sync(0xffffffffu, bend_range, j0 + k);
          amt[k] = __shfl_sync(0xffffffffu, drift_amount, j0 + k);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
        {
          const bool ok = v0 + j0 + k < a.V;
          const size_t off = (size_t)(v0 + j0 + k) * MLB_BLOCK + lane;
          const bool l1 = ok && lb[k].mode == 2, l2 = ok && ld[k].mode == 2;
          b0[k] = l1 ? gb[off] : 0.f;
          b1[k] = l1 ? gb[off + 32] : 0.f;
          d0[k] = l2 ? gd[off] : 0.f;
          d1[k] = l2 ? gd[off + 32] : 0.f;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
        {
          const int j = j0 + k;
          if (v0 + j >= a.V) break;
          const size_t off = (size_t)(v0 + j) * MLB_BLOCK + lane;
          const float yb0 = glide_sample(lb[k], b0[k], lane), yb1 = glide_sample(lb[k], b1[k], lane + 32);
          const float yd0 = glide_sample(ld[k], d0[k], lane), yd1 = glide_sample(ld[k], d1[k], lane + 32);
          if (lb[k].mode >= 1) gb[off] = yb0, gb[off + 32] = yb1;
          if (ld[k].mode >= 1) gd[off] = yd0, gd[off + 32] = yd1;
          if (want_pitch)
          {
            const float k12 = 1.f / 12;
            const float* row = tp + j * MLB_BLOCK + ((((lane >> 2) ^ (j & 7)) << 2) | (lane & 3));
            float p0 = row[0], p1 = row[32];
            p0 = __fadd_rn(p0, __fmul_rn(__fmul_rn(yb0, rng[k]), k12));
            p1 = __fadd_rn(p1, __fmul_rn(__fmul_rn(yb1, rng[k]), k12));
            p0 = __fadd_rn(p0, __fmul_rn(__fmul_rn(yd0, amt[k]), 0.02f));
            p1 = __fadd_rn(p1, __fmul_rn(__fmul_rn(yd1, amt[k]), 0.02f));
            __stcs(planes + off, p0);
            __stcs(planes + off + 32, p1);
          }
        }
      }
    }
    if (a.row_mask & 2u) voice_store_tile(tiles, planes + 1 * plane_floats, v0, a.V, lane);                        // kGate
    if (want_time) voice_store_tile(tiles + 2 * kVoiceTileFloats, planes + 7 * plane_floats, v0, a.V, lane);      // kElapsedTime
    if (a.row_mask & 4u)  // kVoice: voiceIndex - 1 in every sample
    {
      float* const pv = planes + 2 * plane_floats;
#pragma unroll 4
      for (int j = 0; j < 32; ++j)
      {
        if (v0 + j >= a.V) break;
        const float c = __shfl_sync(0xffffffffu, voice_row, j);
        __stcs(pv + (size_t)(v0 + j) * MLB_BLOCK + lane, c);
        __stcs(pv + (size_t)(v0 + j) * MLB_BLOCK + 32 + lane, c);
      }
    }
    // the glide-only rows: kZ(3) kX(4) kY(5) kMod(6) <- z, x, y, mod glides (kZ += the channel-pressure glide in MIDI mode)
    const int glide_of_row[4] = {VG_Z, VG_X, VG_Y, VG_MOD};
#pragma unroll
    for (int rr = 0; rr < 4; ++rr)
    {
      const int row = 3 + rr, gi = glide_of_row[rr];
      float* const gbase = a.grows + (size_t)gi * V * MLB_BLOCK;
      float* const pbase = a.grows + (size_t)VG_PRESSURE * V * MLB_BLOCK;
      const bool with_pressure = gi == VG_Z && a.midi;
      if ((a.row_mask >> row) & 1u)
        glide_row_out(gl[gi].mode, gl[gi].a, gl[gi].b, gbase, with_pressure, gl[VG_PRESSURE].mode, gl[VG_PRESSURE].a,
                      gl[VG_PRESSURE].b, pbase, planes + (size_t)row * plane_floats, v0, a.V, lane);
      else
      {
        glide_advance(gl[gi].mode, gl[gi].a, gl[gi].b, gbase, v0, a.V, lane);  // the glide still advances
        if (with_pressure) glide_advance(gl[VG_PRESSURE].mode, gl[VG_PRESSURE].a, gl[VG_PRESSURE].b, pbase, v0, a.V, lane);
      }
    }
    __syncwarp();  // rows written across lanes are read by their own lane (glide_plan) in the next vector
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) st[VS_PG_CURR + i] = r.pg[i];
  st[VS_PG_PER] = f2u(r.pg_per_f), st[VS_PG_DY] = f2u(r.pg_dy);
  st[VS_VEL] = f2u(r.vel), st[VS_PITCH] = f2u(r.pitch);
  st[VS_AGE] = r.age, st[VS_AGE_STEP] = r.age_step;
  st[VS_BEND] = f2u(cur[0]), st[VS_MOD] = f2u(cur[1]), st[VS_X] = f2u(cur[2]), st[VS_Y] = f2u(cur[3]), st[VS_Z] = f2u(cur[4]);
  st[VS_PRESSURE] = f2u(cur_pressure);
  st[VS_SEED] = seed, st[VS_DRIFT_COUNTER] = (uint32_t)drift_counter, st[VS_NEXT_DRIFT] = (uint32_t)next_drift;
  st[VS_CUR_DRIFT] = f2u(cur_drift);
  if (live)
  {
#pragma unroll
    for (int i = 0; i < VS_COUNT; ++i)
      if (i < VS_GL || i >= VS_VEL) a.state[(size_t)i * V + v] = st[i];
  }
}

// processVector's MPE tail (E:448-460): pitch, x, y, z, mod rows += the rows of the instrument's main voice.
// One thread per float4 of a (block, voice) row; planes [T][n_planes][V][64].
__global__ void __launch_bounds__(256) voice_mpe_add_kernel(float* out, const int32_t* main_voice, int V, int T,
                                                             unsigned row_mask, int n_planes)
{
  const size_t n4 = (size_t)T * V * 16;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
  {
    const int q = (int)(i & 15u);
    const size_t tv = i >> 4;
    const int v = (int)(tv % (size_t)V);
    const size_t t = tv / (size_t)V;
    const int m = main_voice[v];
    if (m < 0) continue;
    const int rows[5] = {0, 3, 4, 5, 6};  // kPitch, kZ, kX, kY, kMod
#pragma unroll
    for (int k = 0; k < 5; ++k)
    {
      if (!((row_mask >> rows[k]) & 1u)) continue;
      float4* plane = reinterpret_cast<float4*>(out + (t * n_planes + rows[k]) * (size_t)V * MLB_BLOCK);
      float4 a = plane[(size_t)v * 16 + q];
      const float4 b = plane[(size_t)m * 16 + q];
      a.x = __fadd_rn(a.x, b.x), a.y = __fadd_rn(a.y, b.y), a.z = __fadd_rn(a.z, b.z), a.w = __fadd_rn(a.w, b.w);
      plane[(size_t)v * 16 + q] = a;
    }
  }
}

}  // namespace mlb
