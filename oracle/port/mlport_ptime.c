/*
 * oracle/port/mlport_ptime.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of AudioContext::ProcessTime (source/app/MLAudioContext.h:23-56, .cpp:16-101) for G
 * instruments, fed by the CSR transport list of mlb_process_time_process_device: the checker of kernel K13.  Built by
 * oracle/ptime.mk with the flags of oracle/port/mlport.c (gcc -O2 -ffp-contract=off -msse2 -mfpmath=sse: one SSE op
 * per binary32 / binary64 operation, round to nearest) into oracle/_port/libmlport_ptime.so.  Pinned against the
 * reference's own AudioContext (oracle/_ref/libmlptime.so) by tests/test_process_time.py.
 *
 * The state is the device bank's: words [MLB_PT_WORDS][G] uint64 in ProcessTime's member order (mlb200.h).
 *
 * Only tests/ and the benchmark tools' parity legs may load this library.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "mlb200.h"

typedef struct
{
  float omega;
  double dpdt, ppq1, phase1, bpm, sr;
  int playing1, active1;
  uint64_t since_prev, since_start;
} clock_t_;

static double bits_d(uint64_t u)
{
  double d;
  memcpy(&d, &u, 8);
  return d;
}
static uint64_t d_bits(double d)
{
  uint64_t u;
  memcpy(&u, &d, 8);
  return u;
}

static void load(clock_t_* c, const uint64_t* w, size_t G, size_t g)
{
  uint32_t o = (uint32_t)w[MLB_PT_OMEGA * G + g];
  memcpy(&c->omega, &o, 4);
  c->dpdt = bits_d(w[MLB_PT_DPDT * G + g]);
  c->ppq1 = bits_d(w[MLB_PT_PPQ_POS1 * G + g]);
  c->phase1 = bits_d(w[MLB_PT_PPQ_PHASE1 * G + g]);
  c->playing1 = w[MLB_PT_PLAYING1 * G + g] != 0;
  c->active1 = w[MLB_PT_ACTIVE1 * G + g] != 0;
  c->since_prev = w[MLB_PT_SAMPLES_PREV * G + g];
  c->since_start = w[MLB_PT_SAMPLES_START * G + g];
  c->bpm = bits_d(w[MLB_PT_BPM * G + g]);
  c->sr = bits_d(w[MLB_PT_SAMPLE_RATE * G + g]);
}

static void save(const clock_t_* c, uint64_t* w, size_t G, size_t g)
{
  uint32_t o;
  memcpy(&o, &c->omega, 4);
  w[MLB_PT_OMEGA * G + g] = o;
  w[MLB_PT_DPDT * G + g] = d_bits(c->dpdt);
  w[MLB_PT_PPQ_POS1 * G + g] = d_bits(c->ppq1);
  w[MLB_PT_PPQ_PHASE1 * G + g] = d_bits(c->phase1);
  w[MLB_PT_PLAYING1 * G + g] = (uint64_t)c->playing1;
  w[MLB_PT_ACTIVE1 * G + g] = (uint64_t)c->active1;
  w[MLB_PT_SAMPLES_PREV * G + g] = c->since_prev;
  w[MLB_PT_SAMPLES_START * G + g] = c->since_start;
  w[MLB_PT_BPM * G + g] = d_bits(c->bpm);
  w[MLB_PT_SAMPLE_RATE * G + g] = d_bits(c->sr);
}

/* setTimeAndRate (.cpp:16-78) */
static void set_time(clock_t_* c, const mlb_transport* u)
{
  const double ppq = u->ppq_pos, bpm = u->bpm;
  if (isnan(ppq) || isinf(ppq) || isnan(bpm) || isinf(bpm)) return;
  c->sr = u->sample_rate;
  c->bpm = bpm;
  const int playing = u->is_playing != 0;
  const int active = (c->ppq1 != ppq) && playing;
  const int just_started = playing && !c->playing1;
  double phase = 0.;
  if (active)
  {
    phase = ppq > 0.f ? ppq - floor(ppq) : ppq;
    c->omega = (float)phase;
    if (just_started)
    {
      c->since_start = 0;
      c->omega = 0.f;
      const double dsdt = 1. / c->sr;
      const double minutes_per_sample = dsdt / 60.;
      c->dpdt = bpm * minutes_per_sample;
    }
    else
    {
      double d = phase - c->phase1;
      if (d < 0.) d += 1.;
      const double r = d / (double)c->since_prev;
      c->dpdt = r < 0. ? 0. : (r > 1. ? 1. : r);
    }
  }
  else
  {
    c->omega = -1.f;
    c->dpdt = 0.;
  }
  c->ppq1 = ppq;
  c->phase1 = phase;
  c->active1 = active;
  c->playing1 = playing;
  c->since_prev = 0;
}

/* G clocks, T blocks: offsets [T][G + 1] into tr; words [MLB_PT_WORDS][G] in / out; out [T][G][64] */
void mlport_process_time(int G, int T, const int32_t* offsets, const mlb_transport* tr, uint64_t* words, float* out)
{
  for (int g = 0; g < G; ++g)
  {
    clock_t_ c;
    load(&c, words, (size_t)G, (size_t)g);
    for (int t = 0; t < T; ++t)
    {
      const int32_t* off = offsets + (size_t)t * (G + 1) + g;
      for (int i = off[0]; i < off[1]; ++i) set_time(&c, tr + i);
      /* processVector (.cpp:88-101) */
      float* row = out + ((size_t)t * G + g) * MLB_BLOCK;
      for (int n = 0; n < MLB_BLOCK; ++n)
      {
        row[n] = c.omega;
        c.omega += c.dpdt;
        if (c.omega > 1.f) c.omega -= 1.f;
      }
      c.since_prev += MLB_BLOCK;
      c.since_start += MLB_BLOCK;
    }
    save(&c, words, (size_t)G, (size_t)g);
  }
}

/* ProcessTime::clear (.cpp:80-85) of every clock */
void mlport_process_time_clear(int G, uint64_t* words)
{
  for (int g = 0; g < G; ++g)
  {
    words[MLB_PT_DPDT * (size_t)G + g] = d_bits(0.);
    words[MLB_PT_PLAYING1 * (size_t)G + g] = 0;
    words[MLB_PT_ACTIVE1 * (size_t)G + g] = 0;
  }
}
