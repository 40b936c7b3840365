/*
 * oracle/port/mlport_ctrl.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of EventsToSignals' smoothed controllers (source/app/MLEventsToSignals.cpp:264-285, 431-435:
 * per vector, the writes of each SmoothedController's inputValue, then output = LinearGlide(inputValue),
 * source/DSP/MLDSPGens.h:433-515) for G instruments x C requested controllers, fed by the CSR change list of
 * mlb_controllers_process_device: the checker of kernel K11.  Built by oracle/ctrl.mk with the flags of
 * oracle/port/mlport.c (gcc -O2 -ffp-contract=off -msse2 -mfpmath=sse: one binary32 SSE op per operation, round to
 * nearest, subnormals kept) into oracle/_port/libmlport_ctrl.so.  Pinned against the complete reference
 * EventsToSignals (oracle/_ref/libmlctrl.so) and tests/golden/controllers.npz by tests/test_controllers.py.
 *
 * The state is the device bank's: words [4][C][G] (inputValue, target, vectorsRemaining, step) and rows [C][G][64];
 * here every row is kept, idle or not.
 *
 * Only tests/, __graft_entry__.smoke() and the benchmark tools' parity legs may load this library.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "mlb200.h"

#define NB MLB_BLOCK

static float bits_f(uint32_t u)
{
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static uint32_t f_bits(float f)
{
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}

/* SmoothedController::process's glide length: setGlideTimeInSamples((float)(int)(sr * 0.02f)), in double */
void mlport_ctrl_glide(float sample_rate, float* per, float* dy)
{
  const int samples = (int)((double)sample_rate * (double)0.02f);
  int n = (int)((float)samples / (float)NB);
  if (n < 1) n = 1;
  *per = (float)n;
  *dy = 1.0f / ((float)n + 0.f);
}

/* LinearGlide::operator()(f) on one controller's state; row = mCurrVec */
static void glide(float f, uint32_t* w_target, uint32_t* w_rem, uint32_t* w_step, float* row, int per, float dy)
{
  float target = bits_f(*w_target), step = bits_f(*w_step);
  int rem = (int32_t)*w_rem;
  if (f != target)
  {
    target = f;
    rem = per;
  }
  if (rem < 0)
  {
  }
  else if (rem == 0)
  {
    for (int n = 0; n < NB; ++n) row[n] = target;
    step = 0.f;
    rem--;
  }
  else if (rem == per)
  {
    const float cv = row[NB - 1];
    step = (target - cv) * dy;
    for (int n = 0; n < NB; ++n) row[n] = cv + (float)(n + 1) * 0.015625f * step;  /* kUnityRampVec * mStepVec */
    rem--;
  }
  else
  {
    for (int n = 0; n < NB; ++n) row[n] = row[n] + step;
    rem--;
  }
  *w_target = f_bits(target), *w_step = f_bits(step), *w_rem = (uint32_t)rem;
}

/* T vectors.  offsets [T][G + 1] into changes; ctrl [C]; words [4][C][G], rows [C][G][64] updated in place;
 * out [T][C][G][64]. */
void mlport_controllers(int G, int C, int T, float sample_rate, const int32_t* ctrl, const int32_t* offsets,
                        const mlb_controller_change* changes, uint32_t* words, float* rows, float* out)
{
  float per_f, dy;
  mlport_ctrl_glide(sample_rate, &per_f, &dy);
  const int per = (int)per_f;
  const size_t CG = (size_t)C * G;
  uint32_t* w_in = words;
  uint32_t* w_target = words + CG;
  uint32_t* w_rem = words + 2 * CG;
  uint32_t* w_step = words + 3 * CG;
  for (int t = 0; t < T; ++t)
  {
    const int32_t* off = offsets + (size_t)t * (G + 1);
    for (int g = 0; g < G; ++g)
      for (int i = off[g]; i < off[g + 1]; ++i)
      {
        const int n = changes[i].controller > 128 ? 128 : changes[i].controller;
        for (int c = 0; c < C; ++c)
          if (ctrl[c] == n) w_in[(size_t)c * G + g] = f_bits(changes[i].value);
      }
    for (int c = 0; c < C; ++c)
      for (int g = 0; g < G; ++g)
      {
        const size_t s = (size_t)c * G + g;
        float* row = rows + s * NB;
        glide(bits_f(w_in[s]), &w_target[s], &w_rem[s], &w_step[s], row, per, dy);
        memcpy(out + (((size_t)t * C + c) * G + g) * NB, row, NB * sizeof(float));
      }
  }
}
