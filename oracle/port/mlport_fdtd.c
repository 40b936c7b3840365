/*
 * oracle/port/mlport_fdtd.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the FDTD membrane of the reference's examples/audio-and-midi/fdtd.cpp, the checker of
 * kernel K9 on machines without the reference tree.  Built by oracle/fdtd.mk with the same flags as
 * oracle/port/mlport.c (gcc -O2 -ffp-contract=off -msse2 -mfpmath=sse: every mul/add is one separately rounded
 * binary32 SSE operation) into oracle/_port/libmlport_fdtd.so.  It is pinned against the example's own text
 * compiled in place (oracle/_ref/libmlfdtd.so) and against tests/golden/fdtd.npz by tests/test_fdtd.py.
 *
 * Only tests/, __graft_entry__.smoke() and the benchmark tools' parity legs may load this library.
 */
#include <math.h>
#include <stddef.h>
#include <string.h>
#include <xmmintrin.h> /* _mm_getcsr / _mm_setcsr: MXCSR FZ + DAZ */

#include "mlb200.h"

#define NB MLB_BLOCK

/* ------------------------------------------------------------------ */
/* K9: the FDTD membrane of examples/audio-and-midi/fdtd.cpp:17-154     */
/* (FDTDState + doFDTDStep2D + processFDTDModel), one instance at a     */
/* time, the sample rate a parameter.  in [T][in_planes][V][64]; state  */
/* [V][2][16][16] (z^-1 interior, then z^-2), read and written back;    */
/* out [T][2][V][64] (pickups L, R).  ftz: the whole call runs with     */
/* MXCSR FZ + DAZ (0x8040), as under UsingFlushDenormalsToZero.         */
#define FD_N MLB_FDTD_SIZE
#define FD_STRIDE (FD_N + 2)
#define FD_CELLS (FD_STRIDE * (FD_N + 2))

static void fdtd_step(const float* u1, const float* u2, float* u0, float kc, float ke, float kk, float kc2, float ke2)
{
  for (int j = 0; j < FD_N; ++j)
  {
    const float* p11 = u1 + FD_STRIDE * j + 1;       /* row j - 1 of the interior */
    const float* p12 = u1 + FD_STRIDE * (j + 1) + 1;
    const float* p13 = u1 + FD_STRIDE * (j + 2) + 1;
    const float* p21 = u2 + FD_STRIDE * j + 1;
    const float* p22 = u2 + FD_STRIDE * (j + 1) + 1;
    const float* p23 = u2 + FD_STRIDE * (j + 2) + 1;
    float* po = u0 + FD_STRIDE * (j + 1) + 1;
    for (int i = 0; i < FD_N; ++i)
    {
      float f = kc * p12[i];
      f += ke * (((p12[i - 1] + p11[i]) + p12[i + 1]) + p13[i]);
      f += kk * (((p11[i - 1] + p11[i + 1]) + p13[i - 1]) + p13[i + 1]);
      f += kc2 * p22[i];
      f += ke2 * (((p22[i - 1] + p21[i]) + p22[i + 1]) + p23[i]);
      po[i] = f;
    }
  }
}

void mlport_fdtd(int V, int T, float sample_rate, int in_planes, int excite_plane, int freq_plane, const float* in,
                 float* state, float* out, int ftz)
{
  const unsigned csr = _mm_getcsr();
  if (ftz) _mm_setcsr(csr | 0x8040u);
  const float kSize = sqrtf(((float)(FD_N * FD_N)) + ((float)(FD_N * FD_N)));
  const float kInputGain = (float)(FD_N * FD_N / 64);
  const float isr = 1.0f / sample_rate;
  float surf[3][FD_CELLS];
  for (int v = 0; v < V; ++v)
  {
    memset(surf, 0, sizeof(surf));
    float *u0 = surf[0], *u1 = surf[1], *u2 = surf[2];
    float* st = state + (size_t)v * 2 * FD_N * FD_N;
    for (int j = 0; j < FD_N; ++j)
      for (int i = 0; i < FD_N; ++i)
      {
        u1[FD_STRIDE * (j + 1) + 1 + i] = st[j * FD_N + i];
        u2[FD_STRIDE * (j + 1) + 1 + i] = st[FD_N * FD_N + j * FD_N + i];
      }
    for (int t = 0; t < T; ++t)
    {
      const float* ex = in + (((size_t)t * in_planes + excite_plane) * V + v) * NB;
      const float* fq = in + (((size_t)t * in_planes + freq_plane) * V + v) * NB;
      float* oL = out + (((size_t)t * 2 + 0) * V + v) * NB;
      float* oR = out + (((size_t)t * 2 + 1) * V + v) * NB;
      for (int n = 0; n < NB; ++n)
      {
        const float Fs = fq[n];
        const float c = kSize * Fs;
        const float T_ = (3.0f / 5.0f) * c;
        float kk = (T_ * T_) * (1.f / 6.f);
        float ke = (T_ * T_) * (2.f / 3.f);
        float kc = 2.f - 4.f * (kk + ke);
        const float s0 = 1.0f, s1 = 1.0f;
        const float ks1 = (s1 * T_) * isr;
        ke += ks1;
        kc += -4.0f * ks1;
        float ke2 = -1.0f * ks1;
        float kc2 = ((s0 * isr) + 4.0f * ks1) - 1.0f;
        const float SK = 1.0f / (1.0f + isr * s0);
        kc *= SK;
        ke *= SK;
        kk *= SK;
        kc2 *= SK;
        ke2 *= SK;
        u1[FD_STRIDE * (1 + 2) + 1 + FD_N / 2] += ex[n] * kInputGain; /* exciter: row 2, column 8 */
        fdtd_step(u1, u2, u0, kc, ke, kk, kc2, ke2);
        oL[n] = u0[FD_STRIDE * (1 + FD_N / 2 + 1) + 1 + 1];          /* pickups: row 9, columns 1 and 15 */
        oR[n] = u0[FD_STRIDE * (1 + FD_N / 2 + 1) + 1 + FD_N - 1];
        float* tmp = u2;
        u2 = u1, u1 = u0, u0 = tmp;
      }
    }
    for (int j = 0; j < FD_N; ++j)
      for (int i = 0; i < FD_N; ++i)
      {
        st[j * FD_N + i] = u1[FD_STRIDE * (j + 1) + 1 + i];
        st[FD_N * FD_N + j * FD_N + i] = u2[FD_STRIDE * (j + 1) + 1 + i];
      }
  }
  if (ftz) _mm_setcsr(csr);
}
