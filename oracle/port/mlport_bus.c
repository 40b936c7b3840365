/*
 * oracle/port/mlport_bus.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the voice sum of the reference's Synth::processVector (source/app/MLSynth.h:36-60),
 * per bus: the checker of kernel K10 at any bus size (the reference's Synth reads at most 16 voices).  Built by
 * oracle/synth.mk with the flags of oracle/port/mlport.c (gcc -O2 -ffp-contract=off -msse2 -mfpmath=sse: every add
 * is one binary32 SSE add, round to nearest, subnormals kept) into oracle/_port/libmlport_bus.so.  Pinned against
 * the reference's own Synth (oracle/_ref/libmlsynth.so) and tests/golden/buses.npz by tests/test_buses.py.
 *
 * Only tests/, __graft_entry__.smoke() and the benchmark tools' parity legs may load this library.
 */
#include <stddef.h>
#include <stdint.h>

#include "mlb200.h"

#define NB MLB_BLOCK

/* rows [T][P][V][64] -> bus [T][P][G][64]: bus g = ((+0 + row first[g]) + row first[g] + 1) + ..., count[g] rows. */
void mlport_buses(int V, int G, int P, int T, const int32_t* first, const int32_t* count, const float* rows,
                  float* bus)
{
  for (size_t tp = 0; tp < (size_t)T * P; ++tp)
    for (int g = 0; g < G; ++g)
    {
      float* out = bus + (tp * G + g) * NB;
      for (int n = 0; n < NB; ++n) out[n] = 0.0f;
      for (int v = first[g]; v < first[g] + count[g]; ++v)
      {
        const float* x = rows + (tp * V + v) * NB;
        for (int n = 0; n < NB; ++n) out[n] += x[n];
      }
    }
}
