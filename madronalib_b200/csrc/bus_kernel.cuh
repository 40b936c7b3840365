// bus_kernel.cuh -- K10: per-instrument output buses, the voice sum of the reference's Synth::processVector
// (source/app/MLSynth.h:36-60) for G instruments at once.
//
// A bus g is the voice range [first[g], first[g] + count[g]) of a V-voice bank.  For every block t, plane p and
// sample n:  bus[t][p][g][n] = ((+0 + x[first]) + x[first + 1]) + ... + x[first + count - 1],  one binary32 add
// per voice, round to nearest, subnormals kept -- what `outputs[i] = DSPVector{0.f}; ... outputs[i] += row`
// does with the default isVoiceActive.  No tree, no atomics, no FTZ: the order is the contract.
//
// One warp per (t, p, g); lane l owns columns 2l and 2l + 1, so each voice row is one coalesced 256-byte warp
// load and the bus row leaves as one 256-byte store.  The adds are serial per column; the loads are not:
// kBusAhead rows are loaded (read-once, so not allocated in L1) before they are added in order.
#pragma once
#include "ops.cuh"

namespace mlb
{
constexpr int kBusWarps = 8;  // (t, p, g) items per 256-thread CTA
constexpr int kBusAhead = 8;  // voice rows in flight per warp

struct BusArgs
{
  const float* rows;     // [T][stride][V][64]: planes 0..P-1 of each block are summed
  float* bus;            // [T][P][G][64]
  const int32_t* first;  // [G]
  const int32_t* count;  // [G]
  int V, G, P, stride;
  long long n_items;     // T * P * G
};

MLB_DEV float2 ld_stream_f2(const float2* p)
{
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}

// ((+0 + x[0]) + x[1]) + ... over `count` voice rows 64 floats apart, from src (this lane's two columns)
MLB_DEV float2 sum_voices(const float2* src, int count)
{
  float2 acc = make_float2(0.f, 0.f);
  for (int i = 0; i < count; i += kBusAhead)
  {
    float2 x[kBusAhead];
#pragma unroll
    for (int u = 0; u < kBusAhead; ++u)
      if (i + u < count) x[u] = ld_stream_f2(src + (size_t)(i + u) * (MLB_BLOCK / 2));
#pragma unroll
    for (int u = 0; u < kBusAhead; ++u)
      if (i + u < count)
      {
        acc.x = __fadd_rn(acc.x, x[u].x);
        acc.y = __fadd_rn(acc.y, x[u].y);
      }
  }
  return acc;
}

__global__ void __launch_bounds__(32 * kBusWarps) bus_sum_kernel(BusArgs a)
{
  const long long w = (long long)blockIdx.x * kBusWarps + (threadIdx.x >> 5);
  if (w >= a.n_items) return;
  const int lane = threadIdx.x & 31;
  const int g = (int)(w % a.G);
  const long long tp = w / a.G;  // t * P + p
  const long long row = tp + (tp / a.P) * (a.stride - a.P);  // t * stride + p
  const int first = __ldg(a.first + g), count = __ldg(a.count + g);
  const float2* src = reinterpret_cast<const float2*>(a.rows + ((size_t)row * a.V + first) * MLB_BLOCK) + lane;
  reinterpret_cast<float2*>(a.bus + (size_t)w * MLB_BLOCK)[lane] = sum_voices(src, count);
}

// The input planes of an instrument graph (Synth::processVector overridden around the base call):
// in [T][P + C][G][64], planes 0..P-1 the bus sums exactly as bus_sum_kernel makes them, planes P..P+C-1 bit copies of
// planes plane0..plane0+C-1 of the voice planes at the bus's first voice (the controllers and the beat phase, which
// every voice of an instrument holds alike).  A copy is a move, not +0 + x, which would turn -0 into +0.
struct InstrumentInputArgs
{
  BusArgs bus;          // bus.bus unused; bus.P: the bus planes
  const float* voice;   // [T][voice_stride][V][64]
  float* in;            // [T][P + C][G][64]
  int voice_stride, plane0, C;
  long long n_items;    // T * (P + C) * G
};

__global__ void __launch_bounds__(32 * kBusWarps) instrument_inputs_kernel(InstrumentInputArgs a)
{
  const long long w = (long long)blockIdx.x * kBusWarps + (threadIdx.x >> 5);
  if (w >= a.n_items) return;
  const int lane = threadIdx.x & 31;
  const BusArgs& b = a.bus;
  const int g = (int)(w % b.G), NI = b.P + a.C;
  const long long tq = w / b.G;
  const long long t = tq / NI;
  const int q = (int)(tq - t * NI);
  const int first = __ldg(b.first + g);
  float2 y;
  if (q < b.P)
    y = sum_voices(reinterpret_cast<const float2*>(b.rows + (((size_t)t * b.stride + q) * b.V + first) * MLB_BLOCK) + lane,
                   __ldg(b.count + g));
  else
    y = ld_stream_f2(reinterpret_cast<const float2*>(
                         a.voice + (((size_t)t * a.voice_stride + a.plane0 + (q - b.P)) * b.V + first) * MLB_BLOCK) +
                     lane);
  reinterpret_cast<float2*>(a.in + (size_t)w * MLB_BLOCK)[lane] = y;
}

}  // namespace mlb
