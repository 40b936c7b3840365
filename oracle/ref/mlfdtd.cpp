// oracle/ref/mlfdtd.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs the reference's own FDTD membrane example (examples/audio-and-midi/fdtd.cpp) for a bank of
// instances.  tests/cpp/make_fdtd_body.py extracts the example's text between `using namespace ml;`
// and `int main(` byte for byte into the git-ignored tests/cpp/_ref/fdtd_body.inc; this file includes it
// inside a namespace and calls its FDTDState, processFDTDModel and processFDTD.  oracle/fdtd.mk compiles
// it together with the reference's MLAudioContext.cpp and the three sources of libmle2s.so, in place, into
// oracle/_ref/libmlfdtd.so.  Nothing from the reference is copied into this repository.
//
// Only tests/, __graft_entry__.smoke() and the benchmark tools' CPU legs may load the library.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <thread>
#include <vector>

#include "MLAudioContext.h"
#include "MLDSPGens.h"
#include "MLDSPOps.h"
#include "MLDSPUtils.h"

namespace fdtd_example
{
using namespace ml;
#include "../../tests/cpp/_ref/fdtd_body.inc"
}  // namespace fdtd_example

using namespace fdtd_example;

extern "C"
{
// V instances, T vectors.  in [T][2][V][64] (plane 0 excitation, plane 1 frequency in cycles per sample);
// state_in / state_out [V][2][16][16] (the interiors of *mpU1, then *mpU2; state_out may equal state_in);
// out [T][2][V][64] (the two rows processFDTDModel returns).  ftz: every processFDTDModel call runs inside the
// reference's UsingFlushDenormalsToZero, taken in the worker thread (MXCSR is per thread).  Returns seconds.
double mlfdtd_run(int V, int T, const float* in, const float* state_in, float* state_out, float* out, int ftz,
                  int nthreads)
{
  constexpr int N = kWidth * kHeight;
  if (nthreads < 1) nthreads = 1;
  nthreads = std::min(nthreads, std::max(1, V));
  auto worker = [&](int v0, int v1)
  {
    for (int v = v0; v < v1; ++v)
    {
      auto st = std::make_unique<FDTDState>();
      const float* si = state_in + (size_t)v * 2 * N;
      for (int j = 0; j < kHeight; ++j)
        for (int i = 0; i < kWidth; ++i)
        {
          (*st->mpU1)[kRowStride * (j + kPadding) + kPadding + i] = si[j * kWidth + i];
          (*st->mpU2)[kRowStride * (j + kPadding) + kPadding + i] = si[N + j * kWidth + i];
        }
      for (int t = 0; t < T; ++t)
      {
        DSPVector x, f;
        load(x, in + (((size_t)t * 2 + 0) * V + v) * kFloatsPerDSPVector);
        load(f, in + (((size_t)t * 2 + 1) * V + v) * kFloatsPerDSPVector);
        DSPVectorArray<2> y;
        if (ftz)
        {
          UsingFlushDenormalsToZero guard;
          y = processFDTDModel(x, f, st.get());
        }
        else
          y = processFDTDModel(x, f, st.get());
        store(y.constRow(0), out + (((size_t)t * 2 + 0) * V + v) * kFloatsPerDSPVector);
        store(y.constRow(1), out + (((size_t)t * 2 + 1) * V + v) * kFloatsPerDSPVector);
      }
      float* so = state_out + (size_t)v * 2 * N;
      for (int j = 0; j < kHeight; ++j)
        for (int i = 0; i < kWidth; ++i)
        {
          so[j * kWidth + i] = (*st->mpU1)[kRowStride * (j + kPadding) + kPadding + i];
          so[N + j * kWidth + i] = (*st->mpU2)[kRowStride * (j + kPadding) + kPadding + i];
        }
    }
  };
  auto t0 = std::chrono::steady_clock::now();
  if (nthreads == 1)
    worker(0, V);
  else
  {
    std::vector<std::thread> th;
    for (int i = 0; i < nthreads; ++i)
      th.emplace_back(worker, (int)((long long)V * i / nthreads), (int)((long long)V * (i + 1) / nthreads));
    for (auto& t : th) t.join();
  }
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// The example itself: n_vectors calls of its own processFDTD with a real AudioContext(0, 2, 48000) and a
// fresh FDTDState.  out [n_vectors][2][64] = ctx.outputs[0], ctx.outputs[1] after each call.
void mlfdtd_example(int n_vectors, float* out)
{
  auto state = std::make_unique<FDTDState>();
  AudioContext ctx(kInputChannels, kOutputChannels, kSampleRate);
  for (int t = 0; t < n_vectors; ++t)
  {
    processFDTD(&ctx, state.get());
    store(ctx.outputs[0], out + ((size_t)t * 2 + 0) * kFloatsPerDSPVector);
    store(ctx.outputs[1], out + ((size_t)t * 2 + 1) * kFloatsPerDSPVector);
  }
}
}  // extern "C"
