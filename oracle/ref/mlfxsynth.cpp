// oracle/ref/mlfxsynth.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// The end-to-end checker of a traced Synth that overrides processVector: G complete, UNMODIFIED reference AudioContext +
// Synth pairs (source/app/MLAudioContext.{h,cpp}, MLSynth.h, the EventsToSignals sources), each an
// AudioContext(0, 3, sample rate) set up by fxSynthSetup and an FxSynth -- the Synth subclass of
// tests/cpp/fx_synth_body.h, the SAME source tests/cpp/test_fx_synth.cpp traces.  Per vector the loop of
// oracle/ref/mltsynth.cpp: updateTime with each transport update of the vector, addInputEvent at t * 64 + frame,
// processVector(t * 64), synth.processVector(inputs, outputs, &ctx), store the three outputs, clearInputEvents.
// oracle/fxsynth.mk compiles this file in place with the reference's MLAudioContext.cpp, MLValue.cpp and the
// EventsToSignals sources into oracle/_ref/libmlfxsynth.so.  Nothing from the reference is copied into this repository.
//
// Only tests/ and tools/ may load the library.
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <memory>
#include <thread>
#include <vector>

#include "MLSynth.h"
#include "mlb200.h"

using namespace ml;
#include "../../tests/cpp/fx_synth_body.h"

namespace
{
constexpr int kOutputs = 3;

void runInstruments(int g0, int g1, int G, int T, int variant, int n_voices, int sample_rate, const int32_t* offsets,
                    const mlb_event* events, const int32_t* time_offsets, const mlb_transport* tr, float* bus)
{
  for (int g = g0; g < g1; ++g)
  {
    auto ctx = std::make_unique<AudioContext>(0, kOutputs, sample_rate);
    auto synth = std::make_unique<FxSynth>(n_voices);
    fxSynthSetup(*ctx, *synth, variant);
    for (int t = 0; t < T; ++t)
    {
      const int32_t* to = time_offsets + (size_t)t * (G + 1) + g;
      for (int i = to[0]; i < to[1]; ++i)
        ctx->updateTime(tr[i].ppq_pos, tr[i].bpm, tr[i].is_playing != 0, tr[i].sample_rate);
      const int32_t* eo = offsets + (size_t)t * (G + 1) + g;
      for (int i = eo[0]; i < eo[1]; ++i)
      {
        Event e;
        e.type = (EventType)events[i].type, e.channel = events[i].channel, e.sourceIdx = events[i].source_idx;
        e.time = t * kFloatsPerDSPVector + events[i].time, e.value1 = events[i].value1, e.value2 = events[i].value2;
        ctx->addInputEvent(e);
      }
      ctx->processVector(t * kFloatsPerDSPVector);
      synth->processVector(ctx->inputs, ctx->outputs, ctx.get());
      for (int o = 0; o < kOutputs; ++o)
        store(ctx->outputs[o], bus + (((size_t)t * kOutputs + o) * G + g) * kFloatsPerDSPVector);
      ctx->clearInputEvents();
    }
  }
}
}  // namespace

extern "C"
{
// G instruments, T vectors of fxSynthSetup(variant) with n_voices voices; the arguments of mltsynth_run, and bus
// [T][3][G][64].  Returns the seconds the instruments took.
double mlfxsynth_run(int G, int T, int variant, int n_voices, int sample_rate, const int32_t* offsets,
                     const mlb_event* events, const int32_t* time_offsets, const mlb_transport* tr, float* bus,
                     int nthreads)
{
  if (nthreads <= 0) nthreads = (int)std::max(1u, std::thread::hardware_concurrency());
  nthreads = std::max(1, std::min(nthreads, G));
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> pool;
  for (int k = 0; k < nthreads; ++k)
    pool.emplace_back(runInstruments, (int)((int64_t)G * k / nthreads), (int)((int64_t)G * (k + 1) / nthreads), G, T,
                      variant, n_voices, sample_rate, offsets, events, time_offsets, tr, bus);
  for (auto& th : pool) th.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
}  // extern "C"
