// oracle/ref/mlpsynth.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// The end-to-end checker of published signals of mlb::tr::TracedSynth: G complete, UNMODIFIED reference AudioContext +
// Synth pairs, each an AudioContext(0, 2, sample rate) set up by publishBodySetup and a PublishSynth -- the Synth
// subclass of tests/cpp/published_body.h, the SAME source tests/cpp/test_published_trace.cpp traces.  Per vector t and
// instrument, as oracle/ref/mltsynth.cpp: addInputEvent at t * 64 + frame, processVector(t * 64),
// synth.processVector(inputs, outputs, &ctx), store the outputs, clearInputEvents.  After the vectors of each call,
// the reads of published_body.h through getPublishedSignals()[name].  oracle/psynth.mk compiles this file in place with
// the reference's MLAudioContext.cpp, MLSignalProcessor.cpp, MLValue.cpp and the EventsToSignals sources into
// oracle/_ref/libmlpsynth.so.  Nothing from the reference is copied into this repository.
//
// Only tests/ may load the library.
#include <algorithm>
#include <cstdint>
#include <memory>
#include <thread>
#include <vector>

#include "MLSynth.h"
#include "mlb200.h"

using namespace ml;
#include "../../tests/cpp/published_body.h"

namespace
{
const char* const kNames[kPublishSignals] = {"scope", "voices", "pitch"};

void runInstruments(int g0, int g1, int G, int T, int variant, int n_voices, int sample_rate, const int32_t* offsets,
                    const mlb_event* events, const int32_t* splits, int n_calls, float* bus, int32_t* counts,
                    float* dest)
{
  for (int g = g0; g < g1; ++g)
  {
    auto ctx = std::make_unique<AudioContext>(0, 2, sample_rate);
    auto synth = std::make_unique<PublishSynth>(n_voices, true);
    publishBodySetup(*ctx, *synth, variant);
    int t = 0;
    for (int call = 0; call < n_calls; ++call)
    {
      for (int t1 = t + splits[call]; t < t1; ++t)
      {
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
        for (int o = 0; o < 2; ++o) store(ctx->outputs[o], bus + (((size_t)t * 2 + o) * G + g) * kFloatsPerDSPVector);
        ctx->clearInputEvents();
      }
      for (int k = 0; k < kPublishSignals; ++k)
      {
        SignalProcessor::PublishedSignal* s = synth->getPublishedSignals()[Path(kNames[k])].get();
        const size_t frames = (size_t)kPublishReadFrames[k];
        float* d = dest + (((size_t)call * kPublishSignals + k) * G + g) * kPublishReadWidth;
        int32_t& c = counts[((size_t)call * kPublishSignals + k) * G + g];
        switch (publishReadMode(call, k))
        {
          case 0: c = (int32_t)s->readLatest(d, frames); break;
          case 1: c = (int32_t)s->read(d, frames); break;
          case 2:
            c = (size_t)s->getReadAvailable() >= frames * s->getNumChannels() ? 1 : 0;
            s->peekLatest(d, frames);
            break;
          default: c = s->getAvailableFrames(); break;
        }
      }
    }
  }
}

template <size_t CH>
void signalRun(int max_frames, int max_voices, int octaves, int n_calls, const int32_t* n_stores, const int32_t* frames,
               const float* rows, const int32_t* modes, const int32_t* req, int32_t* counts, float* dest)
{
  SignalProcessor::PublishedSignal sig(max_frames, max_voices, (int)CH, octaves);
  for (int c = 0, i = 0; c < n_calls; ++c)
  {
    for (int k = 0; k < n_stores[c]; ++k, ++i)
    {
      DSPVectorArray<CH> a;
      for (size_t j = 0; j < CH; ++j)
        for (int n = 0; n < kFloatsPerDSPVector; ++n) a.row((int)j)[n] = rows[((size_t)i * CH + j) * kFloatsPerDSPVector + n];
      sig.writeQuick(a, (size_t)frames[i], 0);
    }
    const size_t want = (size_t)req[c];
    switch (modes[c])
    {
      case 0: counts[c] = (int32_t)sig.readLatest(dest, want); break;
      case 1: counts[c] = (int32_t)sig.read(dest, want); break;
      case 2:
        counts[c] = (size_t)sig.getReadAvailable() >= want * CH ? 1 : 0;
        sig.peekLatest(dest, want);
        break;
      default: counts[c] = sig.getAvailableFrames(); break;
    }
    dest += want * CH;
  }
}
}  // namespace

extern "C"
{
// One reference PublishedSignal(max_frames, max_voices, channels 1..3, octaves) through n_calls calls: call c makes
// n_stores[c] writeQuick calls (store i: the first frames[i] frames of rows [i][channels][64], in order), then one read
// (mode as publishReadMode's: 0 readLatest, 1 read, 2 peekLatest, 3 getAvailableFrames) of req[c] frames into dest,
// req[c] * channels floats per call (the caller zeroes it), and counts[c] as in mlpsynth_run.  Returns 0, -1 for a
// channel count it does not build.
int mlpsynth_signal_run(int max_frames, int max_voices, int channels, int octaves, int n_calls, const int32_t* n_stores,
                        const int32_t* frames, const float* rows, const int32_t* modes, const int32_t* req,
                        int32_t* counts, float* dest)
{
  switch (channels)
  {
    case 1: signalRun<1>(max_frames, max_voices, octaves, n_calls, n_stores, frames, rows, modes, req, counts, dest); return 0;
    case 2: signalRun<2>(max_frames, max_voices, octaves, n_calls, n_stores, frames, rows, modes, req, counts, dest); return 0;
    case 3: signalRun<3>(max_frames, max_voices, octaves, n_calls, n_stores, frames, rows, modes, req, counts, dest); return 0;
    default: return -1;
  }
}

// G instruments, T = sum of splits vectors of publishBodySetup(variant) with n_voices voices, in n_calls calls of
// splits[call] vectors.  Events of instrument g in vector t: events[offsets[t][g] .. offsets[t][g + 1]) (times 0..63
// within the vector).  bus [T][2][G][64]; after each call the reads of published_body.h: counts [calls][3][G], dest
// [calls][3][G][kPublishReadWidth] (zero where a read wrote nothing).  nthreads <= 0: every hardware thread.
void mlpsynth_run(int G, int variant, int n_voices, int sample_rate, const int32_t* offsets, const mlb_event* events,
                  const int32_t* splits, int n_calls, float* bus, int32_t* counts, float* dest, int nthreads)
{
  int T = 0;
  for (int c = 0; c < n_calls; ++c) T += splits[c];
  std::fill(dest, dest + (size_t)n_calls * kPublishSignals * G * kPublishReadWidth, 0.f);
  if (nthreads <= 0) nthreads = (int)std::max(1u, std::thread::hardware_concurrency());
  nthreads = std::max(1, std::min(nthreads, G));
  std::vector<std::thread> pool;
  for (int k = 0; k < nthreads; ++k)
    pool.emplace_back(runInstruments, (int)((int64_t)G * k / nthreads), (int)((int64_t)G * (k + 1) / nthreads), G, T,
                      variant, n_voices, sample_rate, offsets, events, splits, n_calls, bus, counts, dest);
  for (auto& th : pool) th.join();
}
}  // extern "C"
