// oracle/ref/mlptime.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs the reference's own AudioContext::ProcessTime as the checker of kernel K13: one complete, UNMODIFIED
// AudioContext(0, 0, sample rate) per instrument (source/app/MLAudioContext.{h,cpp}), driven the way a plugin drives
// it -- updateTime() with each transport update of the coming vector, processVector(), getBeatPhase() -- with clear()
// where asked.  The private ProcessTime members are read through -fno-access-control, in the device bank's state
// layout (mlb200.h, MLB_PT_*).  oracle/ptime.mk compiles this file in place with the reference's MLAudioContext.cpp,
// MLValue.cpp and the EventsToSignals sources into oracle/_ref/libmlptime.so.  Nothing from the reference is copied
// into this repository.
//
// Only tests/ may load the library.
#include <cstdint>
#include <cstring>
#include <memory>

#include "MLAudioContext.h"
#include "mlb200.h"

using namespace ml;

namespace
{
uint64_t bits(double d)
{
  uint64_t u;
  memcpy(&u, &d, 8);
  return u;
}
}  // namespace

extern "C"
{
// G instruments, T vectors.  The transport updates of instrument g before vector t are
// tr[offsets[t][g] .. offsets[t][g + 1]); clear_before[t] != 0: AudioContext::clear() before vector t's updates.
// out [T][G][64] = getBeatPhase(); words [MLB_PT_WORDS][G] = ProcessTime's members after the last vector.
void mlptime_run(int G, int T, int sample_rate, const int32_t* offsets, const mlb_transport* tr,
                 const int32_t* clear_before, float* out, uint64_t* words)
{
  for (int g = 0; g < G; ++g)
  {
    auto ctx = std::make_unique<AudioContext>(0, 0, sample_rate);
    for (int t = 0; t < T; ++t)
    {
      if (clear_before && clear_before[t]) ctx->clear();
      const int32_t* off = offsets + (size_t)t * (G + 1) + g;
      for (int i = off[0]; i < off[1]; ++i)
        ctx->updateTime(tr[i].ppq_pos, tr[i].bpm, tr[i].is_playing != 0, tr[i].sample_rate);
      ctx->processVector(t * kFloatsPerDSPVector);
      store(ctx->getBeatPhase(), out + ((size_t)t * G + g) * kFloatsPerDSPVector);
    }
    const AudioContext::ProcessTime& p = ctx->currentTime;
    const size_t n = (size_t)G;
    uint32_t o;
    memcpy(&o, &p.omega_, 4);
    words[MLB_PT_OMEGA * n + g] = o;
    words[MLB_PT_DPDT * n + g] = bits(p.dpdt_);
    words[MLB_PT_PPQ_POS1 * n + g] = bits(p.ppqPos1_);
    words[MLB_PT_PPQ_PHASE1 * n + g] = bits(p.ppqPhase1_);
    words[MLB_PT_PLAYING1 * n + g] = p.playing1_ ? 1 : 0;
    words[MLB_PT_ACTIVE1 * n + g] = p.active1_ ? 1 : 0;
    words[MLB_PT_SAMPLES_PREV * n + g] = (uint64_t)p.samplesSincePreviousTime_;
    words[MLB_PT_SAMPLES_START * n + g] = p.samplesSinceStart;
    words[MLB_PT_BPM * n + g] = bits(p.bpm);
    words[MLB_PT_SAMPLE_RATE * n + g] = bits(p.sampleRate);
  }
}
}  // extern "C"
