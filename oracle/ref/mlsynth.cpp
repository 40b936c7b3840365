// oracle/ref/mlsynth.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs the reference's own Synth::processVector (source/app/MLSynth.h:36-60) as the checker of kernel K10, the
// per-instrument output buses.  A Synth subclass whose processVoice does only `outputs[p] += row p of voice
// first + v`; the clearing of the outputs and the loop over the voices, in their order, are the reference's.  One
// Synth(count) and one AudioContext(0, P, sample rate) per bus.  oracle/synth.mk compiles it in place, with the
// reference's MLAudioContext.cpp, MLValue.cpp and the three sources of libmle2s.so, into oracle/_ref/libmlsynth.so.
// Nothing from the reference is copied into this repository.
//
// Only tests/ and the golden writer may load the library.
#include <cstdint>
#include <memory>

#include "MLSynth.h"

namespace
{
using namespace ml;

class RowSumSynth final : public Synth
{
 public:
  RowSumSynth(int nVoices, int first, size_t planeStride) : Synth(nVoices), first_(first), planeStride_(planeStride) {}
  const float* rows = nullptr;  // plane 0 of the current block: [P][V][64] from here

  void processVoice(int v, const EventsToSignals::Voice&, const DSPVectorDynamic&, DSPVectorDynamic& outputs,
                    AudioContext*) override
  {
    for (int p = 0; p < (int)outputs.size(); ++p)
    {
      DSPVector x;
      load(x, rows + p * planeStride_ + (size_t)(first_ + v) * kFloatsPerDSPVector);
      outputs[p] += x;
    }
  }

 private:
  int first_;
  size_t planeStride_;
};
}  // namespace

extern "C"
{
// rows [T][P][V][64] -> bus [T][P][G][64].  Returns 0, or -1 - g for the first bus g with more voices than a
// Synth can read (getInputVoice(v) indexes EventsToSignals' kMaxVoices + 1 voices); nothing is run then.
int mlsynth_buses(int V, int G, int P, int T, const int32_t* first, const int32_t* count, const float* rows, float* bus,
                  int sample_rate)
{
  for (int g = 0; g < G; ++g)
    if (count[g] > (int)EventsToSignals::kMaxVoices) return -1 - g;
  const size_t plane = (size_t)V * kFloatsPerDSPVector;
  for (int g = 0; g < G; ++g)
  {
    RowSumSynth synth(count[g], first[g], plane);
    auto ctx = std::make_unique<AudioContext>(0, (size_t)P, sample_rate);
    for (int t = 0; t < T; ++t)
    {
      synth.rows = rows + (size_t)t * P * plane;
      synth.processVector(ctx->inputs, ctx->outputs, ctx.get());
      for (int p = 0; p < P; ++p)
        store(ctx->outputs[p], bus + (((size_t)t * P + p) * G + g) * kFloatsPerDSPVector);
    }
  }
  return 0;
}
}  // extern "C"
