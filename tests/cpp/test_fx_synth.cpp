// tests/cpp/test_fx_synth.cpp -- a madronalib Synth subclass that overrides processVector (tests/cpp/fx_synth_body.h,
// also compiled against the reference in oracle/ref/mlfxsynth.cpp) traced by mlb::tr::TracedSynth with only the
// namespace changed, the same synth with an override that only calls the base, and the overrides TracedSynth refuses.
//
//   test_fx_synth dump <case>        trace only (no GPU needed), print the banks as JSON
//   test_fx_synth run <case> <instruments> <blocks> <dir> <splits> [<restart list>]
//                                    compile for <instruments> instruments, then process <blocks> vectors in calls of
//                                    the comma-separated <splits> vectors: <dir>/offsets.bin int32 [T][G + 1], events.bin
//                                    (mlb_event), toff.bin int32 [T][G + 1], tr.bin (mlb_transport) in, <dir>/bus.bin
//                                    f32 [T][outputs][G][64] out; after the first call, restart the comma-separated
//                                    instruments of <restart list>
// cases: midi, mpe (fxSynthSetup's variants), fxbase (FxSynth's voices with an override that only calls the base, MIDI,
// two outputs), fxplain (FxPlainSynth, MIDI), body (synth_body.h's BodySynth, MIDI), bodybase (BodySynth with an override that only calls the base),
// and the refusals below.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "mlb200_trace.hpp"

using namespace mlb::tr;  // the reference says: using namespace ml;
#include "fx_synth_body.h"
#include "synth_body.h"

struct BaseOnlySynth : public BodySynth
{
  using BodySynth::BodySynth;
  void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* state) override
  {
    Synth::processVector(inputs, outputs, state);
  }
};

struct FxBaseOnlySynth : public FxSynth
{
  using FxSynth::FxSynth;
  void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* state) override
  {
    Synth::processVector(inputs, outputs, state);
  }
};

// FxSynth's voices and context planes (controllers 73, 1, 74 and the beat phase) without an instrument section: the
// signals FxSynth's section reads are read and dropped, so the banks and time chunks are FxSynth's, the outputs the bus
// rows as they are
struct FxPlainSynth : public FxSynth
{
  using FxSynth::FxSynth;
  void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* state) override
  {
    auto* ctx = static_cast<AudioContext*>(state);
    ctx->getInputController(73);
    Synth::processVector(inputs, outputs, state);
    ctx->getInputController(74);
    ctx->getBeatPhase();
  }
};

// ---------------------------------------------------------------- what TracedSynth refuses
struct RefusedFx : public Synth
{
  std::string how;
  SineGen osc[16];
  SineGen shared;
  DSPVector member;
  const EventsToSignals::Voice* held = nullptr;
  RefusedFx(const std::string& h) : Synth(4), how(h) { publishSignal("level", 64, 1, 1, 0); }
  void processVoice(int v, const EventsToSignals::Voice& voice, const DSPVectorDynamic&, DSPVectorDynamic& outputs,
                    AudioContext*) override
  {
    DSPVector x = osc[v](voice.outputs.constRow(kPitch) * 0.01f) * voice.outputs.constRow(kGate);
    if (how == "heldvoice") held = &voice;
    if (how == "member" || how == "pre") x = x * member;
    if (how == "shared") x = x + shared(DSPVector(0.01f));
    outputs[0] += x;
  }
  void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* state) override
  {
    auto* ctx = static_cast<AudioContext*>(state);
    if (how == "pre") member = ctx->getInputController(1) * 2.f;
    if (how == "param") member = param("wet", 0.5f);
    if (how == "nobase") return;
    DSPVectorDynamic dry(1);
    Synth::processVector(inputs, how == "passed" ? outputs : dry, state);
    if (how == "twice") Synth::processVector(inputs, dry, state);
    if (how == "passed")  // outputs[0] stays bus row 0: accepted
    {
      outputs[1] = outputs[0] * 0.5f;
      return;
    }
    outputs[0] = dry[0];
    if (how == "voice") outputs[0] = dry[0] * ctx->getInputVoice(0).outputs.constRow(kGate);
    if (how == "heldvoice" && held) outputs[0] = dry[0] * held->outputs.constRow(kGate);  // set by the voices' trace
    if (how == "member") outputs[0] = member = dry[0] * 0.5f;
    if (how == "shared") outputs[0] = dry[0] + shared(DSPVector(0.02f));
    if (how == "store") storePublishedSignal("level", dry[0], 64, 0);
    if (how == "stale") outputs[0] = dry[0] + outputs[1];
    if (how != "unassigned") outputs[1] = dry[0] * 0.25f;  // "unassigned" leaves outputs[1] as it was
  }
};
const char* const kRefusals[] = {"nobase", "twice", "voice", "heldvoice", "pre", "member", "shared", "store",
                                 "unassigned", "stale", "param", "passed"};

static bool readAll(const std::string& path, std::vector<char>& v)
{
  FILE* f = std::fopen(path.c_str(), "rb");
  if (!f) return false;
  std::fseek(f, 0, SEEK_END);
  v.resize((size_t)std::ftell(f));
  std::fseek(f, 0, SEEK_SET);
  const size_t n = v.empty() ? 0 : std::fread(v.data(), 1, v.size(), f);
  std::fclose(f);
  return n == v.size();
}

static std::vector<int> parseList(const char* s)
{
  std::vector<int> v;
  for (; s && *s;)
  {
    v.push_back(std::atoi(s));
    const char* c = std::strchr(s, ',');
    s = c ? c + 1 : nullptr;
  }
  return v;
}

int main(int argc, char** argv)
{
  if (argc < 3)
  {
    std::fprintf(stderr, "usage: test_fx_synth dump|run <midi|mpe|fxbase|fxplain|body|bodybase|refusal> ...\n");
    return 2;
  }
  const std::string mode = argv[1], which = argv[2];
  bool refusal = false;
  for (const char* r : kRefusals) refusal = refusal || which == r;
  if (!refusal && which != "midi" && which != "mpe" && which != "fxbase" && which != "fxplain" && which != "body" &&
      which != "bodybase")
    return 2;
  try
  {
    TracedSynth traced;
    std::unique_ptr<Synth> synth;
    std::unique_ptr<AudioContext> ctx;
    if (refusal)
    {
      synth.reset(new RefusedFx(which));
      ctx.reset(new AudioContext(0, 2, 48000));
      ctx->setInputPolyphony(4);
    }
    else if (which == "midi" || which == "mpe" || which == "fxbase" || which == "fxplain")
    {
      auto* s = which == "fxbase"    ? new FxBaseOnlySynth(16)
                : which == "fxplain" ? new FxPlainSynth(16)
                                     : new FxSynth(which == "mpe" ? 15 : 16);
      synth.reset(s);
      ctx.reset(new AudioContext(0, which == "fxbase" || which == "fxplain" ? 2 : 3, 48000));
      fxSynthSetup(*ctx, *s, which == "mpe" ? 1 : 0);
    }
    else
    {
      auto* s = which == "body" ? new BodySynth(16) : new BaseOnlySynth(16);
      synth.reset(s);
      ctx.reset(new AudioContext(0, 2, 48000));
      synthBodySetup(*ctx, *s, 0);
    }
    traced.trace(*synth, *ctx);
    if (refusal)
    {
      std::printf("traced %s: not refused\n", which.c_str());
      return 0;
    }
    if (mode == "dump")
    {
      traced.dump(stdout);
      return 0;
    }
    if (mode == "run" && (argc == 7 || argc == 8))
    {
      const int G = std::atoi(argv[3]), T = std::atoi(argv[4]);
      const std::string dir = argv[5];
      std::vector<char> off, ev, toff, tr;
      if (!readAll(dir + "/offsets.bin", off) || !readAll(dir + "/events.bin", ev) || !readAll(dir + "/toff.bin", toff) ||
          !readAll(dir + "/tr.bin", tr))
        return 3;
      if (off.size() != (size_t)T * (G + 1) * 4 || toff.size() != off.size()) return 3;
      traced.compile(G);
      const size_t nOut = traced.outputs();
      std::vector<float> bus((size_t)T * nOut * G * 64);
      const auto* o = reinterpret_cast<const int32_t*>(off.data());
      const auto* to = reinterpret_cast<const int32_t*>(toff.data());
      const auto* e = reinterpret_cast<const mlb_event*>(ev.data());
      const auto* t = reinterpret_cast<const mlb_transport*>(tr.data());
      const int nEv = (int)(ev.size() / sizeof(mlb_event)), nTr = (int)(tr.size() / sizeof(mlb_transport));
      const std::vector<int> splits = parseList(argv[6]);
      const std::vector<int> restart = argc == 8 ? parseList(argv[7]) : std::vector<int>{};
      int t0 = 0;
      std::string launches;
      for (size_t k = 0; t0 < T; ++k)
      {
        int n = k < splits.size() ? splits[k] : T - t0;
        if (n <= 0 || t0 + n > T) n = T - t0;
        const long long k0 = mlb_kernel_launches();
        traced.process(o + (size_t)t0 * (G + 1), e, nEv, to + (size_t)t0 * (G + 1), t, nTr,
                       bus.data() + (size_t)t0 * nOut * G * 64, n);
        launches += (launches.empty() ? "" : ",") + std::to_string(mlb_kernel_launches() - k0);
        t0 += n;
        if (k == 0 && argc == 8)
        {
          const long long r0 = mlb_kernel_launches();
          traced.restart(restart);
          std::printf("restart launches: %lld\n", mlb_kernel_launches() - r0);
        }
      }
      FILE* f = std::fopen((dir + "/bus.bin").c_str(), "wb");
      std::fwrite(bus.data(), 4, bus.size(), f);
      std::fclose(f);
      std::printf("ran %s: %d instruments x %d voices x %d vectors on %s, instrument graph on %s\nlaunches per call: %s\n",
                  which.c_str(), G, traced.numVoices(), T, traced.kernelName(),
                  traced.hasInstrumentGraph() ? traced.instrumentKernelName() : "(none)", launches.c_str());
      return 0;
    }
  }
  catch (const mlb::Error& e)
  {
    std::printf("mlb error %d: %s\n", e.code, e.what());
    return e.code == MLB_ERR_NO_DEVICE ? 77 : 1;
  }
  return 2;
}
