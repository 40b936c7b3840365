// tests/cpp/test_synth_trace.cpp -- a madronalib Synth subclass (tests/cpp/synth_body.h, also compiled against the
// reference in oracle/ref/mltsynth.cpp) traced by mlb::tr::TracedSynth with only the namespace changed, plus the
// subclasses TracedSynth must refuse.
//
//   test_synth_trace dump <case>        trace only (no GPU needed), print the instrument bank as JSON
//   test_synth_trace run <case> <instruments> <blocks> <dir> <splits>
//                                       compile for <instruments> instruments, then process <blocks> vectors in calls
//                                       of the comma-separated <splits> vectors: <dir>/offsets.bin int32 [T][G + 1],
//                                       events.bin (mlb_event), toff.bin int32 [T][G + 1], tr.bin (mlb_transport) in,
//                                       <dir>/bus.bin f32 [T][2][G][64] out
// cases: midi, mpe, modcc, unison (synthBodySetup's variants 0..3), and the refusals below.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "mlb200_trace.hpp"

using namespace mlb::tr;  // the reference says: using namespace ml;
#include "synth_body.h"

// ---------------------------------------------------------------- what TracedSynth refuses
struct RefusedSynth : public Synth
{
  std::string how;
  SineGen osc[16];
  SineGen shared;
  DSPVector last;
  const EventsToSignals::Voice* held = nullptr;
  RefusedSynth(const std::string& h) : Synth(4), how(h) {}
  bool isVoiceActive(int v, const EventsToSignals::Voice&) override { return how != "inactive" || v != 2; }
  void processVoice(int v, const EventsToSignals::Voice& voice, const DSPVectorDynamic&, DSPVectorDynamic& outputs,
                    AudioContext* ctx) override
  {
    DSPVector x = osc[v](voice.outputs.constRow(kPitch) * 0.01f) * voice.outputs.constRow(kGate);
    if (how == "rescale") outputs[0] = outputs[0] * 0.5f + x;
    if (how == "twice") outputs[0] += x, outputs[0] += x * 0.5f;
    if (how == "assign") outputs[0] = x;
    if (how == "other") outputs[0] += x * ctx->getInputVoice(v == 0 ? 1 : 0).outputs.constRow(kGate);
    if (how == "differ") outputs[0] += v == 1 ? x * x : x;
    if (how == "inactive" || how == "inputs" || how == "polyphony") outputs[0] += x;
    if (how == "controller") outputs[0] += x * ctx->getInputController(129);
    if (how == "shared") outputs[0] += shared(DSPVector(0.01f));
    if (how == "sharedrow") outputs[0] += x + last, last = x;  // one member read and written by every voice
    if (how == "heldvoice")  // a Voice& of an earlier voice, kept and read later
    {
      if (v == 0) held = &voice;
      outputs[0] += x * held->outputs.constRow(kGate);
    }
    if (how == "drift") outputs[0] += x;
  }
};
const char* const kRefusals[] = {"rescale", "twice", "assign", "other", "differ", "inactive", "inputs", "controller",
                                 "polyphony", "shared", "sharedrow", "heldvoice", "drift"};

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

int main(int argc, char** argv)
{
  if (argc < 3)
  {
    std::fprintf(stderr, "usage: test_synth_trace dump|run <midi|mpe|modcc|unison|refusal> ...\n");
    return 2;
  }
  const std::string mode = argv[1], which = argv[2];
  static const char* const variants[] = {"midi", "mpe", "modcc", "unison"};
  int variant = -1;
  for (int k = 0; k < 4; ++k)
    if (which == variants[k]) variant = k;
  bool refusal = false;
  for (const char* r : kRefusals) refusal = refusal || which == r;
  if (variant < 0 && !refusal) return 2;
  try
  {
    TracedSynth traced;
    if (refusal)
    {
      RefusedSynth synth(which);
      AudioContext ctx(which == "inputs" ? 1 : 0, 1, 48000);
      ctx.setInputPolyphony(which == "polyphony" ? 3 : 4);
      if (which == "drift") ctx.setInputDriftAmount(0.5f);
      traced.trace(synth, ctx);
      std::printf("traced %s: not refused\n", which.c_str());
      return 0;
    }
    BodySynth synth(variant == 1 ? 15 : 16);
    AudioContext ctx(0, 2, 48000);
    synthBodySetup(ctx, synth, variant);
    traced.trace(synth, ctx);
    if (mode == "dump")
    {
      traced.dump(stdout);
      return 0;
    }
    if (mode == "run" && argc == 7)
    {
      const int G = std::atoi(argv[3]), T = std::atoi(argv[4]);
      const std::string dir = argv[5];
      std::vector<char> off, ev, toff, tr;
      if (!readAll(dir + "/offsets.bin", off) || !readAll(dir + "/events.bin", ev) || !readAll(dir + "/toff.bin", toff) ||
          !readAll(dir + "/tr.bin", tr))
        return 3;
      if (off.size() != (size_t)T * (G + 1) * 4 || toff.size() != off.size()) return 3;
      traced.compile(G);
      std::vector<float> bus((size_t)T * traced.outs().size() * G * 64);
      const auto* o = reinterpret_cast<const int32_t*>(off.data());
      const auto* to = reinterpret_cast<const int32_t*>(toff.data());
      const auto* e = reinterpret_cast<const mlb_event*>(ev.data());
      const auto* t = reinterpret_cast<const mlb_transport*>(tr.data());
      const int nEv = (int)(ev.size() / sizeof(mlb_event)), nTr = (int)(tr.size() / sizeof(mlb_transport));
      int t0 = 0;
      std::string launches;
      for (const char* s = argv[6]; t0 < T;)
      {
        int n = std::atoi(s);
        if (n <= 0 || t0 + n > T) n = T - t0;
        const long long k0 = mlb_kernel_launches();
        traced.process(o + (size_t)t0 * (G + 1), e, nEv, to + (size_t)t0 * (G + 1), t, nTr,
                       bus.data() + (size_t)t0 * traced.outs().size() * G * 64, n);
        launches += (launches.empty() ? "" : ",") + std::to_string(mlb_kernel_launches() - k0);
        t0 += n;
        const char* c = std::strchr(s, ',');
        s = c ? c + 1 : "";
      }
      FILE* f = std::fopen((dir + "/bus.bin").c_str(), "wb");
      std::fwrite(bus.data(), 4, bus.size(), f);
      std::fclose(f);
      std::printf("ran %s: %d instruments x %d voices x %d vectors on %s\nlaunches per call: %s\n", which.c_str(), G,
                  traced.numVoices(), T, traced.kernelName(), launches.c_str());
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
