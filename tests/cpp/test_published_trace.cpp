// tests/cpp/test_published_trace.cpp -- a madronalib Synth subclass that publishes signals (tests/cpp/published_body.h,
// also compiled against the reference in oracle/ref/mlpsynth.cpp) traced by mlb::tr::TracedSynth with only the
// namespace changed, plus the stores TracedSynth must refuse.
//
//   test_published_trace dump <case>      trace only (no GPU needed), print the instrument bank as JSON
//   test_published_trace run <case> <instruments> <blocks> <dir> <splits>
//                                         compile for <instruments> instruments, then process <blocks> vectors in calls
//                                         of the comma-separated <splits> vectors, each call followed by the reads of
//                                         published_body.h: <dir>/offsets.bin int32 [T][G + 1] and events.bin
//                                         (mlb_event) in; <dir>/bus.bin f32 [T][2][G][64], counts.bin int32
//                                         [calls][3][G], dest.bin f32 [calls][3][G][kPublishReadWidth] out
// cases: midi, mpe, nostore (MIDI without its stores), and the refusals below.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "mlb200_trace.hpp"

using namespace mlb::tr;  // the reference says: using namespace ml;
#include "published_body.h"

// ---------------------------------------------------------------- what TracedSynth refuses
struct RefusedSynth : public Synth
{
  std::string how;
  SineGen osc[16];
  RefusedSynth(const std::string& h) : Synth(2), how(h) { publishSignal("sig", 32, 2, 2, 0); }
  void processVoice(int v, const EventsToSignals::Voice& voice, const DSPVectorDynamic&, DSPVectorDynamic& outputs,
                    AudioContext*) override
  {
    DSPVector x = osc[v](voice.outputs.constRow(kPitch) * 0.01f);
    outputs[0] += x;
    const float host[2] = {0.f, 0.f};
    if (how == "channels") storePublishedSignal("sig", x, 16, v);
    if (how == "frames") storePublishedSignal("sig", concatRows(x, x), 65, v);
    if (how == "maxframes") storePublishedSignal("sig", concatRows(x, x), 33, v);
    if (how == "vert") storePublishedSignal("sig", concatRows(x, x), 16, v), storePublishedSignalVert("sig", host, 2, v);
    if (how == "differ" && v == 1) storePublishedSignal("sig", concatRows(x, x), 16, v);
  }
};
const char* const kRefusals[] = {"channels", "frames", "maxframes", "vert", "differ"};

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

static void writeAll(const std::string& path, const void* p, size_t bytes)
{
  FILE* f = std::fopen(path.c_str(), "wb");
  std::fwrite(p, 1, bytes, f);
  std::fclose(f);
}

int main(int argc, char** argv)
{
  if (argc < 3)
  {
    std::fprintf(stderr, "usage: test_published_trace dump|run <midi|mpe|nostore|refusal> ...\n");
    return 2;
  }
  const std::string mode = argv[1], which = argv[2];
  static const char* const variants[] = {"midi", "mpe", "nostore"};
  int variant = -1;
  for (int k = 0; k < 3; ++k)
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
      AudioContext ctx(0, 1, 48000);
      ctx.setInputPolyphony(2);
      traced.trace(synth, ctx);
      std::printf("traced %s: not refused\n", which.c_str());
      return 0;
    }
    PublishSynth synth(variant == 1 ? 15 : 16, variant != 2);
    AudioContext ctx(0, 2, 48000);
    publishBodySetup(ctx, synth, variant == 2 ? 0 : variant);
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
      std::vector<char> off, ev;
      if (!readAll(dir + "/offsets.bin", off) || !readAll(dir + "/events.bin", ev)) return 3;
      if (off.size() != (size_t)T * (G + 1) * 4) return 3;
      traced.compile(G);
      const size_t nOut = traced.outs().size();
      std::vector<float> bus((size_t)T * nOut * G * 64), dest, row((size_t)G * kPublishReadWidth);
      std::vector<int32_t> counts, c((size_t)G);
      const auto* o = reinterpret_cast<const int32_t*>(off.data());
      const auto* e = reinterpret_cast<const mlb_event*>(ev.data());
      const int nEv = (int)(ev.size() / sizeof(mlb_event));
      static const char* const names[kPublishSignals] = {"scope", "voices", "pitch"};
      int t0 = 0, call = 0;
      std::string launches;
      for (const char* s = argv[6]; t0 < T; ++call)
      {
        int n = std::atoi(s);
        if (n <= 0 || t0 + n > T) n = T - t0;
        const long long k0 = mlb_kernel_launches();
        traced.process(o + (size_t)t0 * (G + 1), e, nEv, nullptr, nullptr, 0, bus.data() + (size_t)t0 * nOut * G * 64, n);
        launches += (launches.empty() ? "" : ",") + std::to_string(mlb_kernel_launches() - k0);
        t0 += n;
        const char* cm = std::strchr(s, ',');
        s = cm ? cm + 1 : "";
        if (variant == 2) continue;
        for (int k = 0; k < kPublishSignals; ++k)
        {
          const int frames = kPublishReadFrames[k], width = frames * (k == 0 ? 2 : 1);
          std::vector<float> d((size_t)G * width, 0.f);
          switch (publishReadMode(call, k))
          {
            case 0: traced.readLatest(names[k], frames, d.data(), c.data()); break;
            case 1: traced.read(names[k], frames, d.data(), c.data()); break;
            case 2: traced.peekLatest(names[k], frames, d.data(), c.data()); break;
            default: traced.availableFrames(names[k], c.data()); break;
          }
          std::fill(row.begin(), row.end(), 0.f);
          for (int g = 0; g < G; ++g)
            std::memcpy(&row[(size_t)g * kPublishReadWidth], &d[(size_t)g * width], (size_t)width * 4);
          dest.insert(dest.end(), row.begin(), row.end());
          counts.insert(counts.end(), c.begin(), c.end());
        }
      }
      writeAll(dir + "/bus.bin", bus.data(), bus.size() * 4);
      writeAll(dir + "/counts.bin", counts.data(), counts.size() * 4);
      writeAll(dir + "/dest.bin", dest.data(), dest.size() * 4);
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
