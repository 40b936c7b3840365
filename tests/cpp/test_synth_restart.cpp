// tests/cpp/test_synth_restart.cpp -- TracedSynth::restart between calls: the Synth subclass of tests/cpp/synth_body.h
// traced as in test_synth_trace, run from raw events, with chosen instruments restarted at chosen call boundaries.
//
//   test_synth_restart run <case> <instruments> <blocks> <dir> <splits> <restarts>
//       as test_synth_trace run (<dir>/offsets.bin, events.bin, toff.bin, tr.bin in, <dir>/bus.bin out), and before
//       the call that starts at vector t, TracedSynth::restart of the instruments listed for t.  <restarts> is
//       "t:g+g+...,t:..." ("t:" restarts an empty list); a t that is not the start of a call is an error.
//       Prints the launches of every call and of every restart.
// cases: midi, mpe (synthBodySetup's variants 0 and 1).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "mlb200_trace.hpp"

using namespace mlb::tr;  // the reference says: using namespace ml;
#include "synth_body.h"

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

// "t:g+g,t:" -> {t: [g, g], t: []}
static std::map<int, std::vector<int>> parseRestarts(const std::string& s)
{
  std::map<int, std::vector<int>> out;
  size_t i = 0;
  while (i < s.size())
  {
    size_t end = s.find(',', i);
    if (end == std::string::npos) end = s.size();
    const std::string item = s.substr(i, end - i);
    const size_t colon = item.find(':');
    std::vector<int>& list = out[std::atoi(item.substr(0, colon).c_str())];
    for (size_t j = colon + 1; j < item.size();)
    {
      size_t k = item.find('+', j);
      if (k == std::string::npos) k = item.size();
      list.push_back(std::atoi(item.substr(j, k - j).c_str()));
      j = k + 1;
    }
    i = end + 1;
  }
  return out;
}

int main(int argc, char** argv)
{
  if (argc != 8 || std::string(argv[1]) != "run")
  {
    std::fprintf(stderr, "usage: test_synth_restart run <midi|mpe> <instruments> <blocks> <dir> <splits> <restarts>\n");
    return 2;
  }
  const std::string which = argv[2];
  if (which != "midi" && which != "mpe") return 2;
  const int variant = which == "mpe" ? 1 : 0;
  try
  {
    TracedSynth traced;
    BodySynth synth(variant == 1 ? 15 : 16);
    AudioContext ctx(0, 2, 48000);
    synthBodySetup(ctx, synth, variant);
    traced.trace(synth, ctx);
    const int G = std::atoi(argv[3]), T = std::atoi(argv[4]);
    const std::string dir = argv[5];
    std::vector<char> off, ev, toff, tr;
    if (!readAll(dir + "/offsets.bin", off) || !readAll(dir + "/events.bin", ev) || !readAll(dir + "/toff.bin", toff) ||
        !readAll(dir + "/tr.bin", tr))
      return 3;
    if (off.size() != (size_t)T * (G + 1) * 4 || toff.size() != off.size()) return 3;
    std::map<int, std::vector<int>> restarts = parseRestarts(argv[7]);
    traced.compile(G);
    std::vector<float> bus((size_t)T * traced.outs().size() * G * 64);
    const auto* o = reinterpret_cast<const int32_t*>(off.data());
    const auto* to = reinterpret_cast<const int32_t*>(toff.data());
    const auto* e = reinterpret_cast<const mlb_event*>(ev.data());
    const auto* t = reinterpret_cast<const mlb_transport*>(tr.data());
    const int nEv = (int)(ev.size() / sizeof(mlb_event)), nTr = (int)(tr.size() / sizeof(mlb_transport));
    int t0 = 0;
    std::string launches, restartLaunches;
    for (const char* s = argv[6]; t0 < T;)
    {
      int n = std::atoi(s);
      if (n <= 0 || t0 + n > T) n = T - t0;
      auto r = restarts.find(t0);
      if (r != restarts.end())
      {
        const long long k0 = mlb_kernel_launches();
        traced.restart(r->second);
        restartLaunches += (restartLaunches.empty() ? "" : ",") + std::to_string(mlb_kernel_launches() - k0);
        restarts.erase(r);
      }
      const long long k0 = mlb_kernel_launches();
      traced.process(o + (size_t)t0 * (G + 1), e, nEv, to + (size_t)t0 * (G + 1), t, nTr,
                     bus.data() + (size_t)t0 * traced.outs().size() * G * 64, n);
      launches += (launches.empty() ? "" : ",") + std::to_string(mlb_kernel_launches() - k0);
      t0 += n;
      const char* c = std::strchr(s, ',');
      s = c ? c + 1 : "";
    }
    if (!restarts.empty())
    {
      std::printf("restart at vector %d: not the start of a call\n", restarts.begin()->first);
      return 2;
    }
    FILE* f = std::fopen((dir + "/bus.bin").c_str(), "wb");
    std::fwrite(bus.data(), 4, bus.size(), f);
    std::fclose(f);
    std::printf("ran %s: %d instruments x %d voices x %d vectors on %s\nlaunches per call: %s\nlaunches per restart: %s\n",
                which.c_str(), G, traced.numVoices(), T, traced.kernelName(), launches.c_str(), restartLaunches.c_str());
    return 0;
  }
  catch (const mlb::Error& e)
  {
    std::printf("mlb error %d: %s\n", e.code, e.what());
    return e.code == MLB_ERR_NO_DEVICE ? 77 : 1;
  }
}
