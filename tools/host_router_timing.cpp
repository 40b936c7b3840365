// host_router_timing.cpp -- wall time of routing a performance with one mlb::VoiceRouter per instrument on one host
// thread, the work mlb_synth_process_routed_host moves to the GPU.  Used by tools/bench_configs.py (--only routed),
// which compiles it into a temporary directory.
//
// Input file (little-endian): int32 G, T, protocol, reps; int32 polyphony[G], first_voice[G], V; int32 offsets
// [T][G + 1]; int32 n_events; mlb_event events[n_events].  Output: one JSON line with the best of `reps` runs, and the
// records [T][V] of the last run in the file named by the second argument.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <vector>

#include "mlb200_events.hpp"

int main(int argc, char** argv)
{
  if (argc != 3) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  auto rd = [&](void* p, size_t n) { return std::fread(p, 1, n, f) == n; };
  int32_t hdr[4], V = 0, n_events = 0;
  if (!rd(hdr, sizeof(hdr))) return 2;
  const int G = hdr[0], T = hdr[1], protocol = hdr[2], reps = hdr[3];
  std::vector<int32_t> poly(G), first(G), offsets((size_t)T * (G + 1));
  if (!rd(poly.data(), G * 4) || !rd(first.data(), G * 4) || !rd(&V, 4) || !rd(offsets.data(), offsets.size() * 4) ||
      !rd(&n_events, 4))
    return 2;
  std::vector<mlb_event> events(n_events);
  if (!rd(events.data(), events.size() * sizeof(mlb_event))) return 2;
  std::fclose(f);
  std::vector<mlb_voice_events> records((size_t)T * V);
  double best = 1e30;
  long long overflow = 0;
  for (int r = 0; r < reps; ++r)
  {
    const auto t0 = std::chrono::steady_clock::now();
    overflow = 0;
    for (int g = 0; g < G; ++g)
    {
      mlb::VoiceRouter router(poly[g], protocol == 1 ? mlb::VoiceRouter::kMPE : mlb::VoiceRouter::kMIDI);
      for (int t = 0; t < T; ++t)
      {
        const int32_t* o = offsets.data() + (size_t)t * (G + 1);
        for (int i = o[g]; i < o[g + 1]; ++i)
        {
          const mlb_event& e = events[i];
          mlb::Event ev;
          ev.type = e.type, ev.channel = e.channel, ev.sourceIdx = e.source_idx, ev.time = t * MLB_BLOCK + e.time;
          ev.value1 = e.value1, ev.value2 = e.value2;
          router.addEvent(ev);
        }
        overflow += router.processVector(t * MLB_BLOCK, records.data() + (size_t)t * V + first[g]);
        router.clearEvents();
      }
    }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    best = std::min(best, ms);
  }
  FILE* out = std::fopen(argv[2], "wb");
  if (!out || std::fwrite(records.data(), sizeof(mlb_voice_events), records.size(), out) != records.size()) return 2;
  std::fclose(out);
  std::printf("{\"host_routing_ms\": %.3f, \"instruments\": %d, \"blocks\": %d, \"events\": %d, \"reps\": %d, "
              "\"overflow\": %lld}\n",
              best, G, T, n_events, reps, overflow);
  return 0;
}
