// oracle/ref/mlctrl.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Runs the reference's own smoothed controllers as the checker of kernel K11: one complete, UNMODIFIED
// EventsToSignals (source/app/MLEventsToSignals.{h,cpp}) per instrument -- setSampleRate, setProtocol,
// setPolyphony, addEvent, processVector -- and reads getController(n).output after every vector.  So the whole
// reference path is exercised: the event sort, the controller-number clamp, the channel-pressure route, the glide
// length and SmoothedController's recalcNeeded.  oracle/ctrl.mk compiles this file in place with the reference's
// MLEventsToSignals.cpp, MLSymbol.cpp and MLText.cpp into oracle/_ref/libmlctrl.so.  Nothing from the reference is
// copied into this repository.
//
// Only tests/ and the golden writer may load the library.
#include <cstdint>
#include <memory>

#include "MLEventsToSignals.h"
#include "mlb200.h"

using namespace ml;

extern "C"
{
// G instruments, T vectors.  The events of instrument g are events[ev_off[g] .. ev_off[g + 1]), times in frames
// from the start of vector 0.  ctrl [C] controller numbers; out [T][C][G][64].
void mlctrl_run(int G, int C, int T, double sample_rate, int protocol, int polyphony, const int32_t* ctrl,
                const int32_t* ev_off, const mlb_event* events, float* out)
{
  for (int g = 0; g < G; ++g)
  {
    auto e2s = std::make_unique<EventsToSignals>();
    if (protocol == 1) e2s->setProtocol(Symbol("MPE"));
    e2s->setSampleRate(sample_rate);
    e2s->setPolyphony((size_t)polyphony);
    for (int i = ev_off[g]; i < ev_off[g + 1]; ++i)
    {
      Event e;
      e.type = events[i].type, e.channel = events[i].channel, e.sourceIdx = events[i].source_idx;
      e.time = events[i].time, e.value1 = events[i].value1, e.value2 = events[i].value2;
      e2s->addEvent(e);
    }
    for (int t = 0; t < T; ++t)
    {
      e2s->processVector(t * kFloatsPerDSPVector);
      for (int c = 0; c < C; ++c)
        store(e2s->getController((size_t)ctrl[c]).output, out + (((size_t)t * C + c) * G + g) * kFloatsPerDSPVector);
    }
  }
}
}  // extern "C"
