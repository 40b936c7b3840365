// mlb200_events.hpp -- host-side event routing in front of the EventsToSignals::Voice bank (K7).
//
// The reference's EventsToSignals (source/app/MLEventsToSignals.{h,cpp}) does two jobs: it ROUTES
// incoming note / controller events to voices (allocation, stealing, unison, sustain pedal --
// MLEventsToSignals.cpp:370-418, 476-960) and it GENERATES the per-voice control rows
// (EventsToSignals::Voice, .cpp:47-263).  The generation runs on the GPU (mlb_voices_*, mlb200.h).
// This header restates the routing for the MIDI protocol as plain host C++ that, per 64-frame vector,
// emits one mlb_voice_events record per voice -- exactly the writeNoteEvent calls and current-value
// writes the reference would have made.  tests/cpp/test_router.cpp checks it against the complete
// reference EventsToSignals on MIDI phrases.
//
// Both protocols of the reference are routed: "MIDI" (key = note number) and "MPE" (key = channel; the
// main voice, voices[0], gets the channel-1 bend and pressure and its rows are added to the channel voices
// by the bank, mlb_voices_set_main_voices).  Not covered: controller 120 "all sound off" (it resets voices
// mid-vector, .cpp:748-755).
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

extern "C" {
#include "mlb200.h"
}

namespace mlb
{
// ml::EventType, source/app/MLEvent.h:14-27
enum EventType : uint8_t
{
  kNull = 0,
  kNoteOn,
  kNoteRetrig,
  kNoteSustain,
  kNoteOff,
  kSustainPedal,
  kController,
  kPitchBend,
  kNotePressure,
  kChannelPressure,
  kProgramChange
};

// ml::Event, source/app/MLEvent.h:31-50
struct Event
{
  uint8_t type{kNull};
  uint8_t channel{0};
  uint16_t sourceIdx{0};  // key or controller number
  int time{0};            // frames from the start of the top-level buffer
  float value1{0};
  float value2{0};
};

class VoiceRouter
{
 public:
  static constexpr int kMaxVoices = 16;         // EventsToSignals::kMaxVoices, .h:47
  static constexpr int kMaxPhysicalKeys = 128;  // .h:49
  static constexpr int kChannelPressureControllerIdx = 128;

  enum Protocol { kMIDI = 0, kMPE = 1 };

  explicit VoiceRouter(int polyphony, Protocol protocol = kMIDI) : protocol_(protocol) { setPolyphony(polyphony); }

  // records written per vector: MIDI: voices 1..polyphony -> records[0..polyphony-1];
  // MPE: voices 0..polyphony (0 = the main voice) -> records[0..polyphony]
  int recordCount() const { return protocol_ == kMPE ? polyphony_ + 1 : polyphony_; }

  // setPolyphony -> clear(), .cpp:312-331
  int setPolyphony(int n)
  {
    events_.clear();
    for (auto& v : voices_) v = VoiceMirror{};
    lastFreeVoiceFound_ = 0;
    polyphony_ = std::min(std::max(n, 0), kMaxVoices);
    return polyphony_;
  }
  int polyphony() const { return polyphony_; }
  void setUnison(bool b) { unison_ = b; }
  void setModCC(int c) { voiceModCC_ = c; }
  bool awake() const { return awake_; }
  int newestVoice() const { return newestVoice_ - 1; }
  int unsupportedEvents() const { return unsupported_; }
  // the writes of SmoothedController inputValues of the last processVector, in the order they were applied:
  // controller events and, in the MIDI protocol, channel pressure (controller 128)
  const std::vector<mlb_controller_change>& controllerChanges() const { return changes_; }

  // addEvent, .cpp:352-368: insert sorted by (time, type)
  void addEvent(const Event& e)
  {
    awake_ = true;
    auto it = std::lower_bound(events_.begin(), events_.end(), e, [](const Event& a, const Event& b)
                               { return a.time != b.time ? a.time < b.time : a.type < b.type; });
    events_.insert(it, e);
  }
  void clearEvents() { events_.clear(); }

  // processVector, .cpp:372-418: route the events in [startTime, startTime + 64) and write one record
  // per voice (records[i] belongs to voice i + 1 of the reference, i < polyphony).  Returns the number
  // of note events that did not fit into a record (MLB_VOICE_MAX_EVENTS per voice and vector).
  // The vector's controller writes are collected on the side (controllerChanges()).
  int processVector(int startTime, mlb_voice_events* records)
  {
    overflow_ = 0;
    changes_.clear();
    records_ = records;
    for (int i = 0; i < recordCount(); ++i) std::memset(&records[i], 0, sizeof(mlb_voice_events));
    const int endTime = startTime + MLB_BLOCK;
    // the buffer is walked by index: a routed event never inserts into it
    for (size_t i = 0; i < events_.size(); ++i)
    {
      if (events_[i].time >= startTime && events_[i].time < endTime)
      {
        Event e = events_[i];
        e.time -= startTime;
        processEvent(e);
      }
    }
    records_ = nullptr;
    return overflow_;
  }

 private:
  struct KeyState  // .h:29-39
  {
    enum State { kOff, kOn, kSustained } state{kOff};
    float pitch{0.f};
    uint32_t noteOnIndex{0};
  };
  struct VoiceMirror  // the Voice members the routing reads back, .h:129,121
  {
    int creatorKeyIdx{0};
    float currentVelocity{0.f};
  };

  // Voice::writeNoteEvent as seen from the router: append to the voice's record, mirror the members
  void writeNoteEvent(int v, const Event& e, int keyIdx, bool doGlide, bool doReset)
  {
    switch (e.type)
    {
      case kNoteOn:
      case kNoteRetrig:
        voices_[v].creatorKeyIdx = keyIdx;
        voices_[v].currentVelocity = e.value2;
        break;
      case kNoteOff:
        voices_[v].creatorKeyIdx = 0;
        voices_[v].currentVelocity = 0.f;
        break;
      default: return;  // kNoteSustain and everything else: the voice ignores it
    }
    if (v > polyphony_ || v < (protocol_ == kMPE ? 0 : 1)) return;  // MIDI: the main voice has no record
    mlb_voice_events& r = record(v);
    if (r.n_events >= MLB_VOICE_MAX_EVENTS)
    {
      ++overflow_;
      return;
    }
    const int k = r.n_events++;
    r.time[k] = (uint8_t)std::min(std::max(e.time, 0), MLB_BLOCK);
    r.type[k] = e.type;
    r.flags[k] = (uint8_t)((doGlide ? MLB_EVF_GLIDE : 0) | (doReset ? MLB_EVF_RESET : 0));
    r.value1[k] = e.value1;
    r.value2[k] = e.value2;
  }
  mlb_voice_events& record(int v) { return records_[protocol_ == kMPE ? v : v - 1]; }
  int keyIndex(const Event& e) const { return protocol_ == kMPE ? e.channel : e.sourceIdx; }  // getKeyIndex, .cpp:20-43
  void setCurrent(int v, unsigned bit, float val)
  {
    mlb_voice_events& r = record(v);
    r.set_mask |= (uint8_t)bit;
    switch (bit)
    {
      case MLB_SET_BEND: r.bend = val; break;
      case MLB_SET_MOD: r.mod = val; break;
      case MLB_SET_X: r.x = val; break;
      case MLB_SET_Y: r.y = val; break;
      case MLB_SET_Z: r.z = val; break;
      case MLB_SET_PRESSURE: r.pressure = val; break;
    }
  }

  void addChange(int ctrl, float val)
  {
    mlb_controller_change c{};
    c.controller = (uint16_t)ctrl;
    c.value = val;
    changes_.push_back(c);
  }

  int countHeldNotes() const  // .cpp:463-474
  {
    int n = 0;
    for (const auto& ks : keyStates_) n += ks.state == KeyState::kOn;
    return n;
  }
  int findFreeVoice()  // .cpp:880-900
  {
    const int highest = polyphony_ + 1;
    int t = lastFreeVoiceFound_;
    for (int i = 1; i < polyphony_ + 1; ++i)
    {
      if (++t >= highest) t = 1;
      if (voices_[t].creatorKeyIdx == 0)
      {
        lastFreeVoiceFound_ = t;
        return t;
      }
    }
    return -1;
  }
  int findNearestVoice(int note) const  // .cpp:910-925
  {
    int r = 0;
    size_t minDist = 128;
    for (int v = 1; v < polyphony_ + 1; ++v)
    {
      const size_t d = (size_t)std::abs(note - voices_[v].creatorKeyIdx);
      if (d < minDist) minDist = d, r = v;
    }
    return r;
  }

  void processEvent(const Event& e)  // .cpp:477-509
  {
    switch (e.type)
    {
      case kNoteOn: noteOn(e); break;
      case kNoteOff: noteOff(e); break;
      case kController: controller(e); break;
      case kPitchBend:  // .cpp:700-735
        if (protocol_ == kMIDI)
          for (int v = 1; v < polyphony_ + 1; ++v) setCurrent(v, MLB_SET_BEND, e.value1);
        else if (e.channel == 1)
          setCurrent(0, MLB_SET_BEND, e.value1);  // the main voice
        else if (e.channel != 0)
          for (int v = 1; v < polyphony_ + 1; ++v)
            if (voices_[v].creatorKeyIdx == e.channel) setCurrent(v, MLB_SET_BEND, e.value1);
        break;
      case kNotePressure:  // .cpp:673-697; ignored in MPE mode
        if (protocol_ == kMIDI)
          for (int v = 1; v < polyphony_ + 1; ++v)
            if (voices_[v].creatorKeyIdx == e.sourceIdx) setCurrent(v, MLB_SET_Z, e.value1);
        break;
      case kChannelPressure:  // .cpp:634-670
        if (protocol_ == kMIDI)  // controllers[128].inputValue, one smoother copy per voice
        {
          addChange(kChannelPressureControllerIdx, e.value1);
          for (int v = 1; v < polyphony_ + 1; ++v) setCurrent(v, MLB_SET_PRESSURE, e.value1);
        }
        else if (e.channel == 1)
          setCurrent(0, MLB_SET_Z, e.value1);
        else if (e.channel != 0)
          for (int v = 1; v < polyphony_ + 1; ++v)
            if (voices_[v].creatorKeyIdx == e.channel) setCurrent(v, MLB_SET_Z, e.value1);
        break;
      case kSustainPedal: sustainPedal(e); break;
      default: break;
    }
  }
  void noteOn(const Event& e)  // .cpp:513-553
  {
    const int keyIdx = keyIndex(e);
    KeyState& ks = keyStates_[keyIdx % kMaxPhysicalKeys];
    ks.state = KeyState::kOn;
    ks.noteOnIndex = currentNoteOnIndex_++;
    ks.pitch = e.value1;
    if (unison_)
    {
      const bool firstNote = countHeldNotes() == 1;
      for (int v = 1; v < polyphony_ + 1; ++v) writeNoteEvent(v, e, keyIdx, !firstNote, firstNote);
      return;
    }
    int v = findFreeVoice();
    if (v >= 1)
      writeNoteEvent(v, e, keyIdx, true, true);
    else
    {
      v = findNearestVoice(e.sourceIdx);  // findVoiceToSteal
      Event f = e;
      f.type = kNoteRetrig;
      writeNoteEvent(v, f, keyIdx, true, true);
    }
    newestVoice_ = v;
  }
  void noteOff(const Event& e)  // .cpp:555-628
  {
    const int keyIdx = keyIndex(e);
    keyStates_[keyIdx % kMaxPhysicalKeys].state = sustainPedalActive_ ? KeyState::kSustained : KeyState::kOff;
    if (unison_)
    {
      if (countHeldNotes() == 0)
      {
        for (int v = 1; v < polyphony_ + 1; ++v) writeNoteEvent(v, e, 0, true, true);
      }
      else if (keyIdx == voices_[1].creatorKeyIdx)
      {
        // fall back to the most recently played key that is still held, without retriggering
        Event send = e;
        send.type = kNoteOn;
        send.value2 = voices_[1].currentVelocity;
        uint32_t maxIndex = 0, recentKey = 0;
        for (int i = 0; i < kMaxPhysicalKeys; ++i)
          if (keyStates_[i].state == KeyState::kOn && keyStates_[i].noteOnIndex > maxIndex)
            maxIndex = keyStates_[i].noteOnIndex, recentKey = (uint32_t)i;
        send.value1 = keyStates_[recentKey].pitch;
        for (int v = 1; v < polyphony_ + 1; ++v) writeNoteEvent(v, send, (int)recentKey, true, true);
      }
      return;
    }
    if (!sustainPedalActive_)
      for (int v = 1; v < polyphony_ + 1; ++v)
        if (voices_[v].creatorKeyIdx == keyIdx) writeNoteEvent(v, e, keyIdx, true, true);  // type stays kNoteOff
  }
  void controller(const Event& e)  // .cpp:737-820
  {
    const float val = e.value1;
    const int ctrl = std::min<int>(e.sourceIdx, kChannelPressureControllerIdx);
    addChange(ctrl, val);  // controllers[ctrl].inputValue = val, before the special cases
    if (ctrl == kChannelPressureControllerIdx && protocol_ == kMIDI)  // controllers[ctrl].inputValue = val
      for (int v = 1; v < polyphony_ + 1; ++v) setCurrent(v, MLB_SET_PRESSURE, val);
    if (ctrl == 120)
    {
      if (val == 0) ++unsupported_;  // all sound off resets the voices mid-vector: not routed
    }
    else if (ctrl == 123)
    {
      if (val == 0)
      {
        Event off = e;
        off.type = kNoteOff;
        for (int v = 0; v < kMaxVoices + 1; ++v) writeNoteEvent(v, off, 0, false, true);  // every voice, .cpp:759-766
      }
    }
    else
      for (int v = 1; v < polyphony_ + 1; ++v)
      {
        if (protocol_ == kMPE && voices_[v].creatorKeyIdx != e.channel) continue;  // MPE: only the channel's voices
        if (ctrl == voiceModCC_) setCurrent(v, MLB_SET_MOD, val);
        if (ctrl == 73)
          setCurrent(v, MLB_SET_X, val);
        else if (ctrl == 74)
          setCurrent(v, MLB_SET_Y, val);
      }
  }
  void sustainPedal(const Event& e)  // .cpp:823-841
  {
    sustainPedalActive_ = e.value1 > 0.5f;
    if (sustainPedalActive_) return;
    for (int v = 1; v < polyphony_ + 1; ++v)
      if (keyStates_[voices_[v].creatorKeyIdx % kMaxPhysicalKeys].state == KeyState::kSustained)
      {
        Event off;  // a default Event: time 0
        off.type = kNoteOff;
        writeNoteEvent(v, off, 0, true, true);
      }
  }

  std::array<VoiceMirror, kMaxVoices + 1> voices_{};
  std::array<KeyState, kMaxPhysicalKeys> keyStates_{};
  std::vector<Event> events_;
  std::vector<mlb_controller_change> changes_;
  mlb_voice_events* records_{nullptr};
  Protocol protocol_{kMIDI};
  int polyphony_{0};
  int lastFreeVoiceFound_{-1};
  int newestVoice_{-1};
  int voiceModCC_{16};
  bool sustainPedalActive_{false};
  bool unison_{false};
  bool awake_{false};
  uint32_t currentNoteOnIndex_{0};
  int overflow_{0};
  int unsupported_{0};
};

}  // namespace mlb
