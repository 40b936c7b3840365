// tests/cpp/published_body.h -- ONE Synth subclass that publishes signals, compiled twice from this very file:
//   * against the reference itself (oracle/ref/mlpsynth.cpp: `using namespace ml;`), G AudioContext + Synth objects, and
//   * against the tracing layer (tests/cpp/test_published_trace.cpp: `using namespace mlb::tr;`).
// Three published signals: "scope" (2 channels, every 2nd frame, a ring of 256 floats that 16 voices overflow in every
// vector) stores a carried, filtered row and the envelope; "voices" (1 channel, every 128th frame, so the written frames
// rotate between voices) stores the gate Voice row as it is; "pitch" (1 channel, every 8th frame) stores the first 17
// frames of a pitch expression.  One store goes to a name that was never published, which stores nothing.
// Variant 0: MIDI; 1: MPE; 2: MIDI with every store removed (the same audio).  After every call both builds make the
// same reads of every instrument's signals (publishReadMode, kPublishReadFrames).
#pragma once

static volatile float kPublishParams[] = {
    0.004f, 0.05f, 0.6f, 0.08f,  // 0-3: ADSR attack, decay, sustain, release
    0.05f, 0.08f, 0.8f,          // 4-6: Lopass omega, its per-voice spread, k
    5.75f, 440.f, 0.3f,          // 7-9: pitch of 440 Hz in octaves, 440, the carried row's feedback
    2.f, 48.f, 0.02f,            // 10-12: pitch bend, MPE pitch bend (semitones), glide (seconds)
};
inline float pbp(int i) { return kPublishParams[i]; }

// the reads after call k: signal s is read with mode (k + s) % 4 -- 0 readLatest, 1 read, 2 peekLatest, 3
// getAvailableFrames -- of kPublishReadFrames[s] frames; each instrument's result is one row of kPublishReadWidth floats
constexpr int kPublishSignals = 3;
constexpr int kPublishReadFrames[kPublishSignals] = {100, 9, 70};
constexpr int kPublishReadWidth = 200;
inline int publishReadMode(int call, int signal) { return (call + signal) % 4; }

class PublishSynth : public Synth
{
 public:
  PublishSynth(int nVoices, bool stores) : Synth(nVoices), stores_(stores) {}

  SineGen sine[16];
  ADSR adsr[16];
  Lopass lp[16];
  DSPVector carried[16];
  float sr = 48000.f;
  bool stores_;

  void init(float sampleRate)
  {
    sr = sampleRate;
    for (int v = 0; v < 16; ++v)
    {
      sine[v].clear();
      adsr[v].coeffs = ADSR::calcCoeffs(pbp(0), pbp(1), pbp(2), pbp(3), sampleRate);
      lp[v].coeffs = Lopass::makeCoeffs(pbp(4) * (1.f + pbp(5) * (float)v), pbp(6));
    }
    publishSignal("scope", 64, 2, 2, 1);
    publishSignal("voices", 64, 4, 1, 7);
    publishSignal("pitch", 17, 16, 1, 3);
  }

  void processVoice(int voiceIndex, const EventsToSignals::Voice& voice, const DSPVectorDynamic& inputs,
                    DSPVectorDynamic& outputs, AudioContext* ctx) override
  {
    const int v = voiceIndex;
    DSPVector pitch = voice.outputs.constRow(kPitch);
    DSPVector gate = voice.outputs.constRow(kGate);
    DSPVector osc = sine[v](exp2(pitch - pbp(7)) * (pbp(8) / sr));
    DSPVector amp = adsr[v](gate);
    DSPVector y = lp[v](osc * amp) + carried[v] * pbp(9);
    carried[v] = y;
    outputs[0] += y;
    outputs[1] += osc * gate;
    if (!stores_) return;
    storePublishedSignal("scope", concatRows(y, amp), 64, v);
    storePublishedSignal("voices", gate, 64, v);
    storePublishedSignal("nowhere", y, 64, v);
    storePublishedSignal("pitch", pitch * 2.f, 17, v);
  }
};

template <class CTX>
inline void publishBodySetup(CTX& ctx, PublishSynth& synth, int variant)
{
  ctx.setInputProtocol(Symbol(variant == 1 ? "MPE" : "MIDI"));
  ctx.setInputPolyphony(synth.getNumVoices());
  ctx.setInputPitchBend(pbp(10));
  ctx.setInputMPEPitchBend(pbp(11));
  ctx.setInputGlideTimeInSeconds(pbp(12));
  synth.init((float)ctx.getSampleRate());
}
