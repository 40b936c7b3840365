// tests/cpp/synth_body.h -- ONE Synth subclass, compiled twice from this very file:
//   * against the reference itself (oracle/ref/mltsynth.cpp: `using namespace ml;`), G AudioContext + Synth objects, and
//   * against the tracing layer (tests/cpp/test_synth_trace.cpp: `using namespace mlb::tr;`), run by mlb::tr::TracedSynth.
// processVoice reads the voice's pitch, gate (velocity), z and mod rows, controllers 1 and 74 and the beat phase:
// pitch -> frequency through exp2 and pow, a SineGen and a SawGen per voice, an ADSR on the gate, a Lopass whose
// cutoff depends on voiceIndex, a detune that depends on voiceIndex, a tempo-synced LFO, a DSPVector member carried
// between vectors, and two outputs.
#pragma once

// Every numeric parameter goes through a volatile read, so that neither build folds a makeCoeffs / calcCoeffs call at
// compile time (see kitchen_body.h).
static volatile float kSynthParams[] = {
    0.004f, 0.05f, 0.6f, 0.08f,  // 0-3: ADSR attack, decay, sustain, release
    0.03f, 0.07f, 0.9f,          // 4-6: Lopass omega, its per-voice spread, k
    5.75f, 440.f, 0.0013f,       // 7-9: pitch of 440 Hz in octaves, 440, detune per voice
    5.5f, 0.4f,                  // 10-11: the saw's pitch offset, its level
    6.2831853f, 0.3f, 0.5f,      // 12-14: the LFO's radians per quarter note, the carried row's feedback, CC 1 depth
    0.25f, 0.2f, 0.1f,           // 15-17: LFO depth, z depth, CC 74 offset
    2.f, 48.f, 0.03f,            // 18-20: pitch bend, MPE pitch bend (semitones), glide (seconds)
};
inline float sbp(int i) { return kSynthParams[i]; }

class BodySynth : public Synth
{
 public:
  explicit BodySynth(int nVoices) : Synth(nVoices) {}

  SineGen sine[16];
  SawGen saw[16];
  ADSR adsr[16];
  Lopass lp[16];
  DSPVector carried[16];  // read before it is written: state between vectors
  float sr = 48000.f;

  void init(float sampleRate)
  {
    sr = sampleRate;
    for (int v = 0; v < 16; ++v)
    {
      sine[v].clear();
      adsr[v].coeffs = ADSR::calcCoeffs(sbp(0), sbp(1), sbp(2), sbp(3), sampleRate);
      lp[v].coeffs = Lopass::makeCoeffs(sbp(4) * (1.f + sbp(5) * (float)v), sbp(6));
    }
  }

  void processVoice(int voiceIndex, const EventsToSignals::Voice& voice, const DSPVectorDynamic& inputs,
                    DSPVectorDynamic& outputs, AudioContext* ctx) override
  {
    const int v = voiceIndex;
    DSPVector pitch = voice.outputs.constRow(kPitch);
    DSPVector gate = voice.outputs.constRow(kGate);
    DSPVector z = voice.outputs.constRow(kZ);
    DSPVector mod = voice.outputs.constRow(kMod);

    // pitch in octaves -> cycles per sample, the sine detuned by voice
    DSPVector cps = exp2(pitch - sbp(7)) * (sbp(8) / sr) * (1.f + sbp(9) * (float)v);
    DSPVector cps2 = pow(DSPVector(2.f), pitch - sbp(10)) * (sbp(8) / sr);
    DSPVector osc = sine[v](cps) + saw[v](cps2) * sbp(11);
    DSPVector amp = adsr[v](gate);

    DSPVector y = lp[v](osc * amp) + carried[v] * sbp(13);
    carried[v] = y;

    DSPVector c1 = ctx->getInputController(1);
    DSPVector c74 = ctx->getInputController(74);
    DSPVector lfo = sin(ctx->getBeatPhase() * sbp(12));

    outputs[0] += y * (c1 * sbp(14) + 1.f) * (lfo * sbp(15) + 1.f);
    outputs[1] += (y * mod + osc * z * sbp(16)) * (c74 + sbp(17));
  }
};

// The instrument's setup.  variant 0: MIDI; 1: MPE; 2: MIDI with mod CC 74; 3: MIDI in unison.  All glide; none
// drifts (mlb::tr::TracedSynth refuses a drift amount above 0).
template <class CTX>
inline void synthBodySetup(CTX& ctx, BodySynth& synth, int variant)
{
  ctx.setInputProtocol(Symbol(variant == 1 ? "MPE" : "MIDI"));
  ctx.setInputPolyphony(synth.getNumVoices());
  ctx.setInputPitchBend(sbp(18));
  ctx.setInputMPEPitchBend(sbp(19));
  ctx.setInputGlideTimeInSeconds(sbp(20));
  if (variant == 2) ctx.setInputModCC(74);
  if (variant == 3) ctx.setInputUnison(true);
  synth.init((float)ctx.getSampleRate());
}
