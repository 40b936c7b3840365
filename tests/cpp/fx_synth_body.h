// tests/cpp/fx_synth_body.h -- ONE Synth subclass that overrides processVector, compiled twice from this very file:
//   * against the reference itself (oracle/ref/mlfxsynth.cpp: `using namespace ml;`), G AudioContext + Synth objects, and
//   * against the tracing layer (tests/cpp/test_fx_synth.cpp: `using namespace mlb::tr;`), run by mlb::tr::TracedSynth.
// processVoice: a detuned SineGen through an ADSR per voice, scaled by controller 1, into two outputs.  processVector:
// controller 73 and a tap of the carried member read before the base call, the base call into a local
// DSPVectorDynamic(2), then the instrument section: a Lopass and a FractionalDelay in a feedback loop through the
// carried member, an Allpass<IntegerDelay> diffuser, controller 74 (read only here) as the wet level, controller 1
// (read by the voices too), a tremolo on the beat phase, and a third output that is bus row 0 as it is.
#pragma once

// Every numeric parameter goes through a volatile read, so that neither build folds a makeCoeffs / calcCoeffs call at
// compile time (see kitchen_body.h).
static volatile float kFxParams[] = {
    0.004f, 0.05f, 0.6f, 0.08f,  // 0-3: ADSR attack, decay, sustain, release
    5.75f, 440.f, 0.0013f,       // 4-6: pitch of 440 Hz in octaves, 440, detune per voice
    0.5f,                        // 7: CC 1 depth
    0.05f, 0.8f,                 // 8-9: the tone Lopass's omega and k
    613.5f, 2048.f, 0.4f,        // 10-12: the delay in samples, its maximum, the feedback
    0.6f, 233.f, 512.f,          // 13-15: the allpass's gain, delay, maximum delay
    3.1415927f, 0.2f, 0.25f,     // 16-18: the tremolo's radians per quarter note, its depth, CC 73 depth
    2.f, 48.f, 0.03f,            // 19-21: pitch bend, MPE pitch bend (semitones), glide (seconds)
    0.3f,                        // 22: the level of the feedback tap read before the base call
};
inline float fxp(int i) { return kFxParams[i]; }

class FxSynth : public Synth
{
 public:
  explicit FxSynth(int nVoices) : Synth(nVoices) {}

  SineGen osc[16];
  ADSR env[16];
  Lopass tone;                  // per instrument
  FractionalDelay delay;
  Allpass<IntegerDelay> diffuser;
  DSPVector fb;                 // carried between vectors
  float sr = 48000.f;

  void init(float sampleRate)
  {
    sr = sampleRate;
    for (int v = 0; v < 16; ++v)
    {
      osc[v].clear();
      env[v].coeffs = ADSR::calcCoeffs(fxp(0), fxp(1), fxp(2), fxp(3), sampleRate);
    }
    tone.coeffs = Lopass::makeCoeffs(fxp(8), fxp(9));
    delay.setMaxDelayInSamples(fxp(11));
    delay.setDelayInSamples(fxp(10));
    diffuser.mGain = fxp(13);
    diffuser.setMaxDelayInSamples(fxp(15));
    diffuser.setDelayInSamples(fxp(14));
  }

  void processVoice(int voiceIndex, const EventsToSignals::Voice& voice, const DSPVectorDynamic& inputs,
                    DSPVectorDynamic& outputs, AudioContext* ctx) override
  {
    const int v = voiceIndex;
    DSPVector cps = exp2(voice.outputs.constRow(kPitch) - fxp(4)) * (fxp(5) / sr) * (1.f + fxp(6) * (float)v);
    DSPVector y = osc[v](cps) * env[v](voice.outputs.constRow(kGate));
    DSPVector c1 = ctx->getInputController(1);
    outputs[0] += y * (c1 * fxp(7) + 1.f);
    outputs[1] += y * voice.outputs.constRow(kZ);
  }

  void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* state) override
  {
    auto* ctx = static_cast<AudioContext*>(state);
    DSPVector pre = ctx->getInputController(73) * fxp(18) + 1.f;
    DSPVector tap = fb * fxp(22);  // the carried member, read before the base call: last vector's delay output
    DSPVectorDynamic dry(2);
    Synth::processVector(inputs, dry, state);  // the voice sum, exactly once
    DSPVector wet = ctx->getInputController(74);
    DSPVector c1 = ctx->getInputController(1);
    fb = delay(tone(dry[0] + fb * fxp(12)));
    outputs[0] = dry[0] * pre + diffuser(fb) * wet * (c1 + 1.f);
    outputs[1] = dry[1] * (sin(ctx->getBeatPhase() * fxp(16)) * fxp(17) + 1.f) + tap;
    outputs[2] = dry[0];
  }
};

// The instrument's setup.  variant 0: MIDI; 1: MPE.  Both glide; neither drifts.
template <class CTX>
inline void fxSynthSetup(CTX& ctx, FxSynth& synth, int variant)
{
  ctx.setInputProtocol(Symbol(variant == 1 ? "MPE" : "MIDI"));
  ctx.setInputPolyphony(synth.getNumVoices());
  ctx.setInputPitchBend(fxp(19));
  ctx.setInputMPEPitchBend(fxp(20));
  ctx.setInputGlideTimeInSeconds(fxp(21));
  synth.init((float)ctx.getSampleRate());
}
