// mlb200_trace.hpp -- the reference's functor / operator spelling on the host, as a TRACING layer.
//
// The reference's hot path is written by its users like this (examples/audio-and-midi/sine.cpp:21-35,
// reverb.cpp:68-123):
//
//     void process(AudioContext* ctx, void* state) {
//       auto s = static_cast<MyState*>(state);
//       ctx->outputs[0] = s->lp(s->osc(220.f / kSampleRate)) * kOutputGain;
//     }
//
// i.e. functor objects held in a state struct, called with DSPVector values, chained with operators
// (MLDSPGens.h:373-381, MLDSPFilters.h:51-153, MLDSPOps.h:337-352, MLSignalProcessBuffer.h:18,
// MLAudioContext.h:23-101).  In namespace mlb::tr the same spellings exist, but a DSPVector is SYMBOLIC:
// running the process function records the DAG of functors it applies instead of computing samples.
// The recorded graph is then compiled into one fused GPU kernel launch per call for V independent
// instances (mlb_graph_*), which is what "source/procs' runtime graph evaluator becomes a launcher"
// means in this project.  So a reference process function is ported by changing
//
//     using namespace ml;      ->      using namespace mlb::tr;
//
// and handing it to mlb::tr::TracedProcessor instead of ml::AudioTask / ml::SignalProcessBuffer.
//
// How state carried between calls is found: the process function is traced TWICE.  A DSPVector member that is
// read before it is assigned (reverb.cpp:34,114-119: mvFeedbackL) still holds, in the second pass, the symbol
// assigned at the end of the first pass; consuming such a stale symbol yields a one-block feedback edge
// (FEEDBACK_READ now, FEEDBACK_WRITE of the same expression at the end of the block).  Functor state
// (phases, filter memories, delay lines) lives on the device per instance; the host functor objects hold only
// what the caller sets before tracing (coeffs, mGain, setMaxDelayInSamples, clear(), setSeed ...).
//
// Scalars: a `float` handed to a functor or mixed with a DSPVector becomes a per-instance PARAM (the
// reference's implicit float -> DSPVector broadcast, MLDSPOps.h:157); `tr::param(name, value)` names one so
// that it can be set per instance afterwards.  Coefficient design (makeCoeffs) runs on the host through
// mlb_coeffs_* = the reference's own libm calls.
//
// A functor object called more than once in a vector -- by Upsample2xFunction<N> (MLDSPFunctional.h:114-160), which runs
// its process function twice, or in an oversampled loop between an Upsampler and a Downsampler -- ticks once per call, as
// the reference's objects do: the further calls record MLB_AGAIN nodes (mlb200.h), same functor, same state.  Functors
// with a delay ring cannot be called again (the graph is refused when trace() lays it out).
//
// Header only; link against libmlb200.so.  No sample arithmetic happens on the CPU here.
#pragma once
#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "mlb200.hpp"
#include "mlb200_host.hpp"

namespace mlb
{
namespace tr
{
// kFloatsPerDSPVector is the global constant of mlb200.hpp (global in the reference too, MLDSPMath.h:8-9)

// ------------------------------------------------------------------------------------------------------
// the recorder

struct TNode
{
  mlb_node node;
  std::vector<float> coef;      // initial value of every coef word (same for all instances until overridden)
  std::vector<uint32_t> state;  // initial value of every state word
  int opIndex = -1;             // position among the user-visible operations of one pass
  std::string name;             // named PARAMs
};

// a further call of an earlier functor (MLB_AGAIN): it owns no words of its own
inline bool isAgain(const mlb_node& n)
{
  return n.iarg < 0 && n.op != MLB_OP_INPUT && n.op != MLB_OP_PARAM && n.op != MLB_OP_FEEDBACK_WRITE;
}

class Recorder
{
 public:
  std::vector<TNode> nodes;
  std::vector<int> outs;
  int epoch = 0;
  int opCounter = 0;
  std::map<int, int> opIndexToNode;    // this pass
  std::map<int, int> feedbackReaders;  // stale opIndex -> FEEDBACK_READ node of this pass
  bool active = false;
  // a functor object called AGAIN in the same vector (allowed inside the second run of a process function by
  // Upsample2xFunction): its next node becomes a further call of its first one (MLB_AGAIN in mlb200.h)
  int repeatDepth = 0;
  int forbidFunctors = 0;       // > 0 inside a Downsample2xFunction's process function (see there)
  int pendingAgain = -1;        // node of the functor's first call in this pass
  int* pendingOwner = nullptr;  // where a functor's first call wants its node index written
  // TracedSynth::trace: the voice being traced, and the voice each functor object was first called by
  int voice = -1;
  std::map<const void*, int>* functorVoice = nullptr;
  // TracedSynth::trace: the one pass whose symbols may be read stale (pass 1 of this voice, while pass 2 runs); -2:
  // none.  -1 (TracedProcessor): any earlier pass.
  int staleEpoch = -1;
  // TracedSynth::trace: the epochs of processVoice's passes, [voiceEpoch0, voiceEpoch1), and whether this recorder
  // traces the instrument section (Synth::processVector around the base call) rather than processVoice
  int voiceEpoch0 = 0, voiceEpoch1 = INT_MAX;
  bool instrument = false;

  // epochs are unique across recorders, so that a symbol of one recorder is never current in another
  static int& lastEpoch()
  {
    static thread_local int e = 0;
    return e;
  }

  static Recorder*& current()
  {
    static thread_local Recorder* r = nullptr;
    return r;
  }
  static Recorder& get()
  {
    Recorder* r = current();
    if (!r || !r->active) throw Error(MLB_ERR_INVALID, "mlb::tr: DSPVector operation outside TracedProcessor::trace()");
    return *r;
  }
  void beginPass()
  {
    epoch = ++lastEpoch();
    nodes.clear();
    outs.clear();
    opCounter = 0;
    opIndexToNode.clear();
    feedbackReaders.clear();
    repeatDepth = 0, forbidFunctors = 0, pendingAgain = -1, pendingOwner = nullptr;
    active = true;
  }
  int addNode(int op, std::initializer_list<int> ins, int iarg = 0, bool userOp = true)
  {
    int nin = 0, nst = 0, nco = 0;
    if (mlb_op_info(op, &nin, &nst, &nco) != MLB_OK) throw Error(MLB_ERR_INVALID, "mlb::tr: unknown op");
    TNode t;
    t.node.op = op;
    for (int k = 0; k < MLB_MAX_INS; ++k) t.node.in[k] = -1;
    int k = 0;
    for (int i : ins) t.node.in[k++] = i;
    if (k != nin && op != MLB_OP_FEEDBACK_WRITE) throw Error(MLB_ERR_INVALID, "mlb::tr: operand count");
    t.node.iarg = iarg;
    t.coef.assign((size_t)nco, 0.f);
    t.state.assign((size_t)nst, 0u);
    if (userOp && (nst > 0 || nco > 0) && (pendingOwner || pendingAgain >= 0))  // the node of the functor that just said once()
    {
      if (pendingAgain >= 0)
      {
        if (nodes[(size_t)pendingAgain].node.op != op)
          throw Error(MLB_ERR_UNSUPPORTED, "mlb::tr: a functor called again in a vector recorded a different operation");
        t.node.iarg = MLB_AGAIN(pendingAgain);
      }
      else
        *pendingOwner = (int)nodes.size();
      pendingAgain = -1, pendingOwner = nullptr;
    }
    if (userOp)
    {
      t.opIndex = opCounter++;
      opIndexToNode[t.opIndex] = (int)nodes.size();
    }
    nodes.push_back(t);
    return (int)nodes.size() - 1;
  }
  // After the second pass: the expression a stale symbol stood for is, in this pass, the node with the same operation
  // index; it is written back at the end of the block.  `fn` names the traced function in the error.
  void closeFeedback(const std::string& fn)
  {
    for (const auto& fr : feedbackReaders)
    {
      auto it = opIndexToNode.find(fr.first);
      if (it == opIndexToNode.end()) throw Error(MLB_ERR_INVALID, ("mlb::tr: " + fn + " is not deterministic between calls").c_str());
      addNode(MLB_OP_FEEDBACK_WRITE, {it->second}, fr.second, false);
    }
  }
};

// ------------------------------------------------------------------------------------------------------
// DSPVector: a symbolic row

class DSPVector
{
 public:
  enum Kind
  {
    kConst,
    kNode
  };
  Kind kind = kConst;
  float k = 0.f;  // kConst: the broadcast value (default-constructed = zero filled, MLDSPOps.h:153)
  int epoch = 0, node = -1, opIndex = -1;

  DSPVector() = default;
  DSPVector(float v) : kind(kConst), k(v) {}  // implicit, like the reference's DSPVectorArray(float)
  DSPVector(double v) : kind(kConst), k((float)v) {}
  DSPVector(int v) : kind(kConst), k((float)v) {}
  DSPVector(size_t v) : kind(kConst), k((float)v) {}
  static DSPVector ofNode(int n)
  {
    Recorder& r = Recorder::get();
    DSPVector d;
    d.kind = kNode, d.epoch = r.epoch, d.node = n, d.opIndex = r.nodes[(size_t)n].opIndex;
    return d;
  }
  // node index of this row in the pass being recorded (constants become PARAMs, stale symbols feedback reads)
  int resolve() const
  {
    Recorder& r = Recorder::get();
    if (kind == kConst)
    {
      const int n = r.addNode(MLB_OP_PARAM, {}, 0, false);
      r.nodes[(size_t)n].coef[0] = k;
      return n;
    }
    if (epoch == r.epoch) return node;
    // a symbol of the previous pass: state the caller keeps between process calls
    if (r.staleEpoch != -1)
    {
      const bool ofVoice = epoch >= r.voiceEpoch0 && epoch < r.voiceEpoch1;
      if (r.instrument)
      {
        if (ofVoice)
          throw Error(MLB_ERR_UNSUPPORTED,
                      "mlb::tr::TracedSynth: Synth::processVector reads, outside the base Synth::processVector call, a "
                      "DSPVector made in processVoice (a Voice& kept past the call, or a voice's member); the instrument "
                      "section sees the voices only through the bus rows the base call leaves in its outputs");
        if (epoch != r.staleEpoch)
          throw Error(MLB_ERR_UNSUPPORTED,
                      "mlb::tr::TracedSynth: Synth::processVector reads a DSPVector made before this trace");
        if (opIndex < 0)
          throw Error(MLB_ERR_UNSUPPORTED,
                      "mlb::tr::TracedSynth: Synth::processVector carries a bus row, controller, beat phase or tr::param "
                      "between vectors as it stands; carry an expression of it (e.g. row * 1.f)");
      }
      else if (!ofVoice)
        throw Error(MLB_ERR_UNSUPPORTED,
                    ("mlb::tr::TracedSynth: voice " + std::to_string(r.voice) +
                     " reads a DSPVector made outside processVoice (before the base Synth::processVector call, or by "
                     "the instrument section); processVoice may read only its own rows, controllers and members")
                        .c_str());
      // a voice's own member is written only in its own two passes; anything older was written by another voice
      else if (epoch != r.staleEpoch)
        throw Error(MLB_ERR_UNSUPPORTED,
                    ("mlb::tr::TracedSynth: voice " + std::to_string(r.voice) +
                     " reads a DSPVector of another voice (a member shared between voices, or another voice's Voice "
                     "rows); a row carried between vectors must be per voice, e.g. DSPVector carried[16]")
                        .c_str());
      else if (opIndex < 0)
        throw Error(MLB_ERR_UNSUPPORTED,
                    ("mlb::tr::TracedSynth: voice " + std::to_string(r.voice) +
                     " carries a Voice row, controller, beat phase or tr::param between vectors as it stands; carry "
                     "an expression of it (e.g. row * 1.f)")
                        .c_str());
    }
    auto it = r.feedbackReaders.find(opIndex);
    if (it != r.feedbackReaders.end()) return it->second;
    const int n = r.addNode(MLB_OP_FEEDBACK_READ, {}, 0, false);
    r.feedbackReaders[opIndex] = n;
    return n;
  }
};

inline DSPVector op1(int op, const DSPVector& a) { return DSPVector::ofNode(Recorder::get().addNode(op, {a.resolve()})); }
inline DSPVector op2(int op, const DSPVector& a, const DSPVector& b)
{
  const int x = a.resolve(), y = b.resolve();
  return DSPVector::ofNode(Recorder::get().addNode(op, {x, y}));
}
inline DSPVector op3(int op, const DSPVector& a, const DSPVector& b, const DSPVector& c)
{
  const int x = a.resolve(), y = b.resolve(), z = c.resolve();
  return DSPVector::ofNode(Recorder::get().addNode(op, {x, y, z}));
}

// a named per-instance scalar, broadcast like DSPVector(float); set per instance with TracedProcessor::setParam
inline DSPVector param(const char* name, float value)
{
  Recorder& r = Recorder::get();
  if (r.instrument)
    throw Error(MLB_ERR_UNSUPPORTED, (std::string("mlb::tr::TracedSynth: tr::param(") + name + ") in Synth::processVector "
                                     "outside the base call: the instrument section has no per-instrument parameters "
                                     "(TracedSynth::setParam sets the voices' only); use a float or a controller")
                                        .c_str());
  const int n = r.addNode(MLB_OP_PARAM, {}, 0, false);
  r.nodes[(size_t)n].coef[0] = value;
  r.nodes[(size_t)n].name = name;
  DSPVector d;
  d.kind = DSPVector::kNode, d.epoch = r.epoch, d.node = n, d.opIndex = -1;
  return d;
}

// operators, MLDSPOps.h:337-352, 370-388 (compound forms)
inline DSPVector operator+(const DSPVector& a, const DSPVector& b) { return op2(MLB_OP_ADD, a, b); }
inline DSPVector operator-(const DSPVector& a, const DSPVector& b) { return op2(MLB_OP_SUBTRACT, a, b); }
inline DSPVector operator*(const DSPVector& a, const DSPVector& b) { return op2(MLB_OP_MULTIPLY, a, b); }
inline DSPVector operator/(const DSPVector& a, const DSPVector& b) { return op2(MLB_OP_DIVIDE, a, b); }
inline DSPVector& operator+=(DSPVector& a, const DSPVector& b) { return a = a + b; }
inline DSPVector& operator-=(DSPVector& a, const DSPVector& b) { return a = a - b; }
inline DSPVector& operator*=(DSPVector& a, const DSPVector& b) { return a = a * b; }
inline DSPVector& operator/=(DSPVector& a, const DSPVector& b) { return a = a / b; }
inline DSPVector operator-(const DSPVector& a) { return DSPVector(0.f) - a; }  // MLDSPOps.h:354-358

#define MLB_TR_OP1(NAME, OP) \
  inline DSPVector NAME(const DSPVector& x) { return op1(OP, x); }
MLB_TR_OP1(sqrt, MLB_OP_SQRT)
MLB_TR_OP1(sqrtApprox, MLB_OP_SQRT_APPROX)
MLB_TR_OP1(abs, MLB_OP_ABS)
MLB_TR_OP1(sign, MLB_OP_SIGN)
MLB_TR_OP1(signBit, MLB_OP_SIGNBIT)
MLB_TR_OP1(sin, MLB_OP_SIN)
MLB_TR_OP1(cos, MLB_OP_COS)
MLB_TR_OP1(log, MLB_OP_LOG)
MLB_TR_OP1(exp, MLB_OP_EXP)
MLB_TR_OP1(log2, MLB_OP_LOG2)
MLB_TR_OP1(exp2, MLB_OP_EXP2)
MLB_TR_OP1(sinApprox, MLB_OP_SIN_APPROX)
MLB_TR_OP1(cosApprox, MLB_OP_COS_APPROX)
MLB_TR_OP1(expApprox, MLB_OP_EXP_APPROX)
MLB_TR_OP1(logApprox, MLB_OP_LOG_APPROX)
MLB_TR_OP1(log2Approx, MLB_OP_LOG2_APPROX)
MLB_TR_OP1(exp2Approx, MLB_OP_EXP2_APPROX)
MLB_TR_OP1(fractionalPart, MLB_OP_FRACTIONAL_PART)
#undef MLB_TR_OP1
#define MLB_TR_OP2(NAME, OP) \
  inline DSPVector NAME(const DSPVector& a, const DSPVector& b) { return op2(OP, a, b); }
MLB_TR_OP2(add, MLB_OP_ADD)
MLB_TR_OP2(subtract, MLB_OP_SUBTRACT)
MLB_TR_OP2(multiply, MLB_OP_MULTIPLY)
MLB_TR_OP2(divide, MLB_OP_DIVIDE)
MLB_TR_OP2(divideApprox, MLB_OP_DIVIDE_APPROX)
MLB_TR_OP2(pow, MLB_OP_POW)
MLB_TR_OP2(powApprox, MLB_OP_POW_APPROX)
MLB_TR_OP2(min, MLB_OP_MIN)
MLB_TR_OP2(max, MLB_OP_MAX)
#undef MLB_TR_OP2
inline DSPVector lerp(const DSPVector& a, const DSPVector& b, const DSPVector& m) { return op3(MLB_OP_LERP, a, b, m); }
inline DSPVector inverseLerp(const DSPVector& a, const DSPVector& b, const DSPVector& m) { return op3(MLB_OP_INVERSE_LERP, a, b, m); }
inline DSPVector clamp(const DSPVector& x, const DSPVector& lo, const DSPVector& hi) { return op3(MLB_OP_CLAMP, x, lo, hi); }
// interpolateDSPVectorLinear(start, end), MLDSPOps.h:986-990
inline DSPVector interpolateDSPVectorLinear(const DSPVector& start, const DSPVector& end) { return op2(MLB_OP_RAMP, start, end); }

// DSPVectorInt: a row of int32 (MLDSPOps.h:370-498).  On the device a row is 64 words either way; the type only says
// how the words are read, as in the reference (whose int and float vectors share their storage layout).
class DSPVectorInt
{
 public:
  DSPVector bits;  // the symbolic row
  DSPVectorInt() : bits(intAsFloat(0)) {}
  explicit DSPVectorInt(int32_t k) : bits(intAsFloat(k)) {}
  static float intAsFloat(int32_t k)
  {
    float f;
    std::memcpy(&f, &k, 4);
    return f;
  }
  static DSPVectorInt of(const DSPVector& d)
  {
    DSPVectorInt y;
    y.bits = d;
    return y;
  }
};
// conversions, MLDSPOps.h:780-820
inline DSPVectorInt roundFloatToInt(const DSPVector& x) { return DSPVectorInt::of(op1(MLB_OP_ROUND_F2I, x)); }
inline DSPVectorInt truncateFloatToInt(const DSPVector& x) { return DSPVectorInt::of(op1(MLB_OP_TRUNC_F2I, x)); }
inline DSPVector intToFloat(const DSPVectorInt& x) { return op1(MLB_OP_INT_TO_FLOAT, x.bits); }
inline DSPVector unsignedIntToFloat(const DSPVectorInt& x) { return op1(MLB_OP_UNSIGNED_TO_FLOAT, x.bits); }
// int arithmetic, MLDSPOps.h:713-714
inline DSPVectorInt addInt32(const DSPVectorInt& a, const DSPVectorInt& b) { return DSPVectorInt::of(op2(MLB_OP_ADD_INT32, a.bits, b.bits)); }
inline DSPVectorInt subtractInt32(const DSPVectorInt& a, const DSPVectorInt& b) { return DSPVectorInt::of(op2(MLB_OP_SUBTRACT_INT32, a.bits, b.bits)); }
// comparisons give all-ones / all-zeros masks, MLDSPOps.h:851-856
#define MLB_TR_CMP(NAME, OP) \
  inline DSPVectorInt NAME(const DSPVector& a, const DSPVector& b) { return DSPVectorInt::of(op2(OP, a, b)); }
MLB_TR_CMP(equal, MLB_OP_EQUAL)
MLB_TR_CMP(notEqual, MLB_OP_NOT_EQUAL)
MLB_TR_CMP(greaterThan, MLB_OP_GREATER_THAN)
MLB_TR_CMP(greaterThanOrEqual, MLB_OP_GREATER_EQUAL)
MLB_TR_CMP(lessThan, MLB_OP_LESS_THAN)
MLB_TR_CMP(lessThanOrEqual, MLB_OP_LESS_EQUAL)
#undef MLB_TR_CMP
// bitwise select(resultIfTrue, resultIfFalse, mask), float and int forms, MLDSPOps.h:886,917
inline DSPVector select(const DSPVector& a, const DSPVector& b, const DSPVectorInt& m) { return op3(MLB_OP_SELECT, a, b, m.bits); }
inline DSPVectorInt select(const DSPVectorInt& a, const DSPVectorInt& b, const DSPVectorInt& m)
{
  return DSPVectorInt::of(op3(MLB_OP_SELECT, a.bits, b.bits, m.bits));
}
// within(x, lo, hi): is x in [lo, hi) -- a mask in a float row, MLDSPOps.h:748
inline DSPVector within(const DSPVector& x, const DSPVector& lo, const DSPVector& hi) { return op3(MLB_OP_WITHIN, x, lo, hi); }

// DSPVectorArray<ROWS>: ROWS symbolic rows (MLDSPOps.h:94-353); rowwise use only
template <size_t ROWS>
class DSPVectorArray
{
  std::array<DSPVector, ROWS> rows_;

 public:
  DSPVectorArray() = default;
  DSPVectorArray(float k) { rows_.fill(DSPVector(k)); }
  DSPVector& row(int j) { return rows_[(size_t)j]; }
  const DSPVector& constRow(int j) const { return rows_[(size_t)j]; }
};
template <size_t A, size_t B>
inline DSPVectorArray<A + B> concatRows(const DSPVectorArray<A>& a, const DSPVectorArray<B>& b)
{
  DSPVectorArray<A + B> y;
  for (size_t i = 0; i < A; ++i) y.row((int)i) = a.constRow((int)i);
  for (size_t i = 0; i < B; ++i) y.row((int)(A + i)) = b.constRow((int)i);
  return y;
}
inline DSPVectorArray<2> concatRows(const DSPVector& a, const DSPVector& b)
{
  DSPVectorArray<2> y;
  y.row(0) = a, y.row(1) = b;
  return y;
}
// ---- DSPVectorArray<ROWS> as a value: rowwise arithmetic, MLDSPOps.h:337-358 ----
#define MLB_TR_ARRAY_OP(SYM, OP)                                                                              \
  template <size_t ROWS>                                                                                      \
  inline DSPVectorArray<ROWS> operator SYM(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b)      \
  {                                                                                                           \
    DSPVectorArray<ROWS> y;                                                                                   \
    for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = op2(OP, a.constRow((int)j), b.constRow((int)j));        \
    return y;                                                                                                 \
  }                                                                                                           \
  template <size_t ROWS>                                                                                      \
  inline DSPVectorArray<ROWS>& operator SYM##=(DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b)        \
  {                                                                                                           \
    return a = a SYM b;                                                                                       \
  }
MLB_TR_ARRAY_OP(+, MLB_OP_ADD)
MLB_TR_ARRAY_OP(-, MLB_OP_SUBTRACT)
MLB_TR_ARRAY_OP(*, MLB_OP_MULTIPLY)
MLB_TR_ARRAY_OP(/, MLB_OP_DIVIDE)
#undef MLB_TR_ARRAY_OP

// the "1" forms, MLDSPOps.h:678-687: the second operand is ONE row, used for every row of the first
#define MLB_TR_ARRAY_OP1(NAME, OP)                                                               \
  template <size_t ROWS>                                                                         \
  inline DSPVectorArray<ROWS> NAME(const DSPVectorArray<ROWS>& a, const DSPVector& b)            \
  {                                                                                              \
    DSPVectorArray<ROWS> y;                                                                      \
    for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = op2(OP, a.constRow((int)j), b);            \
    return y;                                                                                    \
  }
MLB_TR_ARRAY_OP1(add1, MLB_OP_ADD)
MLB_TR_ARRAY_OP1(subtract1, MLB_OP_SUBTRACT)
MLB_TR_ARRAY_OP1(multiply1, MLB_OP_MULTIPLY)
MLB_TR_ARRAY_OP1(divide1, MLB_OP_DIVIDE)
MLB_TR_ARRAY_OP1(divideApprox1, MLB_OP_DIVIDE_APPROX)
MLB_TR_ARRAY_OP1(pow1, MLB_OP_POW)
MLB_TR_ARRAY_OP1(powApprox1, MLB_OP_POW_APPROX)
MLB_TR_ARRAY_OP1(min1, MLB_OP_MIN)
MLB_TR_ARRAY_OP1(max1, MLB_OP_MAX)
#undef MLB_TR_ARRAY_OP1
// lerp of two arrays with one scalar mixture, MLDSPOps.h:753-775
template <size_t ROWS>
inline DSPVectorArray<ROWS> lerp(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b, float m)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = lerp(a.constRow((int)j), b.constRow((int)j), DSPVector(m));
  return y;
}

// ---- row operations, MLDSPOps.h:1056-1359: pure rearrangements of the symbolic rows (no nodes), except addRows ----
// output row j = input row src(j), or a zero row where src(j) < 0
template <size_t OUT, size_t N, class F>
inline DSPVectorArray<OUT> mapRows(const DSPVectorArray<N>& x, F src)
{
  DSPVectorArray<OUT> y;
  for (size_t j = 0; j < OUT; ++j)
  {
    const int k = src((int)j);
    y.row((int)j) = (k >= 0 && k < (int)N) ? x.constRow(k) : DSPVector(0.f);
  }
  return y;
}
template <size_t ROWS, size_t N>
inline DSPVectorArray<ROWS * N> repeatRows(const DSPVectorArray<N>& x)  // the N rows over and over
{
  return mapRows<ROWS * N>(x, [](int j) { return j % (int)N; });
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> repeatRows(const DSPVector& x)  // (a DSPVector is a one-row array in the reference)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = x;
  return y;
}
template <size_t ROWS, size_t N>
inline DSPVectorArray<ROWS> stretchRows(const DSPVectorArray<N>& x)  // nearest input row for every output row
{
  return mapRows<ROWS>(x, [](int j) { return (int)roundf((j * ((float)N - 1.f)) / ((float)ROWS - 1.f)); });
}
template <size_t ROWS, size_t N>
inline DSPVectorArray<ROWS> zeroPadRows(const DSPVectorArray<N>& x)
{
  return mapRows<ROWS>(x, [](int j) { return j < (int)N ? j : -1; });
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> shiftRows(const DSPVectorArray<ROWS>& x, int rowsToShift)  // zeros come in from outside
{
  return mapRows<ROWS>(x, [=](int j) { const int k = j - rowsToShift; return (k >= 0 && k < (int)ROWS) ? k : -1; });
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> rotateRows(const DSPVectorArray<ROWS>& x, int rowsToRotate)
{
  return mapRows<ROWS>(x, [=](int j) { const int m = (int)ROWS; return (((j - rowsToRotate) % m) + m) % m; });
}
template <size_t A, size_t B>
inline DSPVectorArray<A + B> shuffleRows(const DSPVectorArray<A>& a, const DSPVectorArray<B>& b)  // a0 b0 a1 b1 ..., then the rest
{
  DSPVectorArray<A + B> y;
  size_t ja = 0, jb = 0, jy = 0;
  while (ja < A || jb < B)
  {
    if (ja < A) y.row((int)jy++) = a.constRow((int)ja++);
    if (jb < B) y.row((int)jy++) = b.constRow((int)jb++);
  }
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<(ROWS + 1) / 2> evenRows(const DSPVectorArray<ROWS>& x)
{
  return mapRows<(ROWS + 1) / 2>(x, [](int j) { return 2 * j; });
}
template <size_t ROWS>
inline DSPVectorArray<ROWS / 2> oddRows(const DSPVectorArray<ROWS>& x)
{
  return mapRows<ROWS / 2>(x, [](int j) { return 2 * j + 1; });
}
template <size_t A, size_t B, size_t ROWS>
inline DSPVectorArray<B - A> separateRows(const DSPVectorArray<ROWS>& x)  // rows [A, B)
{
  static_assert(B <= ROWS && A < ROWS, "separateRows: range out of bounds");
  return mapRows<B - A>(x, [](int j) { return j + (int)A; });
}
template <size_t ROWS>
inline DSPVector addRows(const DSPVectorArray<ROWS>& x)  // from a zero row, left to right (MLDSPOps.h:1349-1359)
{
  DSPVector y(0.f);
  for (size_t j = 0; j < ROWS; ++j) y = add(y, x.constRow((int)j));
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> rowIndex()  // row j filled with j
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = DSPVector((float)j);
  return y;
}
// columnIndex() = 0, 1, ... 63: exactly interpolateDSPVectorLinear(-1, 63) (interval 1, first value -1 + 1);
// rangeOpen / rangeClosed as the reference composes them from it (MLDSPOps.h:965-982)
inline DSPVector columnIndex() { return interpolateDSPVectorLinear(-1.f, 63.f); }
template <size_t ROWS>
inline DSPVectorArray<ROWS> columnIndex()
{
  return repeatRows<ROWS>(columnIndex());
}
inline DSPVector rangeOpen(float start, float end)
{
  const float interval = (end - start) / (float)kFloatsPerDSPVector;
  return columnIndex() * DSPVector(interval) + DSPVector(start);
}
inline DSPVector rangeClosed(float start, float end)
{
  const float interval = (end - start) / ((float)kFloatsPerDSPVector - 1.f);
  return columnIndex() * DSPVector(interval) + DSPVector(start);
}

// interpolateCoeffsLinear, MLDSPFilters.h:32-44
template <size_t N>
inline DSPVectorArray<N> interpolateCoeffsLinear(const std::array<float, N> c0, const std::array<float, N> c1)
{
  DSPVectorArray<N> vy;
  for (size_t i = 0; i < N; ++i) vy.row((int)i) = interpolateDSPVectorLinear(c0[i], c1[i]);
  return vy;
}

// ------------------------------------------------------------------------------------------------------
// functors.  Each object records ONE node per pass, the first time it is called.

class Functor
{
 protected:
  int lastEpoch_ = 0;
  int firstNode_ = -1;  // the node this object recorded when it was first called in the current pass
  void once()
  {
    Recorder& r = Recorder::get();
    if (r.forbidFunctors > 0)
      throw Error(MLB_ERR_UNSUPPORTED,
                  "mlb::tr: the process function of a Downsample2xFunction must be stateless (its functors would have to "
                  "tick on every second vector only)");
    if (r.functorVoice)
    {
      // in the reference one object shared by two voices ticks once per voice and vector; each lane here has its own
      auto it = r.functorVoice->emplace(this, r.voice).first;
      if (it->second != r.voice && (it->second < 0 || r.voice < 0))  // -1: the instrument section
        throw Error(MLB_ERR_UNSUPPORTED, ("mlb::tr: a functor object is called by voice " +
                                          std::to_string(std::max(it->second, r.voice)) + " and by the instrument "
                                          "section of Synth::processVector; each needs its own")
                                             .c_str());
      if (it->second != r.voice)
        throw Error(MLB_ERR_UNSUPPORTED, ("mlb::tr: a functor object is called by voice " + std::to_string(it->second) +
                                          " and voice " + std::to_string(r.voice) + "; each voice needs its own")
                                             .c_str());
    }
    if (lastEpoch_ == r.epoch)
    {
      // called again in the same vector: the reference object would simply tick once more (a process function run twice
      // by Upsample2xFunction, MLDSPFunctional.h:138-140; an oversampled loop between an Upsampler and a Downsampler).
      // Recorded as a further call of the first node (MLB_AGAIN); a functor with a delay ring cannot be -- trace()
      // reports that when it lays the graph out.
      if (firstNode_ < 0) throw Error(MLB_ERR_UNSUPPORTED, "mlb::tr: this object cannot be called again in the same vector");
      r.pendingAgain = firstNode_, r.pendingOwner = nullptr;
      return;
    }
    lastEpoch_ = r.epoch;
    firstNode_ = -1;
    r.pendingOwner = &firstNode_, r.pendingAgain = -1;
  }
  static TNode& nodeOf(const DSPVector& d) { return Recorder::get().nodes[(size_t)d.node]; }
};

inline float dBToGain(float dB) { return mlb_db_to_gain(dB); }  // MLDSPFilters.h:30

// ---- generators, MLDSPGens.h ----
class NoiseGen : public Functor
{
  uint32_t seed_ = 0;

 public:
  void setSeed(uint32_t s) { seed_ = s; }
  void reset() { seed_ = 0; }
  DSPVector operator()()
  {
    once();
    DSPVector y = DSPVector::ofNode(Recorder::get().addNode(MLB_OP_NOISE, {}));
    nodeOf(y).state[0] = seed_;
    return y;
  }
};
template <int OP>
class PhaseGen : public Functor
{
 protected:
  uint32_t omega32_ = 0;

 public:
  DSPVector operator()(const DSPVector& cyclesPerSample)
  {
    once();
    DSPVector y = op1(OP, cyclesPerSample);
    nodeOf(y).state[0] = omega32_;
    return y;
  }
};
class PhasorGen : public PhaseGen<MLB_OP_PHASOR>
{
 public:
  void clear(uint32_t omega = 0) { omega32_ = omega; }  // MLDSPGens.h:182
};
class SineGen : public PhaseGen<MLB_OP_SINE>
{
 public:
  void clear() { omega32_ = 0xC0000000u; }  // kZeroPhase = -(2 << 29), MLDSPGens.h:375-379
};
class SawGen : public PhaseGen<MLB_OP_SAW>
{
 public:
  void clear() { omega32_ = 0; }
};
class PulseGen : public Functor
{
  uint32_t omega32_ = 0;

 public:
  void clear() { omega32_ = 0; }
  DSPVector operator()(const DSPVector& freq, const DSPVector& width)
  {
    once();
    DSPVector y = op2(MLB_OP_PULSE, freq, width);
    nodeOf(y).state[0] = omega32_;
    return y;
  }
};
class TickGen : public Functor
{
 public:
  DSPVector operator()(const DSPVector& cyclesPerSample)
  {
    once();
    return op1(MLB_OP_TICK, cyclesPerSample);
  }
};
class ImpulseGen : public Functor
{
 public:
  DSPVector operator()(const DSPVector& cyclesPerSample)
  {
    once();
    return op1(MLB_OP_IMPULSE, cyclesPerSample);
  }
};
class OneShotGen : public Functor
{
  bool triggered_ = false;

 public:
  void trigger() { triggered_ = true; }  // MLDSPGens.h:229-233: {mOmega32 0, mGate 1, mOmegaPrev 0}
  DSPVector operator()(const DSPVector& cyclesPerSample)
  {
    once();
    DSPVector y = op1(MLB_OP_ONESHOT, cyclesPerSample);
    if (triggered_) nodeOf(y).state[1] = 1u;
    return y;
  }
};

// ---- SVF family, MLDSPFilters.h:51-442 ----
template <int OP, size_t NC>
class FixedFilter : public Functor
{
 public:
  typedef std::array<float, NC> Coeffs;
  Coeffs coeffs{};
  void clear() {}
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(OP, vx);
    for (size_t i = 0; i < NC; ++i) nodeOf(y).coef[i] = coeffs[i];
    return y;
  }
};
class Lopass : public FixedFilter<MLB_OP_LOPASS, 3>
{
 public:
  typedef DSPVectorArray<3> coeffsVec;
  static Coeffs makeCoeffs(float omega, float k)
  {
    Coeffs c;
    mlb_coeffs_lopass(omega, k, c.data());
    return c;
  }
  using FixedFilter<MLB_OP_LOPASS, 3>::operator();
  // operator()(vx, omega, k), MLDSPFilters.h:136-152: the coefficients are designed per sample.  On the device
  // that is LOPASS_MOD (CUDA sinf instead of glibc's: the stated-tolerance variant, DESIGN.md 5); for
  // bit-exactness design the rows on the host (mlb_coeffs_lopass_vec) and use operator()(vx, coeffsVec).
  DSPVector operator()(const DSPVector& vx, const DSPVector& omega, const DSPVector& k)
  {
    once();
    return op3(MLB_OP_LOPASS_MOD, vx, omega, k);
  }
  // coefficient ROWS g0, g1, g2 (what makeCoeffsVec returns), MLDSPFilters.h:141-149
  DSPVector operator()(const DSPVector& vx, const coeffsVec& vc)
  {
    once();
    const int x = vx.resolve(), a = vc.constRow(0).resolve(), b = vc.constRow(1).resolve(), c = vc.constRow(2).resolve();
    return DSPVector::ofNode(Recorder::get().addNode(MLB_OP_LOPASS_V, {x, a, b, c}));
  }
};
class Hipass : public FixedFilter<MLB_OP_HIPASS, 4>
{
 public:
  static Coeffs makeCoeffs(float omega, float k)
  {
    Coeffs c;
    mlb_coeffs_hipass(omega, k, c.data());
    return c;
  }
};
class Bandpass : public FixedFilter<MLB_OP_BANDPASS, 3>
{
 public:
  static Coeffs makeCoeffs(float omega, float k)
  {
    Coeffs c;
    mlb_coeffs_bandpass(omega, k, c.data());
    return c;
  }
};
class LoShelf : public FixedFilter<MLB_OP_LOSHELF, 5>
{
 public:
  typedef std::array<float, 3> params;  // omega, k, A
  typedef DSPVectorArray<5> _vcoeffs;
  static Coeffs makeCoeffs(params p)
  {
    Coeffs c;
    mlb_coeffs_loshelf(p[0], p[1], p[2], c.data());
    return c;
  }
  static _vcoeffs vcoeffs(const params p0, const params p1) { return interpolateCoeffsLinear<5>(makeCoeffs(p0), makeCoeffs(p1)); }
  using FixedFilter<MLB_OP_LOSHELF, 5>::operator();
  DSPVector operator()(const DSPVector& vx, const _vcoeffs& vc)  // MLDSPFilters.h:304-319
  {
    once();
    int in[6] = {vx.resolve(), 0, 0, 0, 0, 0};
    for (int i = 0; i < 5; ++i) in[1 + i] = vc.constRow(i).resolve();
    return DSPVector::ofNode(Recorder::get().addNode(MLB_OP_LOSHELF_V, {in[0], in[1], in[2], in[3], in[4], in[5]}));
  }
};
class HiShelf : public FixedFilter<MLB_OP_HISHELF, 6>
{
 public:
  typedef std::array<float, 3> params;
  typedef DSPVectorArray<6> _vcoeffs;
  static Coeffs makeCoeffs(params p)
  {
    Coeffs c;
    mlb_coeffs_hishelf(p[0], p[1], p[2], c.data());
    return c;
  }
  static _vcoeffs vcoeffs(const params p0, const params p1) { return interpolateCoeffsLinear<6>(makeCoeffs(p0), makeCoeffs(p1)); }
  using FixedFilter<MLB_OP_HISHELF, 6>::operator();
  DSPVector operator()(const DSPVector& vx, const _vcoeffs& vc)  // MLDSPFilters.h:385-400
  {
    once();
    int in[7] = {vx.resolve(), 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 6; ++i) in[1 + i] = vc.constRow(i).resolve();
    return DSPVector::ofNode(Recorder::get().addNode(MLB_OP_HISHELF_V, {in[0], in[1], in[2], in[3], in[4], in[5], in[6]}));
  }
};
class Bell : public FixedFilter<MLB_OP_BELL, 4>
{
 public:
  static Coeffs makeCoeffs(float omega, float k, float A)
  {
    Coeffs c;
    mlb_coeffs_bell(omega, k, A, c.data());
    return c;
  }
};
class OnePole : public FixedFilter<MLB_OP_ONEPOLE, 2>
{
 public:
  static Coeffs makeCoeffs(float omega)
  {
    Coeffs c;
    mlb_coeffs_onepole(omega, c.data());
    return c;
  }
  static Coeffs passthru() { return {1.f, 0.f}; }
};
class DCBlocker : public FixedFilter<MLB_OP_DCBLOCKER, 1>
{
 public:
  static Coeffs makeCoeffs(float omega) { return {mlb_coeffs_dcblocker(omega)}; }
};
class Differentiator : public FixedFilter<MLB_OP_DIFFERENTIATOR, 0>
{
};
class Integrator : public Functor
{
 public:
  float mLeak = 0.f;  // MLDSPFilters.h:544
  void setLeak(float k) { mLeak = k; }
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_INTEGRATOR, vx);
    nodeOf(y).coef[0] = mLeak;
    return y;
  }
};
class Peak : public Functor
{
 public:
  typedef std::array<float, 2> Coeffs;
  Coeffs coeffs{};
  int peakHoldSamples = 44100;  // MLDSPFilters.h:574
  static Coeffs makeCoeffs(float omega)
  {
    Coeffs c;
    mlb_coeffs_peak(omega, c.data());
    return c;
  }
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_PEAK, vx);
    nodeOf(y).coef[0] = coeffs[0], nodeOf(y).coef[1] = coeffs[1], nodeOf(y).coef[2] = (float)peakHoldSamples;
    return y;
  }
};
class RMS : public FixedFilter<MLB_OP_RMS, 2>
{
 public:
  static Coeffs makeCoeffs(float omega)
  {
    Coeffs c;
    mlb_coeffs_rms(omega, c.data());
    return c;
  }
};
class ADSR : public FixedFilter<MLB_OP_ADSR, 4>
{
 public:
  static Coeffs calcCoeffs(float a, float d, float s, float r, float sr)
  {
    Coeffs c;
    mlb_coeffs_adsr(a, d, s, r, sr, c.data());
    return c;
  }
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_ADSR, vx);
    for (size_t i = 0; i < 4; ++i) nodeOf(y).coef[i] = coeffs[i];
    nodeOf(y).state[7] = 4u;  // segment{off}, MLDSPFilters.h:694
    return y;
  }
};
class Allpass1 : public FixedFilter<MLB_OP_ALLPASS1, 1>
{
 public:
  Allpass1() = default;
  Allpass1(float a) { coeffs = {a}; }  // the reference's only constructor, MLDSPFilters.h:927
  static Coeffs makeCoeffs(float d) { return {mlb_coeffs_allpass1(d)}; }
};

// ---- smoothers, MLDSPGens.h:412-590 ----
class LinearGlide : public Functor
{
  float vectorsPerGlide_ = 32.f, dyPerVector_ = 1.f / 32.f;  // MLDSPGens.h:437-439

 public:
  void setGlideTimeInSamples(float t)
  {
    float c[2];
    mlb_coeffs_glide(t, c);
    vectorsPerGlide_ = c[0], dyPerVector_ = c[1];
  }
  DSPVector operator()(const DSPVector& f)  // the reference takes a float: sample 0 of the operand is used
  {
    once();
    DSPVector y = op1(MLB_OP_GLIDE, f);
    nodeOf(y).coef[0] = vectorsPerGlide_, nodeOf(y).coef[1] = dyPerVector_;
    nodeOf(y).state[2] = 0xFFFFFFFFu;  // mVectorsRemaining{-1}, MLDSPGens.h:440
    return y;
  }
};
class SampleAccurateLinearGlide : public Functor
{
  float samplesPerGlide_ = 32.f, dyPerSample_ = 1.f / 32.f;

 public:
  void setGlideTimeInSamples(float t)
  {
    float c[2];
    mlb_coeffs_sample_glide(t, c);
    samplesPerGlide_ = c[0], dyPerSample_ = c[1];
  }
  DSPVector operator()(const DSPVector& target)  // nextSample(target[n]) for every sample
  {
    once();
    DSPVector y = op1(MLB_OP_SAMPLE_GLIDE, target);
    nodeOf(y).coef[0] = samplesPerGlide_, nodeOf(y).coef[1] = dyPerSample_;
    nodeOf(y).state[3] = 0xFFFFFFFFu;
    return y;
  }
};
class Interpolator1 : public Functor
{
 public:
  DSPVector operator()(const DSPVector& f)
  {
    once();
    return op1(MLB_OP_INTERPOLATOR1, f);
  }
};

// ---- delays, MLDSPFilters.h:803-1155 ----
class IntegerDelay : public Functor
{
  float maxDelay_ = 0.f, delay_ = 0.f;

 public:
  IntegerDelay() = default;
  IntegerDelay(int d) { setMaxDelayInSamples((float)d), setDelayInSamples(d); }
  void setMaxDelayInSamples(float d) { maxDelay_ = d; }
  void setDelayInSamples(int d) { delay_ = (float)d; }
  void clear() {}
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_INTEGER_DELAY, vx);
    nodeOf(y).coef[0] = delay_, nodeOf(y).coef[1] = maxDelay_;
    return y;
  }
  DSPVector operator()(const DSPVector& vx, const DSPVector& vDelay)
  {
    once();
    DSPVector y = op2(MLB_OP_INTEGER_DELAY_VAR, vx, vDelay);
    nodeOf(y).coef[0] = maxDelay_;
    return y;
  }
};
class FractionalDelay : public Functor
{
  float maxDelay_ = 0.f, delay_ = 0.f;

 public:
  void setMaxDelayInSamples(float d) { maxDelay_ = d; }
  void setDelayInSamples(float d) { delay_ = d; }
  void clear() {}
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_FRACTIONAL_DELAY, vx);
    nodeOf(y).coef[0] = delay_, nodeOf(y).coef[1] = maxDelay_;
    return y;
  }
  DSPVector operator()(const DSPVector& vx, const DSPVector& vDelay)
  {
    once();
    DSPVector y = op2(MLB_OP_FRACTIONAL_DELAY_VAR, vx, vDelay);
    nodeOf(y).coef[0] = maxDelay_;
    return y;
  }
};
class PitchbendableDelay : public Functor
{
  float maxDelay_ = 0.f;

 public:
  void setMaxDelayInSamples(float d) { maxDelay_ = d; }
  float maxDelay() const { return maxDelay_; }
  void clear() {}
  DSPVector operator()(const DSPVector& vx, const DSPVector& vDelay)
  {
    once();
    DSPVector y = op2(MLB_OP_PITCHBEND_DELAY, vx, vDelay);
    nodeOf(y).coef[0] = maxDelay_;
    return y;
  }
};
// Allpass<DELAY_TYPE>, MLDSPFilters.h:1111-1155
template <typename DELAY_TYPE>
class Allpass;
template <>
class Allpass<PitchbendableDelay> : public Functor
{
  float maxDelay_ = 0.f;

 public:
  float mGain = 0.f;
  void setMaxDelayInSamples(float d) { maxDelay_ = d; }
  void clear() {}
  DSPVector operator()(const DSPVector& vx, const DSPVector& vDelay)
  {
    once();
    DSPVector y = op2(MLB_OP_ALLPASS_PB, vx, vDelay);
    nodeOf(y).coef[0] = mGain, nodeOf(y).coef[1] = maxDelay_;
    return y;
  }
};
template <>
class Allpass<IntegerDelay> : public Functor
{
  float maxDelay_ = 0.f, delay_ = 0.f;

 public:
  float mGain = 0.f;
  void setMaxDelayInSamples(float d) { maxDelay_ = d; }
  void setDelayInSamples(float d) { delay_ = d; }
  void clear() {}
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_ALLPASS_INT, vx);
    nodeOf(y).coef[0] = mGain, nodeOf(y).coef[1] = delay_, nodeOf(y).coef[2] = maxDelay_;
    return y;
  }
};
template <>
class Allpass<FractionalDelay> : public Functor
{
  float maxDelay_ = 0.f, delay_ = 0.f;

 public:
  float mGain = 0.f;
  void setMaxDelayInSamples(float d) { maxDelay_ = d; }
  void setDelayInSamples(float d) { delay_ = d; }
  void clear() {}
  DSPVector operator()(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_ALLPASS_FRAC, vx);
    nodeOf(y).coef[0] = mGain, nodeOf(y).coef[1] = delay_, nodeOf(y).coef[2] = maxDelay_;
    return y;
  }
};

// FDN<SIZE>, MLDSPFilters.h:1162-1239.  Any SIZE is recorded as what it is made of -- SIZE IntegerDelays fed by the
// vectors kept from the previous call (they become one-block feedback edges like any carried DSPVector member), the
// stereo sums, the Householder step, SIZE OnePoles, the gains -- in the reference's operation order, so with its bits
// (tests/test_oracle_port_vs_ref.py::test_fdn_of_any_size_written_out_with_its_parts).  FDN<8> (below) is ONE node
// with its own kernel.  The delays are sized for exactly their length (the reference never sizes them: SURVEY D7).
template <int SIZE>
class FDN
{
  std::array<IntegerDelay, (size_t)SIZE> delays_;
  std::array<OnePole, (size_t)SIZE> filters_;
  std::array<DSPVector, (size_t)SIZE> lines_;  // mDelayInputVectors: read before they are assigned

 public:
  std::array<float, (size_t)SIZE> mFeedbackGains{};
  void setDelaysInSamples(std::array<float, (size_t)SIZE> times)
  {
    for (int n = 0; n < SIZE; ++n)
    {
      int len = (int)(times[(size_t)n] - (float)kFloatsPerDSPVector);  // one vector of latency is in the feedback edge
      if (len < 1) len = 1;
      delays_[(size_t)n].setMaxDelayInSamples((float)len);
      delays_[(size_t)n].setDelayInSamples(len);
    }
  }
  void setFilterCutoffs(std::array<float, (size_t)SIZE> omegas)
  {
    for (int n = 0; n < SIZE; ++n) filters_[(size_t)n].coeffs = OnePole::makeCoeffs(omegas[(size_t)n]);
  }
  DSPVectorArray<2> operator()(const DSPVector& x)
  {
    for (int n = 0; n < SIZE; ++n) lines_[(size_t)n] = delays_[(size_t)n](lines_[(size_t)n]);
    DSPVector sumR, sumL;  // zero filled
    for (int n = 0; n < (SIZE & ~1); ++n)
    {
      if (n & 1)
        sumL += lines_[(size_t)n];
      else
        sumR += lines_[(size_t)n];
    }
    DSPVector sumOfDelays;
    for (int n = 0; n < SIZE; ++n) sumOfDelays += lines_[(size_t)n];
    sumOfDelays *= DSPVector(2.0f / SIZE);  // the unit-gain Householder matrix: identity minus 2 / SIZE
    for (int n = 0; n < SIZE; ++n)
    {
      DSPVector& line = lines_[(size_t)n];
      line -= sumOfDelays;
      line = filters_[(size_t)n](line) * DSPVector(mFeedbackGains[(size_t)n]);
      line += x;
    }
    return concatRows(sumL, sumR);
  }
};
template <>
class FDN<8> : public Functor
{
  static constexpr int SIZE = 8;
  std::array<float, 8> times_{}, cutoffs_{};

 public:
  std::array<float, 8> mFeedbackGains{{0, 0, 0, 0, 0, 0, 0, 0}};
  void setDelaysInSamples(std::array<float, 8> times) { times_ = times; }
  void setFilterCutoffs(std::array<float, 8> omegas) { cutoffs_ = omegas; }
  DSPVectorArray<2> operator()(const DSPVector& x)
  {
    once();
    DSPVector l = op1(MLB_OP_FDN8, x);
    mlb_coeffs_fdn8(times_.data(), cutoffs_.data(), mFeedbackGains.data(), nodeOf(l).coef.data());
    DSPVector r = DSPVector::ofNode(Recorder::get().addNode(MLB_OP_FDN8_R, {l.node}));
    return concatRows(l, r);
  }
};

// Bank<T, ROWS>, MLDSPFunctional.h:321-360: ROWS processors inside ONE traced instance.  (The batch axis --
// thousands of instances of the whole process function -- is TracedProcessor's run-time `instances`.)
template <class T, size_t ROWS>
class Bank
{
  std::array<T, ROWS> procs_;

 public:
  T& operator[](size_t n) { return procs_[n]; }
  DSPVectorArray<ROWS> operator()()
  {
    DSPVectorArray<ROWS> y;
    for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = procs_[j]();
    return y;
  }
  template <typename... Args>
  DSPVectorArray<ROWS> operator()(const Args&... args)
  {
    DSPVectorArray<ROWS> y;
    for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = procs_[j](args.constRow((int)j)...);
    return y;
  }
};

// HalfBandFilter, MLDSPFilters.h:1245-1310, used directly: one object works in one direction per vector --
// upsampleFirstHalf(x) then upsampleSecondHalf(x) of the same x (two rows at twice the rate), or downsample(x1, x2).
class HalfBandFilter : public Functor
{
  int upNode_ = -1, upEpoch_ = 0;

 public:
  void clear() {}
  DSPVector upsampleFirstHalf(const DSPVector& vx)
  {
    once();
    DSPVector y = op1(MLB_OP_HALFBAND_UP, vx);
    upNode_ = y.node, upEpoch_ = Recorder::get().epoch;
    return y;
  }
  DSPVector upsampleSecondHalf(const DSPVector& /*the same vx*/)
  {
    Recorder& r = Recorder::get();
    if (upEpoch_ != r.epoch || upNode_ < 0)
      throw Error(MLB_ERR_UNSUPPORTED, "mlb::tr: HalfBandFilter::upsampleSecondHalf needs upsampleFirstHalf of the same vector first");
    return DSPVector::ofNode(r.addNode(MLB_OP_HALFBAND_UP_2, {upNode_}));
  }
  DSPVector downsample(const DSPVector& vx1, const DSPVector& vx2)
  {
    once();
    return op2(MLB_OP_HALFBAND_DOWN, vx1, vx2);
  }
};

// TempoLock, MLDSPFilters.h:1478-1579: a phasor locked to the input phasor at the ratio dydx
class TempoLock : public Functor
{
 public:
  void clear() {}
  DSPVector operator()(const DSPVector& x, float dydx, float isr)
  {
    once();
    DSPVector y = op2(MLB_OP_TEMPO_LOCK, x, DSPVector(dydx));
    nodeOf(y).coef[0] = isr;
    nodeOf(y).state[0] = 0xBF800000u;  // _omega{-1.f}: stopped, MLDSPFilters.h:1481
    return y;
  }
};

// Upsample2xFunction<IN_ROWS>, MLDSPFunctional.h:114-160: the input rows upsampled by two half-band filters, the
// process function run on BOTH halves, the two results downsampled to one row.  The functors inside fn are called
// twice per vector, as in the reference (the second call records MLB_AGAIN nodes: same state, ticked again);
// functors with a delay ring cannot be (the graph is then rejected when it is compiled).
template <int IN_ROWS>
class Upsample2xFunction : public Functor
{
  using inputType = DSPVectorArray<(size_t)IN_ROWS>;
  using ProcessFn = std::function<DSPVector(const inputType)>;

 public:
  DSPVector operator()(ProcessFn fn, const inputType& vx)
  {
    once();  // the wrapper's own half-band filters are one-per-vector objects like any functor
    Recorder& r = Recorder::get();
    r.pendingOwner = nullptr, r.pendingAgain = -1;  // (its nodes are recorded here, not through a functor member)
    inputType first, second;
    for (int j = 0; j < IN_ROWS; ++j)
    {
      DSPVector up = op1(MLB_OP_HALFBAND_UP, vx.constRow(j));  // mUppers[j].upsampleFirstHalf
      first.row(j) = up;
      second.row(j) = DSPVector::ofNode(r.addNode(MLB_OP_HALFBAND_UP_2, {up.node}));  // ... upsampleSecondHalf
    }
    const DSPVector y1 = fn(first);
    ++r.repeatDepth;
    DSPVector y2;
    try
    {
      y2 = fn(second);
    }
    catch (...)
    {
      --r.repeatDepth;
      throw;
    }
    --r.repeatDepth;
    return op2(MLB_OP_HALFBAND_DOWN, y1, y2);  // mDowners[0].downsample
  }
  // the one-row form: upper(fn, x) with DSPVector in and out (dspOpsExample.cpp:100-102)
  template <int R = IN_ROWS, typename = typename std::enable_if<R == 1>::type>
  DSPVector operator()(std::function<DSPVector(const DSPVector)> fn, const DSPVector& x)
  {
    inputType in;
    in.row(0) = x;
    return (*this)([&](const inputType a) { return fn(a.constRow(0)); }, in);
  }
};

// Upsampler(octaves) / Downsampler(octaves), MLDSPFilters.h:1316-1473, used inside ONE process function: write a vector,
// read 2^octaves vectors at the higher rate, process them, write them to the Downsampler, read one vector back -- an
// oversampled loop.  Stage j of either cascade owns one half-band filter and runs it 2^j (up) / 2^(octaves-1-j) (down)
// times per vector: the first call records a HALFBAND node, the others MLB_AGAIN calls of it.  (The block-rate-changing
// use -- several process calls per write -- is the mlb_resampler_* bank.)
class Upsampler
{
  int octaves_;
  std::vector<int> firstNode_, firstEpoch_;  // per stage: the filter's first call in the current pass
  std::vector<DSPVector> rows_;
  size_t readIdx_ = 0;

 public:
  explicit Upsampler(int octavesUp) : octaves_(octavesUp), firstNode_((size_t)octavesUp, -1), firstEpoch_((size_t)octavesUp, 0) {}
  void clear() {}
  void write(const DSPVector& x)
  {
    Recorder& r = Recorder::get();
    rows_.assign(1, x);
    for (int j = 0; j < octaves_; ++j)
    {
      std::vector<DSPVector> next;
      for (const DSPVector& src : rows_)
      {
        const int in = src.resolve();
        const bool again = firstEpoch_[(size_t)j] == r.epoch;
        const int up = r.addNode(MLB_OP_HALFBAND_UP, {in}, again ? MLB_AGAIN(firstNode_[(size_t)j]) : 0);
        if (!again) firstNode_[(size_t)j] = up, firstEpoch_[(size_t)j] = r.epoch;
        next.push_back(DSPVector::ofNode(up));
        next.push_back(DSPVector::ofNode(r.addNode(MLB_OP_HALFBAND_UP_2, {up})));
      }
      rows_.swap(next);
    }
    readIdx_ = 0;
  }
  DSPVector read()  // after a write, 1 << octaves reads are available
  {
    if (readIdx_ >= rows_.size()) throw Error(MLB_ERR_INVALID, "mlb::tr: Upsampler::read past the vectors of the last write");
    return rows_[readIdx_++];
  }
};
class Downsampler
{
  int octaves_;
  std::vector<int> firstNode_, firstEpoch_;
  std::vector<DSPVector> buffers_;  // 2 per octave + the output, as in the reference
  uint32_t counter_ = 0;
  int epoch_ = 0;

 public:
  explicit Downsampler(int octavesDown)
      : octaves_(octavesDown), firstNode_((size_t)octavesDown, -1), firstEpoch_((size_t)octavesDown, 0),
        buffers_((size_t)(2 * octavesDown + 1))
  {
  }
  void clear() {}
  bool write(const DSPVector& v)  // true when a new output vector is ready (every 2^octaves writes)
  {
    Recorder& r = Recorder::get();
    if (epoch_ != r.epoch)
    {
      if (counter_ != 0)
        throw Error(MLB_ERR_UNSUPPORTED, "mlb::tr: a Downsampler must be written 2^octaves times in every vector");
      epoch_ = r.epoch;
    }
    if (octaves_ == 0)
    {
      buffers_[0] = v;
      return true;
    }
    buffers_[counter_ & 1u] = v;
    uint32_t mask = 1;
    for (int h = 0; h < octaves_; ++h)
    {
      if (!(counter_ & mask)) break;  // an octave runs when its bit and all lesser bits are 1
      mask <<= 1;
      const bool b1 = (counter_ & mask) != 0;
      const int x1 = buffers_[(size_t)(2 * h)].resolve(), x2 = buffers_[(size_t)(2 * h + 1)].resolve();
      const bool again = firstEpoch_[(size_t)h] == r.epoch;
      const int down = r.addNode(MLB_OP_HALFBAND_DOWN, {x1, x2}, again ? MLB_AGAIN(firstNode_[(size_t)h]) : 0);
      if (!again) firstNode_[(size_t)h] = down, firstEpoch_[(size_t)h] = r.epoch;
      buffers_[(size_t)(2 * h + 2 + (b1 ? 1 : 0))] = DSPVector::ofNode(down);
    }
    counter_ = (counter_ + 1u) & ((1u << octaves_) - 1u);
    return counter_ == 0;
  }
  DSPVector read() const { return buffers_.back(); }
};

// Downsample2xFunction<IN_ROWS>, MLDSPFunctional.h:166-223: on every second vector the input (this vector and the
// buffered previous one) is downsampled, the process function runs on that half-rate vector and its result is upsampled
// into this vector and the next.  Recorded as DOWN2X_IN per input row, fn's nodes, DOWN2X_OUT (mlb200.h).  fn must be
// stateless: its nodes run on every vector here, its functors would have to tick on every second one only.
template <int IN_ROWS>
class Downsample2xFunction : public Functor
{
  using inputType = DSPVectorArray<(size_t)IN_ROWS>;
  using ProcessFn = std::function<DSPVector(const inputType)>;

 public:
  DSPVector operator()(ProcessFn fn, const inputType& vx)
  {
    once();
    Recorder& r = Recorder::get();
    r.pendingOwner = nullptr, r.pendingAgain = -1;
    inputType half;
    for (int j = 0; j < IN_ROWS; ++j) half.row(j) = op1(MLB_OP_DOWN2X_IN, vx.constRow(j));
    ++r.forbidFunctors;
    DSPVector y;
    try
    {
      y = fn(half);
    }
    catch (...)
    {
      --r.forbidFunctors;
      throw;
    }
    --r.forbidFunctors;
    return op1(MLB_OP_DOWN2X_OUT, y);
  }
  template <int R = IN_ROWS, typename = typename std::enable_if<R == 1>::type>
  DSPVector operator()(std::function<DSPVector(const DSPVector)> fn, const DSPVector& x)
  {
    inputType in;
    in.row(0) = x;
    return (*this)([&](const inputType a) { return fn(a.constRow(0)); }, in);
  }
};

// ---- scalar host helpers the examples use (MLDSPProjections.h:15-23,105-123,176-195) ----
struct Interval
{
  float x1, x2;
};
using Projection = std::function<float(float)>;
namespace projections
{
inline Projection log(Interval m)
{
  const float a = m.x1, b = m.x2;
  if (b - a == 0.f) return [=](float) { return a; };
  if (a == 0.f) return [=](float) { return 0.f; };
  return [=](float x) { return a * (powf((b / a), x) - 1) / (b - a); };
}
inline Projection intervalMap(const Interval a, const Interval b, Projection c)
{
  return [=](float x)
  {
    const float scaleA = 1 / (a.x2 - a.x1);
    const float offsetA = (-a.x1) / (a.x2 - a.x1);
    const float scaleB = (b.x2 - b.x1);
    const float offsetB = b.x1;
    return c(x * scaleA + offsetA) * scaleB + offsetB;
  };
}
inline Projection unityToLogParam(Interval paramInterval) { return intervalMap({0, 1}, paramInterval, log(paramInterval)); }
}  // namespace projections

// ------------------------------------------------------------------------------------------------------
// AudioContext / SignalProcessFn (source/app/MLAudioContext.h:23-101, MLSignalProcessBuffer.h:18)

class DSPVectorDynamic
{
  std::vector<DSPVector> rows_;

 public:
  explicit DSPVectorDynamic(size_t n = 0) : rows_(n) {}
  size_t size() const { return rows_.size(); }
  DSPVector& operator[](size_t i) { return rows_[i]; }
  const DSPVector& operator[](size_t i) const { return rows_[i]; }
};
using MainInputs = const DSPVectorDynamic&;
using MainOutputs = DSPVectorDynamic&;

// ---- the synth spelling: EventsToSignals' voice rows (MLEventsToSignals.h:15-26, 46-47, 184) ----
enum VoiceOutputSignals
{
  kPitch = 0,
  kGate,
  kVoice,
  kZ,
  kX,
  kY,
  kMod,
  kElapsedTime,
  kNumVoiceOutputRows
};

class EventsToSignals
{
 public:
  static constexpr size_t kMaxVoices{16};
  struct Voice
  {
    DSPVectorArray<kNumVoiceOutputRows> outputs;  // symbolic: INPUT planes 0..7 of the traced graph
  };
};

using Symbol = std::string;  // what setInputProtocol takes ("MIDI" or "MPE")

// MLSynth.h:16-19, a host scalar
inline float pitchToFrequency(float pitch) { return 440.0f * powf(2.0f, (pitch - 69.0f) / 12.0f); }

// what getInputVoice / getInputController / getBeatPhase return while TracedSynth::trace runs one voice, or (voice -1)
// the instrument section of Synth::processVector
struct SynthPass
{
  static constexpr int kPhasePlane = 1 << 20;  // INPUT iarg of the beat phase until the controller count is known
  static constexpr int kAccPlane = 1 << 21;    // INPUT iarg kAccPlane + i: the accumulator outputs[i] at entry
  static constexpr int kBusPlane = 1 << 22;    // instrument section: kBusPlane + i, bus row i after the base call
  static constexpr int kOutPlane = 1 << 23;    // instrument section: kOutPlane + i, outputs[i] at entry
  int voice = -1;
  std::function<void(DSPVectorDynamic&)> base;  // instrument section: what the base Synth::processVector does
  EventsToSignals::Voice rows;
  std::vector<int>* controllers = nullptr;  // controller numbers in first-use order, over all voices
  std::map<int, int> controllerNode;        // this pass: controller number -> its INPUT node
  int phaseNode = -1;
};

class AudioContext
{
  double sampleRate_ = 0;

 public:
  AudioContext(size_t nInputs, size_t nOutputs, int rate = 0) : sampleRate_(rate), inputs(nInputs), outputs(nOutputs) {}
  double getSampleRate() const { return sampleRate_; }
  void setSampleRate(int r) { sampleRate_ = r; }
  DSPVectorDynamic inputs;
  DSPVectorDynamic outputs;

  // The instrument settings a synth's setup makes (MLAudioContext.h:76-98): recorded here, applied to every instrument
  // by TracedSynth::compile.  The defaults are EventsToSignals' (MLEventsToSignals.h:213-228).
  struct InputSettings
  {
    int polyphony = 0;
    bool mpe = false;
    bool unison = false;
    int modCC = 16;
    float pitchBend = 7.f, mpePitchBend = 24.f, glideSeconds = 0.f, driftAmount = 0.f;
  };
  InputSettings input;
  void setInputPolyphony(int voices) { input.polyphony = voices; }
  void setInputProtocol(const Symbol& p)
  {
    if (p != "MIDI" && p != "MPE") throw Error(MLB_ERR_INVALID, ("mlb::tr: protocol " + p + " is not MIDI or MPE").c_str());
    input.mpe = p == "MPE";
  }
  void setInputUnison(bool u) { input.unison = u; }
  void setInputModCC(int p) { input.modCC = p; }
  void setInputPitchBend(float p) { input.pitchBend = p; }
  void setInputMPEPitchBend(float p) { input.mpePitchBend = p; }
  void setInputGlideTimeInSeconds(float s) { input.glideSeconds = s; }
  void setInputDriftAmount(float d) { input.driftAmount = d; }

  // the voice's rows, a smoothed controller, the beat phase: symbolic rows (INPUT planes 0..7, 8 + k, 8 + C)
  const EventsToSignals::Voice& getInputVoice(int n)
  {
    if (!pass_) throw Error(MLB_ERR_INVALID, "mlb::tr: getInputVoice outside TracedSynth::trace()");
    if (pass_->voice < 0)
      throw Error(MLB_ERR_UNSUPPORTED, ("mlb::tr::TracedSynth: getInputVoice(" + std::to_string(n) + ") outside the base "
                                        "Synth::processVector call; the instrument section sees the voices only through "
                                        "the bus rows the base call leaves in its outputs")
                                           .c_str());
    if (n != pass_->voice)
      throw Error(MLB_ERR_UNSUPPORTED, ("mlb::tr: voice " + std::to_string(pass_->voice) + " reads the rows of voice " +
                                        std::to_string(n) + "; a voice may read only its own rows")
                                           .c_str());
    return pass_->rows;
  }
  DSPVector getInputController(size_t n) const
  {
    if (!pass_) throw Error(MLB_ERR_INVALID, "mlb::tr: getInputController outside TracedSynth::trace()");
    if (n > 128)
      throw Error(MLB_ERR_INVALID, ("mlb::tr: controller " + std::to_string(n) + " is above 128 (EventsToSignals has 129)").c_str());
    auto it = pass_->controllerNode.find((int)n);
    if (it == pass_->controllerNode.end())
    {
      std::vector<int>& list = *pass_->controllers;
      size_t k = 0;
      while (k < list.size() && list[k] != (int)n) ++k;
      if (k == list.size()) list.push_back((int)n);
      Recorder& r = Recorder::get();
      it = pass_->controllerNode.emplace((int)n, r.addNode(MLB_OP_INPUT, {}, MLB_VOICE_ROWS + (int)k, false)).first;
    }
    return DSPVector::ofNode(it->second);
  }
  DSPVector getBeatPhase()
  {
    if (!pass_) throw Error(MLB_ERR_INVALID, "mlb::tr: getBeatPhase outside TracedSynth::trace()");
    if (pass_->phaseNode < 0) pass_->phaseNode = Recorder::get().addNode(MLB_OP_INPUT, {}, SynthPass::kPhasePlane, false);
    return DSPVector::ofNode(pass_->phaseNode);
  }

  SynthPass* pass_ = nullptr;  // set by TracedSynth::trace
};
using SignalProcessFn = void (*)(AudioContext*, void*);

using Path = std::string;  // the name of a published signal (the reference's ml::Path, made from a string)

// A published signal as publishSignal declared it, and one storePublishedSignal call as TracedSynth::trace recorded it
struct PublishDecl
{
  Path name;
  int maxFrames, maxVoices, channels, octavesDown;
};
struct PublishStore
{
  int signal;             // index into the declarations
  int frames;
  std::vector<int> rows;  // the `channels` rows stored: node indices of the pass being recorded
};

// MLSignalProcessor.h: the base of Synth, reduced to what a Synth subclass uses
class SignalProcessor
{
 public:
  SignalProcessor() {}
  virtual ~SignalProcessor() {}
  virtual void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* stateData = nullptr) {}
  virtual void setSampleRate(double sr) { sampleRate_ = sr; }
  const std::vector<PublishDecl>& publishedSignals() const { return published_; }

 protected:
  double sampleRate_{0};

  // MLSignalProcessor.h:184-188: declares the signal (publishing a name again replaces its declaration)
  void publishSignal(Path signalName, int maxFrames, int maxVoices, int channels, int octavesDown)
  {
    const std::string what = "mlb::tr: publishSignal(" + signalName + "): ";
    if (maxFrames < 1 || maxVoices < 1 || channels < 1 || channels > (int)kFloatsPerDSPVector)
      throw Error(MLB_ERR_UNSUPPORTED, (what + "maxFrames and maxVoices must be at least 1 and channels in 1..64").c_str());
    if (octavesDown < 0 || octavesDown > 30)
      throw Error(MLB_ERR_UNSUPPORTED, (what + "octavesDown " + std::to_string(octavesDown) + " is not in 0..30").c_str());
    for (PublishDecl& d : published_)
      if (d.name == signalName)
      {
        d = PublishDecl{signalName, maxFrames, maxVoices, channels, octavesDown};
        return;
      }
    published_.push_back(PublishDecl{signalName, maxFrames, maxVoices, channels, octavesDown});
  }

  // MLSignalProcessor.h:193-201: inside TracedSynth::trace, records the rows as graph outputs of the voice; a name that
  // was never published stores nothing, as in the reference
  template <size_t CHANNELS>
  void storePublishedSignal(Path signalName, const DSPVectorArray<CHANNELS>& inputVec, int frames, int voice)
  {
    (void)voice;
    int s = 0;
    while (s < (int)published_.size() && published_[(size_t)s].name != signalName) ++s;
    if (s == (int)published_.size()) return;
    const PublishDecl& d = published_[(size_t)s];
    const std::string what = "mlb::tr: storePublishedSignal(" + signalName + "): ";
    if (!publishStores_)
      throw Error(inSynthTrace_ ? MLB_ERR_UNSUPPORTED : MLB_ERR_INVALID,
                  (what + (inSynthTrace_ ? "outside processVoice; only a voice publishes" : "outside TracedSynth::trace()"))
                      .c_str());
    if ((int)CHANNELS != d.channels)
      throw Error(MLB_ERR_UNSUPPORTED, (what + "a DSPVectorArray<" + std::to_string(CHANNELS) + "> into a signal of " +
                                        std::to_string(d.channels) + " channels (the reference's rotate buffer would be "
                                        "mis-sized)").c_str());
    if (frames < 0 || frames > (int)kFloatsPerDSPVector)
      throw Error(MLB_ERR_UNSUPPORTED, (what + "frames " + std::to_string(frames) + " is not in 0..64").c_str());
    if (frames > d.maxFrames)
      throw Error(MLB_ERR_UNSUPPORTED, (what + "frames " + std::to_string(frames) + " is above maxFrames " +
                                        std::to_string(d.maxFrames) + " (the reference writes past its rotate buffer)")
                                           .c_str());
    PublishStore st{s, frames, {}};
    for (size_t j = 0; j < CHANNELS; ++j) st.rows.push_back(inputVec.constRow((int)j).resolve());
    publishStores_->push_back(st);
  }
  // one row: the reference's DSPVector is a DSPVectorArray<1>
  void storePublishedSignal(Path signalName, const DSPVector& inputVec, int frames, int voice)
  {
    DSPVectorArray<1> a;
    a.row(0) = inputVec;
    storePublishedSignal(signalName, a, frames, voice);
  }

  // MLSignalProcessor.h:203-210: takes a host pointer, which has no symbolic form
  void storePublishedSignalVert(Path signalName, const float*, int, int)
  {
    throw Error(MLB_ERR_UNSUPPORTED, ("mlb::tr: storePublishedSignalVert(" + signalName +
                                      ") takes a host pointer and cannot be traced; store a DSPVectorArray with "
                                      "storePublishedSignal")
                                         .c_str());
  }

 private:
  friend class TracedSynth;
  std::vector<PublishDecl> published_;
  std::vector<PublishStore>* publishStores_ = nullptr;  // set by TracedSynth::trace while processVoice runs
  bool inSynthTrace_ = false;                           // set by TracedSynth::trace for the whole trace
};

// Synth (MLSynth.h:26-93): subclasses implement processVoice; TracedSynth traces it once per voice
class Synth : public SignalProcessor
{
 public:
  static constexpr int kDefaultNumVoices = 8;
  static constexpr int kNumVoices = 8;

  Synth(int numVoices = kDefaultNumVoices) : numVoices_(numVoices) {}
  virtual ~Synth() = default;

  void processVector(const DSPVectorDynamic& inputs, DSPVectorDynamic& outputs, void* stateData) override
  {
    auto* audioContext = static_cast<AudioContext*>(stateData);
    if (!audioContext) return;
    if (audioContext->pass_ && audioContext->pass_->base)  // TracedSynth::trace: every voice, then the bus rows
    {
      audioContext->pass_->base(outputs);
      return;
    }
    for (int i = 0; i < (int)outputs.size(); ++i) outputs[i] = DSPVector{0.f};
    int activeCount = 0;
    for (int v = 0; v < numVoices_; ++v)
    {
      const auto& voice = audioContext->getInputVoice(v);
      if (isVoiceActive(v, voice))
      {
        activeCount++;
        processVoice(v, voice, inputs, outputs, audioContext);
      }
    }
    activeVoiceCount_ = activeCount;
  }

  virtual void processVoice(int voiceIndex, const EventsToSignals::Voice& voice, const DSPVectorDynamic& inputs,
                            DSPVectorDynamic& outputs, AudioContext* audioContext) = 0;
  virtual bool isVoiceActive(int voiceIndex, const EventsToSignals::Voice& voice) { return true; }
  int getActiveVoiceCount() const { return activeVoiceCount_; }
  int getNumVoices() const { return numVoices_; }
  virtual bool hasActiveVoices() const { return activeVoiceCount_ > 0; }

 protected:
  int numVoices_;
  int activeVoiceCount_ = 0;
};

// ------------------------------------------------------------------------------------------------------
// what TracedProcessor and TracedSynth share

// Records into `rec` for the lifetime of the scope.  On exit, normal or thrown, the recorder stops, the previous one
// is current again and the context no longer answers for a synth voice.
class TraceScope
{
  Recorder& rec_;
  Recorder* prev_;
  AudioContext& ctx_;

 public:
  TraceScope(Recorder& rec, AudioContext& ctx) : rec_(rec), prev_(Recorder::current()), ctx_(ctx) { Recorder::current() = &rec; }
  ~TraceScope()
  {
    rec_.active = false;
    Recorder::current() = prev_;
    ctx_.pass_ = nullptr;
  }
  TraceScope(const TraceScope&) = delete;
  TraceScope& operator=(const TraceScope&) = delete;
};

// Lay the traced graph out once at trace time: that is where a functor with a delay ring that is called again is
// refused.  The bank lays it out again when it is compiled.
inline void checkLayout(const std::vector<mlb_node>& nodes)
{
  mlb_layout layout;
  check(mlb_graph_layout(nodes.data(), (int)nodes.size(), &layout, nullptr, nullptr));
}

// the initial coefficient and state words of traced node `node` into one row of the bank
inline void loadWords(DeviceBank& bank, int node, int row, const TNode& t)
{
  if (isAgain(t.node)) return;  // the words belong to the functor's first call
  for (size_t k = 0; k < t.coef.size(); ++k) bank.setCoef(node, (int)k, row, t.coef[k]);
  for (size_t k = 0; k < t.state.size(); ++k) bank.setStateWord(node, (int)k, row, t.state[k]);
}

// coefficient or state words as a JSON list body of decimal bit patterns: an exact round trip
template <class Word>
inline void printWords(FILE* f, const std::vector<Word>& words)
{
  static_assert(sizeof(Word) == 4, "32-bit words");
  for (size_t k = 0; k < words.size(); ++k)
  {
    uint32_t u;
    std::memcpy(&u, &words[k], 4);
    std::fprintf(f, "%s%u", k ? ", " : "", u);
  }
}

// ------------------------------------------------------------------------------------------------------
// TracedProcessor: trace a SignalProcessFn, compile it for `instances` independent copies, run it on the GPU.

class TracedProcessor
{
  Recorder rec_;
  std::vector<mlb_node> nodes_;
  std::vector<int32_t> outs_;
  std::map<std::string, int> named_;
  std::unique_ptr<DeviceBank> bank_;
  size_t nIn_ = 0, nOut_ = 0;
  std::unique_ptr<BatchedSignalProcessBuffer> buffer_;

  DeviceBank& bank() const
  {
    if (!bank_) throw Error(MLB_ERR_INVALID, "mlb::tr: compile() first");
    return *bank_;
  }

  void runPass(AudioContext* ctx, SignalProcessFn fn, void* state)
  {
    rec_.beginPass();
    for (size_t i = 0; i < ctx->inputs.size(); ++i)
      ctx->inputs[i] = DSPVector::ofNode(rec_.addNode(MLB_OP_INPUT, {}, (int)i));
    fn(ctx, state);
  }

 public:
  TracedProcessor() = default;
  TracedProcessor(const TracedProcessor&) = delete;
  TracedProcessor& operator=(const TracedProcessor&) = delete;

  // Record the graph `fn` builds (host only: works without a GPU).
  void trace(AudioContext* ctx, SignalProcessFn fn, void* state)
  {
    {
      TraceScope scope(rec_, *ctx);
      runPass(ctx, fn, state);  // pass 1: discovers which symbols survive the call
      runPass(ctx, fn, state);  // pass 2: the graph; stale symbols of pass 1 become feedback edges
      rec_.closeFeedback("process function");
      nOut_ = ctx->outputs.size();
      for (size_t i = 0; i < nOut_; ++i) rec_.outs.push_back(ctx->outputs[i].resolve());
    }
    nIn_ = ctx->inputs.size();
    nodes_.clear();
    for (const TNode& t : rec_.nodes) nodes_.push_back(t.node);
    outs_.assign(rec_.outs.begin(), rec_.outs.end());
    checkLayout(nodes_);
    named_.clear();
    for (size_t i = 0; i < rec_.nodes.size(); ++i)
      if (!rec_.nodes[i].name.empty()) named_[rec_.nodes[i].name] = (int)i;
  }

  size_t nodeCount() const { return nodes_.size(); }
  const std::vector<mlb_node>& nodes() const { return nodes_; }
  const std::vector<int32_t>& outs() const { return outs_; }
  size_t inputs() const { return nIn_; }
  size_t outputs() const { return nOut_; }

  // Write the traced graph as JSON (nodes, outs, initial coefficient and state words): lets a test or a tool
  // rebuild it elsewhere (tests/test_trace.py feeds it to the CPU checkers).
  void dump(FILE* f) const
  {
    std::fprintf(f, "{\"n_in\": %zu, \"nodes\": [", nIn_);
    for (size_t i = 0; i < rec_.nodes.size(); ++i)
    {
      const TNode& t = rec_.nodes[i];
      std::fprintf(f, "%s{\"op\": %d, \"in\": [", i ? ", " : "", t.node.op);
      for (int k = 0; k < MLB_MAX_INS; ++k) std::fprintf(f, "%s%d", k ? ", " : "", t.node.in[k]);
      std::fprintf(f, "], \"iarg\": %d, \"coef\": [", t.node.iarg);
      const bool again = isAgain(t.node);
      if (!again) printWords(f, t.coef);
      std::fprintf(f, "], \"state\": [");
      if (!again) printWords(f, t.state);
      std::fprintf(f, "], \"name\": \"%s\"}", t.name.c_str());
    }
    std::fprintf(f, "], \"outs\": [");
    for (size_t i = 0; i < outs_.size(); ++i) std::fprintf(f, "%s%d", i ? ", " : "", outs_[i]);
    std::fprintf(f, "]}\n");
  }

  // Create the device bank: `instances` independent copies of the traced process function (needs a GPU).
  void compile(int instances, unsigned flags = MLB_GRAPH_EXACT)
  {
    if (nodes_.empty()) throw Error(MLB_ERR_INVALID, "mlb::tr: trace() first");
    bank_.reset();  // the old graph's device memory is freed before the new graph's is allocated
    bank_.reset(new DeviceBank(nodes_, outs_, instances, flags));
    for (size_t i = 0; i < rec_.nodes.size(); ++i)
      for (int v = 0; v < instances; ++v) loadWords(*bank_, (int)i, v, rec_.nodes[i]);
    commit();
  }
  void commit() { bank().commit(); }
  int instances() const { return bank_ ? bank_->rows() : 0; }
  const char* kernelName() const { return bank_ ? bank_->kernelName() : ""; }
  // per-instance value of a tr::param(name, ...) scalar; call commit() after a batch of changes
  void setParam(const std::string& name, int instance, float value)
  {
    auto it = named_.find(name);
    if (it == named_.end()) throw Error(MLB_ERR_INVALID, "mlb::tr: no such param");
    bank().setParam(it->second, instance, value);
  }
  // per-instance coefficient / state word of node `node` (indices as in nodes())
  void setCoef(int node, int word, int instance, float value) { bank().setCoef(node, word, instance, value); }
  void setStateWord(int node, int word, int instance, uint32_t value) { bank().setStateWord(node, word, instance, value); }

  // Restart the listed instances between two calls: from the next vector each runs as a newly constructed copy of the
  // process function (its state words as the last commit() uploaded them, its delay memory empty, its parameters
  // kept); the others are untouched.  One launch, none for an empty list.  Frames the process() streaming shim has
  // already computed and buffered are not recalled: they come out of the next process() call as before.
  void restart(const std::vector<int>& instances) { bank().reset(std::vector<int32_t>(instances.begin(), instances.end())); }

  // n_blocks successive process calls for every instance in ONE kernel launch.
  // in [T][inputs][instances][64], out [T][outputs][instances][64], mix [T][outputs][64] (sum over instances).
  void processBlocks(const float* in, float* out, float* mix, int nBlocks) { bank().process(in, out, mix, nBlocks); }

  // SignalProcessBuffer::process for ONE instance's I/O (source/app/MLSignalProcessBuffer.cpp:36-90): any host
  // buffer size; every vector the callback needs is computed by one launch.  With instances > 1 the outputs are
  // the mix bus (sum over instances, Synth::processVector's accumulate, source/app/MLSynth.h:36-60) and every
  // instance receives the same external inputs.
  void process(const float** externalInputs, float** externalOutputs, int nFrames, int maxFrames = 4096)
  {
    DeviceBank& bank = this->bank();
    if (!buffer_) buffer_.reset(new BatchedSignalProcessBuffer(nIn_, nOut_, (size_t)maxFrames));
    std::vector<float>& bin = bcast_;
    const int instances = bank.rows();
    buffer_->process(externalInputs, externalOutputs, nFrames,
                     [&](const float* in, float* out, int nVec)
                     {
                       const float* src = in;
                       if (nIn_ && instances > 1)
                       {
                         bin.resize((size_t)nVec * nIn_ * instances * MLB_BLOCK);
                         for (size_t r = 0; r < (size_t)nVec * nIn_; ++r)
                           for (int v = 0; v < instances; ++v)
                             std::memcpy(&bin[(r * instances + v) * MLB_BLOCK], in + r * MLB_BLOCK, MLB_BLOCK * 4);
                         src = bin.data();
                       }
                       if (instances > 1)
                         bank.process(nIn_ ? src : nullptr, nullptr, out, nVec);
                       else
                         bank.process(nIn_ ? src : nullptr, out, nullptr, nVec);
                     });
  }

 private:
  std::vector<float> bcast_;
};

// ------------------------------------------------------------------------------------------------------
// TracedSynth: trace a Synth subclass's processVoice, compile it for G instruments, run it from raw events.
//
// processVoice is traced once per voice (two passes each, as TracedProcessor::trace, so carried DSPVector members
// become feedback edges).  At entry every outputs[i] is an accumulator; a voice must leave it untouched or end it as
// the accumulator plus ONE expression x.  Graph output i is x (or a +0 row), and the bus kernel sums the voices of an
// instrument as ((+0 + x0) + x1) + ..., which is what Synth::processVector's `outputs[i] = 0; outputs[i] += ...` gives
// in voice order.  All voices must record the same nodes; their coefficient and state words may differ (a cutoff
// that depends on voiceIndex) and become per-lane words.  The graph's INPUT planes follow contract E: the Voice rows
// at 0..7, the controllers at 8 + k in first-use order, the beat phase after them.
//
// processVoice runs inside the base Synth::processVector, which trace() reaches through synth.processVector.  An
// override that calls the base once and works on the bus rows it leaves (an effects section per instrument) becomes a
// second graph, over instrument lanes, on the bus rows, the controllers and the beat phase (DESIGN.md, "Instrument
// stage"); a synth without such a section builds none.
class TracedSynth
{
  struct VoiceGraph
  {
    std::vector<TNode> nodes;
    std::vector<int32_t> outs;
    std::vector<PublishStore> stores;  // rows: nodes of this graph
  };
  struct InstrumentGraph
  {
    std::vector<TNode> nodes;  // none: Synth::processVector is the base's, its outputs the bus rows
    std::vector<int32_t> outs;
    int planes = 0;  // INPUT planes: the bus rows, the controllers, the beat phase
  };
  std::vector<VoiceGraph> voices_;  // one per synth voice
  InstrumentGraph instrument_;
  size_t busPlanes_ = 0;  // the outputs Synth::processVector hands to the base call
  std::vector<mlb_node> nodes_;
  std::vector<int32_t> outs_;
  std::vector<PublishDecl> published_;  // the synth's publishSignal declarations
  std::vector<int32_t> pubOuts_;        // graph outputs after outs_: the stored rows, store by store
  std::vector<int> controllers_;
  bool phase_ = false;
  AudioContext::InputSettings settings_;
  double sampleRate_ = 0;
  int numVoices_ = 0;
  size_t nOut_ = 0;

  int instruments_ = 0, lanesPer_ = 0;
  std::unique_ptr<RouterBank> routers_;
  std::unique_ptr<VoiceBank> voiceBank_;
  std::unique_ptr<ControllerBank> ctrl_;
  std::unique_ptr<ProcessTimeBank> times_;
  std::unique_ptr<Buses> buses_;
  std::unique_ptr<DeviceBank> bank_;  // the graph over every lane
  std::unique_ptr<PublishedBank> pubBank_;
  std::unique_ptr<DeviceBank> ibank_;  // the instrument graph over the instruments, if there is one
  std::vector<int64_t> overflow_;  // the router bank's overflow counts after the last call

  DeviceBank& bank() const
  {
    if (!bank_) throw Error(MLB_ERR_INVALID, "mlb::tr::TracedSynth: compile() first");
    return *bank_;
  }

  [[noreturn]] static void refuse(int v, const std::string& what)
  {
    throw Error(MLB_ERR_UNSUPPORTED, ("mlb::tr::TracedSynth: voice " + std::to_string(v) + " " + what).c_str());
  }

  // the pass's graph without the accumulators and unread Voice rows; out i = x, or -1 for an untouched output; the
  // stored rows of `stores` are kept and renumbered
  static VoiceGraph extract(const Recorder& rec, const std::vector<int>& acc, const std::vector<int>& fin, int v,
                            std::vector<PublishStore> stores)
  {
    const int n = (int)rec.nodes.size(), nOut = (int)acc.size();
    std::vector<char> drop((size_t)n, 0);
    std::vector<int> accOf((size_t)n, -1), x((size_t)nOut, -1);
    for (int i = 0; i < nOut; ++i) drop[(size_t)acc[(size_t)i]] = 1, accOf[(size_t)acc[(size_t)i]] = i;
    const auto name = [](int i) { return "outputs[" + std::to_string(i) + "]"; };
    for (int i = 0; i < nOut; ++i)
    {
      const int f = fin[(size_t)i];
      if (f == acc[(size_t)i]) continue;  // untouched
      const mlb_node& m = rec.nodes[(size_t)f].node;
      if (m.op == MLB_OP_ADD && m.in[0] == acc[(size_t)i] && !drop[(size_t)f])
      {
        drop[(size_t)f] = 1, x[(size_t)i] = m.in[1];
        continue;
      }
      if (m.op == MLB_OP_ADD && m.in[0] >= 0 && rec.nodes[(size_t)m.in[0]].node.op == MLB_OP_ADD &&
          rec.nodes[(size_t)m.in[0]].node.in[0] == acc[(size_t)i])
        refuse(v, "adds twice into " + name(i) + ": (acc + a) + b is not one bus term; add one expression");
      if (accOf[(size_t)f] >= 0) refuse(v, "assigns " + name(accOf[(size_t)f]) + " to " + name(i));
      bool reads = false;
      for (const TNode& t : rec.nodes)
        for (int k = 0; k < MLB_MAX_INS; ++k) reads = reads || t.node.in[k] == acc[(size_t)i];
      if (reads)
        refuse(v, "reads or rescales the accumulator " + name(i) + "; only " + name(i) + " += x (accumulator + x) is "
                  "allowed: x + " + name(i) + " keeps x's NaN payload where the reference keeps the accumulator's");
      refuse(v, "assigns " + name(i) + " = x; a voice adds into its outputs: " + name(i) + " += x");
    }
    std::vector<int> uses((size_t)n, 0);
    for (int j = 0; j < n; ++j)
    {
      if (drop[(size_t)j]) continue;
      const mlb_node& m = rec.nodes[(size_t)j].node;
      for (int k = 0; k < MLB_MAX_INS; ++k)
      {
        const int s = m.in[k];
        if (s < 0) continue;
        if (accOf[(size_t)s] >= 0) refuse(v, "reads or rescales the accumulator " + name(accOf[(size_t)s]));
        if (drop[(size_t)s]) refuse(v, "reads an output after adding into it");
        ++uses[(size_t)s];
      }
    }
    for (int i = 0; i < nOut; ++i)
    {
      const int s = x[(size_t)i];
      if (s < 0) continue;
      if (accOf[(size_t)s] >= 0) refuse(v, "adds the accumulator " + name(accOf[(size_t)s]) + " into " + name(i));
      if (drop[(size_t)s]) refuse(v, "adds one output into another");
      ++uses[(size_t)s];
    }
    for (const PublishStore& st : stores)
      for (int s : st.rows)
      {
        if (accOf[(size_t)s] >= 0) refuse(v, "publishes the accumulator " + name(accOf[(size_t)s]));
        if (drop[(size_t)s]) refuse(v, "publishes an output after adding into it");
        ++uses[(size_t)s];
      }
    for (int j = 0; j < n; ++j)  // Voice rows the voice does not read
    {
      const mlb_node& m = rec.nodes[(size_t)j].node;
      if (m.op == MLB_OP_INPUT && m.iarg < MLB_VOICE_ROWS && uses[(size_t)j] == 0) drop[(size_t)j] = 1;
    }
    VoiceGraph vg;
    const std::vector<int> idx = keepNodes(rec.nodes, drop, vg.nodes);
    for (int i = 0; i < nOut; ++i) vg.outs.push_back(x[(size_t)i] < 0 ? -1 : idx[(size_t)x[(size_t)i]]);
    for (PublishStore& st : stores)
      for (int& s : st.rows) s = idx[(size_t)s];
    vg.stores = std::move(stores);
    return vg;
  }

  // the nodes not dropped, renumbered (operands, feedback writes, further calls); returns old index -> new (-1: dropped)
  static std::vector<int> keepNodes(const std::vector<TNode>& nodes, const std::vector<char>& drop, std::vector<TNode>& kept)
  {
    std::vector<int> idx(nodes.size(), -1);
    for (size_t j = 0; j < nodes.size(); ++j)
      if (!drop[j]) idx[j] = (int)kept.size(), kept.push_back(nodes[j]);
    for (TNode& t : kept)
    {
      for (int k = 0; k < MLB_MAX_INS; ++k)
        if (t.node.in[k] >= 0) t.node.in[k] = idx[(size_t)t.node.in[k]];
      if (t.node.op == MLB_OP_FEEDBACK_WRITE) t.node.iarg = idx[(size_t)t.node.iarg];
      else if (isAgain(t.node)) t.node.iarg = MLB_AGAIN(idx[(size_t)MLB_AGAIN_TARGET(t.node.iarg)]);
    }
    return idx;
  }

  // The instrument section (Synth::processVector around the base call) as a graph over instrument lanes.  Its INPUT
  // planes: the P bus rows, the C controllers, the beat phase.  No nodes when the section only hands `outputs` to the
  // base call: the outputs are then the bus rows as they are.
  static InstrumentGraph instrumentGraph(const Recorder& rec, size_t P, size_t nOut, size_t C, bool phase)
  {
    const std::string pv = "mlb::tr::TracedSynth: Synth::processVector ";
    const int n = (int)rec.nodes.size();
    const auto entry = [&](int j)  // i if node j is outputs[i] at entry (the reference's: the previous vector's), or -1
    {
      const mlb_node& m = rec.nodes[(size_t)j].node;
      return m.op == MLB_OP_INPUT && m.iarg >= SynthPass::kOutPlane ? m.iarg - SynthPass::kOutPlane : -1;
    };
    const auto stale = [&](int i)
    {
      return Error(MLB_ERR_UNSUPPORTED, (pv + "reads outputs[" + std::to_string(i) + "] before assigning it; in the "
                                              "reference it still holds the previous vector's output").c_str());
    };
    std::vector<int> uses((size_t)n, 0);
    for (const TNode& t : rec.nodes)
      for (int k = 0; k < MLB_MAX_INS; ++k)
        if (t.node.in[k] >= 0)
        {
          if (entry(t.node.in[k]) >= 0) throw stale(entry(t.node.in[k]));
          ++uses[(size_t)t.node.in[k]];
        }
    for (size_t i = 0; i < rec.outs.size(); ++i)
    {
      const int e = entry(rec.outs[i]);
      if (e == (int)i)
        throw Error(MLB_ERR_UNSUPPORTED,
                    (pv + "leaves outputs[" + std::to_string(i) + "] unassigned: it is neither handed to the base "
                          "Synth::processVector nor assigned after it, so in the reference it holds the previous "
                          "vector's value").c_str());
      if (e >= 0) throw stale(e);
      ++uses[(size_t)rec.outs[i]];
    }
    std::vector<char> drop((size_t)n, 0);  // INPUT nodes nothing reads: outputs at entry, bus rows passed through
    size_t kept = 0;
    for (int j = 0; j < n; ++j)
      kept += !(drop[(size_t)j] = rec.nodes[(size_t)j].node.op == MLB_OP_INPUT && uses[(size_t)j] == 0);
    InstrumentGraph ig;
    bool passThrough = P == nOut && kept == nOut;
    for (size_t i = 0; i < nOut && passThrough; ++i)
    {
      const mlb_node& m = rec.nodes[(size_t)rec.outs[i]].node;
      passThrough = m.op == MLB_OP_INPUT && m.iarg == SynthPass::kBusPlane + (int)i;
    }
    if (passThrough) return ig;
    const std::vector<int> idx = keepNodes(rec.nodes, drop, ig.nodes);
    for (TNode& t : ig.nodes)
      if (t.node.op == MLB_OP_INPUT)
        t.node.iarg = t.node.iarg == SynthPass::kPhasePlane ? (int)(P + C)
                      : t.node.iarg >= SynthPass::kBusPlane ? t.node.iarg - SynthPass::kBusPlane
                                                            : (int)P + t.node.iarg - MLB_VOICE_ROWS;
    for (int32_t o : rec.outs) ig.outs.push_back(idx[(size_t)o]);
    // an output that is an input row as it is, or that an earlier output already is, leaves through a copy of its own,
    // select(x, x, x) (bitwise: exactly x): each graph output is a distinct node
    std::vector<char> isOut(ig.nodes.size(), 0);
    for (int32_t& o : ig.outs)
    {
      if (ig.nodes[(size_t)o].node.op == MLB_OP_INPUT || isOut[(size_t)o])
      {
        TNode c;
        c.node.op = MLB_OP_SELECT;
        for (int k = 0; k < MLB_MAX_INS; ++k) c.node.in[k] = k < 3 ? o : -1;
        c.node.iarg = 0;
        o = (int32_t)ig.nodes.size();
        ig.nodes.push_back(c);
        isOut.push_back(0);
      }
      isOut[(size_t)o] = 1;
    }
    ig.planes = (int)(P + C) + (phase ? 1 : 0);
    std::vector<mlb_node> m;
    for (const TNode& t : ig.nodes) m.push_back(t.node);
    checkLayout(m);
    return ig;
  }

  static bool sameStructure(const VoiceGraph& a, const VoiceGraph& b, std::string& where)
  {
    if (a.nodes.size() != b.nodes.size()) return where = "a different number of nodes", false;
    if (a.outs != b.outs) return where = "different outputs", false;
    if (a.stores.size() != b.stores.size()) return where = "a different number of published stores", false;
    for (size_t k = 0; k < a.stores.size(); ++k)
      if (a.stores[k].signal != b.stores[k].signal || a.stores[k].frames != b.stores[k].frames ||
          a.stores[k].rows != b.stores[k].rows)
        return where = "published store " + std::to_string(k), false;
    for (size_t j = 0; j < a.nodes.size(); ++j)
    {
      const mlb_node &p = a.nodes[j].node, &q = b.nodes[j].node;
      bool same = p.op == q.op && p.iarg == q.iarg && a.nodes[j].name == b.nodes[j].name;
      for (int k = 0; k < MLB_MAX_INS; ++k) same = same && p.in[k] == q.in[k];
      if (!same) return where = "node " + std::to_string(j), false;
    }
    return true;
  }

  // synth voice of lane j of an instrument (MPE lane 0 is the main voice, which no voice reads: voice 0's words)
  int laneVoice(int j) const
  {
    const int v = settings_.mpe ? j - 1 : j;
    return v >= 0 && v < numVoices_ ? v : 0;
  }
  int lane(int instrument, int voice) const { return instrument * lanesPer_ + (settings_.mpe ? 1 : 0) + voice; }

 public:
  TracedSynth() = default;
  TracedSynth(const TracedSynth&) = delete;
  TracedSynth& operator=(const TracedSynth&) = delete;

  // Record processVoice for every voice of `synth` (host only: works without a GPU).  `ctx` carries the instrument
  // settings the synth's setup made (setInputPolyphony, ...) and the sample rate; its outputs are the synth's outputs.
  void trace(Synth& synth, AudioContext& ctx)
  {
    const int V = synth.getNumVoices();
    const int P = ctx.input.polyphony;
    if (ctx.inputs.size() != 0)
      throw Error(MLB_ERR_UNSUPPORTED, "mlb::tr::TracedSynth: the synth has audio inputs; only synths without inputs are traced");
    if (V < 1) throw Error(MLB_ERR_INVALID, "mlb::tr::TracedSynth: the synth has no voices");
    if (P < V || P > (int)EventsToSignals::kMaxVoices)
      throw Error(MLB_ERR_UNSUPPORTED,
                  ("mlb::tr::TracedSynth: polyphony " + std::to_string(P) + " must be in [getNumVoices() = " +
                   std::to_string(V) + ", 16]: EventsToSignals runs only voices 1..polyphony; call setInputPolyphony(" +
                   std::to_string(V) + ")")
                      .c_str());
    if (ctx.input.driftAmount != 0.f)
      throw Error(MLB_ERR_UNSUPPORTED,
                  ("mlb::tr::TracedSynth: drift amount " + std::to_string(ctx.input.driftAmount) +
                   " is not 0: EventsToSignals starts an instrument's voices, drift included, only at its first event "
                   "(awake_), and the device Voice bank runs them from the first vector; call setInputDriftAmount(0)")
                      .c_str());
    if (ctx.input.modCC < 0 || ctx.input.modCC > 127)
      throw Error(MLB_ERR_INVALID, ("mlb::tr::TracedSynth: mod CC " + std::to_string(ctx.input.modCC) + " is not in 0..127").c_str());
    Recorder rec, irec;  // processVoice's, and the instrument section's (Synth::processVector around the base call)
    std::map<const void*, int> functorVoice;
    std::vector<int> controllers;
    bool phase = false;
    std::vector<VoiceGraph> graphs;
    std::vector<SynthPass> passes((size_t)V);  // kept for the whole trace: a Voice& held by a later voice stays valid
    std::vector<PublishStore> stores;          // this pass's storePublishedSignal calls
    SynthPass ipass;                           // the instrument section's: no voice
    int ipassIndex = 0, baseCalls = 0;
    size_t nBus = 0;             // the outputs handed to the base call: the bus rows
    bool baseOnOutputs = false;  // the base call was handed `outputs` itself
    const std::string pv = "mlb::tr::TracedSynth: Synth::processVector ";
    // processVoice for every voice, two passes each, into `outputs` (what the base call was handed)
    const auto traceVoices = [&](DSPVectorDynamic& outputs)
    {
      TraceScope scope(rec, ctx);
      struct StoreSink  // where the synth's stores are recorded, while processVoice runs
      {
        SignalProcessor& sp;
        ~StoreSink() { sp.publishStores_ = nullptr; }
      } sink{synth};
      synth.publishStores_ = &stores;
      rec.functorVoice = &functorVoice;
      rec.voiceEpoch0 = Recorder::lastEpoch() + 1;
      for (int v = 0; v < V; ++v)
      {
        SynthPass& pass = passes[(size_t)v];
        std::vector<int> acc, fin;
        rec.voice = v;
        for (int p = 0; p < 2; ++p)  // pass 1 finds which symbols survive the call; pass 2 is the graph
        {
          rec.staleEpoch = p == 0 ? -2 : rec.epoch;  // pass 2 may read what pass 1 of this voice left
          rec.beginPass();
          stores.clear();
          pass.voice = v;
          pass.controllers = &controllers;
          pass.controllerNode.clear();
          pass.phaseNode = -1;
          for (int r = 0; r < kNumVoiceOutputRows; ++r)
            pass.rows.outputs.row(r) = DSPVector::ofNode(rec.addNode(MLB_OP_INPUT, {}, r, false));
          acc.clear();
          for (size_t i = 0; i < outputs.size(); ++i)
          {
            acc.push_back(rec.addNode(MLB_OP_INPUT, {}, SynthPass::kAccPlane + (int)i, false));
            outputs[i] = DSPVector::ofNode(acc.back());
          }
          ctx.pass_ = &pass;
          if (!synth.isVoiceActive(v, ctx.getInputVoice(v)))
            refuse(v, "is not active (isVoiceActive returned false); every voice is processed on every vector");
          synth.processVoice(v, ctx.getInputVoice(v), ctx.inputs, outputs, &ctx);
          ctx.pass_ = nullptr;
        }
        rec.closeFeedback("processVoice");
        fin.clear();
        for (size_t i = 0; i < outputs.size(); ++i) fin.push_back(outputs[i].resolve());
        phase = phase || pass.phaseNode >= 0;
        graphs.push_back(extract(rec, acc, fin, v, stores));
        std::string where;
        if (v > 0 && !sameStructure(graphs[0], graphs.back(), where))
          refuse(v, "records a different graph from voice 0 (" + where +
                        "); voices may differ in coefficients and state only");
      }
    };
    // Synth::processVector, traced twice as TracedProcessor::trace does (carried members become feedback edges).  The
    // base call leaves bus row i in its outputs[i]; in the second pass it first traces the voices, so that a voice
    // reading what the first pass's instrument section left in a member is caught.  The controller planes follow
    // first use in that second pass.
    {
      TraceScope scope(irec, ctx);
      struct TraceFlag
      {
        SignalProcessor& sp;
        ~TraceFlag() { sp.inSynthTrace_ = false; }
      } flag{synth};
      synth.inSynthTrace_ = true;
      irec.instrument = true;
      irec.voiceEpoch0 = irec.voiceEpoch1 = 0;  // no voice symbol exists until the base call traces the voices
      irec.functorVoice = &functorVoice;
      ipass.controllers = &controllers;
      ipass.base = [&](DSPVectorDynamic& outputs)
      {
        if (++baseCalls > 1)
          throw Error(MLB_ERR_UNSUPPORTED, (pv + "calls the base Synth::processVector more than once in a vector; it "
                                                 "must call it exactly once").c_str());
        if (ipassIndex == 0)
          nBus = outputs.size(), baseOnOutputs = &outputs == &ctx.outputs;
        else
        {
          if (outputs.size() != nBus || (&outputs == &ctx.outputs) != baseOnOutputs)
            throw Error(MLB_ERR_INVALID, (pv + "is not deterministic between calls").c_str());
          traceVoices(outputs);
          irec.voiceEpoch0 = rec.voiceEpoch0, irec.voiceEpoch1 = Recorder::lastEpoch() + 1;
        }
        ctx.pass_ = &ipass;
        for (size_t i = 0; i < outputs.size(); ++i)
          outputs[i] = DSPVector::ofNode(irec.addNode(MLB_OP_INPUT, {}, SynthPass::kBusPlane + (int)i, false));
      };
      for (ipassIndex = 0; ipassIndex < 2; ++ipassIndex)
      {
        irec.staleEpoch = ipassIndex == 0 ? -2 : irec.epoch;
        irec.beginPass();
        baseCalls = 0;
        controllers.clear();
        ipass.controllerNode.clear();
        ipass.phaseNode = -1;
        for (size_t i = 0; i < ctx.outputs.size(); ++i)
          ctx.outputs[i] = DSPVector::ofNode(irec.addNode(MLB_OP_INPUT, {}, SynthPass::kOutPlane + (int)i, false));
        ctx.pass_ = &ipass;
        synth.processVector(ctx.inputs, ctx.outputs, &ctx);
        if (baseCalls == 0)
          throw Error(MLB_ERR_UNSUPPORTED, (pv + "does not call the base Synth::processVector, which runs the voices; "
                                                 "it must call it exactly once").c_str());
      }
      phase = phase || ipass.phaseNode >= 0;
      ctx.pass_ = nullptr;
      irec.closeFeedback("Synth::processVector");
      for (size_t i = 0; i < ctx.outputs.size(); ++i) irec.outs.push_back(ctx.outputs[i].resolve());
    }
    InstrumentGraph ig = instrumentGraph(irec, nBus, ctx.outputs.size(), controllers.size(), phase);
    // the beat phase after the controllers; untouched outputs read one shared +0 row
    const int phasePlane = MLB_VOICE_ROWS + (int)controllers.size();
    for (VoiceGraph& vg : graphs)
    {
      for (TNode& t : vg.nodes)
        if (t.node.op == MLB_OP_INPUT && t.node.iarg == SynthPass::kPhasePlane) t.node.iarg = phasePlane;
      int zero = -1;
      for (int32_t& o : vg.outs)
        if (o < 0)
        {
          if (zero < 0)
          {
            TNode z;
            z.node.op = MLB_OP_PARAM;
            for (int k = 0; k < MLB_MAX_INS; ++k) z.node.in[k] = -1;
            z.node.iarg = 0;
            z.coef.assign(1, 0.f);
            zero = (int)vg.nodes.size();
            vg.nodes.push_back(z);
          }
          o = zero;
        }
    }
    // every stored row leaves the graph through a copy of its own, select(x, x, x) (bitwise: exactly x), so that a row
    // stored twice, stored and also added into an output, or a Voice row stored as it is, is one distinct output each
    std::vector<int32_t> pubOuts;
    for (VoiceGraph& vg : graphs)
    {
      pubOuts.clear();
      for (const PublishStore& st : vg.stores)
        for (int s : st.rows)
        {
          TNode c;
          c.node.op = MLB_OP_SELECT;
          for (int k = 0; k < MLB_MAX_INS; ++k) c.node.in[k] = k < 3 ? s : -1;
          c.node.iarg = 0;
          pubOuts.push_back((int32_t)vg.nodes.size());
          vg.nodes.push_back(c);
        }
    }
    published_ = synth.publishedSignals();
    instrument_ = std::move(ig);
    busPlanes_ = nBus;
    pubOuts_ = pubOuts;
    voices_ = std::move(graphs);
    controllers_ = controllers;
    phase_ = phase;
    settings_ = ctx.input;
    sampleRate_ = ctx.getSampleRate();
    numVoices_ = V;
    nOut_ = ctx.outputs.size();
    nodes_.clear();
    for (const TNode& t : voices_[0].nodes) nodes_.push_back(t.node);
    outs_ = voices_[0].outs;
    checkLayout(nodes_);
  }

  const std::vector<mlb_node>& nodes() const { return nodes_; }
  const std::vector<int32_t>& outs() const { return outs_; }
  const std::vector<int>& controllers() const { return controllers_; }
  const std::vector<PublishDecl>& published() const { return published_; }
  const std::vector<PublishStore>& stores() const { return voices_.at(0).stores; }
  const std::vector<int32_t>& publishedOuts() const { return pubOuts_; }
  bool readsBeatPhase() const { return phase_; }
  size_t outputs() const { return nOut_; }
  size_t busPlanes() const { return busPlanes_; }
  bool hasInstrumentGraph() const { return !instrument_.nodes.empty(); }
  const AudioContext::InputSettings& settings() const { return settings_; }
  int numVoices() const { return numVoices_; }
  // lanes of one instrument: polyphony voices, plus the MPE main voice first
  int lanesPerInstrument() const { return settings_.polyphony + (settings_.mpe ? 1 : 0); }

  // JSON: nodes (with every voice's coefficient and state words), outs, controllers, beat phase, settings -- what a
  // test or a tool needs to rebuild the instrument bank elsewhere (tests/test_synth_trace.py).
  void dump(FILE* f) const
  {
    const AudioContext::InputSettings& s = settings_;
    std::fprintf(f, "{\"n_voices\": %d, \"sample_rate\": %.17g, \"polyphony\": %d, \"mpe\": %d, \"unison\": %d, "
                    "\"mod_cc\": %d, \"pitch_bend\": %.9g, \"mpe_pitch_bend\": %.9g, \"glide_seconds\": %.9g, "
                    "\"drift_amount\": %.9g, \"phase\": %d, \"controllers\": [",
                 numVoices_, sampleRate_, s.polyphony, (int)s.mpe, (int)s.unison, s.modCC, s.pitchBend, s.mpePitchBend,
                 s.glideSeconds, s.driftAmount, (int)phase_);
    for (size_t k = 0; k < controllers_.size(); ++k) std::fprintf(f, "%s%d", k ? ", " : "", controllers_[k]);
    std::fprintf(f, "], \"nodes\": [");
    for (size_t i = 0; i < nodes_.size(); ++i)
    {
      const mlb_node& m = nodes_[i];
      std::fprintf(f, "%s{\"op\": %d, \"in\": [", i ? ", " : "", m.op);
      for (int k = 0; k < MLB_MAX_INS; ++k) std::fprintf(f, "%s%d", k ? ", " : "", m.in[k]);
      std::fprintf(f, "], \"iarg\": %d, \"name\": \"%s\", \"coef\": [", m.iarg, voices_[0].nodes[i].name.c_str());
      const bool again = isAgain(m);
      for (size_t v = 0; v < voices_.size(); ++v)
      {
        std::fprintf(f, "%s[", v ? ", " : "");
        if (!again) printWords(f, voices_[v].nodes[i].coef);
        std::fprintf(f, "]");
      }
      std::fprintf(f, "], \"state\": [");
      for (size_t v = 0; v < voices_.size(); ++v)
      {
        std::fprintf(f, "%s[", v ? ", " : "");
        if (!again) printWords(f, voices_[v].nodes[i].state);
        std::fprintf(f, "]");
      }
      std::fprintf(f, "]}");
    }
    std::fprintf(f, "], \"outs\": [");
    for (size_t i = 0; i < outs_.size(); ++i) std::fprintf(f, "%s%d", i ? ", " : "", outs_[i]);
    std::fprintf(f, "]");
    if (!published_.empty())  // a synth that publishes: its declarations, voice 0's store items, their graph outputs
    {
      std::fprintf(f, ", \"published\": [");
      for (size_t s = 0; s < published_.size(); ++s)
      {
        const PublishDecl& d = published_[s];
        std::fprintf(f, "%s{\"name\": \"%s\", \"max_frames\": %d, \"max_voices\": %d, \"channels\": %d, "
                        "\"octaves_down\": %d}", s ? ", " : "", d.name.c_str(), d.maxFrames, d.maxVoices, d.channels,
                     d.octavesDown);
      }
      std::fprintf(f, "], \"stores\": [");
      const std::vector<PublishStore>& st = voices_[0].stores;
      for (size_t k = 0; k < st.size(); ++k)
      {
        std::fprintf(f, "%s{\"signal\": %d, \"frames\": %d, \"rows\": [", k ? ", " : "", st[k].signal, st[k].frames);
        for (size_t j = 0; j < st[k].rows.size(); ++j) std::fprintf(f, "%s%d", j ? ", " : "", st[k].rows[j]);
        std::fprintf(f, "]}");
      }
      std::fprintf(f, "], \"published_outs\": [");
      for (size_t i = 0; i < pubOuts_.size(); ++i) std::fprintf(f, "%s%d", i ? ", " : "", pubOuts_[i]);
      std::fprintf(f, "]");
    }
    if (hasInstrumentGraph())  // the instrument section: its graph over instrument lanes, one set of words for all
    {
      const InstrumentGraph& ig = instrument_;
      std::fprintf(f, ", \"instrument\": {\"planes\": %d, \"bus_planes\": %zu, \"nodes\": [", ig.planes, busPlanes_);
      for (size_t i = 0; i < ig.nodes.size(); ++i)
      {
        const TNode& t = ig.nodes[i];
        std::fprintf(f, "%s{\"op\": %d, \"in\": [", i ? ", " : "", t.node.op);
        for (int k = 0; k < MLB_MAX_INS; ++k) std::fprintf(f, "%s%d", k ? ", " : "", t.node.in[k]);
        std::fprintf(f, "], \"iarg\": %d, \"name\": \"%s\", \"coef\": [", t.node.iarg, t.name.c_str());
        const bool again = isAgain(t.node);
        if (!again) printWords(f, t.coef);
        std::fprintf(f, "], \"state\": [");
        if (!again) printWords(f, t.state);
        std::fprintf(f, "]}");
      }
      std::fprintf(f, "], \"outs\": [");
      for (size_t i = 0; i < ig.outs.size(); ++i) std::fprintf(f, "%s%d", i ? ", " : "", ig.outs[i]);
      std::fprintf(f, "]}");
    }
    std::fprintf(f, "}\n");
  }

  // Create the banks for `instruments` instruments (needs a GPU): the router and Voice bank over
  // instruments x lanesPerInstrument() lanes, the controller and beat-phase banks if processVoice reads them, the
  // graph over every lane, and one bus per instrument over its getNumVoices() voices (never the MPE main voice).
  void compile(int instruments, unsigned flags = MLB_GRAPH_EXACT)
  {
    if (nodes_.empty()) throw Error(MLB_ERR_INVALID, "mlb::tr::TracedSynth: trace() first");
    if (instruments < 1) throw Error(MLB_ERR_INVALID, "mlb::tr::TracedSynth: instruments must be positive");
    ibank_.reset(), pubBank_.reset(), bank_.reset(), buses_.reset(), times_.reset(), ctrl_.reset(), voiceBank_.reset(),
        routers_.reset();
    const AudioContext::InputSettings& s = settings_;
    const int G = instruments, NR = lanesPerInstrument(), V = G * NR;
    instruments_ = G, lanesPer_ = NR;
    std::vector<int32_t> poly((size_t)G, s.polyphony), first((size_t)G), unison((size_t)G, s.unison ? 1 : 0),
        modCC((size_t)G, s.modCC), busFirst((size_t)G), busCount((size_t)G, numVoices_);
    std::vector<int32_t> vi((size_t)V), mainVoice((size_t)V, -1), inst((size_t)V);
    std::vector<float> glide((size_t)V, s.glideSeconds), drift((size_t)V, s.driftAmount), bend((size_t)V, s.pitchBend);
    for (int g = 0; g < G; ++g)
    {
      first[(size_t)g] = g * NR, busFirst[(size_t)g] = lane(g, 0);
      for (int j = 0; j < NR; ++j)
      {
        const size_t l = (size_t)(g * NR + j);
        vi[l] = s.mpe ? j : j + 1;
        inst[l] = g;
        if (s.mpe && j > 0) mainVoice[l] = g * NR, bend[l] = s.mpePitchBend;
      }
    }
    const float sr = (float)sampleRate_;
    routers_.reset(new RouterBank(G, s.mpe ? 1 : 0, poly.data(), first.data(), V, unison.data(), modCC.data()));
    voiceBank_.reset(new VoiceBank(V, sr, vi.data(), glide.data(), drift.data(), bend.data(), s.mpe ? 0u : MLB_VOICES_MIDI));
    if (s.mpe) voiceBank_->setMainVoices(mainVoice.data());
    if (!controllers_.empty())
    {
      ctrl_.reset(new ControllerBank(G, sr, s.mpe ? 1 : 0, controllers_.data(), (int)controllers_.size()));
      ctrl_->setVoiceMap(inst.data(), V);
    }
    if (phase_)
    {
      times_.reset(new ProcessTimeBank(G, sampleRate_));
      times_->setVoiceMap(inst.data(), V);
    }
    std::vector<int32_t> outs = outs_;  // the audio outputs, then the published rows
    outs.insert(outs.end(), pubOuts_.begin(), pubOuts_.end());
    bank_.reset(new DeviceBank(nodes_, outs, V, flags));
    buses_.reset(new Buses(V, G, busFirst.data(), busCount.data()));
    if (!published_.empty())
    {
      std::vector<mlb_published_signal> sig;
      for (const PublishDecl& d : published_) sig.push_back({d.maxFrames, d.maxVoices, d.channels, d.octavesDown});
      std::vector<mlb_published_store> st;
      for (const PublishStore& k : voices_[0].stores) st.push_back({k.signal, k.frames});
      pubBank_.reset(new PublishedBank(V, G, busFirst.data(), busCount.data(), sig, st));
    }
    if (hasInstrumentGraph())
    {
      std::vector<mlb_node> in;
      for (const TNode& t : instrument_.nodes) in.push_back(t.node);
      ibank_.reset(new DeviceBank(in, instrument_.outs, G, flags));
      for (size_t i = 0; i < in.size(); ++i)
        for (int g = 0; g < G; ++g) loadWords(*ibank_, (int)i, g, instrument_.nodes[i]);
      ibank_->commit();
    }
    overflow_.assign((size_t)G, 0);
    for (size_t i = 0; i < nodes_.size(); ++i)
      for (int l = 0; l < V; ++l) loadWords(*bank_, (int)i, l, voices_[(size_t)laneVoice(l % NR)].nodes[i]);
    commit();
  }
  void commit() { bank().commit(); }
  int instruments() const { return instruments_; }
  const char* kernelName() const { return bank_ ? bank_->kernelName() : ""; }
  // the instrument graph's kernel ("" without an instrument graph)
  const char* instrumentKernelName() const { return ibank_ ? ibank_->kernelName() : ""; }

  // per-instrument, per-voice value of a tr::param(name, ...) scalar; call commit() after a batch of changes
  void setParam(const std::string& name, int instrument, int voice, float value)
  {
    DeviceBank& bank = this->bank();
    if (instrument < 0 || instrument >= instruments_ || voice < 0 || voice >= numVoices_)
      throw Error(MLB_ERR_INVALID, "mlb::tr::TracedSynth: no such instrument or voice");
    for (size_t i = 0; i < nodes_.size(); ++i)
      if (voices_[0].nodes[i].name == name)
      {
        bank.setParam((int)i, lane(instrument, voice), value);
        return;
      }
    throw Error(MLB_ERR_INVALID, ("mlb::tr::TracedSynth: no param named " + name).c_str());
  }

  // nBlocks vectors of every instrument: raw events (offsets [nBlocks][instruments + 1] into events, times 0..63 in
  // the vector) and, if processVoice reads the beat phase, host transport updates (timeOffsets [nBlocks][instruments + 1]
  // into transports) in; bus [nBlocks][outputs][instruments][64] out -- what each instrument's Synth::processVector
  // writes to its outputs.  Routing, Voice rows, controllers, beat phase, graph and bus sum run on the device
  // (mlb_synth_process_context_host); state carries over from call to call.
  void process(const int32_t* offsets, const mlb_event* events, int nEvents, const int32_t* timeOffsets,
               const mlb_transport* transports, int nTransports, float* bus, int nBlocks)
  {
    mlb_graph* graph = bank().handle();
    if (ibank_)  // the instrument graph on the bus sums in every time chunk (K14 before it)
      check(mlb_synth_process_instrument_host(
          routers_->handle(), voiceBank_->handle(), ctrl_ ? ctrl_->handle() : nullptr, times_ ? times_->handle() : nullptr,
          graph, buses_->handle(), pubBank_ && pubBank_->planes() > 0 ? pubBank_->handle() : nullptr, ibank_->handle(),
          offsets, events, nEvents, times_ ? timeOffsets : nullptr, times_ ? transports : nullptr,
          times_ ? nTransports : 0, bus, nBlocks));
    else if (pubBank_ && pubBank_->planes() > 0)  // K14 after the bus sum in every time chunk
      check(mlb_synth_process_published_host(
          routers_->handle(), voiceBank_->handle(), ctrl_ ? ctrl_->handle() : nullptr, times_ ? times_->handle() : nullptr,
          graph, buses_->handle(), pubBank_->handle(), offsets, events, nEvents, times_ ? timeOffsets : nullptr,
          times_ ? transports : nullptr, times_ ? nTransports : 0, bus, nBlocks));
    else
      check(mlb_synth_process_context_host(routers_->handle(), voiceBank_->handle(), ctrl_ ? ctrl_->handle() : nullptr,
                                           times_ ? times_->handle() : nullptr, graph, buses_->handle(), offsets, events,
                                           nEvents, times_ ? timeOffsets : nullptr, times_ ? transports : nullptr,
                                           times_ ? nTransports : 0, nullptr, nullptr, bus, nBlocks));
    // A voice's record holds MLB_VOICE_MAX_EVENTS note events per vector (in unison every note event goes to every
    // voice); the router drops and counts the rest, where the reference's Voice would have written them all.
    std::vector<int64_t> overflow((size_t)instruments_);
    routers_->counters(overflow.data(), nullptr);
    overflow.swap(overflow_);
    for (int g = 0; g < instruments_; ++g)
      if (overflow[(size_t)g] != overflow_[(size_t)g])
        throw Error(MLB_ERR_UNSUPPORTED,
                    ("mlb::tr::TracedSynth: instrument " + std::to_string(g) + ": " +
                     std::to_string(overflow_[(size_t)g] - overflow[(size_t)g]) +
                     " note events found their voice's record full (" + std::to_string(MLB_VOICE_MAX_EVENTS) +
                     " per voice and vector) and were dropped; this call's bus rows differ from the reference")
                        .c_str());
  }

  // Restart the listed instruments between two process() calls: from the next vector each behaves as a newly
  // constructed AudioContext + Synth set up as at trace time (the reference's `ctxs[g] = make_unique<AudioContext>(..);
  // synths[g] = make_unique<...>(..)`), fed only the events and transport updates from then on; the others are
  // untouched, bit for bit.  The graph lanes go back to the words of the last commit(), so setParam values stay.  One
  // launch per bank that holds state (routers, Voice rows, controllers and beat phase if built, graph, published
  // signals and instrument graph if built), none for an empty list; an instrument out of range throws before anything is written.
  void restart(const std::vector<int>& instruments)
  {
    DeviceBank& bank = this->bank();
    const std::vector<int32_t> inst(instruments.begin(), instruments.end());
    std::vector<int32_t> lanes;
    for (int g : instruments)
      for (int j = 0; j < lanesPer_; ++j) lanes.push_back(g * lanesPer_ + j);
    routers_->reset(inst);  // first: it refuses an instrument out of range before any bank is written
    voiceBank_->reset(lanes);
    if (ctrl_) ctrl_->reset(inst);
    if (times_) times_->reset(inst);
    bank.reset(lanes);
    if (pubBank_) pubBank_->reset(inst);
    if (ibank_) ibank_->reset(inst);
  }

  // getPublishedSignals()[name]->readLatest(dest, frames) of every instrument in one call (MLSignalProcessor.cpp:19-28):
  // dest [instruments][frames * channels] (what a read does not fill is zero), counts [instruments] the floats read.
  void readLatest(const Path& name, int frames, float* dest, int32_t* counts)
  {
    publishedBank().read(signalIndex(name), MLB_PUBLISHED_READ_LATEST, frames, dest, counts);
  }
  // ...->read(dest, frames): the oldest frames, consumed; counts the floats read
  void read(const Path& name, int frames, float* dest, int32_t* counts)
  {
    publishedBank().read(signalIndex(name), MLB_PUBLISHED_READ, frames, dest, counts);
  }
  // ...->peekLatest(dest, frames): the newest frames, nothing consumed; counts 1 where they were copied, 0 where fewer
  // were available (the reference copies nothing then, and dest stays zero here)
  void peekLatest(const Path& name, int frames, float* dest, int32_t* counts)
  {
    publishedBank().read(signalIndex(name), MLB_PUBLISHED_PEEK, frames, dest, counts);
  }
  // ...->getAvailableFrames() into counts [instruments]
  void availableFrames(const Path& name, int32_t* counts)
  {
    publishedBank().read(signalIndex(name), MLB_PUBLISHED_AVAILABLE, 0, nullptr, counts);
  }

 private:
  PublishedBank& publishedBank() const
  {
    if (!pubBank_)
      throw Error(MLB_ERR_INVALID, bank_ ? "mlb::tr::TracedSynth: the synth publishes no signal"
                                         : "mlb::tr::TracedSynth: compile() first");
    return *pubBank_;
  }
  int signalIndex(const Path& name) const
  {
    for (size_t s = 0; s < published_.size(); ++s)
      if (published_[s].name == name) return (int)s;
    throw Error(MLB_ERR_INVALID, ("mlb::tr::TracedSynth: no published signal named " + name).c_str());
  }
};

}  // namespace tr
}  // namespace mlb
