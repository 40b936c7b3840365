/*
 * mlb200.h -- C ABI of the H100-native (sm_90a) DSPVector voice-chain engine.
 *
 * This is the drop-in boundary for ONE hot path of madronalib: the DSPVector
 * processing chain (generators -> stateful filters -> elementwise ops) batched
 * over many independent voices.  The reference has no FFI for this path (it is
 * header-only C++ templates), so each entry point below cites the reference
 * interface it stands in for.  Everything here is plain C: pointers, sizes and
 * int status codes; no C++ or torch types cross the boundary.
 *
 * Vocabulary follows the reference:
 *   block   = one DSPVector = kFloatsPerDSPVector = 64 samples
 *             (reference: source/DSP/MLDSPMath.h:8-9)
 *   row     = 64 contiguous f32 (256 B); a DSPVectorArray<ROWS> is ROWS rows
 *             (reference: source/DSP/MLDSPOps.h:94-127)
 *   voice   = one independent processor instance = one row of a Bank<T,ROWS>
 *             (reference: source/DSP/MLDSPFunctional.h:321-360)
 *   graph   = a fixed DAG of generator / filter / op nodes evaluated once per
 *             block for every voice (what a user's SignalProcessFn does with
 *             functors; reference: source/app/MLSignalProcessBuffer.h:18,
 *             examples/audio-and-midi/sine.cpp:21-43; the absent source/procs
 *             runtime graph, source/procs/MLProcMultiply.cpp:29-46)
 *
 * Signal layout (all f32, little endian), for T blocks and V voices:
 *   inputs   in [T][n_in ][V][64]   -- plane (t,k) is exactly the
 *                                      DSPVectorArray<V> a Bank::operator()
 *                                      receives as argument k on block t
 *   outputs  out[T][n_out][V][64]   -- plane (t,c) is the DSPVectorArray<V>
 *                                      a Bank would return for output c
 *   mix bus  mix[T][n_out][64]      -- sum over voices of each output plane
 *                                      (reference: addRows, MLDSPOps.h:1349-1359;
 *                                       Synth::processVector, source/app/MLSynth.h:36-60)
 *
 * Per-voice state and coefficients are struct-of-arrays of 32-bit words:
 *   state[n_state_words][V]  (u32 / f32 bit patterns), coef[n_coef_words][V] (f32)
 * Word order = node order, then slot order as listed in MLB_OP_TABLE below.
 */
#ifndef MLB200_H
#define MLB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MLB_BLOCK 64           /* kFloatsPerDSPVector, MLDSPMath.h:8-9 */
#define MLB_MAX_INS 7         /* signal inputs of a node: x + up to 6 coefficient rows (HiShelf::_vcoeffs) */
#define MLB_FDN_LINES 8        /* FDN<8>, MLDSPFilters.h:1162 */
#define MLB_ABI_VERSION 2     /* 2: MLB_MAX_INS 3 -> 7 (sizeof(mlb_node) 20 -> 36), coefficient-row filters */

/* ---- status codes (the reference has no error channel; SURVEY 8b) ---- */
enum {
  MLB_OK = 0,
  MLB_ERR_INVALID = 1,   /* bad argument / malformed graph */
  MLB_ERR_CUDA = 2,      /* CUDA runtime / driver error (see mlb_last_error) */
  MLB_ERR_NO_DEVICE = 3, /* no usable sm_90 device: there is NO CPU fallback */
  MLB_ERR_ALLOC = 4,
  MLB_ERR_UNSUPPORTED = 5
};

/*
 * Node table: X(NAME, id, n_in, n_state, n_coef)
 *   n_in    signal inputs (rows produced by earlier nodes)
 *   n_state per-voice 32-bit state words carried block to block
 *   n_coef  per-voice f32 coefficient words
 * Citations: G = source/DSP/MLDSPGens.h, F = source/DSP/MLDSPFilters.h,
 *            O = source/DSP/MLDSPOps.h, M = source/DSP/MLDSPMathSSE.h
 */
#define MLB_OP_TABLE(X)                                                                  \
  /* sources */                                                                          \
  X(INPUT, 0, 0, 0, 0)          /* external signal row in[t][iarg][v][:]             */ \
  X(PARAM, 1, 0, 0, 1)          /* per-voice float -> DSPVector broadcast, O:157     */ \
  /* generators */                                                                       \
  X(NOISE, 2, 0, 1, 0)          /* NoiseGen, G:109-148; state: mSeed                 */ \
  X(PHASOR, 3, 1, 1, 0)         /* PhasorGen(freq), G:177-203; state: mOmega32       */ \
  X(SINE, 4, 1, 1, 0)           /* SineGen(freq), G:316-338,373-381; state: mOmega32 */ \
  X(SAW, 5, 1, 1, 0)            /* SawGen(freq), G:285-311,362-369,395-402           */ \
  X(PULSE, 6, 2, 1, 0)          /* PulseGen(freq,width), G:342-358,383-393           */ \
  X(TICK, 7, 1, 1, 0)           /* TickGen(freq), G:24-47; state: mOmega (f32)       */ \
  X(ONESHOT, 8, 1, 3, 0)        /* OneShotGen(freq), G:221-252; state mOmega32,mGate,*/ \
                                /* mOmegaPrev; trigger() = set_state {0,1,0}         */ \
  X(IMPULSE, 9, 1, 2, 0)        /* ImpulseGen(freq), G:53-103: a 17-tap Blackman-windowed sinc fired at every  */ \
                                /* phase wrap; state _omega (f32), _outputCounter (i32; 0 at construction)     */ \
  /* SVF family ("Biquad" stand-ins) -- state: ic1eq, ic2eq */                           \
  X(LOPASS, 10, 1, 2, 3)        /* F:51-133   coef g0,g1,g2                          */ \
  X(HIPASS, 11, 1, 2, 4)        /* F:155-197  coef g0,g1,g2,k                        */ \
  X(BANDPASS, 12, 1, 2, 3)      /* F:199-240  coef g0,g1,g2                          */ \
  X(LOSHELF, 13, 1, 2, 5)       /* F:242-302  coef a1,a2,a3,m1,m2                    */ \
  X(HISHELF, 14, 1, 2, 6)       /* F:321-383  coef a1,a2,a3,m0,m1,m2                 */ \
  X(BELL, 15, 1, 2, 4)          /* F:402-442  coef a1,a2,a3,m1                       */ \
  /* one-pole family */                                                                  \
  X(ONEPOLE, 16, 1, 1, 2)       /* F:446-481  state y1; coef a0,b1                   */ \
  X(DCBLOCKER, 17, 1, 2, 1)     /* F:489-513  state x1,y1; coef c                    */ \
  X(DIFFERENTIATOR, 18, 1, 1, 0)/* F:517-535  state x1                               */ \
  X(INTEGRATOR, 19, 1, 1, 1)    /* F:539-558  state y1; coef leak                    */ \
  /* FDN<8>: mono in -> stereo out.  Output row of FDN8 is sumL, FDN8_R(in=fdn) is   */ \
  /* sumR (concatRows(sumL,sumR), F:1237).  state: 8 OnePole y1.  coef: 8x a0,b1,    */ \
  /* 8 feedback gains, 8 delay lengths (float-valued ints).  Delay rings + carried   */ \
  /* mDelayInputVectors live in separate delay memory (mlb_graph_delay_bytes).       */ \
  X(FDN8, 20, 1, 8, 32)         /* F:1162-1239                                       */ \
  X(FDN8_R, 21, 1, 0, 0)                                                                 \
  /* envelope followers / envelopes / one-sample allpass */                              \
  X(PEAK, 22, 1, 2, 3)          /* F:562-615 state y1,peakHoldCounter(i32); coef a0, */ \
                                /* b1,peakHoldSamples (float-valued int)             */ \
  X(RMS, 23, 1, 1, 2)           /* F:619-653 state y1; coef a0,b1                    */ \
  X(ADSR, 24, 1, 8, 4)          /* F:657-797 state y,y1,x1,threshold,target,k,amp,   */ \
                                /* segment(i32; 4 = off); coef ka,kd,s,kr            */ \
  X(ALLPASS1, 25, 1, 2, 1)      /* F:918-964 state x1,y1; coef a                     */ \
  /* control-rate smoothers: the scalar argument is sample 0 of the operand row      */ \
  X(GLIDE, 26, 1, 3, 2)         /* LinearGlide(float), G:433-515; state step,target, */ \
                                /* mVectorsRemaining(i32, -1 idle); coef             */ \
                                /* mVectorsPerGlide (float-valued int), mDyPerVector;*/ \
                                /* mCurrVec is a 64-float row in delay memory        */ \
  X(INTERPOLATOR1, 27, 1, 1, 0) /* G:412-424 state currentValue                      */ \
  X(SAMPLE_GLIDE, 28, 1, 4, 2)  /* SampleAccurateLinearGlide::nextSample per sample, */ \
                                /* G:517-590; state curr,step,target,remaining(i32); */ \
                                /* coef mSamplesPerGlide (float-valued int),         */ \
                                /* mDyPerSample                                      */ \
  /* unary float ops, O:584-614,825 */                                                   \
  X(SQRT, 30, 1, 0, 0)                                                                   \
  X(SQRT_APPROX, 31, 1, 0, 0)                                                            \
  X(ABS, 32, 1, 0, 0)                                                                    \
  X(SIGN, 33, 1, 0, 0)                                                                   \
  X(SIGNBIT, 34, 1, 0, 0)                                                                \
  X(SIN, 35, 1, 0, 0)                                                                    \
  X(COS, 36, 1, 0, 0)                                                                    \
  X(LOG, 37, 1, 0, 0)                                                                    \
  X(EXP, 38, 1, 0, 0)                                                                    \
  X(LOG2, 39, 1, 0, 0)                                                                   \
  X(EXP2, 40, 1, 0, 0)                                                                   \
  X(SIN_APPROX, 41, 1, 0, 0)                                                             \
  X(COS_APPROX, 42, 1, 0, 0)                                                             \
  X(EXP_APPROX, 43, 1, 0, 0)                                                             \
  X(LOG_APPROX, 44, 1, 0, 0)                                                             \
  X(LOG2_APPROX, 45, 1, 0, 0)                                                            \
  X(EXP2_APPROX, 46, 1, 0, 0)                                                            \
  X(FRACTIONAL_PART, 47, 1, 0, 0)                                                        \
  /* binary float ops, O:640-649 */                                                      \
  X(ADD, 50, 2, 0, 0)                                                                    \
  X(SUBTRACT, 51, 2, 0, 0)                                                               \
  X(MULTIPLY, 52, 2, 0, 0)                                                               \
  X(DIVIDE, 53, 2, 0, 0)                                                                 \
  X(DIVIDE_APPROX, 54, 2, 0, 0)                                                          \
  X(POW, 55, 2, 0, 0)                                                                    \
  X(POW_APPROX, 56, 2, 0, 0)                                                             \
  X(MIN, 57, 2, 0, 0)                                                                    \
  X(MAX, 58, 2, 0, 0)                                                                    \
  /* ternary float ops, O:744-748 */                                                     \
  X(LERP, 60, 3, 0, 0)                                                                   \
  X(INVERSE_LERP, 61, 3, 0, 0)                                                           \
  X(CLAMP, 62, 3, 0, 0)                                                                  \
  X(WITHIN, 63, 3, 0, 0)                                                                 \
  /* conversions, O:796-797,819-820 (int rows are 32-bit patterns in f32 storage) */     \
  X(ROUND_F2I, 70, 1, 0, 0)                                                              \
  X(TRUNC_F2I, 71, 1, 0, 0)                                                              \
  X(INT_TO_FLOAT, 72, 1, 0, 0)                                                           \
  X(UNSIGNED_TO_FLOAT, 73, 1, 0, 0)                                                      \
  /* comparisons -> all-ones / zero masks, O:851-856 */                                  \
  X(EQUAL, 80, 2, 0, 0)                                                                  \
  X(NOT_EQUAL, 81, 2, 0, 0)                                                              \
  X(GREATER_THAN, 82, 2, 0, 0)                                                           \
  X(GREATER_EQUAL, 83, 2, 0, 0)                                                          \
  X(LESS_THAN, 84, 2, 0, 0)                                                              \
  X(LESS_EQUAL, 85, 2, 0, 0)                                                             \
  /* select(a, b, mask) bitwise, O:886,917; int add/sub O:713-714 */                     \
  X(SELECT, 90, 3, 0, 0)                                                                 \
  X(ADD_INT32, 91, 2, 0, 0)                                                              \
  X(SUBTRACT_INT32, 92, 2, 0, 0)                                                         \
  /* ---- delay-memory ops (ids >= 100).  Rings and 64-float rows live in the graph's  */ \
  /* delay memory (MLB_OP_MEM_TABLE below), zeroed by mlb_graph_set_coefs /           */ \
  /* mlb_graph_clear_delays.  "maxDelay" is the argument the caller would hand to the */ \
  /* functor's own setMaxDelayInSamples; the ring of voice v has                      */ \
  /* 1 << bitsToContain(floor(maxDelay_v') + 64) samples (F:822-830).                 */ \
  X(INTEGER_DELAY, 100, 1, 0, 2)      /* IntegerDelay(vx), F:834-875; coef delay      */ \
                                      /* (float-valued int), maxDelay                 */ \
  X(INTEGER_DELAY_VAR, 101, 2, 0, 1)  /* IntegerDelay(x, delay), F:877-896; coef      */ \
                                      /* maxDelay                                     */ \
  X(FRACTIONAL_DELAY, 102, 1, 2, 2)   /* FractionalDelay(vx), F:971-1030; state       */ \
                                      /* allpass x1,y1; coef delay, maxDelay          */ \
  X(FRACTIONAL_DELAY_VAR, 103, 2, 2, 1) /* FractionalDelay(vx, vDelay), F:1033-1042   */ \
  X(PITCHBEND_DELAY, 104, 2, 8, 1)    /* PitchbendableDelay(x, vDelay), F:1079-1105;  */ \
                                      /* state 2 x {x1,y1,intDelay(i32),apCoeff};     */ \
                                      /* coef maxDelay                                */ \
  X(ALLPASS_INT, 105, 1, 0, 3)        /* Allpass<IntegerDelay>(x), F:1111-1143; coef  */ \
                                      /* mGain, delay, maxDelay                       */ \
  X(ALLPASS_FRAC, 106, 1, 2, 3)       /* Allpass<FractionalDelay>(x); state x1,y1     */ \
  X(ALLPASS_PB, 107, 2, 8, 2)         /* Allpass<PitchbendableDelay>(x, vDelay),      */ \
                                      /* F:1145-1154; state as PITCHBEND_DELAY; coef  */ \
                                      /* mGain, maxDelay                              */ \
  /* one-block feedback edge (a DSPVector member kept between processVector calls,    */ \
  /* examples/audio-and-midi/reverb.cpp:34,115-116): FEEDBACK_READ yields the row     */ \
  /* stored by the FEEDBACK_WRITE of the previous block (zero at start);              */ \
  /* FEEDBACK_WRITE(in0).iarg = node index of its FEEDBACK_READ; it passes in0 on.    */ \
  X(FEEDBACK_READ, 108, 0, 0, 0)                                                         \
  X(FEEDBACK_WRITE, 109, 1, 0, 0)                                                        \
  /* ---- resampler primitives (SURVEY 8f row 4): HalfBandFilter, F:1245-1310.  State:   */ \
  /* the four Allpass1 {x1,y1} pairs apa0, apa1, apb0, apb1, then b1 (9 words).          */ \
  /* HALFBAND_UP(x) = upsampleFirstHalf(x); HALFBAND_UP_2(in = that node) =              */ \
  /* upsampleSecondHalf(x) of the SAME filter (two rows at twice the rate);              */ \
  /* HALFBAND_DOWN(x1, x2) = downsample(x1, x2) (two rows in, one row out).              */ \
  /* Upsample2xFunction(fn, x) (MLDSPFunctional.h:114-160) is (fn's functors: MLB_AGAIN) */ \
  /* HALFBAND_DOWN(fn(HALFBAND_UP(x)), fn(HALFBAND_UP_2(x))).                            */ \
  X(HALFBAND_UP, 110, 1, 9, 0)                                                           \
  X(HALFBAND_UP_2, 111, 1, 0, 0)                                                         \
  X(HALFBAND_DOWN, 112, 2, 9, 0)                                                         \
  /* Downsample2xFunction(fn, x) (MLDSPFunctional.h:166-223) with a stateless fn, as a node pair around  */ \
  /* fn's nodes: DOWN2X_IN(x) yields downsample(mInputBuffer, x) on every second block (phase 1) and   */ \
  /* stores x on the others; DOWN2X_OUT(fn(...)) returns upsampleFirstHalf on phase-1 blocks and the   */ \
  /* buffered second half on the others.  State: HalfBandFilter (9 words) + mPhase; one member row     */ \
  /* each (mInputBuffer / mOutputBuffer).  fn's nodes run on every block; their rows on phase-0 blocks */ \
  /* are never used.                                                                                   */ \
  X(DOWN2X_IN, 114, 1, 10, 0)                                                            \
  X(DOWN2X_OUT, 115, 1, 10, 0)                                                           \
  /* TempoLock(x, dydx, isr), F:1478-1579: in0 = input phasor row, in1 = ratio (sample   */ \
  /* 0 of the row); state _omega, _x1v (fresh: _omega = -1); coef isr                    */ \
  X(TEMPO_LOCK, 113, 2, 2, 1)                                                            \
  /* ---- filters whose coefficients are SIGNAL ROWS (one value per sample), i.e. the modulated /  */ \
  /* swept forms of the reference.  in0 = audio, in1.. = the coefficient rows in the order of the   */ \
  /* reference's coeffNames enums; a PARAM operand is a constant row.  state: ic1eq, ic2eq.         */ \
  /* The rows are designed on the host with the reference's own libm calls (mlb_coeffs_lopass_vec = */ \
  /* Lopass::makeCoeffsVec, mlb_interpolate_coeffs_linear = interpolateCoeffsLinear of two          */ \
  /* makeCoeffs results = LoShelf/HiShelf::vcoeffs) or on the device from two endpoints (RAMP).     */ \
  X(LOPASS_V, 116, 4, 2, 0)     /* Lopass::operator()(vx, omega, k) after its makeCoeffsVec,         */ \
                                /* F:136-152: in1..3 = rows g0, g1, g2                               */ \
  X(LOSHELF_V, 117, 6, 2, 0)    /* LoShelf::operator()(vx, vc), F:304-319: rows a1,a2,a3,m1,m2       */ \
  X(HISHELF_V, 118, 7, 2, 0)    /* HiShelf::operator()(vx, vc), F:385-400: rows a1,a2,a3,m0,m1,m2    */ \
  /* Lopass::operator()(vx, omega, k) with makeCoeffsVec evaluated ON THE DEVICE (F:97-115: clamps,  */ \
  /* two sinf and one division per sample).  CUDA sinf is not glibc sinf: this node is the           */ \
  /* "approximate variant" of LOPASS_V with a stated tolerance (DESIGN.md 5), never bit-exact.      */ \
  X(LOPASS_MOD, 119, 3, 2, 0)                                                                        \
  /* interpolateDSPVectorLinear(start, end), O:986-990: row[n] = n * ((end - start) / 64) +          */ \
  /* (start + (end - start) / 64); the scalar arguments are sample 0 of the operand rows (or PARAMs). */ \
  /* One RAMP per coefficient = interpolateCoeffsLinear (F:32-44) on the device.                     */ \
  X(RAMP, 120, 2, 0, 0)

/* Delay memory per voice: X(NAME, n_rows, n_rings) -- 64-float rows and rings.
 * PitchbendableDelay's two FractionalDelays are fed the same input on every sample
 * (F:1101-1103), so their two rings always hold identical data: one ring serves both. */
#define MLB_OP_MEM_TABLE(X) \
  X(GLIDE, 1, 0)            \
  X(INTEGER_DELAY, 0, 1)    \
  X(INTEGER_DELAY_VAR, 0, 1)\
  X(FRACTIONAL_DELAY, 0, 1) \
  X(FRACTIONAL_DELAY_VAR, 0, 1) \
  X(PITCHBEND_DELAY, 0, 1)  \
  X(ALLPASS_INT, 1, 1)      \
  X(ALLPASS_FRAC, 1, 1)     \
  X(ALLPASS_PB, 1, 1)       \
  X(FEEDBACK_READ, 1, 0)    \
  X(DOWN2X_IN, 1, 0)        \
  X(DOWN2X_OUT, 1, 0)

/* ids in [MLB_OP_MAP_FIRST, MLB_OP_MAP_END) are the stateless elementwise ops (mlb_map_*) */
#define MLB_OP_MAP_FIRST 30
#define MLB_OP_MAP_END 100

typedef enum mlb_op {
#define MLB_X_ENUM(NAME, id, nin, nst, nco) MLB_OP_##NAME = id,
  MLB_OP_TABLE(MLB_X_ENUM)
#undef MLB_X_ENUM
  MLB_OP__END = 121
} mlb_op;

/* One node of a voice graph.  in[] index earlier nodes (topological order). */
typedef struct mlb_node {
  int32_t op;               /* mlb_op */
  int32_t in[MLB_MAX_INS];  /* producer node indices, -1 = unused */
  int32_t iarg;             /* INPUT: external input plane index k; FEEDBACK_WRITE: its FEEDBACK_READ node;
                               a functor node: 0, or MLB_AGAIN(t) (below) */
} mlb_node;

/* The same functor OBJECT called again in the same vector: a node with iarg = MLB_AGAIN(t) is a further call of
 * the functor of the earlier node t (same op, itself not an AGAIN node) on other inputs.  It owns no state,
 * coefficient or member-row words: it reads and writes those of node t, so the functor ticks once per call in node
 * order -- what happens to the functors inside a process function that Upsample2xFunction runs twice per vector
 * (MLDSPFunctional.h:114-160: fn(upsampled first half), fn(upsampled second half); the reference's tutorial wraps a
 * sine generator this way, examples/tutorial/dspOpsExample.cpp:100-102).  Allowed for ops that have state or
 * coefficients and no ring in delay memory (a ring's write index is the vector count, MLDSPFilters.h:836-851 run
 * once per vector), and not for INPUT / PARAM / FEEDBACK_* / FDN8* / HALFBAND_UP_2 / DOWN2X_*.  (HALFBAND_UP and
 * HALFBAND_DOWN may be: the stages of an Upsampler(octaves) / Downsampler(octaves) run their one filter several times per
 * vector, MLDSPFilters.h:1345-1372,1427-1448; a HALFBAND_UP called again gets its own HALFBAND_UP_2.)  Such graphs run on
 * the graph interpreter; node t and its AGAIN nodes are kept in one pipeline stage. */
#define MLB_AGAIN(t) (-1 - (t))
#define MLB_AGAIN_TARGET(iarg) (-1 - (iarg))

/* Word offsets of every node inside the state / coef SoA. */
typedef struct mlb_layout {
  int32_t n_state_words;
  int32_t n_coef_words;
  int32_t n_inputs;   /* 1 + max iarg over INPUT nodes, 0 if none */
} mlb_layout;

/* op metadata (pure host functions, no GPU needed) */
int mlb_op_info(int op, int* n_in, int* n_state, int* n_coef); /* MLB_OK or MLB_ERR_INVALID */
const char* mlb_op_name(int op);
/* validate a graph and compute its SoA layout; state_off/coef_off may be NULL,
 * else they receive n_nodes word offsets each. */
int mlb_graph_layout(const mlb_node* nodes, int n_nodes, mlb_layout* layout,
                     int32_t* state_off, int32_t* coef_off);

/* ---- coefficient design on the host (glibc libm, same as the reference) ----
 * Each writes the node's coef words for ONE voice.  Cited reference makeCoeffs:
 * Lopass F:85-95, Hipass F:168-178, Bandpass F:212-222, LoShelf F:270-281,
 * HiShelf F:350-362, Bell F:415-425, OnePole F:458-462, DCBlocker F:498,
 * dBToGain F:30. */
void mlb_coeffs_lopass(float omega, float k, float out3[3]);
void mlb_coeffs_hipass(float omega, float k, float out4[4]);
void mlb_coeffs_bandpass(float omega, float k, float out3[3]);
void mlb_coeffs_loshelf(float omega, float k, float A, float out5[5]);
void mlb_coeffs_hishelf(float omega, float k, float A, float out6[6]);
void mlb_coeffs_bell(float omega, float k, float A, float out4[4]);
void mlb_coeffs_onepole(float omega, float out2[2]);
float mlb_coeffs_dcblocker(float omega);
float mlb_db_to_gain(float dB);
/* Peak::makeCoeffs F:578-582, RMS::makeCoeffs F:632-636 (a0, b1); ADSR::calcCoeffs F:676-683
 * (ka, kd, s, kr); Allpass1::makeCoeffs F:936-941; LinearGlide::setGlideTimeInSamples G:443-448
 * and SampleAccurateLinearGlide::setGlideTimeInSamples G:527-532 (count as float, 1/count). */
void mlb_coeffs_peak(float omega, float out2[2]);
void mlb_coeffs_rms(float omega, float out2[2]);
void mlb_coeffs_adsr(float a, float d, float s, float r, float sr, float out4[4]);
float mlb_coeffs_allpass1(float d);
void mlb_coeffs_glide(float time_in_samples, float out2[2]);
/* ImpulseGen's table (its constructor, G:64-78): normalize(sinc(0.25) * blackman), 17 taps, host libm */
void mlb_impulse_table(float out17[17]);
void mlb_coeffs_sample_glide(float time_in_samples, float out2[2]);
/* FDN<8>::setDelaysInSamples / setFilterCutoffs / mFeedbackGains, F:1171-1191.
 * Fills the 32 coef words of an FDN8 node for one voice:
 * [0..7]=a0, [8..15]=b1, [16..23]=feedback gain, [24..31]=len=max(1,int(time)-64). */
void mlb_coeffs_fdn8(const float times[8], const float cutoffs[8], const float gains[8],
                     float out32[32]);

/* The same designs for n voices in one call (pure host): op = MLB_OP_LOPASS / HIPASS / BANDPASS / LOSHELF /
 * HISHELF / BELL / ONEPOLE; omega[n], k[n] (unused for ONEPOLE), A[n] (shelves and bell only);
 * out[n_coef][n] in the SoA layout of mlb_graph_set_coefs. */
int mlb_coeffs_batch(int op, size_t n, const float* omega, const float* k, const float* A, float* out);

/* Lopass::makeCoeffsVec(omega, k), F:97-115, for ONE 64-sample block: clamps omega to <= 0.5 and k to
 * >= 0.01 (min/max with the reference's operand order), then the per-sample makeCoeffs formula with host
 * libm sinf.  out3x64 = rows g0, g1, g2 (the in1..3 rows of a LOPASS_V node). */
void mlb_coeffs_lopass_vec(const float omega[64], const float k[64], float out3x64[3 * 64]);
/* the same for n_rows blocks: omega, k [n_rows][64] -> out [n_rows][3][64] */
void mlb_coeffs_lopass_vec_n(const float* omega, const float* k, float* out, size_t n_rows);
/* interpolateCoeffsLinear(c0, c1), F:32-44: row i = interpolateDSPVectorLinear(c0[i], c1[i]) (O:986-990).
 * With c0 / c1 from mlb_coeffs_loshelf / mlb_coeffs_hishelf this is LoShelf/HiShelf::vcoeffs(p0, p1)
 * (F:283-286, 364-367).  out = [n_coeffs][64]. */
void mlb_interpolate_coeffs_linear(const float* c0, const float* c1, int n_coeffs, float* out);

/* ---- device / context ---- */
/* One device per process (the multi-GPU model is one process per GPU): mlb_init(other) while graphs, voice
 * banks, bus layouts, resamplers, FDTD banks or mix buses of the current device are alive returns MLB_ERR_INVALID.
 * Entry points make the library's device current on the calling thread. */
int mlb_init(int device);          /* select device, check sm_90; MLB_ERR_NO_DEVICE if absent */
int mlb_device_count(void);        /* 0 when no GPU: callers must fail loudly, not fall back */
const char* mlb_last_error(void);  /* thread-local message of the last failing call */
int mlb_abi_version(void);
long long mlb_kernel_launches(void); /* count of kernels this library launched (process-wide) */
int mlb_live_handles(void);          /* handles of the kinds mlb_init counts that are alive now (process-wide) */

/* ---- block-rate resamplers (SURVEY 8f row 4) -------------------------------------------------
 * Upsampler(octaves) / Downsampler(octaves), source/DSP/MLDSPFilters.h:1316-1473: cascades of
 * HalfBandFilters that change the number of blocks -- every input block of an Upsampler gives
 * 2^octaves output blocks (write, then 2^octaves reads); a Downsampler gives one output block per
 * 2^octaves input blocks (write returns true).  One object per voice, V voices per call.
 * in [n_blocks_in][V][64]; out [n_blocks_out][V][64] with n_blocks_out = n_blocks_in << octaves (up)
 * or the number of completed groups (down; the write counter carries over between calls and
 * *n_blocks_out reports it).  octaves in [1, 4] (the reference leaves _numBuffers unset at 0). */
typedef struct mlb_resampler mlb_resampler;
enum { MLB_RESAMPLE_UP = 0, MLB_RESAMPLE_DOWN = 1 };
int mlb_resampler_create(int direction, int octaves, int n_voices, mlb_resampler** out);
int mlb_resampler_destroy(mlb_resampler* r);
int mlb_resampler_clear(mlb_resampler* r);   /* Upsampler::clear / Downsampler::clear */
int mlb_resampler_process_host(mlb_resampler* r, const float* in_host, float* out_host, int n_blocks_in,
                               int* n_blocks_out);
int mlb_resampler_process_device(mlb_resampler* r, const float* in_dev, float* out_dev, int n_blocks_in,
                                 int* n_blocks_out, void* stream);

/* ---- FDTD membrane banks (K9) ---------------------------------------------------------------
 * V independent 16 x 16 finite-difference membranes = V x (FDTDState + processFDTDModel) of the reference's
 * examples/audio-and-midi/fdtd.cpp:26-154: per sample, the coefficients are designed from the frequency
 * sample (cycles per sample), the excitation sample times 4 is added to the z^-1 surface at row 2, column 8,
 * one explicit step of the 3 x 3 stencil over the z^-1 and z^-2 surfaces gives the new surface (fixed zero
 * boundary), and its cells at row 9, columns 1 and 15 are the L and R outputs.  Bit-exact: every op is one
 * separately rounded binary32 op in the reference's order.  One kernel launch per call. */
typedef struct mlb_fdtd mlb_fdtd;        /* V membranes = V FDTDState + processFDTDModel, fdtd.cpp:26-154 */
#define MLB_FDTD_SIZE 16                 /* kWidth = kHeight */
#define MLB_FDTD_FTZ 1u                  /* every FP op flushes subnormals, as under UsingFlushDenormalsToZero */
/* inputs are [T][in_planes][V][64]; rows excite_plane / freq_plane (cycles per sample) are read, so a graph's
 * or a Voice bank's output buffer can be passed as-is.  State after create/clear: all surfaces zero. */
int mlb_fdtd_create(int n_instances, float sample_rate, int in_planes, int excite_plane, int freq_plane,
                    unsigned flags, mlb_fdtd** out);
int mlb_fdtd_destroy(mlb_fdtd* f);
int mlb_fdtd_clear(mlb_fdtd* f);
int mlb_fdtd_get_state(mlb_fdtd* f, float* host);        /* [V][2][16][16]: z^-1 interior, then z^-2 */
int mlb_fdtd_set_state(mlb_fdtd* f, const float* host);
int mlb_fdtd_process_device(mlb_fdtd* f, const float* in_dev, float* out_dev /* [T][2][V][64] L,R */,
                            int n_blocks, void* stream);
int mlb_fdtd_process_host(mlb_fdtd* f, const float* in_host, float* out_host, int n_blocks);

/* ---- EventsToSignals::Voice bank (SURVEY 8f row 3) ---------------------------------------
 * The step BEFORE the chain: the reference's EventsToSignals (source/app/MLEventsToSignals.h:43-236)
 * turns note / controller events into 8 control rows per voice.  Its event routing (voice
 * allocation, stealing, unison, MPE: MLEventsToSignals.cpp:476-960) is host-side control logic and
 * stays with the caller; what is built here is the per-voice signal generator
 * EventsToSignals::Voice (beginProcess / writeNoteEvent / endProcess, .cpp:97-263) for V voices at
 * once: sample-accurate gate and pitch (SampleAccurateLinearGlide), vector-accurate bend / mod /
 * x / y / z / drift glides (LinearGlide), elapsed time, pitch drift (RandomScalarSource).
 * Per voice and block the caller hands over one 72-byte record instead of 256-byte rows. */
#define MLB_VOICE_ROWS 8          /* kPitch, kGate, kVoice, kZ, kX, kY, kMod, kElapsedTime (.h:16-27) */
#define MLB_VOICE_MAX_EVENTS 4    /* note events one voice can take per 64-frame vector */
enum {                            /* = ml::EventType (source/app/MLEvent.h:14-27) */
  MLB_EV_NULL = 0, MLB_EV_NOTE_ON = 1, MLB_EV_NOTE_RETRIG = 2, MLB_EV_NOTE_SUSTAIN = 3, MLB_EV_NOTE_OFF = 4
};
enum { MLB_EVF_GLIDE = 1, MLB_EVF_RESET = 2 };                  /* writeNoteEvent(e, key, doGlide, doReset) */
enum { MLB_SET_BEND = 1, MLB_SET_MOD = 2, MLB_SET_X = 4, MLB_SET_Y = 8, MLB_SET_Z = 16, MLB_SET_PRESSURE = 32 };
typedef struct mlb_voice_events {  /* what ONE Voice receives during ONE vector */
  uint8_t n_events;                          /* <= MLB_VOICE_MAX_EVENTS, in time order */
  uint8_t set_mask;                          /* which of bend/mod/x/y/z were written this vector */
  uint8_t pad[2];
  uint8_t time[MLB_VOICE_MAX_EVENTS];        /* Event::time, frame offset in the vector (clamped to 64) */
  uint8_t type[MLB_VOICE_MAX_EVENTS];        /* MLB_EV_* */
  uint8_t flags[MLB_VOICE_MAX_EVENTS];       /* MLB_EVF_* */
  float value1[MLB_VOICE_MAX_EVENTS];        /* Event::value1 = pitch */
  float value2[MLB_VOICE_MAX_EVENTS];        /* Event::value2 = velocity */
  float bend, mod, x, y, z;                  /* currentPitchBend, currentMod, currentX/Y/Z when set */
  float pressure;                            /* MIDI channel pressure = controllers[128].inputValue (.cpp:601-606) */
} mlb_voice_events;                          /* 72 bytes */
/* flags for mlb_voices_create */
#define MLB_VOICES_MIDI 1u  /* processVector's MIDI tail (.cpp:440-447): z row += the smoothed channel-pressure
                             * controller (SmoothedController, .cpp:274-285), one copy per voice */


/* Event routing in front of the bank (host only, no GPU needed): the C face of mlb::VoiceRouter
 * (include/mlb200_events.hpp) = EventsToSignals::addEvent / processVector / processEvent... for the MIDI
 * (protocol 0) and MPE (protocol 1) protocols (MLEventsToSignals.cpp:352-418, 476-960).
 * mlb_router_process_vector writes mlb_router_record_count() records: MIDI: voice i+1 -> records[i];
 * MPE: voice i -> records[i] (0 = the main voice).  Returns the number of note events that did not fit
 * (MLB_VOICE_MAX_EVENTS per voice and vector), or a negative value on a null argument. */
typedef struct mlb_router mlb_router;
typedef struct mlb_event {   /* ml::Event, source/app/MLEvent.h:31-50 */
  uint8_t type;              /* ml::EventType: 1 note on, 4 note off, 5 sustain pedal, 6 controller, 7 pitch bend,
                                8 note pressure, 9 channel pressure */
  uint8_t channel;
  uint16_t source_idx;       /* key or controller number */
  int32_t time;              /* frames from the start of the top-level buffer */
  float value1, value2;
} mlb_event;
mlb_router* mlb_router_create(int polyphony, int protocol);
void mlb_router_destroy(mlb_router* r);
void mlb_router_set_unison(mlb_router* r, int on);
void mlb_router_add_event(mlb_router* r, const mlb_event* e);
void mlb_router_clear_events(mlb_router* r);
int mlb_router_record_count(const mlb_router* r);
/* events the router saw but does not route (CC 120 "all sound off" resets voices in mid-vector,
 * MLEventsToSignals.cpp:748-755: not built), since creation; -1 on null */
int mlb_router_unsupported_count(const mlb_router* r);
void mlb_router_set_mod_cc(mlb_router* r, int cc);   /* EventsToSignals::setModCC (.h:80) */
int mlb_router_process_vector(mlb_router* r, int start_time, mlb_voice_events* records);
/* One write of a SmoothedController's inputValue (EventsToSignals::controllers[n], MLEventsToSignals.h:170-180):
 * a controller event writes controllers[min(source_idx, 128)] (.cpp:743-744, before the CC 120 / 123 cases), and in
 * the MIDI protocol a channel-pressure event writes controller 128 (.cpp:643-652). */
typedef struct mlb_controller_change {
  uint16_t controller;       /* 0..128; larger numbers are read as 128 */
  uint16_t pad;
  float value;
} mlb_controller_change;     /* 8 bytes */
/* The controller writes of the last mlb_router_process_vector, in the order the reference applies them.  Copies at
 * most `cap` of them to `out` (which may be NULL when cap is 0) and returns how many there were; -1 on null. */
int mlb_router_controller_changes(const mlb_router* r, mlb_controller_change* out, int cap);

typedef struct mlb_voices mlb_voices;  /* opaque: V Voice objects on the device */

/* V voices after Voice() + reset() + setSampleRate(sr) + setPitchGlideInSeconds + setDriftAmount
 * (.cpp:47-95).  voice_index[v] = Voice::voiceIndex (seeds the drift source with index * 232 and
 * gives the kVoice row = index - 1, .cpp:61,292); pitch_bend[v] = the semitone range handed to
 * endProcess (.cpp:422-428).  Arrays are per voice, host memory. */
int mlb_voices_create(int n_voices, float sample_rate, const int32_t* voice_index, const float* pitch_glide_seconds,
                      const float* drift_amount, const float* pitch_bend, unsigned flags, mlb_voices** out);
int mlb_voices_destroy(mlb_voices* vb);
/* processVector's MPE tail (.cpp:448-460): the pitch, x, y, z and mod rows of a channel voice get the rows of
 * its instrument's main voice (voices[0]) added.  mlb_voices_set_main_voices names, per voice, the index of
 * its main voice in the bank, or -1 (main voices themselves, or no MPE).  The rows involved must be in
 * row_mask. */
int mlb_voices_set_main_voices(mlb_voices* vb, const int32_t* main_voice);
/* n_blocks vectors: beginProcess, the block's events, endProcess, for every voice.
 * events_host [n_blocks][V]; out_host [n_blocks][MLB_VOICE_ROWS][V][64] (rows whose bit is clear in
 * row_mask are not written; bit r = row r).  One kernel launch. */
int mlb_voices_process_host(mlb_voices* vb, const mlb_voice_events* events_host, float* out_host,
                            int n_blocks, unsigned row_mask);
/* same with device-resident buffers, asynchronous on `stream`; the out planes have the layout of
 * graph inputs, so they can be handed to mlb_graph_process_device as-is. */
int mlb_voices_process_device(mlb_voices* vb, const mlb_voice_events* events_dev, float* out_dev,
                              int n_blocks, unsigned row_mask, void* stream);

/* ---- stateless elementwise ops on device or host buffers (K3) ----
 * y[i] = op(x1[i], x2[i], x3[i]) for n_rows*64 elements; unused inputs NULL.
 * Stands in for every DEFINE_OP* function of MLDSPOps.h:567-918 applied to a
 * DSPVectorArray<n_rows>.  *_device: pointers are device memory, async on
 * `stream` (a cudaStream_t passed as void*).  *_host: pointers are host memory;
 * the call copies in, launches, copies out and synchronises. */
int mlb_map_device(int op, const float* x1, const float* x2, const float* x3, float* y,
                   size_t n_rows, void* stream);
int mlb_map_host(int op, const float* x1, const float* x2, const float* x3, float* y,
                 size_t n_rows);
/* mlb_map_host stages through a process-wide pool of device buffers that only grows: number of times the
 * pool was (re)allocated so far (stays constant once the largest operand size has been seen). */
long long mlb_map_host_allocations(void);

/* ---- voice graphs: Bank<>-shaped batched processors ---- */
typedef struct mlb_graph mlb_graph; /* opaque; owns device state, coefs, delay memory */

/* flags for mlb_graph_create */
#define MLB_GRAPH_EXACT 0u        /* bit-exact with the reference SSE path (default) */
#define MLB_GRAPH_FAST 1u         /* allow FMA contraction (stated tolerance, see DESIGN.md) */
#define MLB_GRAPH_FORCE_GENERIC 2u /* skip fused specialisations, use the graph interpreter kernel */
#define MLB_GRAPH_SINGLE_STAGE 4u  /* interpreter: one CTA per voice group, no stage pipeline across CTAs */

/* Create a graph for n_voices voices on the current device.
 * outs[n_out] = node indices whose rows are written to out planes / mix bus.
 * Stands in for declaring Bank<T,ROWS> members / functor structs
 * (MLDSPFunctional.h:321-326; examples/audio-and-midi/sine.cpp:17-19). */
int mlb_graph_create(const mlb_node* nodes, int n_nodes, const int32_t* outs, int n_out,
                     int n_voices, unsigned flags, mlb_graph** out_graph);
int mlb_graph_destroy(mlb_graph* g);
/* Input buffers normally hold 1 + (highest INPUT plane index) planes per block.  A caller whose buffer has
 * more planes per block -- the 8 planes of a Voice bank's output, of which a graph reads two -- declares the
 * real count here (n_planes >= the graph's own; call before processing). */
int mlb_graph_set_input_planes(mlb_graph* g, int n_planes);
/* Leave n_sms SMs out of the persistent chain grid (default 0) so that kernels of an overlapped
 * collective -- the NCCL all-reduce of the mix bus in a multi-GPU run -- can be resident next to it
 * (ours; the reference is single-device). */
int mlb_graph_reserve_sms(mlb_graph* g, int n_sms);
int mlb_graph_layout_of(const mlb_graph* g, mlb_layout* layout);
/* name of the kernel variant chosen ("fused:sine_lopass_gain", "generic", ...) */
const char* mlb_graph_kernel_name(const mlb_graph* g);

/* Upload / download SoA words for ALL voices: host buffers of n_words*V words.
 * set_coefs stands in for assigning `coeffs` members (F:80,166,...);
 * set_state / get_state for clear()/setSeed()/reading state members
 * (G:116,182,379; F:66-70,478-480). */
int mlb_graph_set_coefs(mlb_graph* g, const float* coef_host /*[n_coef_words][V]*/);
int mlb_graph_set_state(mlb_graph* g, const uint32_t* state_host /*[n_state_words][V]*/);
int mlb_graph_get_state(mlb_graph* g, uint32_t* state_host);
/* zero delay memory + delay write index (IntegerDelay::clear, F:832; FDN carried vectors) */
int mlb_graph_clear_delays(mlb_graph* g);
size_t mlb_graph_delay_bytes(const mlb_graph* g);

/* Process n_blocks blocks for all voices.  Stands in for n_blocks successive
 * Bank::operator() calls (MLDSPFunctional.h:328-337) / SignalProcessFn
 * invocations (MLSignalProcessBuffer.cpp:57-78) fused into ONE kernel launch.
 * Any of in/out/mix may be NULL when the graph has no INPUT nodes / the caller
 * does not want that product.  _device: device pointers, async on stream.
 * _host: host pointers (pinned or pageable); H2D, launch, D2H, synchronise. */
int mlb_graph_process_device(mlb_graph* g, const float* in_dev, float* out_dev, float* mix_dev,
                             int n_blocks, void* stream);
int mlb_graph_process_host(mlb_graph* g, const float* in_host, float* out_host, float* mix_host,
                           int n_blocks);

/* ---- multi-GPU mix bus (SURVEY 8e): one process per GPU, voices sharded, the ONLY exchange is the sum of the
 * per-rank mix buses (Synth::processVector's accumulate, source/app/MLSynth.h:36-60, continued over GPUs).
 * With a mix bus attached, mlb_graph_process_* delivers in `mix` the sum over ALL ranks: the kernel that
 * finishes the local sum writes it into every peer's exchange buffer over NVLink (CUDA IPC peer memory),
 * raises per-plane flags, waits for the peers' flags and adds the world's rows in rank order -- bit-identical
 * on every rank, no NCCL call, no extra launch.  Set-up: every rank creates its bus, the 64-byte handles are
 * exchanged by whatever means the host has (torch.distributed all_gather in bench.py), every rank connects.
 * Every rank must then issue the same sequence of process calls (as with any collective).
 * max_floats = largest n_blocks * n_out * 64 a call will reduce. */
typedef struct mlb_mixbus mlb_mixbus;
int mlb_mixbus_create(int rank, int world, size_t max_floats, mlb_mixbus** out);
int mlb_mixbus_handle(mlb_mixbus* bus, void* out64);              /* this rank's cudaIpcMemHandle_t (64 bytes) */
int mlb_mixbus_connect(mlb_mixbus* bus, const void* handles);     /* [world][64], rank order */
int mlb_mixbus_destroy(mlb_mixbus* bus);
int mlb_graph_attach_mixbus(mlb_graph* g, mlb_mixbus* bus);       /* NULL detaches */
/* Asynchronous exchange (choose before the first process call, same on every rank): the kernel on the caller's
 * stream only leaves this rank's sums in a local staging block; writing them to the peers, waiting for the peers'
 * rows and adding them runs in one small kernel on the bus's own stream while the caller's stream already
 * computes the next call (what an async NCCL all-reduce gives, without NCCL; up to four calls may be in flight).  `mix` of a mlb_graph_process_device call is then complete only after
 * mlb_graph_mix_wait(g, stream) -- which makes `stream` wait for the most recent call's completion -- so use
 * one `mix` buffer per call in flight.  mlb_graph_process_host always returns finished results. */
int mlb_mixbus_set_async(mlb_mixbus* bus, int on);
/* The same for ONE GPU (and in front of the exchange on several): with mix_async on, mlb_graph_process_device leaves only
 * the chain kernel on the caller's stream; the reduction of the per-group partials into `mix` (mix_reduce_kernel, 3 % of a
 * config-A step) runs on the graph's own stream beside the next call's kernel, from partials double-buffered by call
 * parity.  `mix` of a call is complete after mlb_graph_mix_wait(g, stream); use one `mix` buffer per call in flight. */
int mlb_graph_set_mix_async(mlb_graph* g, int on);
int mlb_graph_mix_wait(mlb_graph* g, void* stream);

/* Duration in milliseconds of the most recent chain kernel launched by
 * process_device, measured with CUDA events on the launching stream
 * (blocks until that launch has finished). */
int mlb_graph_last_kernel_ms(mlb_graph* g, float* ms);
/* Number of voice slices the most recent mlb_graph_process_host call was pipelined over
 * (H2D / kernel / D2H on three streams); 1 = a single launch, -1 = null graph.  Large fused banks
 * are sliced when the PCIe traffic of the call reaches MLB_HOST_SLICE_MIN_MB (env, default 32) MiB. */
int mlb_graph_last_host_slices(const mlb_graph* g);

/* The graph interpreter's host-side plan, without a device (tests, tools): the pipeline stage of every node (-1 for
 * nodes that run in no stage, e.g. PARAM), the number of stages and of 8.5-KB shared-memory row slots the program needs,
 * for an H100 SXM (132 SMs, 227 KB) unless mlb_init has seen another device; MLB_STAGES (env) forces the stage count as it
 * does for mlb_graph_create.  Fails like mlb_graph_create does when the graph cannot be planned (too many live rows,
 * a stage depending on too many stages).  Any pointer may be NULL. */
int mlb_graph_plan(const mlb_node* nodes, int n_nodes, const int32_t* outs, int n_out, int n_voices, unsigned flags,
                   int32_t* stage_of, int32_t* n_stages, int32_t* n_row_slots);


/* Events -> signals -> chain in one call, host buffers, only the event records going up ("contract E"):
 * what a synth built on the reference does per top-level buffer -- EventsToSignals::processVector
 * (MLEventsToSignals.cpp:383-470), then Synth::processVector's loop of processVoice calls reading the
 * voice.outputs rows and accumulating into the outputs (MLSynth.h:36-60,67-71) -- for all voices of the
 * bank.  The graph's INPUT plane r is Voice row r (kPitch = 0, kGate = 1, ... MLEventsToSignals.h:14-26);
 * the bank generates exactly the rows the graph reads, on the device, into the graph's input buffer.
 * events_host [n_blocks][V] (72 B per voice and vector instead of 256 B per input row); out_host
 * [n_blocks][n_out][V][64] or NULL; mix_host [n_blocks][n_out][64] or NULL.  Pipelined over time chunks
 * (MLB_SYNTH_CHUNK_BLOCKS, env; default: rows of a chunk <= 1 GiB) on three streams; returns when the host
 * buffers are complete; mlb_graph_last_host_slices() then reports the number of chunks.
 * MLB_ERR_INVALID when the bank and the graph differ in voice count or the graph reads no Voice row. */
int mlb_synth_process_host(mlb_voices* vb, mlb_graph* g, const mlb_voice_events* events_host,
                           float* out_host, float* mix_host, int n_blocks);

/* ---- Per-instrument output buses (K10) ---------------------------------------------------------
 * A reference Synth owns at most 16 voices (EventsToSignals::kMaxVoices, MLEventsToSignals.h:47), so a bank of V
 * voices is in practice many instruments.  A bus layout is G voice ranges [first[g], first[g] + count[g]): a count
 * of 0 gives a bus of +0; ranges may leave gaps (MPE: Synth reads getInputVoice(v) = voices[v + 1], so an
 * instrument's main voice is not summed) and may overlap.  For every block t, plane p, bus g and sample n:
 *   bus[t][p][g][n] = ((+0 + x[first]) + x[first + 1]) + ... + x[first + count - 1]
 * one binary32 add per voice in voice order, subnormals kept: Synth::processVector (MLSynth.h:36-60) with the
 * default isVoiceActive, bit for bit.  The bus rows [T][P][G][64] have the layout of a G-voice graph's input. */
typedef struct mlb_buses mlb_buses;   /* G per-instrument output buses over a V-voice bank (Synth::processVector, MLSynth.h:36-60) */
/* Validates the layout on the host (MLB_ERR_INVALID names the offending bus) and uploads it.  A live layout counts
 * toward mlb_init's one-device rule. */
int mlb_buses_create(int n_voices, int n_buses, const int32_t* first_voice, const int32_t* voice_count, mlb_buses** out);
int mlb_buses_destroy(mlb_buses* b);
/* rows_dev [T][n_planes][V][64] -> bus_dev [T][n_planes][G][64]; one launch, no allocation, no synchronisation */
int mlb_buses_sum_device(mlb_buses* b, const float* rows_dev, float* bus_dev, int n_planes, int n_blocks, void* stream);
/* contract E with per-instrument output: event records in, bus rows [T][n_out][G][64] out; voice rows never leave HBM.
 * The pipeline of mlb_synth_process_host; the graph's rows of one time chunk go to a device scratch of one chunk
 * and are summed into buses on the graph's stream right after the graph.  MLB_ERR_INVALID when the bank, graph and
 * buses differ in voice count, the graph has no outputs or reads no Voice row. */
int mlb_synth_process_buses_host(mlb_voices* vb, mlb_graph* g, mlb_buses* b, const mlb_voice_events* events_host,
                                 float* bus_host, int n_blocks);

/* ---- Smoothed MIDI controllers (K11) -----------------------------------------------------------
 * Every reference EventsToSignals (one per instrument) owns 129 SmoothedControllers (MLEventsToSignals.h:50,170-180):
 * per vector each runs output = LinearGlide(inputValue) (MLDSPGens.h:433-515, .cpp:431-435) with a glide of
 * int(sr * 0.02) samples truncated to whole vectors (.cpp:274-285), and a process function reads the rows through
 * AudioContext::getInputController(n).  A controller bank holds G instruments x C requested controllers (numbers
 * 0..128, any order, no repeats): only these are stored and produced; writes to the others are ignored.
 * Input per block t: the changes of instrument g are changes[offsets[t][g] .. offsets[t][g + 1]) (offsets
 * [T][G + 1] int32, indexes into `changes`), in event order: the last write to a controller in a block wins, and
 * an inputValue persists across blocks.  The rows are the reference's bit for bit, -0, +-inf, NaN and subnormals
 * included.  Output [T][n_planes][N][64]: controller k of the list goes to plane plane0 + k; N = G (instrument rows)
 * or, after mlb_controllers_set_voice_map, N = V, every voice getting its instrument's row (+0 for a voice of no
 * instrument): the layout of a voice graph's INPUT planes. */
typedef struct mlb_controllers mlb_controllers;
/* protocol: 0 MIDI, 1 MPE (mlb_router_create's); it must match the voice bank's MLB_VOICES_MIDI flag in
 * mlb_synth_process_controllers_host.  Arguments are validated on the host; MLB_ERR_INVALID names the offending
 * controller.  A live bank counts toward mlb_init's one-device rule. */
int mlb_controllers_create(int n_instruments, float sample_rate, int protocol, const int32_t* controllers,
                           int n_controllers, mlb_controllers** out);
int mlb_controllers_destroy(mlb_controllers* cb);
int mlb_controllers_clear(mlb_controllers* cb);   /* every controller back to inputValue = target = 0, idle */
/* state words [4][C][G] uint32: inputValue, LinearGlide::mTargetValue, mVectorsRemaining (int32), step (the float
 * bits of mStepVec); rows [C][G][64] = LinearGlide::mCurrVec.  get_state returns an idle glide's (remaining < 0)
 * row as its target, and set_state reads only the rows of moving glides: an idle row always equals its target. */
int mlb_controllers_get_state(mlb_controllers* cb, uint32_t* words, float* rows);
int mlb_controllers_set_state(mlb_controllers* cb, const uint32_t* words, const float* rows);
/* voice_instrument[V]: the instrument of each voice, or -1; NULL goes back to instrument rows */
int mlb_controllers_set_voice_map(mlb_controllers* cb, const int32_t* voice_instrument, int n_voices);
/* one launch for n_blocks vectors, no allocation, no synchronisation (capturable into a CUDA graph) */
int mlb_controllers_process_device(mlb_controllers* cb, const int32_t* offsets_dev,
                                   const mlb_controller_change* changes_dev, float* out_dev, int plane0, int n_planes,
                                   int n_blocks, void* stream);
/* host buffers: offsets are checked (non-decreasing per block, within [0, n_changes]) before anything is copied */
int mlb_controllers_process_host(mlb_controllers* cb, const int32_t* offsets_host,
                                 const mlb_controller_change* changes_host, int n_changes, float* out_host,
                                 int plane0, int n_planes, int n_blocks);
/* Contract E with controller planes (AudioContext::getInputController(n) -> graph INPUT planes): the graph's input
 * per block is the 8 Voice rows, then the C controller rows in the bank's list order (INPUT plane 8 + k is
 * controller k of the list).  events_host [T][V] as for mlb_synth_process_host; ctrl_offsets_host [T][G + 1] into
 * ctrl_changes_host, checked before anything is copied; out_host [T][n_out][V][64] or NULL; mix_host [T][n_out][64]
 * or NULL.  The pipeline of mlb_synth_process_host; returns when its copies are finished, also on failure.
 * MLB_ERR_INVALID when the bank, the controller bank's voice map (mlb_controllers_set_voice_map) and the graph differ
 * in voice count, the protocols differ (MPE bank vs MLB_VOICES_MIDI), or the graph reads a plane beyond 8 + C - 1. */
int mlb_synth_process_controllers_host(mlb_voices* vb, mlb_controllers* cb, mlb_graph* g,
                                       const mlb_voice_events* events_host, const int32_t* ctrl_offsets_host,
                                       const mlb_controller_change* ctrl_changes_host, float* out_host,
                                       float* mix_host, int n_blocks);

#ifdef __cplusplus
}
#endif
#endif /* MLB200_H */
