// mlb200.cu -- host side of the C ABI declared in include/mlb200.h.
//
// Owns device memory for per-voice state / coefficients / delay lines, recognises linear
// chains that have a fused sm_90a kernel (chain_kernel.cuh), builds the TMA tensor maps
// and launches ONE kernel per process call.  Everything else goes through the graph
// interpreter kernel (generic_kernel.cuh).  There is no CPU compute path in this library:
// without an sm_90 device every processing entry point returns MLB_ERR_NO_DEVICE.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/mlb200.h"
#include "chain_kernel.cuh"
#include "fdn_kernel.cuh"
#include "voice_kernel.cuh"
#include "resample_kernel.cuh"
#include "fdtd_kernel.cuh"
#include "bus_kernel.cuh"
#include "controller_kernel.cuh"
#include "generic_kernel.cuh"

using namespace mlb;

// ------------------------------------------------------------------------------------------
// errors, counters

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

static int fail(int code, const char* fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CU_CHECK(expr)                                                                      \
  do                                                                                        \
  {                                                                                         \
    cudaError_t e__ = (expr);                                                               \
    if (e__ != cudaSuccess)                                                                 \
      return fail(MLB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),   \
                  __FILE__, __LINE__);                                                      \
  } while (0)

// return the MLB_* code of a failing call of this library
#define MLB_TRY(expr)                \
  do                                 \
  {                                  \
    const int rc__ = (expr);         \
    if (rc__ != MLB_OK) return rc__; \
  } while (0)

// The return of a host entry point that has enqueued anything, whatever rc says: wait for every stream the call used,
// so that no copy still reads or writes the caller's buffers after it returns.  The first error wins.
static int drain(int rc, std::initializer_list<cudaStream_t> streams)
{
  for (cudaStream_t s : streams)
    if (const cudaError_t e = cudaStreamSynchronize(s); e != cudaSuccess && rc == MLB_OK)
      rc = fail(MLB_ERR_CUDA, "stream synchronise: %s", cudaGetErrorString(e));
  return rc;
}

// ------------------------------------------------------------------------------------------
// owners of device memory, streams, events and live-handle counts: move-only, failures reported by the explicit
// alloc / create calls (no exception crosses the C ABI).  A default-constructed owner makes no CUDA runtime call,
// not even when it is destroyed: mlb_graph_plan builds a host-only graph.

// graphs, voice banks, bus layouts, resamplers, FDTD banks and mix buses alive (they hold pointers of g_device)
static std::atomic<int> g_live_handles{0};

// One cudaMalloc allocation of T and its size in bytes.
template <class T>
class DevBuf
{
 public:
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); return *this; }
  ~DevBuf() { reset(); }
  // frees the old allocation first; empty after a failure
  int alloc(size_t bytes, const char* what)
  {
    reset();
    const cudaError_t e = cudaMalloc(&p_, bytes);
    if (e != cudaSuccess)
    {
      p_ = nullptr;
      cudaGetLastError();
      return fail(MLB_ERR_ALLOC, "cudaMalloc of %zu B %s failed: %s", bytes, what, cudaGetErrorString(e));
    }
    bytes_ = bytes;
    return MLB_OK;
  }
  // grow only: nothing is copied
  int ensure(size_t bytes, const char* what) { return bytes <= bytes_ ? MLB_OK : alloc(bytes, what); }
  void reset()
  {
    if (p_) cudaFree(p_);
    p_ = nullptr, bytes_ = 0;
  }
  T* get() const { return p_; }
  size_t bytes() const { return bytes_; }

 private:
  T* p_ = nullptr;
  size_t bytes_ = 0;
};

// One cudaStream_t or cudaEvent_t.  create() is a no-op once it has succeeded, so that a handle can create what it
// needs on first use (mlb_graph_set_mix_async).
template <class H>
class CudaObj
{
 public:
  CudaObj() = default;
  CudaObj(CudaObj&& o) noexcept { std::swap(h_, o.h_); }
  CudaObj& operator=(CudaObj&& o) noexcept { std::swap(h_, o.h_); return *this; }
  ~CudaObj() { if (h_) destroy(h_); }
  int create(unsigned flags)
  {
    const cudaError_t e = h_ ? cudaSuccess : make(&h_, flags);
    if (e == cudaSuccess) return MLB_OK;
    h_ = nullptr;
    const char* kind = std::is_same<H, cudaStream_t>::value ? "stream" : "event";
    return fail(MLB_ERR_CUDA, "creating a CUDA %s failed: %s", kind, cudaGetErrorString(e));
  }
  H get() const { return h_; }

 private:
  static cudaError_t make(cudaStream_t* s, unsigned flags) { return cudaStreamCreateWithFlags(s, flags); }
  static cudaError_t make(cudaEvent_t* e, unsigned flags) { return cudaEventCreateWithFlags(e, flags); }
  static void destroy(cudaStream_t s) { cudaStreamDestroy(s); }
  static void destroy(cudaEvent_t e) { cudaEventDestroy(e); }
  H h_ = nullptr;
};
using Stream = CudaObj<cudaStream_t>;
using Event = CudaObj<cudaEvent_t>;

// A handle's place in g_live_handles, from arm() until destruction.  Only the *_create entry points arm it.
class LiveCount
{
 public:
  LiveCount() = default;
  LiveCount(LiveCount&& o) noexcept { std::swap(armed_, o.armed_); }
  LiveCount& operator=(LiveCount&& o) noexcept { std::swap(armed_, o.armed_); return *this; }
  ~LiveCount() { if (armed_) --g_live_handles; }
  void arm()
  {
    if (!armed_) ++g_live_handles;
    armed_ = true;
  }

 private:
  bool armed_ = false;
};

extern "C" const char* mlb_last_error(void) { return g_err; }
extern "C" int mlb_abi_version(void) { return MLB_ABI_VERSION; }
extern "C" long long mlb_kernel_launches(void) { return g_launches.load(); }
extern "C" int mlb_live_handles(void) { return g_live_handles.load(); }

// ------------------------------------------------------------------------------------------
// op metadata and graph layout (host only)

extern "C" int mlb_op_info(int op, int* n_in, int* n_state, int* n_coef)
{
  switch (op)
  {
#define MLB_X_INFO(NAME, id, nin, nst, nco) \
  case id:                                  \
    if (n_in) *n_in = nin;                  \
    if (n_state) *n_state = nst;            \
    if (n_coef) *n_coef = nco;              \
    return MLB_OK;
    MLB_OP_TABLE(MLB_X_INFO)
#undef MLB_X_INFO
  }
  return MLB_ERR_INVALID;
}

extern "C" const char* mlb_op_name(int op)
{
  switch (op)
  {
#define MLB_X_NAME(NAME, id, nin, nst, nco) \
  case id: return #NAME;
    MLB_OP_TABLE(MLB_X_NAME)
#undef MLB_X_NAME
  }
  return "?";
}

// delay memory of an op: 64-float member rows and IntegerDelay rings per voice (MLB_OP_MEM_TABLE)
static void op_mem(int op, int* n_rows, int* n_rings);

// MLB_AGAIN (mlb200.h): may a node of this op be a further call of an earlier functor?
static bool again_allowed(int op)
{
  int nin = 0, nst = 0, nco = 0, rows = 0, rings = 0;
  if (mlb_op_info(op, &nin, &nst, &nco) != MLB_OK) return false;
  op_mem(op, &rows, &rings);
  if (rings != 0 || (nst == 0 && nco == 0)) return false;
  switch (op)
  {
    case MLB_OP_INPUT: case MLB_OP_PARAM: case MLB_OP_FEEDBACK_READ: case MLB_OP_FEEDBACK_WRITE: case MLB_OP_FDN8:
    case MLB_OP_FDN8_R: case MLB_OP_HALFBAND_UP_2: case MLB_OP_DOWN2X_IN: case MLB_OP_DOWN2X_OUT:
      return false;  // (a HALFBAND_UP called again has its own HALFBAND_UP_2 reading ITS second row)
    default: return true;
  }
}
// the node whose functor node i calls again, or -1
static int again_target(const mlb_node* nodes, int i)
{
  const int op = nodes[i].op;
  if (op == MLB_OP_INPUT || op == MLB_OP_PARAM || op == MLB_OP_FEEDBACK_WRITE) return -1;  // iarg has its own meaning / none
  return nodes[i].iarg < 0 ? MLB_AGAIN_TARGET(nodes[i].iarg) : -1;
}

extern "C" int mlb_graph_layout(const mlb_node* nodes, int n_nodes, mlb_layout* layout,
                                int32_t* state_off, int32_t* coef_off)
{
  if (!nodes || n_nodes <= 0 || !layout) return fail(MLB_ERR_INVALID, "null graph");
  int ns = 0, nc = 0, nin_planes = 0, n_fdn = 0;
  for (int i = 0; i < n_nodes; ++i)
  {
    int nin, nst, nco;
    if (mlb_op_info(nodes[i].op, &nin, &nst, &nco) != MLB_OK)
      return fail(MLB_ERR_INVALID, "node %d: unknown op %d", i, nodes[i].op);
    for (int k = 0; k < MLB_MAX_INS; ++k)
    {
      const int src = nodes[i].in[k];
      if (k < nin)
      {
        if (src < 0 || src >= i)
          return fail(MLB_ERR_INVALID, "node %d (%s): input %d must be an earlier node", i,
                      mlb_op_name(nodes[i].op), k);
      }
      else if (src != -1)
        return fail(MLB_ERR_INVALID, "node %d (%s): unused input %d must be -1", i,
                    mlb_op_name(nodes[i].op), k);
    }
    if (nodes[i].op == MLB_OP_INPUT)
    {
      if (nodes[i].iarg < 0 || nodes[i].iarg >= 64)
        return fail(MLB_ERR_INVALID, "node %d: INPUT plane %d out of range", i, nodes[i].iarg);
      nin_planes = std::max(nin_planes, nodes[i].iarg + 1);
    }
    if (nodes[i].op == MLB_OP_FDN8_R && nodes[nodes[i].in[0]].op != MLB_OP_FDN8)
      return fail(MLB_ERR_INVALID, "node %d: FDN8_R must read an FDN8 node", i);
    if (nodes[i].op == MLB_OP_HALFBAND_UP_2 && nodes[nodes[i].in[0]].op != MLB_OP_HALFBAND_UP)
      return fail(MLB_ERR_INVALID, "node %d: HALFBAND_UP_2 must read a HALFBAND_UP node", i);
    if (nodes[i].op == MLB_OP_FDN8) ++n_fdn;
    if (nodes[i].op == MLB_OP_FEEDBACK_WRITE)
    {
      const int rd = nodes[i].iarg;
      if (rd < 0 || rd >= i || nodes[rd].op != MLB_OP_FEEDBACK_READ)
        return fail(MLB_ERR_INVALID, "node %d: FEEDBACK_WRITE.iarg must name an earlier FEEDBACK_READ node", i);
      for (int q = 0; q < i; ++q)
        if (nodes[q].op == MLB_OP_FEEDBACK_WRITE && nodes[q].iarg == rd)
          return fail(MLB_ERR_INVALID, "node %d: FEEDBACK_READ %d already has a FEEDBACK_WRITE (node %d)", i, rd, q);
    }
    const int again = again_target(nodes, i);
    if (again >= 0)
    {
      if (!again_allowed(nodes[i].op))
        return fail(MLB_ERR_INVALID, "node %d (%s): iarg %d -- this op cannot be called again in a vector (MLB_AGAIN)", i,
                    mlb_op_name(nodes[i].op), nodes[i].iarg);
      if (again >= i || nodes[again].op != nodes[i].op || again_target(nodes, again) >= 0)
        return fail(MLB_ERR_INVALID, "node %d (%s): MLB_AGAIN(%d) must name an earlier node of the same op that is not "
                    "itself an AGAIN node", i, mlb_op_name(nodes[i].op), again);
      // a further call of node `again`: its words, no words of its own
      if (state_off) state_off[i] = state_off[again];
      if (coef_off) coef_off[i] = coef_off[again];
      continue;
    }
    if (state_off) state_off[i] = ns;
    if (coef_off) coef_off[i] = nc;
    ns += nst;
    nc += nco;
  }
  if (n_fdn > 1) return fail(MLB_ERR_UNSUPPORTED, "at most one FDN8 node per graph");
  layout->n_state_words = ns;
  layout->n_coef_words = nc;
  layout->n_inputs = nin_planes;
  return MLB_OK;
}

// ------------------------------------------------------------------------------------------
// coefficient design on the host with glibc libm -- the same calls the reference makes, so
// coefficients are bit-identical by construction (SURVEY 8c "third-party arithmetic").

static const float kPiF = 3.1415926535897932384626433f;     // ScalarMath.h:24
static const float kTwoPiF = 6.2831853071795864769252867f;  // ScalarMath.h:23

static void svf_g(float omega, float k, float* g0, float* g1, float* g2)
{
  volatile float piOmega = kPiF * omega;
  volatile float s1 = sinf(piOmega);
  volatile float s2 = sinf(2.0f * piOmega);
  volatile float nrm = 1.0f / (2.f + k * s2);
  *g0 = s2 * nrm;
  volatile float a = -2.f * s1 * s1;
  volatile float b = k * s2;
  volatile float c = a - b;
  *g1 = c * nrm;
  volatile float d = 2.0f * s1 * s1;
  *g2 = d * nrm;
}
extern "C" void mlb_coeffs_lopass(float omega, float k, float o[3]) { svf_g(omega, k, &o[0], &o[1], &o[2]); }
extern "C" void mlb_coeffs_hipass(float omega, float k, float o[4])
{
  svf_g(omega, k, &o[0], &o[1], &o[2]);
  o[3] = k;
}
extern "C" void mlb_coeffs_bandpass(float omega, float k, float o[3]) { svf_g(omega, k, &o[0], &o[1], &o[2]); }
extern "C" void mlb_coeffs_loshelf(float omega, float k, float A, float r[5])
{
  volatile float piOmega = kPiF * omega;
  volatile float g = tanf(piOmega) / sqrtf(A);
  volatile float t0 = g + k;
  volatile float t1 = g * t0;
  volatile float t2 = 1.f + t1;
  r[0] = 1.f / t2;
  r[1] = g * r[0];
  r[2] = g * r[1];
  volatile float am1 = A - 1.f;
  r[3] = k * am1;
  volatile float aa = A * A;
  r[4] = aa - 1.f;
}
extern "C" void mlb_coeffs_hishelf(float omega, float k, float A, float r[6])
{
  volatile float piOmega = kPiF * omega;
  volatile float g = tanf(piOmega) * sqrtf(A);
  volatile float t0 = g + k;
  volatile float t1 = g * t0;
  volatile float t2 = 1.f + t1;
  r[0] = 1.f / t2;
  r[1] = g * r[0];
  r[2] = g * r[1];
  r[3] = A * A;
  volatile float oma = 1.f - A;
  volatile float koma = k * oma;
  r[4] = koma * A;
  volatile float aa = A * A;
  r[5] = 1.f - aa;
}
extern "C" void mlb_coeffs_bell(float omega, float k, float A, float r[4])
{
  volatile float kc = k / A;
  volatile float piOmega = kPiF * omega;
  volatile float g = tanf(piOmega);
  volatile float t0 = g + kc;
  volatile float t1 = g * t0;
  volatile float t2 = 1.f + t1;
  volatile float a1 = 1.f / t2;
  volatile float a2 = g * a1;
  volatile float a3 = g * a2;
  volatile float aa = A * A;
  volatile float aam1 = aa - 1.f;
  r[0] = a1, r[1] = a2, r[2] = a3, r[3] = kc * aam1;
}
extern "C" void mlb_coeffs_onepole(float omega, float r[2])
{
  volatile float arg = -omega * kTwoPiF;
  volatile float x = expf(arg);
  r[0] = 1.f - x;
  r[1] = x;
}
extern "C" float mlb_coeffs_dcblocker(float omega) { return cosf(omega); }
extern "C" float mlb_db_to_gain(float dB)
{
  volatile float e = dB / 40.f;
  return powf(10.f, e);
}
extern "C" void mlb_coeffs_peak(float omega, float r[2]) { mlb_coeffs_onepole(omega, r); }
extern "C" void mlb_coeffs_rms(float omega, float r[2]) { mlb_coeffs_onepole(omega, r); }
extern "C" void mlb_coeffs_adsr(float a, float d, float s, float rel, float sr, float o[4])
{
  const float minSegmentTime = 0.0002f;
  volatile float invSr = 1.0f / sr;
  volatile float num = kTwoPiF * invSr;
  o[0] = num / (a > minSegmentTime ? a : minSegmentTime);
  o[1] = num / (d > minSegmentTime ? d : minSegmentTime);
  o[2] = s;
  o[3] = num / (rel > minSegmentTime ? rel : minSegmentTime);
}
extern "C" float mlb_coeffs_allpass1(float d)
{
  volatile float xm1 = d - 1.f;
  volatile float t0 = -0.53f * xm1;
  volatile float t1 = 0.24f * xm1;
  volatile float t2 = t1 * xm1;
  return t0 + t2;
}
// ImpulseGen's constructor, G:64-78 (window: MLDSPUtils.h:22-35; normalize / sum: MLDSPOps.h:995-1049 with
// vecSumH's (v0 + v2) + (v1 + v3) order, MLDSPMathSSE.h:246-251)
extern "C" void mlb_impulse_table(float t17[17])
{
  float row[MLB_BLOCK];
  memset(row, 0, sizeof(row));
  for (int i = 0; i < 17; ++i)
  {
    volatile float m = (1.f - 0.f) / (16.f - 0.f);
    volatile float x = m * ((float)i - 0.f) + 0.f;
    volatile float c1 = cosf(kTwoPiF * x);
    volatile float c2 = cosf(2.f * kTwoPiF * x);
    volatile float w0 = 0.5f * c1;
    volatile float w1 = 0.42f - w0;
    volatile float w2 = 0.08f * c2;
    volatile float w = w1 + w2;
    const int idx = i - 8;
    volatile float pi_x = kTwoPiF * 0.25f * (float)idx;
    volatile float sinc = (idx == 0) ? 1.f : sinf(pi_x) / pi_x;
    row[i] = sinc * w;
  }
  volatile float sum = 0.f;
  for (int n = 0; n < MLB_BLOCK; n += 4)
  {
    volatile float a = row[n] + row[n + 2];
    volatile float b = row[n + 1] + row[n + 3];
    volatile float ab = a + b;
    sum = sum + ab;
  }
  for (int i = 0; i < 17; ++i) t17[i] = row[i] / sum;
}
extern "C" void mlb_coeffs_glide(float t, float o[2])
{
  int n = (int)(t / (float)MLB_BLOCK);
  if (n < 1) n = 1;
  o[0] = (float)n;
  o[1] = 1.0f / ((float)n + 0.f);
}
extern "C" void mlb_coeffs_sample_glide(float t, float o[2])
{
  int n = (int)t;
  if (n < 1) n = 1;
  o[0] = (float)n;
  o[1] = 1.0f / (float)n;
}
// Lopass::makeCoeffsVec, F:97-115 (clamps by _mm_min_ps / _mm_max_ps operand order, then per-sample makeCoeffs)
extern "C" void mlb_coeffs_lopass_vec(const float omega[64], const float k[64], float out[3 * 64])
{
  for (int n = 0; n < MLB_BLOCK; ++n)
  {
    const float om = omega[n] < 0.5f ? omega[n] : 0.5f;  // min(omega, DSPVector(0.5f))
    const float kk = k[n] > 0.01f ? k[n] : 0.01f;        // max(k, DSPVector(0.01f))
    svf_g(om, kk, &out[n], &out[MLB_BLOCK + n], &out[2 * MLB_BLOCK + n]);
  }
}
extern "C" void mlb_coeffs_lopass_vec_n(const float* omega, const float* k, float* out, size_t n_rows)
{
  for (size_t r = 0; r < n_rows; ++r)
    mlb_coeffs_lopass_vec(omega + r * MLB_BLOCK, k + r * MLB_BLOCK, out + r * 3 * MLB_BLOCK);
}
// interpolateCoeffsLinear, F:32-44; interpolateDSPVectorLinear, O:986-990 (columnIndex() * interval + (start + interval))
extern "C" void mlb_interpolate_coeffs_linear(const float* c0, const float* c1, int n_coeffs, float* out)
{
  for (int i = 0; i < n_coeffs; ++i)
  {
    volatile float diff = c1[i] - c0[i];
    volatile float interval = diff / (float)MLB_BLOCK;
    volatile float base = c0[i] + interval;
    for (int n = 0; n < MLB_BLOCK; ++n)
    {
      volatile float ramp = (float)n * interval;
      out[(size_t)i * MLB_BLOCK + n] = ramp + base;
    }
  }
}

// n voices at once: out[word][n] (the SoA layout of mlb_graph_set_coefs).  kind = the node op.
extern "C" int mlb_coeffs_batch(int op, size_t n, const float* omega, const float* k, const float* A, float* out)
{
  if (!omega || !out) return fail(MLB_ERR_INVALID, "null argument");
  int nco = 0;
  switch (op)
  {
    case MLB_OP_LOPASS: case MLB_OP_BANDPASS: nco = 3; break;
    case MLB_OP_HIPASS: case MLB_OP_BELL: nco = 4; break;
    case MLB_OP_LOSHELF: nco = 5; break;
    case MLB_OP_HISHELF: nco = 6; break;
    case MLB_OP_ONEPOLE: nco = 2; break;
    default: return fail(MLB_ERR_INVALID, "mlb_coeffs_batch: op %d has no omega/k/A coefficient design", op);
  }
  if (op != MLB_OP_ONEPOLE && !k) return fail(MLB_ERR_INVALID, "k is null");
  if ((op == MLB_OP_BELL || op == MLB_OP_LOSHELF || op == MLB_OP_HISHELF) && !A) return fail(MLB_ERR_INVALID, "A is null");
  for (size_t v = 0; v < n; ++v)
  {
    float c[6];
    switch (op)
    {
      case MLB_OP_LOPASS: mlb_coeffs_lopass(omega[v], k[v], c); break;
      case MLB_OP_BANDPASS: mlb_coeffs_bandpass(omega[v], k[v], c); break;
      case MLB_OP_HIPASS: mlb_coeffs_hipass(omega[v], k[v], c); break;
      case MLB_OP_BELL: mlb_coeffs_bell(omega[v], k[v], A[v], c); break;
      case MLB_OP_LOSHELF: mlb_coeffs_loshelf(omega[v], k[v], A[v], c); break;
      case MLB_OP_HISHELF: mlb_coeffs_hishelf(omega[v], k[v], A[v], c); break;
      default: mlb_coeffs_onepole(omega[v], c); break;
    }
    for (int w = 0; w < nco; ++w) out[(size_t)w * n + v] = c[w];
  }
  return MLB_OK;
}
extern "C" void mlb_coeffs_fdn8(const float times[8], const float cutoffs[8], const float gains[8],
                                float out32[32])
{
  for (int n = 0; n < 8; ++n)
  {
    float c[2];
    mlb_coeffs_onepole(cutoffs[n], c);
    out32[n] = c[0];
    out32[8 + n] = c[1];
    out32[16 + n] = gains[n];
    // FDN::setDelaysInSamples, F:1173-1183: int len = times[n] - 64; len = max(1, len)
    int len = (int)(times[n] - (float)MLB_BLOCK);
    out32[24 + n] = (float)std::max(1, len);
  }
}

// ------------------------------------------------------------------------------------------
// device

static int g_device = -1;
static int g_sm_count = 0;
static size_t g_smem_optin = 0;
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

extern "C" int mlb_device_count(void)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess)
  {
    cudaGetLastError();
    return 0;
  }
  return n;
}

extern "C" int mlb_init(int device)
{
  int n = mlb_device_count();
  if (n <= 0)
    return fail(MLB_ERR_NO_DEVICE,
                "no CUDA device visible: this library has no CPU fallback (sm_90a kernels only)");
  if (device < 0 || device >= n) return fail(MLB_ERR_INVALID, "device %d out of range (%d)", device, n);
  // one device per process (one process per GPU is the multi-GPU model, DESIGN.md 6): retargeting while
  // handles of the current device are alive would leave them with foreign pointers
  if (g_device >= 0 && device != g_device && g_live_handles.load() > 0)
    return fail(MLB_ERR_INVALID, "mlb_init(%d): %d handle(s) of device %d are still alive (one device per process)",
                device, g_live_handles.load(), g_device);
  CU_CHECK(cudaSetDevice(device));
  cudaDeviceProp p;
  CU_CHECK(cudaGetDeviceProperties(&p, device));
  if (p.major != 9 || p.minor != 0)
    return fail(MLB_ERR_NO_DEVICE, "device %d is sm_%d%d; this library ships sm_90a code only",
                device, p.major, p.minor);
  g_sm_count = p.multiProcessorCount;
  g_smem_optin = p.sharedMemPerBlockOptin;
  if (!g_encode)
  {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CU_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !fn)
      return fail(MLB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    g_encode = (EncodeTiledFn)fn;
  }
  {
    float table[17];
    mlb_impulse_table(table);  // ImpulseGen's windowed sinc, host libm
    CU_CHECK(cudaMemcpyToSymbol(c_impulse_table, table, sizeof(table)));
  }
  // mix_reduce_kernel runs between two chain kernels that need the maximum shared-memory carve-out: keep the
  // SMs in that configuration instead of switching the L1 / shared split twice per step
  cudaFuncSetAttribute((const void*)mix_reduce_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                       (int)cudaSharedmemCarveoutMaxShared);
  g_device = device;
  return MLB_OK;
}

static int ensure_init()
{
  if (g_device >= 0)
  {
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != g_device) cudaSetDevice(g_device);
    return MLB_OK;
  }
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess)
  {
    cudaGetLastError();
    dev = 0;
  }
  return mlb_init(dev);
}

// Tensor map over planes of [V][64] f32 that moves FULL 256-byte rows yet lands as two
// 128B-swizzled half tiles: dims {32 samples, V voices, 2 halves, n_planes} with strides
// {256 B, 128 B, plane} and box {32, 32, 2, 1} (8 KB per TMA op).
static int make_block_map(CUtensorMap* map, const float* base, int V, long long n_planes,
                          long long plane_stride_floats)
{
  cuuint64_t dims[4] = {(cuuint64_t)kTileSamples, (cuuint64_t)V, 2, (cuuint64_t)n_planes};
  cuuint64_t strides[3] = {(cuuint64_t)MLB_BLOCK * 4, (cuuint64_t)kTileSamples * 4,
                           (cuuint64_t)plane_stride_floats * 4};
  cuuint32_t box[4] = {(cuuint32_t)kTileSamples, (cuuint32_t)kTileVoices, 2, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MLB_ERR_CUDA, "cuTensorMapEncodeTiled failed: %d", (int)r);
  return MLB_OK;
}

// Encoded tensor maps are pure functions of (base, V, planes, plane stride): a graph keeps the few it has
// built (an audio callback re-uses the same buffers call after call), so a steady-state process call does
// no driver work besides the launches.
struct MapKey
{
  const void* base;
  int V;
  long long n_planes, stride;
  bool operator==(const MapKey& o) const { return base == o.base && V == o.V && n_planes == o.n_planes && stride == o.stride; }
};
struct MapCache
{
  static constexpr int kEntries = 40;  // 2 maps x 16 host slices + device-path buffers
  MapKey key[kEntries];
  CUtensorMap map[kEntries];
  int n = 0, next = 0;
  long long hits = 0, misses = 0;
};
static int cached_block_map(MapCache* c, CUtensorMap* out, const float* base, int V, long long n_planes,
                            long long plane_stride_floats)
{
  const MapKey k{base, V, n_planes, plane_stride_floats};
  for (int i = 0; i < c->n; ++i)
    if (c->key[i] == k)
    {
      *out = c->map[i];
      ++c->hits;
      return MLB_OK;
    }
  int rc = make_block_map(out, base, V, n_planes, plane_stride_floats);
  if (rc != MLB_OK) return rc;
  const int slot = c->n < MapCache::kEntries ? c->n++ : (c->next++ % MapCache::kEntries);
  c->key[slot] = k;
  c->map[slot] = *out;
  ++c->misses;
  return MLB_OK;
}
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per kernel and size, not once per launch
static int ensure_func_smem(const void* fn, size_t smem)
{
  static std::mutex mu;
  static std::vector<std::pair<const void*, size_t>> seen;
  std::lock_guard<std::mutex> lock(mu);
  for (auto& e : seen)
    if (e.first == fn)
    {
      if (e.second >= smem) return MLB_OK;
      CU_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      e.second = smem;
      return MLB_OK;
    }
  CU_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // every kernel of this library wants the SM's L1 / shared split at "maximum shared": the rings of several CTAs
  // (or one 197-KB CTA) per SM set the occupancy, and kernels that follow each other then never make the SM switch
  CU_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
  seen.emplace_back(fn, smem);
  return MLB_OK;
}

// ------------------------------------------------------------------------------------------
// fused chain registry

typedef void (*ChainKernelFn)(const CUtensorMap, const CUtensorMap, const ChainArgs);
struct FusedEntry
{
  int gen, src, f1, f2, gain, exact;
  ChainKernelFn fn;
  const char* name;
  bool has_in;
  int n_planes;  // 8-KB planes a ring stage holds (Chain::NP): the input row and/or coefficient rows
  ChainKernelFn team_fn;  // two-warp team variant for small banks (chain_team_kernel), or nullptr
};
template <class P>
static constexpr ChainKernelFn team_fn_of()
{
  if constexpr (P::SPLIT)
    return chain_team_kernel<P>;
  else
    return nullptr;
}

#define N_ (-1)
// (GEN, SRC, F1, F2, GAIN)
#define MLB_FUSED_LIST(X)                                                   \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_LOPASS, N_, true)   /* config 1 / A */   \
  X(MLB_OP_SINE, SRC_PARAM, MLB_OP_LOPASS, N_, true)   /* contract S / M */ \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_LOPASS, N_, false)  /* config 2 */       \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_HIPASS, N_, false)                       \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_BANDPASS, N_, false)                     \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_LOSHELF, N_, false)                      \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_HISHELF, N_, false)                      \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_BELL, N_, false)                         \
  X(MLB_OP_PHASOR, SRC_INPUT, MLB_OP_LOPASS, MLB_OP_ONEPOLE, false) /* config 3 */ \
  X(MLB_OP_SINE, SRC_INPUT, N_, N_, false)                                  \
  X(MLB_OP_PHASOR, SRC_INPUT, N_, N_, false)                                \
  X(MLB_OP_SAW, SRC_INPUT, N_, N_, false)                                   \
  X(MLB_OP_NOISE, SRC_NONE, N_, N_, false)                                  \
  X(MLB_OP_NOISE, SRC_NONE, MLB_OP_LOPASS, N_, true)                        \
  X(N_, SRC_INPUT, MLB_OP_LOPASS, N_, false)                                \
  X(N_, SRC_INPUT, MLB_OP_ONEPOLE, N_, false)                               \
  X(N_, SRC_INPUT, MLB_OP_DCBLOCKER, N_, false)                             \
  /* swept filter: coefficient ROWS as three more input planes (20 B per voice-sample) */ \
  X(MLB_OP_SINE, SRC_INPUT, MLB_OP_LOPASS_V, N_, true)                      \
  X(MLB_OP_SINE, SRC_PARAM, MLB_OP_LOPASS_V, N_, true)                      \
  X(N_, SRC_INPUT, MLB_OP_LOPASS_V, N_, false)

static const FusedEntry g_fused[] = {
#define MLB_X_ENTRY(G, S, F1, F2, GN)                                                          \
  {G, S, F1, F2, GN, 1, chain_kernel<Chain<G, S, F1, F2, GN, true>>, #G "+" #F1 "+" #F2 "+" #GN, \
   S == SRC_INPUT, Chain<G, S, F1, F2, GN, true>::NP, team_fn_of<Chain<G, S, F1, F2, GN, true>>()}, \
      {G, S, F1, F2, GN, 0, chain_kernel<Chain<G, S, F1, F2, GN, false>>,                        \
       #G "+" #F1 "+" #F2 "+" #GN "(fast)", S == SRC_INPUT, Chain<G, S, F1, F2, GN, false>::NP,    \
       team_fn_of<Chain<G, S, F1, F2, GN, false>>()},
    MLB_FUSED_LIST(MLB_X_ENTRY)
#undef MLB_X_ENTRY
};

// ------------------------------------------------------------------------------------------
// graph object

enum GraphKind
{
  KIND_FUSED = 0,
  KIND_FDN = 1,
  KIND_GENERIC = 2
};

struct mlb_graph
{
  // declared first, so released last: the buffers below are freed first, and cudaFree waits for the device
  LiveCount live;
  static constexpr int kMaxHostSlices = 64;
  Stream stream, s_h2d, s_d2h;  // staging for the host entry point
  Event ev_up[kMaxHostSlices], ev_k[kMaxHostSlices];
  Event ev0, ev1;
  // asynchronous mix bus (mlb_graph_set_mix_async): mix_reduce_kernel (and the multi-GPU exchange) run on s_mix,
  // beside the next call's chain kernel; the per-group partials are double-buffered by call parity
  Stream s_mix;
  Event ev_main, ev_mixdone[4];

  std::vector<mlb_node> nodes;
  std::vector<int32_t> outs;
  std::vector<int32_t> st_off, co_off;
  mlb_layout layout{};
  int V = 0;
  unsigned flags = 0;
  bool exact = true;
  int kind = KIND_GENERIC;
  std::string kernel_name;

  // device SoA
  DevBuf<uint32_t> d_state;
  DevBuf<float> d_coef;
  std::vector<float> h_coef;  // host mirror (ring sizing, FDN descriptors)

  // fused chain
  const FusedEntry* fused = nullptr;
  ChainArgs cargs{};

  // FM3 -> FDN8 specialisation
  FdnArgs fargs{};

  // generic interpreter
  std::vector<GNode> gnodes;   // stage programs back to back (imports + nodes)
  DevBuf<GNode> d_gnodes;
  int scratch_slot = 0;
  std::vector<GStage> gstages;
  DevBuf<GStage> d_gstages;
  int n_stages = 1, n_chan = 0;
  DevBuf<unsigned> d_gsync;  // [0] ticket, [1 + s*G + g] blocks finished by stage s of group g
  DevBuf<float> d_chan;      // channel planes [T][n_chan][V][64]

  int n_slots = 0;

  // FDN delay memory
  int fdn_node = -1;
  DevBuf<float> d_ring, d_carry;
  int ring_len = 0;
  long long blocks_done = 0;
  int reserved_sms = 0;
  // delay memory of the section-8(f) functors: member rows [V][64] and rings [V][stride] per node
  bool has_dmem = false;
  DevBuf<float> d_dmem;
  size_t dmem_floats = 0;
  std::vector<unsigned> ring_stride;  // per node, 0 = no ring

  // chain scheduler words, all maintained by the kernels themselves (see ChainArgs)
  DevBuf<unsigned> d_sched;
  int launch_chunks = 1;  // chunks per group of the most recent launch (all slices of one host call agree)

  // mix bus partials
  DevBuf<float> d_partial;

  // staging for the host entry point
  DevBuf<float> d_in, d_out, d_mix;
  bool timed = false;
  int last_host_slices = 0;  // voice slices of the most recent mlb_graph_process_host call (1 = one launch)
  MapCache maps;
  int mix_async = 0;
  unsigned mix_seq = 0;
  bool mix_pending = false;
  float* partial_cur = nullptr;  // the partial buffer of the call being issued
  struct mlb_mixbus* bus = nullptr;  // multi-GPU: the mix bus is all-reduced over peer memory inside mix_reduce_kernel
};

// delay memory of an op: 64-float member rows and IntegerDelay rings per voice (MLB_OP_MEM_TABLE)
static void op_mem(int op, int* n_rows, int* n_rings)
{
  *n_rows = *n_rings = 0;
  switch (op)
  {
#define MLB_X_MEM(NAME, rows, rings) \
  case MLB_OP_##NAME: *n_rows = rows, *n_rings = rings; break;
    MLB_OP_MEM_TABLE(MLB_X_MEM)
#undef MLB_X_MEM
    default: break;
  }
}

static bool is_filter(int op)
{
  switch (op)
  {
    case MLB_OP_LOPASS:
    case MLB_OP_HIPASS:
    case MLB_OP_BANDPASS:
    case MLB_OP_LOSHELF:
    case MLB_OP_HISHELF:
    case MLB_OP_BELL:
    case MLB_OP_ONEPOLE:
    case MLB_OP_DCBLOCKER:
    case MLB_OP_DIFFERENTIATOR:
    case MLB_OP_INTEGRATOR: return true;
  }
  return false;
}
static bool is_vfilter(int op) { return op == MLB_OP_LOPASS_V || op == MLB_OP_LOSHELF_V || op == MLB_OP_HISHELF_V; }
static bool is_gen1(int op)
{
  return op == MLB_OP_SINE || op == MLB_OP_PHASOR || op == MLB_OP_SAW || op == MLB_OP_TICK;
}

// Recognise  out = [gain *] F2( F1( GEN(src) ) )  and fill g->cargs index maps.
static bool has_again_nodes(const mlb_graph* g);
static bool match_fused_chain(mlb_graph* g)
{
  if (has_again_nodes(g)) return false;  // a functor called twice per vector: interpreter only
  if (g->outs.size() != 1) return false;
  const auto& N = g->nodes;
  std::vector<char> used(N.size(), 0);
  int y = g->outs[0];
  int gain_node = -1;
  if (N[y].op == MLB_OP_MULTIPLY)
  {
    const int a = N[y].in[0], b = N[y].in[1];
    used[y] = 1;
    if (N[b].op == MLB_OP_PARAM && N[a].op != MLB_OP_PARAM)
      gain_node = b, y = a;
    else if (N[a].op == MLB_OP_PARAM && N[b].op != MLB_OP_PARAM)
      gain_node = a, y = b;
    else
      return false;
    used[gain_node] = 1;
  }
  int filt[2] = {-1, -1};
  int nf = 0;
  while (is_filter(N[y].op) || is_vfilter(N[y].op))
  {
    if (nf == 2) return false;
    filt[nf++] = y;
    used[y] = 1;
    y = N[y].in[0];
  }
  // filt[] is output-side first: reverse into signal order
  int f1 = -1, f2 = -1;
  if (nf == 1) f1 = filt[0];
  if (nf == 2) f1 = filt[1], f2 = filt[0];
  int gen = -1, src = SRC_NONE, src_node = -1, gen_node = -1;
  if (is_gen1(N[y].op))
  {
    gen = N[y].op, gen_node = y;
    used[y] = 1;
    src_node = N[y].in[0];
  }
  else if (N[y].op == MLB_OP_NOISE)
  {
    gen = MLB_OP_NOISE, gen_node = y;
    used[y] = 1;
  }
  else
    src_node = y;
  if (src_node >= 0)
  {
    used[src_node] = 1;
    if (N[src_node].op == MLB_OP_INPUT)
      src = SRC_INPUT;
    else if (N[src_node].op == MLB_OP_PARAM)
      src = SRC_PARAM;
    else
      return false;
  }
  // a coefficient-row filter is fused only as F1, with every coefficient row an external INPUT plane
  if (f2 >= 0 && is_vfilter(N[f2].op)) return false;
  if (f1 >= 0 && is_vfilter(N[f1].op))
  {
    int nin = 0;
    mlb_op_info(N[f1].op, &nin, nullptr, nullptr);
    for (int k = 1; k < nin; ++k)
    {
      if (N[N[f1].in[k]].op != MLB_OP_INPUT) return false;
      used[N[f1].in[k]] = 1;
    }
  }
  for (char u : used)
    if (!u) return false;  // every node must be on the chain (unused stateful nodes still tick)
  const int f1op = f1 >= 0 ? N[f1].op : -1, f2op = f2 >= 0 ? N[f2].op : -1;
  for (const FusedEntry& e : g_fused)
  {
    if (e.gen == gen && e.src == src && e.f1 == f1op && e.f2 == f2op &&
        e.gain == (gain_node >= 0 ? 1 : 0) && e.exact == (g->exact ? 1 : 0))
    {
      g->fused = &e;
      ChainArgs& c = g->cargs;
      memset(&c, 0, sizeof(c));
      int si = 0, ci = 0;
      auto add_state = [&](int node)
      {
        int nst = 0;
        mlb_op_info(N[node].op, nullptr, &nst, nullptr);
        for (int k = 0; k < nst; ++k) c.st_idx[si++] = g->st_off[node] + k;
      };
      auto add_coef = [&](int node)
      {
        int nco = 0;
        mlb_op_info(N[node].op, nullptr, nullptr, &nco);
        for (int k = 0; k < nco; ++k) c.co_idx[ci++] = g->co_off[node] + k;
      };
      if (gen_node >= 0) add_state(gen_node);
      if (f1 >= 0) add_state(f1);
      if (f2 >= 0) add_state(f2);
      if (src == SRC_PARAM) add_coef(src_node);
      if (f1 >= 0) add_coef(f1);
      if (f2 >= 0) add_coef(f2);
      if (gain_node >= 0) add_coef(gain_node);
      c.in_plane = (src == SRC_INPUT) ? N[src_node].iarg : 0;
      if (f1 >= 0 && is_vfilter(N[f1].op))
      {
        int nin = 0;
        mlb_op_info(N[f1].op, &nin, nullptr, nullptr);
        for (int k = 1; k < nin; ++k) c.cv_plane[k - 1] = N[N[f1].in[k]].iarg;
      }
      g->kernel_name = std::string("fused:") + e.name;
      return true;
    }
  }
  return false;
}

static bool has_again_nodes(const mlb_graph* g)
{
  for (int i = 0; i < (int)g->nodes.size(); ++i)
    if (again_target(g->nodes.data(), i) >= 0) return true;
  return false;
}
static int env_int(const char* name, int dflt);
// ops with two output rows (the second is read through the paired *_R / *_2 op)
static bool is_dual(int op) { return op == MLB_OP_FDN8 || op == MLB_OP_HALFBAND_UP; }
static bool is_second(int op) { return op == MLB_OP_FDN8_R || op == MLB_OP_HALFBAND_UP_2; }

// Relative cost of one node-block in the interpreter (used only to balance pipeline stages).
static int node_cost(int op)
{
  if (op == MLB_OP_PARAM || op == MLB_OP_INPUT || op == MLB_OP_FDN8_R || op == MLB_OP_HALFBAND_UP_2) return 0;
  if (op >= MLB_OP_MAP_FIRST && op < MLB_OP_MAP_END) return 2;
  switch (op)
  {
    case MLB_OP_ONEPOLE:
    case MLB_OP_DIFFERENTIATOR:
    case MLB_OP_INTEGRATOR:
    case MLB_OP_DCBLOCKER:
    case MLB_OP_RMS:
    case MLB_OP_ALLPASS1: return 8;
    case MLB_OP_FDN8: return 200;
    case MLB_OP_ALLPASS_PB:
    case MLB_OP_PITCHBEND_DELAY: return 40;
    case MLB_OP_ALLPASS_INT:
    case MLB_OP_ALLPASS_FRAC:
    case MLB_OP_FRACTIONAL_DELAY:
    case MLB_OP_FRACTIONAL_DELAY_VAR:
    case MLB_OP_INTEGER_DELAY_VAR: return 20;
    case MLB_OP_FEEDBACK_READ:
    case MLB_OP_FEEDBACK_WRITE:
    case MLB_OP_INTEGER_DELAY:
    case MLB_OP_GLIDE:
    case MLB_OP_INTERPOLATOR1: return 4;
    default: return 16;  // SVF family, generators, envelopes
  }
}

// Build the interpreter program (DESIGN.md K5).  The node list is cut into S contiguous *stages*
// (balanced by node_cost); stage s of voice group g is run by its own one-warp CTA for all T
// blocks, so a graph with few voices still fills the machine: stage s works on block t while
// stage s+1 works on block t-1 (a software pipeline across CTAs).  A row that crosses a stage
// boundary travels through a *channel* plane in global memory [T][n_chan][V][64]; per-(stage,
// group) progress words order the producer's stores before the consumer's loads.  Inside a stage
// rows live in shared-memory slots allocated by liveness, as before.  S = 1 is the plain
// single-CTA-per-group interpreter.
static int build_generic(mlb_graph* g)
{
  const auto& N = g->nodes;
  const int n = (int)N.size();
  const int n_groups = (g->V + 31) / 32;
  std::vector<int> out_plane(n, -1);
  for (size_t c = 0; c < g->outs.size(); ++c)
  {
    if (out_plane[g->outs[c]] >= 0)
      return fail(MLB_ERR_UNSUPPORTED, "a node may appear only once in outs");
    out_plane[g->outs[c]] = (int)c;
  }
  // ---- choose the number of stages ----
  long long total_cost = 0;
  int n_real = 0;
  for (int i = 0; i < n; ++i)
  {
    total_cost += node_cost(N[i].op);
    if (node_cost(N[i].op) > 0) ++n_real;
  }
  int S = 1;
  {
    // one warp per scheduler: a second warp on a scheduler halves the pace of both (tools/ubench/dep_latency.cu
    // measures what a lone warp pays per dependent instruction), and every extra stage costs a block of pipeline fill
    const int target_warps = g_sm_count * 4;
    S = (target_warps + n_groups - 1) / n_groups;
    S = std::min(S, std::max(1, n_real / 3));
    S = std::min(S, 64);
    S = env_int("MLB_STAGES", S);
    S = std::min(std::max(S, 1), std::max(1, n_real));
    if (g->flags & MLB_GRAPH_SINGLE_STAGE) S = 1;
  }
  // ---- cut points: stage_of[i], contiguous, balanced by cost ----
  // A feedback loop (FEEDBACK_READ ... its FEEDBACK_WRITE) stays inside one stage: the reader of
  // block t+1 would otherwise wait for a CTA with a LARGER ticket, which need not be resident.
  std::vector<char> no_cut(n, 0);
  for (int q = 0; q < n; ++q)
  {
    if (N[q].op == MLB_OP_FEEDBACK_WRITE)
      for (int i = N[q].iarg; i < q; ++i) no_cut[i] = 1;
    if (is_second(N[q].op))  // FDN8_R / HALFBAND_UP_2 alias the second row of their producer: same stage
      for (int i = N[q].in[0]; i < q; ++i) no_cut[i] = 1;
    // MLB_AGAIN: the calls of one functor share its state words, which a node loads and stores once per vector --
    // they must run in node order inside one CTA
    if (again_target(N.data(), q) >= 0)
      for (int i = again_target(N.data(), q); i < q; ++i) no_cut[i] = 1;
  }
  std::vector<int> stage_of(n, 0);
  {
    long long acc = 0;
    int s = 0;
    for (int i = 0; i < n; ++i)
    {
      stage_of[i] = s;
      acc += node_cost(N[i].op);
      // close the stage once it holds its share of the cost (and a real node)
      if (s < S - 1 && !no_cut[i] && acc * S >= total_cost * (s + 1) && node_cost(N[i].op) > 0) ++s;
    }
    S = stage_of[n - 1] + 1;
  }
  // ---- channels: one per node whose row is read in a later stage (INPUT rows are re-read from `in`) ----
  std::vector<int> chan_of(n, -1);
  int n_chan = 0;
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < MLB_MAX_INS; ++k)
    {
      const int src = N[i].in[k];
      if (src < 0 || stage_of[src] == stage_of[i]) continue;
      if (N[src].op == MLB_OP_PARAM || N[src].op == MLB_OP_INPUT) continue;
      if (chan_of[src] < 0) chan_of[src] = n_chan++;
    }
  // ---- per-stage programs ----
  g->gnodes.clear();
  g->gstages.assign(S, GStage{});
  int max_slots = 1;
  for (int s = 0; s < S; ++s)
  {
    GStage& st = g->gstages[s];
    st.node_begin = (int)g->gnodes.size();
    std::vector<int> members;
    for (int i = 0; i < n; ++i)
      if (stage_of[i] == s) members.push_back(i);
    // rows produced outside this stage and read inside it
    std::vector<int> ext;
    for (int i : members)
      for (int k = 0; k < MLB_MAX_INS; ++k)
      {
        const int src = N[i].in[k];
        if (src < 0 || stage_of[src] == s || N[src].op == MLB_OP_PARAM) continue;
        if (std::find(ext.begin(), ext.end(), src) == ext.end()) ext.push_back(src);
      }
    // producer stages this stage must wait for (block t), and feedback partners
    auto add_wait = [&](int ws)
    {
      if (ws == s) return true;
      for (int q = 0; q < st.n_wait; ++q)
        if (st.wait_stage[q] == ws) return true;
      if (st.n_wait == GStage::kMaxWait) return false;
      st.wait_stage[st.n_wait++] = ws;
      return true;
    };
    auto add_fbwait = [&](int ws)
    {
      if (ws == s) return true;
      for (int q = 0; q < st.n_fbwait; ++q)
        if (st.fbwait_stage[q] == ws) return true;
      if (st.n_fbwait == GStage::kMaxWait) return false;
      st.fbwait_stage[st.n_fbwait++] = ws;
      return true;
    };
    bool ok = true;
    for (int src : ext)
      if (N[src].op != MLB_OP_INPUT) ok = ok && add_wait(stage_of[src]);
    for (int i : members)
    {
      // a FEEDBACK_READ at block t needs its writer's block t-1; the writer must not overwrite the
      // row before the reader of the same block has taken it
      if (N[i].op == MLB_OP_FEEDBACK_READ)
        for (int q = 0; q < n; ++q)
          if (N[q].op == MLB_OP_FEEDBACK_WRITE && N[q].iarg == i) ok = ok && add_fbwait(stage_of[q]);
      if (N[i].op == MLB_OP_FEEDBACK_WRITE) ok = ok && add_wait(stage_of[N[i].iarg]);
    }
    if (!ok) return fail(MLB_ERR_UNSUPPORTED, "stage %d of the interpreter program depends on too many stages", s);

    // liveness inside the stage: local index -> last local reader
    const int n_ext = (int)ext.size(), n_loc = n_ext + (int)members.size();
    auto local_of = [&](int node)
    {
      for (int e = 0; e < n_ext; ++e)
        if (ext[e] == node) return e;
      for (size_t m = 0; m < members.size(); ++m)
        if (members[m] == node) return n_ext + (int)m;
      return -1;
    };
    std::vector<int> last_use(n_loc, -1), slot(n_loc, -1), slot2(n_loc, -1);
    for (size_t m = 0; m < members.size(); ++m)
      for (int k = 0; k < MLB_MAX_INS; ++k)
      {
        const int src = N[members[m]].in[k];
        if (src < 0 || N[src].op == MLB_OP_PARAM) continue;
        last_use[local_of(src)] = n_ext + (int)m;
      }
    std::vector<int> free_slots;
    int n_slots = 0;
    auto alloc = [&]()
    {
      if (!free_slots.empty())
      {
        int q = free_slots.back();
        free_slots.pop_back();
        return q;
      }
      return n_slots++;
    };
    for (int li = 0; li < n_loc; ++li)
    {
      GNode gn{};
      const bool is_ext = li < n_ext;
      const int node = is_ext ? ext[li] : members[li - n_ext];
      gn.src_node = is_ext ? -1 : node;
      gn.out_slot = gn.out_slot2 = -1;
      gn.out_plane = -1;
      gn.chan_out = -1;
      for (int k = 0; k < MLB_MAX_INS; ++k) gn.in_kind[k] = OPERAND_NONE, gn.in_ref[k] = 0;
      if (is_ext)
      {
        // import: re-read an external input plane, or load the producer's channel plane
        if (N[node].op == MLB_OP_INPUT)
          gn.op = MLB_OP_INPUT, gn.iarg = N[node].iarg;
        else
          gn.op = MLB_OP_IMPORT_ROW, gn.iarg = chan_of[node];
        slot[li] = alloc();
      }
      else
      {
        gn.op = N[node].op;
        gn.st_off = g->st_off[node];
        gn.co_off = g->co_off[node];
        gn.iarg = N[node].iarg;
        gn.out_plane = out_plane[node];
        gn.chan_out = chan_of[node];
        for (int k = 0; k < MLB_MAX_INS; ++k)
        {
          const int src = N[node].in[k];
          if (src < 0) continue;
          if (N[src].op == MLB_OP_PARAM)
            gn.in_kind[k] = OPERAND_PARAM, gn.in_ref[k] = g->co_off[src];
          else
            gn.in_kind[k] = OPERAND_SLOT, gn.in_ref[k] = slot[local_of(src)];
        }
        // allocate the output slot BEFORE freeing inputs: nodes never run in place
        if (is_second(N[node].op))
          slot[li] = slot2[local_of(N[node].in[0])];
        else if (N[node].op != MLB_OP_PARAM)
          slot[li] = alloc();
        if (is_dual(N[node].op)) slot2[li] = alloc();
      }
      gn.out_slot = slot[li];
      gn.out_slot2 = slot2[li];
      g->gnodes.push_back(gn);
      // release rows whose last reader is this node
      for (int j = 0; j < li; ++j)
      {
        const int nj = j < n_ext ? ext[j] : members[j - n_ext];
        if (slot[j] < 0 || is_second(N[nj].op)) continue;
        if (last_use[j] == li) free_slots.push_back(slot[j]);
        if (is_dual(N[nj].op) && j >= n_ext)
        {
          // second row is read only through FDN8_R nodes; free it when their last reader ran
          int lu = -1;
          bool has_r = false;
          for (int q = j + 1; q < n_loc; ++q)
          {
            const int nq = q < n_ext ? ext[q] : members[q - n_ext];
            if (q >= n_ext && is_second(N[nq].op) && N[nq].in[0] == nj)
            {
              has_r = true;
              lu = std::max(lu, std::max(last_use[q], q));
            }
          }
          if (has_r && lu == li) free_slots.push_back(slot2[j]);
        }
      }
      // a dual-output node whose second row nobody in this stage reads gives that row back at once
      if (!is_ext && is_dual(N[node].op))
      {
        bool has_r = false;
        for (int q = li + 1; q < n_loc; ++q)
        {
          const int nq = q < n_ext ? ext[q] : members[q - n_ext];
          if (q >= n_ext && is_second(N[nq].op) && N[nq].in[0] == node) has_r = true;
        }
        if (!has_r) free_slots.push_back(slot2[li]);
      }
      // a row nobody in this stage reads can be recycled right after it was written out
      if (slot[li] >= 0 && last_use[li] < 0 && !(li >= n_ext && is_second(N[node].op)))
        free_slots.push_back(slot[li]);
    }
    st.node_end = (int)g->gnodes.size();
    max_slots = std::max(max_slots, n_slots);
  }
  g->n_slots = std::max(1, max_slots);
  g->scratch_slot = g->n_slots;
  for (int i = 0; i < n; ++i)
    if (N[i].op == MLB_OP_PITCHBEND_DELAY || N[i].op == MLB_OP_ALLPASS_PB || N[i].op == MLB_OP_ALLPASS_INT ||
        N[i].op == MLB_OP_ALLPASS_FRAC)
    {
      g->n_slots += 3;  // delay input + two tap streams (cp.async destinations)
      break;
    }
  g->n_stages = S;
  g->n_chan = n_chan;
  const size_t smem = (size_t)g->n_slots * kSlotBytes;
  if (smem > g_smem_optin)
    return fail(MLB_ERR_UNSUPPORTED, "graph needs %d live rows (%zu B shared memory > %zu)",
                g->n_slots, smem, g_smem_optin);
  g->kernel_name = std::string(g->exact ? "generic" : "generic(fast)") + "[" + std::to_string(S) + " stages, " +
                   std::to_string(g->n_slots) + " rows]";
  return MLB_OK;
}

static int size_functor_memory(mlb_graph* g);

// The interpreter's host-side plan for a graph, WITHOUT a device: which pipeline stage every node goes to and how many
// shared-memory row slots the program needs (assuming an H100 SXM: 132 SMs, 227 KB of shared memory per CTA, unless a device
// has been initialised).  The same build_generic() that mlb_graph_create runs; lets the planner's rules -- a feedback
// loop, a paired second row, a functor and its MLB_AGAIN calls stay in one stage; the row pool fits -- be tested on a CPU.
extern "C" int mlb_graph_plan(const mlb_node* nodes, int n_nodes, const int32_t* outs, int n_out, int n_voices,
                              unsigned flags, int32_t* stage_of, int32_t* n_stages, int32_t* n_row_slots)
{
  if (n_voices <= 0) return fail(MLB_ERR_INVALID, "n_voices must be positive");
  if (n_out < 0 || (n_out > 0 && !outs)) return fail(MLB_ERR_INVALID, "bad outs");
  mlb_layout lay;
  std::vector<int32_t> so(std::max(1, n_nodes)), co(std::max(1, n_nodes));
  int rc = mlb_graph_layout(nodes, n_nodes, &lay, so.data(), co.data());
  if (rc != MLB_OK) return rc;
  for (int c = 0; c < n_out; ++c)
    if (outs[c] < 0 || outs[c] >= n_nodes) return fail(MLB_ERR_INVALID, "outs[%d] out of range", c);
  const int sm_saved = g_sm_count;
  const size_t smem_saved = g_smem_optin;
  if (g_sm_count == 0) g_sm_count = 132;
  if (g_smem_optin == 0) g_smem_optin = 232448;
  mlb_graph g;  // host fields only: nothing here touches the CUDA runtime
  g.nodes.assign(nodes, nodes + n_nodes);
  g.outs.assign(outs, outs + n_out);
  g.st_off = so, g.co_off = co, g.layout = lay;
  g.V = n_voices, g.flags = flags, g.exact = !(flags & MLB_GRAPH_FAST);
  rc = build_generic(&g);
  g_sm_count = sm_saved, g_smem_optin = smem_saved;
  if (rc != MLB_OK) return rc;
  if (stage_of)
  {
    for (int i = 0; i < n_nodes; ++i) stage_of[i] = -1;  // PARAM nodes and the like belong to no stage
    for (int s = 0; s < (int)g.gstages.size(); ++s)
      for (int k = g.gstages[s].node_begin; k < g.gstages[s].node_end; ++k)
        if (g.gnodes[k].src_node >= 0) stage_of[g.gnodes[k].src_node] = s;
  }
  if (n_stages) *n_stages = g.n_stages;
  if (n_row_slots) *n_row_slots = g.n_slots;
  return MLB_OK;
}

extern "C" int mlb_graph_create(const mlb_node* nodes, int n_nodes, const int32_t* outs, int n_out,
                                int n_voices, unsigned flags, mlb_graph** out_graph)
{
  if (!out_graph) return fail(MLB_ERR_INVALID, "out_graph is null");
  *out_graph = nullptr;
  if (n_voices <= 0) return fail(MLB_ERR_INVALID, "n_voices must be positive");
  if (n_out < 0 || (n_out > 0 && !outs)) return fail(MLB_ERR_INVALID, "bad outs");
  mlb_layout lay;
  std::vector<int32_t> so(std::max(1, n_nodes)), co(std::max(1, n_nodes));
  int rc = mlb_graph_layout(nodes, n_nodes, &lay, so.data(), co.data());
  if (rc != MLB_OK) return rc;
  for (int c = 0; c < n_out; ++c)
    if (outs[c] < 0 || outs[c] >= n_nodes) return fail(MLB_ERR_INVALID, "outs[%d] out of range", c);
  rc = ensure_init();
  if (rc != MLB_OK) return rc;

  std::unique_ptr<mlb_graph> owner(new mlb_graph);
  mlb_graph* g = owner.get();
  g->live.arm();
  g->nodes.assign(nodes, nodes + n_nodes);
  g->outs.assign(outs, outs + n_out);
  g->st_off = so;
  g->co_off = co;
  g->layout = lay;
  g->V = n_voices;
  g->flags = flags;
  g->exact = !(flags & MLB_GRAPH_FAST);
  for (int i = 0; i < n_nodes; ++i)
  {
    if (nodes[i].op == MLB_OP_FDN8) g->fdn_node = i;
    int rows, rings;
    op_mem(nodes[i].op, &rows, &rings);
    if (rows || rings) g->has_dmem = true;
  }
  g->ring_stride.assign(n_nodes, 0u);

  const size_t V = (size_t)n_voices;
  MLB_TRY(g->d_state.alloc(std::max<size_t>(1, lay.n_state_words) * V * 4, "voice state"));
  MLB_TRY(g->d_coef.alloc(std::max<size_t>(1, lay.n_coef_words) * V * 4, "voice coefficients"));
  // [0] unit counter, [1 + g] finished chunks of group g, [1 + G] finished units, [2 + G] progress base
  MLB_TRY(g->d_sched.alloc(((V + 31) / 32 + 3) * 4, "scheduler words"));
  CU_CHECK(cudaMemset(g->d_sched.get(), 0, g->d_sched.bytes()));
  CU_CHECK(cudaMemset(g->d_state.get(), 0, g->d_state.bytes()));
  // state of freshly constructed functors: zeros, except the "idle" markers
  for (int i = 0; i < n_nodes; ++i)
  {
    int word = -1;
    uint32_t val = 0;
    if (nodes[i].op == MLB_OP_ADSR) word = 7, val = 4u;                   // segment{off}, F:694
    if (nodes[i].op == MLB_OP_GLIDE) word = 2, val = 0xFFFFFFFFu;         // mVectorsRemaining{-1}, G:440
    if (nodes[i].op == MLB_OP_SAMPLE_GLIDE) word = 3, val = 0xFFFFFFFFu;  // mSamplesRemaining{-1}, G:524
    if (nodes[i].op == MLB_OP_TEMPO_LOCK) word = 0, val = 0xBF800000u;    // _omega{-1.f}, F:1481
    if (word < 0) continue;
    std::vector<uint32_t> fill(V, val);
    CU_CHECK(cudaMemcpy(g->d_state.get() + (size_t)(so[i] + word) * V, fill.data(), V * 4, cudaMemcpyHostToDevice));
  }
  CU_CHECK(cudaMemset(g->d_coef.get(), 0, g->d_coef.bytes()));
  g->h_coef.assign((size_t)lay.n_coef_words * V, 0.f);
  for (Stream* s : {&g->stream, &g->s_h2d, &g->s_d2h}) MLB_TRY(s->create(cudaStreamNonBlocking));
  for (int i = 0; i < mlb_graph::kMaxHostSlices; ++i)
  {
    MLB_TRY(g->ev_up[i].create(cudaEventDisableTiming));
    MLB_TRY(g->ev_k[i].create(cudaEventDisableTiming));
  }
  MLB_TRY(g->ev0.create(cudaEventDefault));
  MLB_TRY(g->ev1.create(cudaEventDefault));

  bool matched = false;
  if (!(flags & MLB_GRAPH_FORCE_GENERIC))
  {
    matched = match_fused_chain(g);
    if (matched) g->kind = KIND_FUSED;
    if (!matched && !has_again_nodes(g) && match_fm3_fdn8(g->nodes, g->outs, g->st_off, g->co_off, &g->fargs))
    {
      matched = true;
      g->kind = KIND_FDN;
      g->kernel_name = g->exact ? "fused:fm3_fdn8" : "fused:fm3_fdn8(fast)";
    }
  }
  if (!matched)
  {
    g->kind = KIND_GENERIC;
    MLB_TRY(build_generic(g));
    MLB_TRY(g->d_gnodes.alloc(sizeof(GNode) * g->gnodes.size(), "graph program"));
    MLB_TRY(g->d_gstages.alloc(sizeof(GStage) * g->gstages.size(), "graph program"));
    MLB_TRY(g->d_gsync.alloc((1 + (size_t)g->n_stages * ((V + 31) / 32)) * 4, "graph program"));
    CU_CHECK(cudaMemcpy(g->d_gnodes.get(), g->gnodes.data(), g->d_gnodes.bytes(), cudaMemcpyHostToDevice));
    CU_CHECK(cudaMemcpy(g->d_gstages.get(), g->gstages.data(), g->d_gstages.bytes(), cudaMemcpyHostToDevice));
    MLB_TRY(size_functor_memory(g));
  }
  *out_graph = owner.release();
  return MLB_OK;
}

extern "C" int mlb_graph_destroy(mlb_graph* g)
{
  delete g;
  return MLB_OK;
}

extern "C" int mlb_graph_set_input_planes(mlb_graph* g, int n_planes)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  int need = 0;
  for (const mlb_node& n : g->nodes)
    if (n.op == MLB_OP_INPUT) need = std::max(need, n.iarg + 1);
  if (n_planes < need || n_planes > 64)
    return fail(MLB_ERR_INVALID, "n_planes must be in [%d, 64] for this graph", need);
  g->layout.n_inputs = n_planes;
  return MLB_OK;
}
extern "C" int mlb_graph_reserve_sms(mlb_graph* g, int n_sms)
{
  if (!g || n_sms < 0) return fail(MLB_ERR_INVALID, "bad argument");
  g->reserved_sms = n_sms;
  return MLB_OK;
}
extern "C" int mlb_graph_layout_of(const mlb_graph* g, mlb_layout* layout)
{
  if (!g || !layout) return fail(MLB_ERR_INVALID, "null");
  *layout = g->layout;
  return MLB_OK;
}
extern "C" const char* mlb_graph_kernel_name(const mlb_graph* g) { return g ? g->kernel_name.c_str() : ""; }

// (re)allocate FDN delay memory when the coefficient upload changes the longest delay
static int size_delay_memory(mlb_graph* g)
{
  if (g->fdn_node < 0) return MLB_OK;
  const size_t V = (size_t)g->V;
  const int base = g->co_off[g->fdn_node] + 24;
  int max_len = 1;
  for (int l = 0; l < 8; ++l)
    for (size_t v = 0; v < V; ++v)
    {
      const float f = g->h_coef[(size_t)(base + l) * V + v];
      if (!(f >= 1.0f) || f > 16777216.0f || f != std::floor(f))
        return fail(MLB_ERR_INVALID, "FDN8 delay length coef must be an integer >= 1 (voice %zu line %d: %g)",
                    v, l, (double)f);
      max_len = std::max(max_len, (int)f);
    }
  // IntegerDelay::setMaxDelayInSamples, F:822-830: size = 1 << bitsToContain(dMax + 64)
  int ring = 1;
  while (ring < max_len + MLB_BLOCK) ring <<= 1;
  if (ring != g->ring_len)
  {
    g->d_ring.reset();
    g->d_carry.reset();
    MLB_TRY(g->d_ring.alloc(V * 8 * (size_t)ring * 4, "delay memory"));
    MLB_TRY(g->d_carry.alloc(V * 8 * MLB_BLOCK * 4, "delay memory"));
    g->ring_len = ring;
    return mlb_graph_clear_delays(g);
  }
  return MLB_OK;
}

// Lay out (and, when a ring grows or shrinks, reallocate and clear) the delay memory of the
// section-8(f) functors.  Ring of voice v of a node: 1 << bitsToContain(floor(maxDelay_v') + 64)
// samples (IntegerDelay::setMaxDelayInSamples, F:822-830; maxDelay' = maxDelay - 64 inside an
// Allpass<>, F:1125-1128); every voice of a node gets the stride of the node's longest ring and
// uses its own mask inside it.
static int size_functor_memory(mlb_graph* g)
{
  if (!g->has_dmem) return MLB_OK;
  const size_t V = (size_t)g->V;
  const int n = (int)g->nodes.size();
  std::vector<unsigned> stride(n, 0u);
  std::vector<unsigned long long> row_off(n, 0ull), ring_off(n, 0ull);
  unsigned long long total = 0;
  for (int i = 0; i < n; ++i)
  {
    int rows, rings, nco = 0;
    const int op = g->nodes[i].op;
    op_mem(op, &rows, &rings);
    mlb_op_info(op, nullptr, nullptr, &nco);
    if (again_target(g->nodes.data(), i) >= 0)  // MLB_AGAIN: the member row of the functor's first call (no rings, by rule)
    {
      row_off[i] = row_off[again_target(g->nodes.data(), i)];
      continue;
    }
    if (rows)
    {
      row_off[i] = total;
      total += (unsigned long long)V * MLB_BLOCK;
    }
    if (rings)
    {
      const bool in_allpass = (op == MLB_OP_ALLPASS_INT || op == MLB_OP_ALLPASS_FRAC || op == MLB_OP_ALLPASS_PB);
      const float* md = g->h_coef.data() + (size_t)(g->co_off[i] + nco - 1) * V;  // last coef word = maxDelay
      int dmax = 0;
      for (size_t v = 0; v < V; ++v)
      {
        const float m = md[v] - (in_allpass ? (float)MLB_BLOCK : 0.f);
        if (!(m >= 0.f) || m > 16777216.0f)
        {
          if (md[v] == 0.f) continue;  // coefficients not set yet: smallest ring
          return fail(MLB_ERR_INVALID, "node %d (%s): maxDelay coef of voice %zu is %g (need %s <= maxDelay <= 2^24)", i,
                      mlb_op_name(op), v, (double)md[v], in_allpass ? "64" : "0");
        }
        dmax = std::max(dmax, (int)std::floor(m));
      }
      unsigned ring = 1;
      while (ring < (unsigned)(dmax + MLB_BLOCK)) ring <<= 1;
      stride[i] = ring;
      ring_off[i] = total;
      total += (unsigned long long)V * ring;
    }
  }
  for (int i = 0; i < n; ++i)  // FEEDBACK_WRITE stores into its FEEDBACK_READ's row
    if (g->nodes[i].op == MLB_OP_FEEDBACK_WRITE) row_off[i] = row_off[g->nodes[i].iarg];
  const bool relayout = (total != g->dmem_floats) || (stride != g->ring_stride);
  if (!relayout) return MLB_OK;
  g->dmem_floats = 0;
  MLB_TRY(g->d_dmem.alloc(std::max<unsigned long long>(total, 1) * 4, "delay memory"));
  g->dmem_floats = (size_t)total;
  g->ring_stride = stride;
  for (GNode& gn : g->gnodes)
  {
    if (gn.src_node < 0) continue;
    gn.ring_stride = stride[gn.src_node];
    gn.row_off = row_off[gn.src_node];
    gn.ring_off = ring_off[gn.src_node];
  }
  CU_CHECK(cudaMemcpy(g->d_gnodes.get(), g->gnodes.data(), g->d_gnodes.bytes(), cudaMemcpyHostToDevice));
  return mlb_graph_clear_delays(g);
}

extern "C" int mlb_graph_set_coefs(mlb_graph* g, const float* coef_host)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  if (g->layout.n_coef_words == 0) return MLB_OK;
  if (!coef_host) return fail(MLB_ERR_INVALID, "null coefs");
  const size_t bytes = (size_t)g->layout.n_coef_words * g->V * 4;
  // the sizing passes read the host mirror: hand them the new values, put the old ones back when they are
  // rejected so that the mirror never disagrees with the device copy.  NOTE: a change of any ring size
  // re-lays-out the delay memory and clears ALL delay state of the graph (rings, member rows, write index).
  std::vector<float> old(g->h_coef);
  memcpy(g->h_coef.data(), coef_host, bytes);
  int rc = size_delay_memory(g);
  if (rc == MLB_OK) rc = size_functor_memory(g);
  if (rc != MLB_OK)
  {
    g->h_coef.swap(old);
    return rc;
  }
  CU_CHECK(cudaMemcpy(g->d_coef.get(), coef_host, bytes, cudaMemcpyHostToDevice));
  return MLB_OK;
}
extern "C" int mlb_graph_set_state(mlb_graph* g, const uint32_t* state_host)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  if (g->layout.n_state_words == 0) return MLB_OK;
  if (!state_host) return fail(MLB_ERR_INVALID, "null state");
  CU_CHECK(cudaMemcpy(g->d_state.get(), state_host, (size_t)g->layout.n_state_words * g->V * 4,
                      cudaMemcpyHostToDevice));
  return MLB_OK;
}
extern "C" int mlb_graph_get_state(mlb_graph* g, uint32_t* state_host)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  if (g->layout.n_state_words == 0) return MLB_OK;
  if (!state_host) return fail(MLB_ERR_INVALID, "null state");
  CU_CHECK(cudaDeviceSynchronize());
  CU_CHECK(cudaMemcpy(state_host, g->d_state.get(), (size_t)g->layout.n_state_words * g->V * 4,
                      cudaMemcpyDeviceToHost));
  return MLB_OK;
}
extern "C" int mlb_graph_clear_delays(mlb_graph* g)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  g->blocks_done = 0;
  if (g->d_ring.get())
  {
    CU_CHECK(cudaMemset(g->d_ring.get(), 0, (size_t)g->V * 8 * g->ring_len * 4));
    CU_CHECK(cudaMemset(g->d_carry.get(), 0, (size_t)g->V * 8 * MLB_BLOCK * 4));
  }
  if (g->d_dmem.get()) CU_CHECK(cudaMemset(g->d_dmem.get(), 0, g->dmem_floats * 4));
  return MLB_OK;
}
extern "C" size_t mlb_graph_delay_bytes(const mlb_graph* g)
{
  if (!g) return 0;
  size_t bytes = g->dmem_floats * 4;
  if (g->d_ring.get()) bytes += (size_t)g->V * 8 * ((size_t)g->ring_len + MLB_BLOCK) * 4;
  return bytes;
}

// ------------------------------------------------------------------------------------------
// multi-GPU mix bus over peer memory (one process per GPU; buffers shared through CUDA IPC)

struct mlb_mixbus
{
  // declared first, so released after the exchange buffer (whose cudaFree waits for the device)
  LiveCount live;
  static constexpr int kStage = 4;  // calls whose exchange may still be pending on the side stream
  Event ev_done[kStage], ev_posted;
  Stream side;                    // completion on a side stream (mlb_mixbus_set_async)
  int rank = 0, world = 1;
  size_t n_floats = 0;   // floats per slot
  DevBuf<char> base;     // one allocation: xchg [2][world][n_floats] f32, then flags [2][world][flag_planes()] u32
  void* peer_base[kMaxBusRanks] = {};
  bool connected = false;
  unsigned seq = 0;
  int async = 0;
  bool done_pending = false;
  int flag_planes() const { return (int)(n_floats / MLB_BLOCK); }  // flag words per (parity, rank)
  size_t xchg_bytes() const { return (size_t)2 * world * n_floats * 4; }
  size_t flag_bytes() const { return (size_t)2 * world * flag_planes() * 4; }
  size_t stage_bytes() const { return (size_t)kStage * n_floats * 4; }
  size_t total_bytes() const { return xchg_bytes() + 2 * flag_bytes() + stage_bytes(); }  // slots, flags, acks, staging
};

extern "C" int mlb_mixbus_create(int rank, int world, size_t max_floats, mlb_mixbus** out)
{
  if (!out) return fail(MLB_ERR_INVALID, "out is null");
  *out = nullptr;
  if (world < 1 || world > kMaxBusRanks || rank < 0 || rank >= world || max_floats == 0 || (max_floats % MLB_BLOCK))
    return fail(MLB_ERR_INVALID, "mlb_mixbus_create: need 0 <= rank < world <= %d and max_floats a multiple of 64", kMaxBusRanks);
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  std::unique_ptr<mlb_mixbus> b(new mlb_mixbus);
  b->live.arm();
  b->rank = rank, b->world = world, b->n_floats = max_floats;
  MLB_TRY(b->base.alloc(b->total_bytes(), "exchange buffer"));
  CU_CHECK(cudaMemset(b->base.get(), 0, b->total_bytes()));
  CU_CHECK(cudaDeviceSynchronize());
  b->peer_base[rank] = b->base.get();
  b->connected = (world == 1);
  MLB_TRY(b->side.create(cudaStreamNonBlocking));
  // The exchange kernel runs BESIDE the next call's chain kernel, whose CTAs need the SM configured for the
  // maximum shared-memory carve-out: a resident CTA that prefers another L1 / shared split keeps the chain CTA
  // off its SM until it has finished.  Ask for the same split.
  cudaFuncSetAttribute((const void*)mixbus_exchange_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                       (int)cudaSharedmemCarveoutMaxShared);
  MLB_TRY(b->ev_posted.create(cudaEventDisableTiming));
  for (Event& e : b->ev_done) MLB_TRY(e.create(cudaEventDisableTiming));
  *out = b.release();
  return MLB_OK;
}
extern "C" int mlb_mixbus_handle(mlb_mixbus* b, void* out64)
{
  if (!b || !out64) return fail(MLB_ERR_INVALID, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  cudaIpcMemHandle_t h;
  CU_CHECK(cudaIpcGetMemHandle(&h, b->base.get()));
  memcpy(out64, &h, 64);
  return MLB_OK;
}
extern "C" int mlb_mixbus_connect(mlb_mixbus* b, const void* handles)
{
  if (!b || !handles) return fail(MLB_ERR_INVALID, "null argument");
  for (int r = 0; r < b->world; ++r)
  {
    if (r == b->rank || b->peer_base[r]) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + (size_t)r * 64, 64);
    CU_CHECK(cudaIpcOpenMemHandle(&b->peer_base[r], h, cudaIpcMemLazyEnablePeerAccess));
  }
  b->connected = true;
  return MLB_OK;
}
extern "C" int mlb_mixbus_destroy(mlb_mixbus* b)
{
  if (!b) return MLB_OK;
  cudaDeviceSynchronize();
  for (int r = 0; r < b->world; ++r)
    if (r != b->rank && b->peer_base[r]) cudaIpcCloseMemHandle(b->peer_base[r]);
  delete b;
  return MLB_OK;
}
extern "C" int mlb_mixbus_set_async(mlb_mixbus* b, int on)
{
  if (!b) return fail(MLB_ERR_INVALID, "null bus");
  if (b->seq != 0 && (on != 0) != (b->async != 0))
    return fail(MLB_ERR_INVALID, "mlb_mixbus_set_async: choose the mode before the first process call");
  b->async = on ? 1 : 0;
  return MLB_OK;
}
extern "C" int mlb_graph_mix_wait(mlb_graph* g, void* stream)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  mlb_mixbus* b = g->bus;
  if (g->mix_async && g->mix_pending)
    CU_CHECK(cudaStreamWaitEvent((cudaStream_t)stream, g->ev_mixdone[g->mix_seq & 3u].get(), 0));
  if (b && b->async && b->done_pending)
    CU_CHECK(cudaStreamWaitEvent((cudaStream_t)stream, b->ev_done[b->seq % mlb_mixbus::kStage].get(), 0));
  return MLB_OK;
}
extern "C" int mlb_graph_attach_mixbus(mlb_graph* g, mlb_mixbus* b)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  if (b && !b->connected) return fail(MLB_ERR_INVALID, "mix bus is not connected to its peers yet");
  g->bus = b;
  return MLB_OK;
}
// kernel arguments of the next call's exchange (advances the call counter)
static int bus_args(mlb_graph* g, int n_planes, MixBusArgs* a, cudaStream_t stream)
{
  memset(a, 0, sizeof(*a));
  a->world = 1;
  mlb_mixbus* b = g->bus;
  if (!b || b->world <= 1) return MLB_OK;
  if ((size_t)n_planes * MLB_BLOCK > b->n_floats)
    return fail(MLB_ERR_INVALID, "mix bus holds %zu floats per rank, this call needs %zu", b->n_floats,
                (size_t)n_planes * MLB_BLOCK);
  a->rank = b->rank, a->world = b->world;
  a->seq = ++b->seq;
  a->n_floats = (int)b->n_floats, a->n_planes_cap = b->flag_planes();
  for (int r = 0; r < b->world; ++r)
  {
    a->xchg[r] = (float*)b->peer_base[r];
    a->flags[r] = (unsigned*)((char*)b->peer_base[r] + b->xchg_bytes());
    a->acks[r] = (unsigned*)((char*)b->peer_base[r] + b->xchg_bytes() + b->flag_bytes());
  }
  a->async = b->async;
  if (b->async)
  {
    // staging block of this call; its previous user (four calls ago) must have been exchanged
    a->stage = (float*)(b->base.get() + b->xchg_bytes() + 2 * b->flag_bytes()) + (size_t)(a->seq % mlb_mixbus::kStage) * b->n_floats;
    if (a->seq > (unsigned)mlb_mixbus::kStage)
      CU_CHECK(cudaStreamWaitEvent(stream, b->ev_done[a->seq % mlb_mixbus::kStage].get(), 0));
  }
  return MLB_OK;
}
// async mode: the exchange on the bus's side stream, ordered after the local sums on `stream`
static int bus_complete(mlb_graph* g, const MixBusArgs& ba, int n_planes, float* mix_dev, cudaStream_t stream)
{
  mlb_mixbus* b = g->bus;
  if (!b || b->world <= 1 || !b->async) return MLB_OK;
  CU_CHECK(cudaEventRecord(b->ev_posted.get(), stream));
  CU_CHECK(cudaStreamWaitEvent(b->side.get(), b->ev_posted.get(), 0));
  mixbus_exchange_kernel<<<(n_planes + kExchangePlanesPerCta - 1) / kExchangePlanesPerCta,
                           64 * kExchangePlanesPerCta, 0, b->side.get()>>>(mix_dev, ba, n_planes);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  CU_CHECK(cudaEventRecord(b->ev_done[ba.seq % mlb_mixbus::kStage].get(), b->side.get()));
  b->done_pending = true;
  return MLB_OK;
}

// The mix bus of a call of T blocks whose kernels left their per-group partials in g->partial_cur on `stream`: the
// reduction into mix_dev and the multi-GPU exchange; with `leave` they run on s_mix, beside the next call's kernel.
static int mix_tail(mlb_graph* g, float* mix_dev, int T, bool leave, cudaStream_t stream)
{
  const int n_groups = (g->V + 31) / 32, n_planes = T * std::max<int>(1, (int)g->outs.size());
  cudaStream_t ms = leave ? g->s_mix.get() : stream;
  if (leave)
  {
    CU_CHECK(cudaEventRecord(g->ev_main.get(), stream));
    CU_CHECK(cudaStreamWaitEvent(ms, g->ev_main.get(), 0));
  }
  float* scratch = g->partial_cur + (size_t)n_planes * n_groups * MLB_BLOCK;
  MixBusArgs ba;
  MLB_TRY(bus_args(g, n_planes, &ba, ms));
  // (asynchronous mode: 1024-thread CTAs do not fit beside a resident chain CTA and run in the gaps between chain
  // kernels; 256-thread CTAs that DO run beside it slow the HBM-bound chain kernel down by what they read.  The
  // reduction costs bandwidth, not latency.)
  mix_reduce_kernel<<<n_planes, dim3(MLB_BLOCK, 16), 0, ms>>>(g->partial_cur, scratch, mix_dev, n_groups, ba);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  if (leave)
  {
    CU_CHECK(cudaEventRecord(g->ev_mixdone[g->mix_seq & 3u].get(), ms));
    g->mix_pending = true;
  }
  return bus_complete(g, ba, n_planes, mix_dev, ms);
}

static int env_int(const char* name, int dflt)
{
  const char* s = getenv(name);
  return (s && *s) ? atoi(s) : dflt;
}

static int ensure_partial(mlb_graph* g, int T, int n_groups)
{
  // per-group partials followed by the per-chunk scratch of mix_reduce_kernel
  const size_t n_chunks = ((size_t)n_groups + kMixChunkGroups - 1) / kMixChunkGroups;
  const size_t one = (size_t)T * std::max<size_t>(1, g->outs.size()) * ((size_t)n_groups + n_chunks) * MLB_BLOCK * 4;
  const size_t need = one * (g->mix_async ? 2 : 1);  // async: two buffers, alternating by call parity
  if (need > g->d_partial.bytes() && g->mix_pending)
    cudaStreamSynchronize(g->s_mix.get());  // nothing may still read the old buffers
  MLB_TRY(g->d_partial.ensure(need, "mix partials"));
  g->partial_cur = g->d_partial.get();
  return MLB_OK;
}

// Launch the fused chain kernel for the voice slice [va, vb) (va a multiple of 32) of the bank.
// in_dev / out_dev are the FULL planes [T][in_planes][V][64] / [T][1][V][64]; the tensor maps, SoA
// pointers, mix partials and progress words are offset to the slice.
static int launch_chain_slice(mlb_graph* g, const float* in_dev, int in_planes, float* out_dev, bool want_mix, int T,
                              cudaStream_t stream, int va, int vb, int force_chunks = 0)
{
  const FusedEntry& e = *g->fused;
  const int V = g->V, Vs = vb - va;
  const int groups_total = (V + 31) / 32, n_groups = (Vs + 31) / 32;
  int rc;
  ChainArgs a = g->cargs;
  a.state = g->d_state.get() + va;
  a.coef = g->d_coef.get() + va;
  a.mix_partial = want_mix ? g->partial_cur + (size_t)(va / 32) * MLB_BLOCK : nullptr;
  a.V = Vs;
  a.T = T;
  a.v_stride = V;
  a.n_in_planes = std::max(1, in_planes);
  a.n_out_planes = 1;
  a.out_plane = 0;
  a.n_groups = n_groups;
  a.groups_stride = groups_total;
  a.write_out = out_dev ? 1 : 0;
  // Small banks: a TEAM of two warps per voice group (generator | filter pipeline, chain_team_kernel):
  // with fewer than ~4 groups per SM a lone warp per group is latency-bound, and the chain is the
  // only axis left to split.  One 64-thread CTA per group, static assignment, no scheduler words.
  // Up to 4 teams per SM (5-stage rings, 41 KB each); beyond that one warp per group.
  const int teams_per_sm = (n_groups + g_sm_count - 1) / g_sm_count;
  if (e.team_fn && teams_per_sm <= 4 && env_int("MLB_CHAIN_TEAM", 1) != 0)
  {
    // 3 S named barriers + barrier 0 <= 16  ->  S <= 5
    const int S = std::min(std::max(env_int("MLB_TEAM_STAGES", 5), 4), 5);
    a.stages = S;
    a.chunk_blocks = T, a.n_chunks = 1;
    a.sched = g->d_sched.get(), a.progress = g->d_sched.get() + 1 + va / 32;
    a.done = g->d_sched.get() + 1 + groups_total, a.base_word = g->d_sched.get() + 2 + groups_total;
    g->launch_chunks = 1;
    const size_t smem = (size_t)S * kBlockBytes + (size_t)S * 8;
    CUtensorMap in_map, out_map;
    memset(&in_map, 0, sizeof(in_map));
    memset(&out_map, 0, sizeof(out_map));
    if (e.has_in)
    {
      rc = cached_block_map(&g->maps, &in_map, in_dev + (size_t)va * MLB_BLOCK, Vs, (long long)T * a.n_in_planes,
                            (long long)V * MLB_BLOCK);
      if (rc != MLB_OK) return rc;
    }
    if (out_dev)
    {
      rc = cached_block_map(&g->maps, &out_map, out_dev + (size_t)va * MLB_BLOCK, Vs, (long long)T,
                            (long long)V * MLB_BLOCK);
      if (rc != MLB_OK) return rc;
    }
    rc = ensure_func_smem((const void*)e.team_fn, smem);
    if (rc != MLB_OK) return rc;
    static unsigned long long* d_prof = nullptr;
    const bool prof = env_int("MLB_TEAM_PROF", 0) != 0;
    if (prof && !d_prof) cudaMalloc(&d_prof, 64);
    a.prof = prof ? d_prof : nullptr;
    a.n_sms = g_sm_count;
    const int team_threads = teams_per_sm <= 2 ? 128 : 96;  // see chain_team_kernel: role rotation only pays up to 2 teams per SM
    e.team_fn<<<n_groups, team_threads, smem, stream>>>(in_map, out_map, a);
    ++g_launches;
    CU_CHECK(cudaGetLastError());
    if (prof)
    {
      unsigned long long h[5];
      cudaStreamSynchronize(stream);
      cudaMemcpy(h, d_prof, sizeof(h), cudaMemcpyDeviceToHost);
      const double n = (double)T * MLB_BLOCK;
      int occ = -1;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)e.team_fn, 96, smem);
      fprintf(stderr, "team launch: %d groups, S = %d, %zu B smem, occupancy %d CTAs/SM\n", n_groups, S, smem, occ);
      fprintf(stderr, "team prof (cycles per sample, CTA 0): G wait %.1f compute %.1f | F wait %.1f compute %.1f\n",
              h[0] / n, h[1] / n, h[2] / n, h[3] / n);
    }
    return MLB_OK;
  }
  // Launch shape (DESIGN.md "occupancy").  The grid is persistent: one CTA of W warps per SM,
  // each warp owns a ring of S 8-KB blocks and pulls (group, chunk) work units from an atomic
  // queue.  W is a multiple of 4 so the four SM sub-partitions carry equal warp counts; small
  // banks simply get one warp per group.
  const size_t budget = (size_t)g_smem_optin - 64;
  const size_t stage_bytes = (size_t)std::max(1, e.n_planes) * kBlockBytes;  // a ring stage holds n_planes blocks
  const int w_cap = std::min(kChainMaxWarps, (int)(budget / (2 * (stage_bytes + 8))));  // warps whose 2-stage rings fit
  // Three regimes (n_groups = 32-voice groups of this launch):
  //   * up to 8 warps per SM cover every group (n_groups <= 8 * SMs): W = ceil(n_groups / SMs) warps per
  //     CTA, every warp owns ONE group for the whole launch (n_chunks = 1): no state hopping, no progress waits,
  //     and the spare shared memory deepens each warp's ring.  (Cutting such a launch into time chunks adds no
  //     parallelism -- a group's chunks are serial anyway -- it only idles the warps beyond n_groups.)
  //   * more groups: W = 12 (3 per SM sub-partition, 2-stage rings, 197 KB), work units = (group, chunk of the
  //     launch's blocks) so that SM-to-SM speed differences and the tail stay balanced (a static one group per
  //     warp leaves the tail to the slowest SM).
  int W, S;
  const bool one_warp_per_group = n_groups <= g_sm_count * std::min(w_cap, 8);
  if (one_warp_per_group)
    W = std::max(1, (n_groups + g_sm_count - 1) / g_sm_count);
  else
    W = std::min(12, w_cap);
  W = env_int("MLB_CHAIN_WARPS", W);
  W = std::min(std::max(W, 1), kChainMaxWarps);
  S = 2;
  if (e.n_planes > 0)
  {
    S = (int)(budget / ((size_t)W * (stage_bytes + 8)));
    S = std::min(std::max(S, 2), 6);
    S = env_int("MLB_CHAIN_STAGES", S);
    S = std::min(std::max(S, 2), 12);
  }
  a.stages = S;
  // work units: (group, chunk of blocks).  Aim at >= 6 units per resident warp so the tail of
  // the dynamic schedule costs < 1/6 of a unit column; chunks never shorter than 8 blocks.
  {
    const int n_warps_resident = g_sm_count * W;
    int n_chunks = (int)((6LL * n_warps_resident + n_groups - 1) / n_groups);
    n_chunks = std::min(std::max(n_chunks, 1), std::max(1, T / 8));
    if (one_warp_per_group && n_groups <= n_warps_resident) n_chunks = 1;
    n_chunks = env_int("MLB_CHAIN_CHUNKS", n_chunks);
    if (force_chunks > 0) n_chunks = force_chunks;  // all slices of one call must agree
    n_chunks = std::min(std::max(n_chunks, 1), T);
    a.chunk_blocks = (T + n_chunks - 1) / n_chunks;
    a.n_chunks = (T + a.chunk_blocks - 1) / a.chunk_blocks;
    a.sched = g->d_sched.get();
    a.progress = g->d_sched.get() + 1 + va / 32;
    a.done = g->d_sched.get() + 1 + groups_total;
    a.base_word = g->d_sched.get() + 2 + groups_total;
    g->launch_chunks = a.n_chunks;
  }
  const size_t smem = (size_t)W * S * stage_bytes + (size_t)W * S * 8;
  if (smem > g_smem_optin) return fail(MLB_ERR_INVALID, "chain launch needs %zu B shared memory", smem);
  const int ctas_per_sm = std::max<size_t>(1, (size_t)(227 * 1024) / (smem + 1024));
  // the grid is persistent and fills every SM's shared memory; a caller that overlaps a collective
  // (the mix-bus all-reduce of a multi-GPU run) keeps a few SMs free for its kernels
  const int sms = std::max(1, g_sm_count - std::max(0, g->reserved_sms));
  int n_ctas = std::min((n_groups + W - 1) / W, sms * ctas_per_sm);
  n_ctas = std::min(std::max(env_int("MLB_CHAIN_CTAS", n_ctas), 1), (n_groups + W - 1) / W);
  CUtensorMap in_map, out_map;
  memset(&in_map, 0, sizeof(in_map));
  memset(&out_map, 0, sizeof(out_map));
  if (e.n_planes > 0)
  {
    rc = cached_block_map(&g->maps, &in_map, in_dev + (size_t)va * MLB_BLOCK, Vs, (long long)T * a.n_in_planes,
                          (long long)V * MLB_BLOCK);
    if (rc != MLB_OK) return rc;
  }
  if (out_dev)
  {
    rc = cached_block_map(&g->maps, &out_map, out_dev + (size_t)va * MLB_BLOCK, Vs, (long long)T,
                          (long long)V * MLB_BLOCK);
    if (rc != MLB_OK) return rc;
  }
  rc = ensure_func_smem((const void*)e.fn, smem);
  if (rc != MLB_OK) return rc;
  e.fn<<<n_ctas, W * 32, smem, stream>>>(in_map, out_map, a);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}

// The checks of a graph call that need no device; the host entry points run them before they enqueue anything.
static int graph_check(const mlb_graph* g, int n_blocks, int in_planes, const void* in, bool wants_output)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive");
  if (in_planes > 0 && !in) return fail(MLB_ERR_INVALID, "graph has INPUT nodes but in is null");
  if (g->outs.empty() && wants_output) return fail(MLB_ERR_INVALID, "graph has no outputs");
  if (g->fdn_node >= 0 && !g->d_ring.get())
    return fail(MLB_ERR_INVALID, "FDN8 graph: call mlb_graph_set_coefs before processing");
  return MLB_OK;
}

// The FM3 -> FDN8 kernel; with the mix bus, the per-group partials of its two output planes after it.
static int launch_fdn(mlb_graph* g, const float* in, int in_planes, float* out, bool want_mix, int T,
                      cudaStream_t stream)
{
  const int V = g->V, n_groups = (V + 31) / 32;
  // outputs are needed for the mix bus even when the caller does not want them
  float* planes = out;
  if (!planes)
  {
    MLB_TRY(g->d_out.ensure((size_t)T * 2 * V * MLB_BLOCK * 4, "staging"));
    planes = g->d_out.get();
  }
  const int rc = launch_fm3_fdn8(g->fargs, g->exact, g->d_state.get(), g->d_coef.get(), g->d_ring.get(), g->d_carry.get(),
                                 g->ring_len, g->blocks_done, in, planes, V, T, std::max(1, in_planes), stream);
  if (rc != MLB_OK) return fail(rc, "fdn8 launch failed: %s", cudaGetErrorString(cudaGetLastError()));
  ++g_launches;
  if (want_mix)
  {
    mix_partial_from_planes_kernel<<<dim3(n_groups, T * 2), MLB_BLOCK, 0, stream>>>(planes, g->partial_cur, V,
                                                                                    n_groups);
    ++g_launches;
  }
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}

// The graph interpreter kernel.
static int launch_generic(mlb_graph* g, const float* in, int in_planes, float* out, bool want_mix, int T,
                          cudaStream_t stream)
{
  const int V = g->V, n_groups = (V + 31) / 32;
  GenericArgs a;
  memset(&a, 0, sizeof(a));
  a.nodes = g->d_gnodes.get();
  a.n_nodes = (int)g->gnodes.size();
  a.state = g->d_state.get();
  a.coef = g->d_coef.get();
  a.in = in;
  a.out = out;
  a.mix_partial = want_mix ? g->partial_cur : nullptr;
  a.V = V, a.T = T, a.n_in = std::max(1, in_planes), a.n_out = std::max<int>(1, (int)g->outs.size());
  a.n_groups = n_groups, a.n_slots = g->n_slots;
  a.fdn_ring = g->d_ring.get(), a.fdn_carry = g->d_carry.get(), a.fdn_ring_len = g->ring_len;
  a.blocks_done = g->blocks_done;
  a.dmem = g->d_dmem.get();
  a.scratch_slot = g->scratch_slot;
  a.stages = g->d_gstages.get();
  a.n_stages = g->n_stages;
  a.n_chan = g->n_chan;
  a.sync = g->d_gsync.get();
  if (g->n_chan > 0) MLB_TRY(g->d_chan.ensure((size_t)T * g->n_chan * V * MLB_BLOCK * 4, "staging"));
  a.chan = g->d_chan.get();
  const int grid = n_groups * g->n_stages;
  CU_CHECK(cudaMemsetAsync(g->d_gsync.get(), 0, (1 + (size_t)grid) * 4, stream));
  const size_t smem = (size_t)g->n_slots * kSlotBytes;
  void (*const fn)(const GenericArgs) = g->exact ? generic_graph_kernel<true> : generic_graph_kernel<false>;
  CU_CHECK(cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  fn<<<grid, 32, smem, stream>>>(a);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}

// One call of the graph on device buffers; `in` is [T][in_planes][V][64]: the graph's own plane count from
// mlb_graph_process_device, the Voice rows (MLB_VOICE_ROWS) from contract E.
static int graph_process(mlb_graph* g, const float* in, int in_planes, float* out, float* mix, int T,
                         cudaStream_t stream)
{
  MLB_TRY(graph_check(g, T, in_planes, in, out || mix));
  MLB_TRY(ensure_init());
  if (mix)
  {
    MLB_TRY(ensure_partial(g, T, (g->V + 31) / 32));
    if (g->mix_async)
    {
      // this call's partial buffer; its previous user (two calls ago) must have been reduced
      ++g->mix_seq;
      g->partial_cur = g->d_partial.get() + (size_t)(g->mix_seq & 1u) * (g->d_partial.bytes() / 8);
      if (g->mix_seq > 2u) CU_CHECK(cudaStreamWaitEvent(stream, g->ev_mixdone[(g->mix_seq - 2u) & 3u].get(), 0));
    }
  }

  // the timing events are skipped while `stream` is being captured into a CUDA graph
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CU_CHECK(cudaStreamIsCapturing(stream, &cap));
  const bool capturing = (cap != cudaStreamCaptureStatusNone);
  if (capturing && (g->fdn_node >= 0 || g->has_dmem || (g->bus && g->bus->world > 1) || (g->mix_async && mix)))
    return fail(MLB_ERR_UNSUPPORTED, "CUDA-graph capture of a process call is supported for graphs without delay "
                                     "memory and without a mix bus (their call counters are kernel arguments)");
  if (!capturing) CU_CHECK(cudaEventRecord(g->ev0.get(), stream));
  if (g->kind == KIND_FUSED)
    MLB_TRY(launch_chain_slice(g, in, in_planes, out, mix != nullptr, T, stream, 0, g->V));
  else if (g->kind == KIND_FDN)
    MLB_TRY(launch_fdn(g, in, in_planes, out, mix != nullptr, T, stream));
  else
    MLB_TRY(launch_generic(g, in, in_planes, out, mix != nullptr, T, stream));
  if (!capturing)
  {
    CU_CHECK(cudaEventRecord(g->ev1.get(), stream));
    g->timed = true;
  }
  if (g->fdn_node >= 0 || g->has_dmem) g->blocks_done += T;
  // asynchronous mix bus (mlb_graph_set_mix_async): the reduction leaves the caller's stream
  return mix ? mix_tail(g, mix, T, g->mix_async != 0, stream) : MLB_OK;
}

extern "C" int mlb_graph_process_device(mlb_graph* g, const float* in_dev, float* out_dev,
                                        float* mix_dev, int n_blocks, void* stream)
{
  return graph_process(g, in_dev, g ? g->layout.n_inputs : 0, out_dev, mix_dev, n_blocks, (cudaStream_t)stream);
}

extern "C" int mlb_graph_set_mix_async(mlb_graph* g, int on)
{
  if (!g) return fail(MLB_ERR_INVALID, "null graph");
  if (g->mix_pending) CU_CHECK(cudaStreamSynchronize(g->s_mix.get()));
  g->mix_pending = false;
  if (on)
  {
    MLB_TRY(g->s_mix.create(cudaStreamNonBlocking));
    MLB_TRY(g->ev_main.create(cudaEventDisableTiming));
    for (Event& e : g->ev_mixdone) MLB_TRY(e.create(cudaEventDisableTiming));
  }
  g->mix_async = on ? 1 : 0;
  return MLB_OK;
}

// The three-stream pipeline of the host entry points over the pieces [a, b) = [p * per, min(total, (p + 1) * per)) of
// `total` voices or blocks: piece p goes up on s_h2d (if `up`), runs on the graph's stream once it is there (ev_up[p])
// and goes down on s_d2h (if `down`) once it has run (ev_k[p]), so that the upload of piece p + 1, the kernels of
// piece p and the download of piece p - 1 overlap (PCIe is full duplex).  Steps are called as step(a, b, stream).
// The caller drains the three streams whatever this returns.
template <class Up, class Run, class Down>
static int host_pipeline(mlb_graph* g, int total, int per, bool up, bool down, Up upload, Run run, Down download)
{
  const int n = (total + per - 1) / per;
  if (n > mlb_graph::kMaxHostSlices)
    return fail(MLB_ERR_INVALID, "%d pieces exceed the %d of one host call", n, mlb_graph::kMaxHostSlices);
  g->last_host_slices = 0;
  for (int p = 0; p < n; ++p)
  {
    const int a = p * per, b = std::min(total, a + per);
    if (up)
    {
      CU_CHECK(upload(a, b, g->s_h2d.get()));
      CU_CHECK(cudaEventRecord(g->ev_up[p].get(), g->s_h2d.get()));
      CU_CHECK(cudaStreamWaitEvent(g->stream.get(), g->ev_up[p].get(), 0));
    }
    MLB_TRY(run(a, b, g->stream.get()));
    if (down)
    {
      CU_CHECK(cudaEventRecord(g->ev_k[p].get(), g->stream.get()));
      CU_CHECK(cudaStreamWaitEvent(g->s_d2h.get(), g->ev_k[p].get(), 0));
      CU_CHECK(download(a, b, g->s_d2h.get()));
    }
    g->last_host_slices = p + 1;
  }
  return MLB_OK;
}

extern "C" int mlb_graph_process_host(mlb_graph* g, const float* in_host, float* out_host,
                                      float* mix_host, int n_blocks)
{
  const int n_in = g ? g->layout.n_inputs : 0;
  MLB_TRY(graph_check(g, n_blocks, n_in, in_host, out_host || mix_host));
  MLB_TRY(ensure_init());
  const size_t V = (size_t)g->V, T = (size_t)n_blocks, n_out = g->outs.size();
  const size_t in_bytes = T * n_in * V * MLB_BLOCK * 4, out_bytes = T * n_out * V * MLB_BLOCK * 4;
  const size_t mix_bytes = T * n_out * MLB_BLOCK * 4;
  if (n_in) MLB_TRY(g->d_in.ensure(in_bytes, "staging"));
  if (out_host) MLB_TRY(g->d_out.ensure(out_bytes, "staging"));
  if (mix_host) MLB_TRY(g->d_mix.ensure(mix_bytes, "staging"));
  float* d_in = n_in ? g->d_in.get() : nullptr;
  float* d_out = out_host ? g->d_out.get() : nullptr;
  float* d_mix = mix_host ? g->d_mix.get() : nullptr;
  cudaStream_t s = g->stream.get();
  // Large fused banks: pipelined over voice slices (host_pipeline).
  const int n_slices = std::min(env_int("MLB_HOST_SLICES", 16), (int)mlb_graph::kMaxHostSlices);
  // Only planes that really cross PCIe count: a mix-only call (out_host == NULL) moves 256 B per
  // block and must stay ONE launch -- 16 slice launches of a 4096-voice bank are latency-bound.
  const size_t pcie_bytes = in_bytes + (out_host ? out_bytes : 0);
  const size_t slice_min_bytes = (size_t)env_int("MLB_HOST_SLICE_MIN_MB", 32) << 20;
  const bool sliced = g->kind == KIND_FUSED && n_slices > 1 && g->V >= 4096 && pcie_bytes >= slice_min_bytes;
  // a slice [va, vb) of n planes is the strided window [T * n][va:vb][64] of the planes
  auto window = [&](float* dst, const float* src, size_t n, int va, int vb, cudaMemcpyKind kind, cudaStream_t st)
  {
    const size_t pitch = V * MLB_BLOCK * 4, at = (size_t)va * MLB_BLOCK;
    return cudaMemcpy2DAsync(dst + at, pitch, src + at, pitch, (size_t)(vb - va) * MLB_BLOCK * 4, T * n, kind, st);
  };
  const int rc = [&]() -> int
  {
    if (!sliced)
    {
      g->last_host_slices = 1;
      if (n_in) CU_CHECK(cudaMemcpyAsync(d_in, in_host, in_bytes, cudaMemcpyHostToDevice, s));
      MLB_TRY(graph_process(g, d_in, n_in, d_out, d_mix, n_blocks, s));
      if (out_host) CU_CHECK(cudaMemcpyAsync(out_host, d_out, out_bytes, cudaMemcpyDeviceToHost, s));
      if (mix_host) MLB_TRY(mlb_graph_mix_wait(g, s));  // async mix bus: the completion runs on a side stream
      if (mix_host) CU_CHECK(cudaMemcpyAsync(mix_host, d_mix, mix_bytes, cudaMemcpyDeviceToHost, s));
      return MLB_OK;
    }
    if (mix_host) MLB_TRY(ensure_partial(g, n_blocks, (g->V + 31) / 32));
    if (mix_host) MLB_TRY(mlb_graph_mix_wait(g, s));  // an asynchronous reduce may still read the partials
    CU_CHECK(cudaEventRecord(g->ev0.get(), s));
    const int per = ((g->V + n_slices - 1) / n_slices + 31) / 32 * 32;
    MLB_TRY(host_pipeline(
        g, g->V, per, n_in != 0, out_host != nullptr,
        [&](int va, int vb, cudaStream_t st) { return window(d_in, in_host, n_in, va, vb, cudaMemcpyHostToDevice, st); },
        [&](int va, int vb, cudaStream_t st)
        {
          // every slice takes the chunk count of the first slice's launch
          return launch_chain_slice(g, d_in, n_in, d_out, mix_host != nullptr, n_blocks, st, va, vb,
                                    va ? g->launch_chunks : 0);
        },
        [&](int va, int vb, cudaStream_t st) { return window(out_host, d_out, n_out, va, vb, cudaMemcpyDeviceToHost, st); }));
    CU_CHECK(cudaEventRecord(g->ev1.get(), s));
    g->timed = true;
    if (mix_host)
    {
      // the reduction stays on `s`: this call waits for it anyway, and the slices wrote their partials to the first
      // buffer, whatever the call parity of the asynchronous mix bus
      MLB_TRY(mix_tail(g, d_mix, n_blocks, false, s));
      MLB_TRY(mlb_graph_mix_wait(g, s));
      CU_CHECK(cudaMemcpyAsync(mix_host, d_mix, mix_bytes, cudaMemcpyDeviceToHost, s));
    }
    return MLB_OK;
  }();
  return sliced ? drain(rc, {g->s_h2d.get(), s, g->s_d2h.get()}) : drain(rc, {s});
}

extern "C" int mlb_graph_last_host_slices(const mlb_graph* g) { return g ? g->last_host_slices : -1; }

extern "C" int mlb_graph_last_kernel_ms(mlb_graph* g, float* ms)
{
  if (!g || !ms) return fail(MLB_ERR_INVALID, "null");
  if (!g->timed) return fail(MLB_ERR_INVALID, "no launch recorded yet");
  CU_CHECK(cudaEventSynchronize(g->ev1.get()));
  CU_CHECK(cudaEventElapsedTime(ms, g->ev0.get(), g->ev1.get()));
  return MLB_OK;
}

// ------------------------------------------------------------------------------------------
// stateless elementwise ops

extern "C" int mlb_map_device(int op, const float* x1, const float* x2, const float* x3, float* y,
                              size_t n_rows, void* stream)
{
  int nin, nst, nco;
  if (mlb_op_info(op, &nin, &nst, &nco) != MLB_OK || nst != 0 || nco != 0 || nin < 1 ||
      op == MLB_OP_FDN8_R)
    return fail(MLB_ERR_INVALID, "op %d is not a stateless elementwise op", op);
  if (!x1 || !y || (nin >= 2 && !x2) || (nin >= 3 && !x3)) return fail(MLB_ERR_INVALID, "null operand");
  if (n_rows == 0) return MLB_OK;
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  const size_t n4 = n_rows * (MLB_BLOCK / 4);
  const int threads = 256;
  const size_t want = (n4 + threads - 1) / threads;
  const int blocks = (int)std::min<size_t>(want, (size_t)g_sm_count * 16);
  MapKernelFn fn = map_kernel_for(op);
  if (!fn) return fail(MLB_ERR_INVALID, "op %d has no map kernel", op);
  fn<<<blocks, threads, 0, (cudaStream_t)stream>>>((const float4*)x1, nin >= 2 ? (const float4*)x2 : nullptr,
                                                   nin >= 3 ? (const float4*)x3 : nullptr, (float4*)y, n4);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}

// Device staging of mlb_map_host: four buffers (three operands + result) that only ever grow, so that the
// host value-type operators (`a + b` on two mlb::DSPVectors) do not allocate after their first use.
#include <mutex>
namespace
{
struct MapPool
{
  std::mutex mu;
  float* d[4] = {nullptr, nullptr, nullptr, nullptr};
  size_t cap = 0;
  cudaStream_t stream = nullptr;
  long long allocations = 0;
};
MapPool g_map_pool;
}  // namespace
extern "C" long long mlb_map_host_allocations(void) { return g_map_pool.allocations; }

extern "C" int mlb_map_host(int op, const float* x1, const float* x2, const float* x3, float* y,
                            size_t n_rows)
{
  int nin, nst, nco;
  if (mlb_op_info(op, &nin, &nst, &nco) != MLB_OK || !map_kernel_for(op))
    return fail(MLB_ERR_INVALID, "op %d is not a stateless elementwise op", op);
  if (n_rows == 0) return MLB_OK;
  if (!x1 || !y || (nin >= 2 && !x2) || (nin >= 3 && !x3)) return fail(MLB_ERR_INVALID, "null operand");
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  const size_t bytes = n_rows * MLB_BLOCK * 4;
  MapPool& P = g_map_pool;
  std::lock_guard<std::mutex> lock(P.mu);
  if (!P.stream) CU_CHECK(cudaStreamCreateWithFlags(&P.stream, cudaStreamNonBlocking));
  if (bytes > P.cap)
  {
    const size_t want = std::max(bytes, std::max<size_t>(P.cap * 2, (size_t)64 << 10));
    for (float*& p : P.d)
    {
      cudaFree(p);
      p = nullptr;
    }
    P.cap = 0;
    for (float*& p : P.d)
      if (cudaMalloc(&p, want) != cudaSuccess) return fail(MLB_ERR_ALLOC, "cudaMalloc of %zu B failed", want);
    P.cap = want;
    ++P.allocations;
  }
  const float* h[3] = {x1, x2, x3};
  rc = [&]() -> int
  {
    for (int k = 0; k < nin && k < 3; ++k)
      CU_CHECK(cudaMemcpyAsync(P.d[k], h[k], bytes, cudaMemcpyHostToDevice, P.stream));
    MLB_TRY(mlb_map_device(op, P.d[0], nin >= 2 ? P.d[1] : nullptr, nin >= 3 ? P.d[2] : nullptr, P.d[3], n_rows,
                           P.stream));
    CU_CHECK(cudaMemcpyAsync(y, P.d[3], bytes, cudaMemcpyDeviceToHost, P.stream));
    return MLB_OK;
  }();
  return drain(rc, {P.stream});
}


// ------------------------------------------------------------------------------------------
// EventsToSignals::Voice bank (K7, voice_kernel.cuh)

struct mlb_voices
{
  // declared first, so released last: the buffers below are freed first, and cudaFree waits for the device
  LiveCount live;
  Stream stream;
  int V = 0;
  float sr = 0.f;
  float gl_per = 0.f, gl_dy = 0.f, dr_per = 0.f, dr_dy = 0.f, pc_per = 0.f, pc_dy = 0.f;
  unsigned flags = 0;
  DevBuf<uint32_t> d_state;
  DevBuf<float> d_coef, d_grows;
  DevBuf<int32_t> d_main;  // MPE: index of each voice's main voice, or -1
  DevBuf<mlb_voice_events> d_ev;
  DevBuf<float> d_out;
};

extern "C" int mlb_voices_destroy(mlb_voices* vb)
{
  delete vb;
  return MLB_OK;
}

extern "C" int mlb_voices_create(int n_voices, float sample_rate, const int32_t* voice_index,
                                 const float* pitch_glide_seconds, const float* drift_amount,
                                 const float* pitch_bend, unsigned flags, mlb_voices** out)
{
  if (!out) return fail(MLB_ERR_INVALID, "out is null");
  *out = nullptr;
  if (n_voices <= 0 || !(sample_rate > 0.f) || !voice_index || !pitch_glide_seconds || !drift_amount || !pitch_bend)
    return fail(MLB_ERR_INVALID, "bad argument");
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  const size_t V = (size_t)n_voices;
  std::unique_ptr<mlb_voices> vb(new mlb_voices);
  vb->live.arm();
  vb->V = n_voices;
  vb->sr = sample_rate;
  // the recalc block of the first beginProcess (MLEventsToSignals.cpp:92-113), done once here
  const double sr = (double)sample_rate;
  float c[2];
  mlb_coeffs_glide((float)(sr * 0.02f), c);  // kGlideTimeSeconds
  vb->gl_per = c[0], vb->gl_dy = c[1];
  mlb_coeffs_glide((float)(sr * 8.0f), c);   // kDriftTimeSeconds
  vb->dr_per = c[0], vb->dr_dy = c[1];
  mlb_coeffs_glide((float)(int)(sr * 0.02f), c);  // SmoothedController::process, .cpp:278-280
  vb->pc_per = c[0], vb->pc_dy = c[1];
  vb->flags = flags;
  std::vector<uint32_t> st((size_t)VS_COUNT * V, 0u);
  std::vector<float> co((size_t)VC_COUNT * V, 0.f);
  auto fbits = [](float f)
  {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
  };
  for (size_t v = 0; v < V; ++v)
  {
    const int glide_samples = (int)(sr * pitch_glide_seconds[v]);  // pitchGlideTimeInSamples, :97
    float sg[2];
    mlb_coeffs_sample_glide((float)glide_samples, sg);             // pitchGlide.setGlideTimeInSamples, :101
    st[(size_t)VS_PG_REM * V + v] = 0xFFFFFFFFu;                    // mSamplesRemaining{-1}
    st[(size_t)VS_PG_PER * V + v] = fbits(sg[0]);
    st[(size_t)VS_PG_DY * V + v] = fbits(sg[1]);
    for (int g = 0; g < VG_COUNT; ++g)                              // reset(): setValue(0) on all but the drift glide, :80-84
      st[(size_t)(VS_GL + 4 * g + 2) * V + v] = (g == VG_DRIFT || g == VG_PRESSURE) ? 0xFFFFFFFFu : 0u;
    st[(size_t)VS_SEED * V + v] = (uint32_t)(voice_index[v] * 232);  // :62
    co[(size_t)VC_GLIDE_SAMPLES * V + v] = (float)glide_samples;
    co[(size_t)VC_DRIFT_AMOUNT * V + v] = drift_amount[v];
    co[(size_t)VC_BEND_RANGE * V + v] = pitch_bend[v];
    co[(size_t)VC_VOICE_ROW * V + v] = (float)voice_index[v] - 1;   // :292
  }
  MLB_TRY(vb->d_state.alloc(st.size() * 4, "voice bank"));
  MLB_TRY(vb->d_coef.alloc(co.size() * 4, "voice bank"));
  MLB_TRY(vb->d_grows.alloc((size_t)VG_COUNT * V * MLB_BLOCK * 4, "voice bank"));
  CU_CHECK(cudaMemcpy(vb->d_state.get(), st.data(), st.size() * 4, cudaMemcpyHostToDevice));
  CU_CHECK(cudaMemcpy(vb->d_coef.get(), co.data(), co.size() * 4, cudaMemcpyHostToDevice));
  CU_CHECK(cudaMemset(vb->d_grows.get(), 0, vb->d_grows.bytes()));
  MLB_TRY(vb->stream.create(cudaStreamNonBlocking));
  *out = vb.release();
  return MLB_OK;
}

extern "C" int mlb_voices_set_main_voices(mlb_voices* vb, const int32_t* main_voice)
{
  if (!vb) return fail(MLB_ERR_INVALID, "null voice bank");
  if (!main_voice)
  {
    vb->d_main.reset();
    return MLB_OK;
  }
  for (int v = 0; v < vb->V; ++v)
    if (main_voice[v] >= vb->V || (main_voice[v] >= 0 && main_voice[main_voice[v]] >= 0))
      return fail(MLB_ERR_INVALID, "main_voice[%d] = %d is not a main voice of this bank", v, main_voice[v]);
  MLB_TRY(vb->d_main.ensure((size_t)vb->V * 4, "main-voice table"));
  CU_CHECK(cudaMemcpy(vb->d_main.get(), main_voice, (size_t)vb->V * 4, cudaMemcpyHostToDevice));
  return MLB_OK;
}

// out_dev [T][out_planes][V][64]: the Voice rows in planes 0..7 of each block (contract E with controller planes
// leaves room for the controller rows after them)
static int voices_launch(mlb_voices* vb, const mlb_voice_events* events_dev, float* out_dev, int n_blocks,
                         unsigned row_mask, int out_planes, void* stream)
{
  if (!vb || !events_dev || (!out_dev && (row_mask & 0xFFu))) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive");
  VoiceArgs a;
  a.ev = events_dev;
  a.out = out_dev;
  a.out_block = (size_t)out_planes * vb->V * MLB_BLOCK;
  a.state = vb->d_state.get();
  a.coef = vb->d_coef.get();
  a.grows = vb->d_grows.get();
  a.V = vb->V, a.T = n_blocks;
  a.row_mask = row_mask & 0xFFu;
  a.sr = vb->sr;
  a.gl_per = vb->gl_per, a.gl_dy = vb->gl_dy, a.dr_per = vb->dr_per, a.dr_dy = vb->dr_dy;
  a.pc_per = vb->pc_per, a.pc_dy = vb->pc_dy;
  a.midi = (vb->flags & MLB_VOICES_MIDI) ? 1 : 0;
  // warps x {gate, pitch (, elapsed time)} 8 KB row tiles; up to 7 warps per CTA and two CTAs per SM (14 warps, the
  // most whose tiles fit in an SM's shared memory); 6 by default, measured faster on an H100 (voice_kernel.cuh)
  const bool want_time = (row_mask & 128u) != 0;
  const int wpc_max = want_time ? kVoiceWarpsPerCtaTime : kVoiceWarpsPerCta;
  const int wpc = env_int("MLB_VOICE_WARPS", want_time ? kVoiceWarpsPerCtaTime : kVoiceWarpsPerCtaDefault);
  if (wpc < 1 || wpc > wpc_max) return fail(MLB_ERR_INVALID, "MLB_VOICE_WARPS must be in [1, %d]", wpc_max);
  const size_t smem = (size_t)wpc * (want_time ? 3 : 2) * kVoiceTileFloats * sizeof(float);
  const void* fn = want_time ? (const void*)voice_bank_kernel<true> : (const void*)voice_bank_kernel<false>;
  {
    int rc = ensure_func_smem(fn, smem);
    if (rc != MLB_OK) return rc;
  }
  const int n_warps = (vb->V + 31) / 32;
  if (want_time)
    voice_bank_kernel<true><<<(n_warps + wpc - 1) / wpc, 32 * wpc, smem, (cudaStream_t)stream>>>(a);
  else
    voice_bank_kernel<false><<<(n_warps + wpc - 1) / wpc, 32 * wpc, smem, (cudaStream_t)stream>>>(a);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  if (vb->d_main.get() && (a.row_mask & 0x79u))  // MPE: add the main voices' pitch / z / x / y / mod rows
  {
    const size_t n4 = (size_t)n_blocks * vb->V * 16;
    const int grid = (int)std::min<size_t>((n4 + 255) / 256, (size_t)g_sm_count * 16);
    voice_mpe_add_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(out_dev, vb->d_main.get(), vb->V, n_blocks, a.row_mask,
                                                                  out_planes);
    ++g_launches;
    CU_CHECK(cudaGetLastError());
  }
  return MLB_OK;
}

extern "C" int mlb_voices_process_device(mlb_voices* vb, const mlb_voice_events* events_dev, float* out_dev,
                                         int n_blocks, unsigned row_mask, void* stream)
{
  return voices_launch(vb, events_dev, out_dev, n_blocks, row_mask, MLB_VOICE_ROWS, stream);
}

extern "C" int mlb_voices_process_host(mlb_voices* vb, const mlb_voice_events* events_host, float* out_host,
                                       int n_blocks, unsigned row_mask)
{
  if (!vb || !events_host) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive");
  row_mask &= 0xFFu;
  if (row_mask && !out_host) return fail(MLB_ERR_INVALID, "out is null");
  const size_t V = (size_t)vb->V, T = (size_t)n_blocks;
  const size_t ev_bytes = T * V * sizeof(mlb_voice_events), out_bytes = T * MLB_VOICE_ROWS * V * MLB_BLOCK * 4;
  MLB_TRY(vb->d_ev.ensure(ev_bytes, "staging"));
  MLB_TRY(vb->d_out.ensure(out_bytes, "staging"));
  cudaStream_t s = vb->stream.get();
  const int rc = [&]() -> int
  {
    CU_CHECK(cudaMemcpyAsync(vb->d_ev.get(), events_host, ev_bytes, cudaMemcpyHostToDevice, s));
    MLB_TRY(mlb_voices_process_device(vb, vb->d_ev.get(), vb->d_out.get(), n_blocks, row_mask, s));
    const size_t plane = V * MLB_BLOCK * 4;
    if (row_mask == 0xFFu)
      CU_CHECK(cudaMemcpyAsync(out_host, vb->d_out.get(), out_bytes, cudaMemcpyDeviceToHost, s));
    else
      for (size_t t = 0; t < T; ++t)
        for (int r = 0; r < MLB_VOICE_ROWS; ++r)
          if (row_mask & (1u << r))
            CU_CHECK(cudaMemcpyAsync(reinterpret_cast<char*>(out_host) + (t * MLB_VOICE_ROWS + r) * plane,
                                     reinterpret_cast<char*>(vb->d_out.get()) + (t * MLB_VOICE_ROWS + r) * plane,
                                     plane, cudaMemcpyDeviceToHost, s));
    return MLB_OK;
  }();
  return drain(rc, {s});
}


// Events -> signals -> chain with nothing but the event records crossing PCIe ("contract E"):
// the Voice bank writes the rows the graph reads (EventsToSignals::processVector,
// MLEventsToSignals.cpp:383-470) into a device buffer that IS the graph's input (the bank's out planes
// have the layout of graph inputs, plane r = row r), and the graph runs on it in the same stream.
// Pipelined over TIME chunks by host_pipeline -- blocks are contiguous in every buffer involved, and both
// the bank and the graph carry their state from launch to launch -- so that the H2D copy of chunk c+1's
// records, the kernels of chunk c and the D2H copy of chunk c-1's output rows overlap.
// mlb_synth_process_buses_host runs the same pipeline with the bus kernel (K10) after the graph.

// The checks both contract-E entry points share; *row_mask = the Voice rows the graph reads.
// n_planes: the input planes per block, the 8 Voice rows and any controller planes after them.
static int synth_check(const mlb_voices* vb, const mlb_graph* g, const mlb_voice_events* events_host, int n_blocks,
                       bool wants_output, unsigned* row_mask, int n_planes = MLB_VOICE_ROWS)
{
  if (!vb || !g || !events_host) return fail(MLB_ERR_INVALID, "null argument");
  MLB_TRY(graph_check(g, n_blocks, n_planes, events_host, wants_output));
  if (vb->V != g->V) return fail(MLB_ERR_INVALID, "voice bank has %d voices, graph has %d", vb->V, g->V);
  *row_mask = 0;
  bool reads = false;
  for (const mlb_node& n : g->nodes)
    if (n.op == MLB_OP_INPUT)
    {
      if (n.iarg < 0 || n.iarg >= n_planes)
        return n_planes == MLB_VOICE_ROWS
                   ? fail(MLB_ERR_INVALID, "graph INPUT plane %d is not a Voice row (0..%d)", n.iarg, MLB_VOICE_ROWS - 1)
                   : fail(MLB_ERR_INVALID, "graph INPUT plane %d is not a Voice row or controller plane (0..%d)", n.iarg,
                          n_planes - 1);
      if (n.iarg < MLB_VOICE_ROWS) *row_mask |= 1u << n.iarg;
      reads = true;
    }
  if (!reads) return fail(MLB_ERR_INVALID, "graph reads no Voice row (no INPUT node)");
  return MLB_OK;
}

// Blocks per time chunk: rows of one chunk stay under ~1 GB (8 planes per block are addressed, only the masked
// ones are touched), and a call has at most kMaxHostSlices chunks.
static int synth_chunk_blocks(const mlb_graph* g, int n_blocks, int n_planes = MLB_VOICE_ROWS)
{
  int Tc = env_int("MLB_SYNTH_CHUNK_BLOCKS", 0);
  if (Tc <= 0) Tc = (int)std::max<size_t>(1, ((size_t)1 << 30) / (n_planes * (size_t)g->V * MLB_BLOCK * 4));
  Tc = std::min<int>(Tc, n_blocks);
  return std::max<int>(Tc, (n_blocks + mlb_graph::kMaxHostSlices - 1) / mlb_graph::kMaxHostSlices);
}

extern "C" int mlb_synth_process_host(mlb_voices* vb, mlb_graph* g, const mlb_voice_events* events_host,
                                      float* out_host, float* mix_host, int n_blocks)
{
  unsigned row_mask;
  MLB_TRY(synth_check(vb, g, events_host, n_blocks, out_host || mix_host, &row_mask));
  MLB_TRY(ensure_init());
  const size_t V = (size_t)g->V, T = (size_t)n_blocks, n_out = g->outs.size();
  const int Tc = synth_chunk_blocks(g, n_blocks);
  if (out_host) MLB_TRY(g->d_out.ensure(T * n_out * V * MLB_BLOCK * 4, "staging"));
  if (mix_host) MLB_TRY(g->d_mix.ensure(T * n_out * MLB_BLOCK * 4, "staging"));
  MLB_TRY(vb->d_ev.ensure(T * V * sizeof(mlb_voice_events), "staging"));
  MLB_TRY(vb->d_out.ensure((size_t)Tc * MLB_VOICE_ROWS * V * MLB_BLOCK * 4, "staging"));
  const size_t row_floats = n_out * V * MLB_BLOCK;  // output rows per block
  const int rc = [&]() -> int
  {
    MLB_TRY(host_pipeline(
        g, n_blocks, Tc, true, out_host != nullptr,
        [&](int t0, int t1, cudaStream_t s)
        {
          return cudaMemcpyAsync(vb->d_ev.get() + t0 * V, events_host + t0 * V, (t1 - t0) * V * sizeof(mlb_voice_events),
                                 cudaMemcpyHostToDevice, s);
        },
        [&](int t0, int t1, cudaStream_t s) -> int
        {
          MLB_TRY(mlb_voices_process_device(vb, vb->d_ev.get() + t0 * V, vb->d_out.get(), t1 - t0, row_mask, s));
          return graph_process(g, vb->d_out.get(), MLB_VOICE_ROWS, out_host ? g->d_out.get() + t0 * row_floats : nullptr,
                               mix_host ? g->d_mix.get() + t0 * n_out * MLB_BLOCK : nullptr, t1 - t0, s);
        },
        [&](int t0, int t1, cudaStream_t s)
        {
          return cudaMemcpyAsync(out_host + t0 * row_floats, g->d_out.get() + t0 * row_floats,
                                 (t1 - t0) * row_floats * 4, cudaMemcpyDeviceToHost, s);
        }));
    if (mix_host) MLB_TRY(mlb_graph_mix_wait(g, g->stream.get()));
    if (mix_host)
      CU_CHECK(cudaMemcpyAsync(mix_host, g->d_mix.get(), T * n_out * MLB_BLOCK * 4, cudaMemcpyDeviceToHost, g->stream.get()));
    return MLB_OK;
  }();
  return drain(rc, {g->s_h2d.get(), g->stream.get(), g->s_d2h.get()});
}

// ------------------------------------------------------------------------------------------
// Per-instrument output buses (K10, bus_kernel.cuh)

struct mlb_buses
{
  LiveCount live;
  int V = 0, G = 0;
  DevBuf<int32_t> d_table;  // [2][G]: first voice, voice count
  DevBuf<float> d_out;      // bus rows of mlb_synth_process_buses_host, [T][n_out][G][64]
};

extern "C" int mlb_buses_destroy(mlb_buses* b)
{
  delete b;
  return MLB_OK;
}

extern "C" int mlb_buses_create(int n_voices, int n_buses, const int32_t* first_voice, const int32_t* voice_count,
                                mlb_buses** out)
{
  if (!out) return fail(MLB_ERR_INVALID, "out is null");
  *out = nullptr;
  if (n_voices <= 0) return fail(MLB_ERR_INVALID, "n_voices must be positive (got %d)", n_voices);
  if (n_buses < 1) return fail(MLB_ERR_INVALID, "n_buses must be positive (got %d)", n_buses);
  if (!first_voice || !voice_count) return fail(MLB_ERR_INVALID, "null layout table");
  for (int g = 0; g < n_buses; ++g)
    if (first_voice[g] < 0 || voice_count[g] < 0 || (int64_t)first_voice[g] + voice_count[g] > n_voices)
      return fail(MLB_ERR_INVALID, "bus %d: first voice %d, count %d is not a range of the %d voices", g,
                  first_voice[g], voice_count[g], n_voices);
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  std::unique_ptr<mlb_buses> b(new mlb_buses);
  b->live.arm();
  b->V = n_voices, b->G = n_buses;
  const size_t bytes = (size_t)n_buses * sizeof(int32_t);
  MLB_TRY(b->d_table.alloc(2 * bytes, "bus layout"));
  if (cudaMemcpy(b->d_table.get(), first_voice, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(b->d_table.get() + n_buses, voice_count, bytes, cudaMemcpyHostToDevice) != cudaSuccess)
    return fail(MLB_ERR_CUDA, "upload of bus layout failed");
  *out = b.release();
  return MLB_OK;
}

extern "C" int mlb_buses_sum_device(mlb_buses* b, const float* rows_dev, float* bus_dev, int n_planes, int n_blocks,
                                    void* stream)
{
  if (!b || !rows_dev || !bus_dev) return fail(MLB_ERR_INVALID, "null argument");
  if (n_planes <= 0) return fail(MLB_ERR_INVALID, "n_planes must be positive (got %d)", n_planes);
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive (got %d)", n_blocks);
  BusArgs a;
  a.rows = rows_dev, a.bus = bus_dev, a.first = b->d_table.get(), a.count = b->d_table.get() + b->G;
  a.V = b->V, a.G = b->G;
  a.n_items = (long long)n_blocks * n_planes * b->G;
  const long long grid = (a.n_items + kBusWarps - 1) / kBusWarps;
  if (grid > 0x7FFFFFFFLL) return fail(MLB_ERR_INVALID, "%lld bus rows exceed one launch", a.n_items);
  bus_sum_kernel<<<(unsigned)grid, 32 * kBusWarps, 0, (cudaStream_t)stream>>>(a);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}

// Contract E with per-instrument output: the graph's rows of a chunk go to a device scratch of one chunk (g->d_out),
// the bus kernel sums them on the same stream right after the graph, and only the bus rows come back.
extern "C" int mlb_synth_process_buses_host(mlb_voices* vb, mlb_graph* g, mlb_buses* b,
                                            const mlb_voice_events* events_host, float* bus_host, int n_blocks)
{
  unsigned row_mask;
  MLB_TRY(synth_check(vb, g, events_host, n_blocks, true, &row_mask));
  if (!b || !bus_host) return fail(MLB_ERR_INVALID, "null argument");
  if (b->V != g->V) return fail(MLB_ERR_INVALID, "buses are laid over %d voices, graph has %d", b->V, g->V);
  MLB_TRY(ensure_init());
  const size_t V = (size_t)g->V, T = (size_t)n_blocks, n_out = g->outs.size(), G = (size_t)b->G;
  const int Tc = synth_chunk_blocks(g, n_blocks);
  MLB_TRY(g->d_out.ensure((size_t)Tc * n_out * V * MLB_BLOCK * 4, "staging"));
  MLB_TRY(b->d_out.ensure(T * n_out * G * MLB_BLOCK * 4, "staging"));
  MLB_TRY(vb->d_ev.ensure(T * V * sizeof(mlb_voice_events), "staging"));
  MLB_TRY(vb->d_out.ensure((size_t)Tc * MLB_VOICE_ROWS * V * MLB_BLOCK * 4, "staging"));
  const size_t bus_floats = n_out * G * MLB_BLOCK;  // bus rows per block
  const int rc = host_pipeline(
      g, n_blocks, Tc, true, true,
      [&](int t0, int t1, cudaStream_t s)
      {
        return cudaMemcpyAsync(vb->d_ev.get() + t0 * V, events_host + t0 * V, (t1 - t0) * V * sizeof(mlb_voice_events),
                               cudaMemcpyHostToDevice, s);
      },
      [&](int t0, int t1, cudaStream_t s) -> int
      {
        MLB_TRY(mlb_voices_process_device(vb, vb->d_ev.get() + t0 * V, vb->d_out.get(), t1 - t0, row_mask, s));
        MLB_TRY(graph_process(g, vb->d_out.get(), MLB_VOICE_ROWS, g->d_out.get(), nullptr, t1 - t0, s));
        return mlb_buses_sum_device(b, g->d_out.get(), b->d_out.get() + t0 * bus_floats, (int)n_out, t1 - t0, s);
      },
      [&](int t0, int t1, cudaStream_t s)
      {
        return cudaMemcpyAsync(bus_host + t0 * bus_floats, b->d_out.get() + t0 * bus_floats, (t1 - t0) * bus_floats * 4,
                               cudaMemcpyDeviceToHost, s);
      });
  return drain(rc, {g->s_h2d.get(), g->stream.get(), g->s_d2h.get()});
}

// ------------------------------------------------------------------------------------------
// Smoothed MIDI controllers (K11, controller_kernel.cuh)

struct mlb_controllers
{
  // declared first, so released last: the buffers below are freed first, and cudaFree waits for the device
  LiveCount live;
  Stream stream;
  int G = 0, C = 0, protocol = 0;
  int V = 0;  // voices of the voice map; 0: instrument rows
  float per_f = 0.f, dy = 0.f;
  DevBuf<int32_t> d_ctrl;   // [C] controller numbers
  DevBuf<uint32_t> d_state; // [CS_COUNT][C][G]
  DevBuf<float> d_rows;     // [C][G][64]
  DevBuf<int32_t> d_vmap;   // [G + 2] offsets, then [V] voices grouped by instrument, the unmapped ones last
  DevBuf<int32_t> d_off;    // staging of the host entry points
  DevBuf<mlb_controller_change> d_ch;
  DevBuf<float> d_out;
};

extern "C" int mlb_controllers_destroy(mlb_controllers* cb)
{
  delete cb;
  return MLB_OK;
}

extern "C" int mlb_controllers_clear(mlb_controllers* cb)
{
  if (!cb) return fail(MLB_ERR_INVALID, "null controller bank");
  const size_t CG = (size_t)cb->C * cb->G;
  std::vector<uint32_t> st((size_t)CS_COUNT * CG, 0u);
  std::fill_n(st.begin() + CS_REM * CG, CG, 0xFFFFFFFFu);  // LinearGlide::mVectorsRemaining{-1}
  CU_CHECK(cudaMemcpy(cb->d_state.get(), st.data(), st.size() * 4, cudaMemcpyHostToDevice));
  CU_CHECK(cudaMemset(cb->d_rows.get(), 0, cb->d_rows.bytes()));
  return MLB_OK;
}

extern "C" int mlb_controllers_create(int n_instruments, float sample_rate, int protocol, const int32_t* controllers,
                                      int n_controllers, mlb_controllers** out)
{
  if (!out) return fail(MLB_ERR_INVALID, "out is null");
  *out = nullptr;
  if (n_instruments <= 0) return fail(MLB_ERR_INVALID, "n_instruments must be positive (got %d)", n_instruments);
  if (!(sample_rate > 0.f)) return fail(MLB_ERR_INVALID, "sample_rate must be positive (got %g)", sample_rate);
  if (protocol != 0 && protocol != 1) return fail(MLB_ERR_INVALID, "protocol must be 0 (MIDI) or 1 (MPE), got %d", protocol);
  if (!controllers) return fail(MLB_ERR_INVALID, "null controller list");
  if (n_controllers < 1 || n_controllers > 129)
    return fail(MLB_ERR_INVALID, "n_controllers must be in 1..129 (got %d)", n_controllers);
  int seen[129];
  std::fill_n(seen, 129, -1);
  for (int k = 0; k < n_controllers; ++k)
  {
    const int n = controllers[k];
    if (n < 0 || n > 128) return fail(MLB_ERR_INVALID, "controller %d (list index %d) is not in 0..128", n, k);
    if (seen[n] >= 0)
      return fail(MLB_ERR_INVALID, "controller %d is requested twice (list indexes %d and %d)", n, seen[n], k);
    seen[n] = k;
  }
  MLB_TRY(ensure_init());
  std::unique_ptr<mlb_controllers> cb(new mlb_controllers);
  cb->live.arm();
  cb->G = n_instruments, cb->C = n_controllers, cb->protocol = protocol;
  // SmoothedController::process (.cpp:274-285): int glideTimeInSamples = sr * kControllerGlideTimeSeconds in double
  float c[2];
  mlb_coeffs_glide((float)(int)((double)sample_rate * (double)0.02f), c);
  cb->per_f = c[0], cb->dy = c[1];
  const size_t CG = (size_t)n_controllers * n_instruments;
  MLB_TRY(cb->d_ctrl.alloc((size_t)n_controllers * 4, "controller list"));
  MLB_TRY(cb->d_state.alloc((size_t)CS_COUNT * CG * 4, "controller bank"));
  MLB_TRY(cb->d_rows.alloc(CG * MLB_BLOCK * 4, "controller bank"));
  CU_CHECK(cudaMemcpy(cb->d_ctrl.get(), controllers, (size_t)n_controllers * 4, cudaMemcpyHostToDevice));
  MLB_TRY(mlb_controllers_clear(cb.get()));
  MLB_TRY(cb->stream.create(cudaStreamNonBlocking));
  *out = cb.release();
  return MLB_OK;
}

extern "C" int mlb_controllers_get_state(mlb_controllers* cb, uint32_t* words, float* rows)
{
  if (!cb || !words || !rows) return fail(MLB_ERR_INVALID, "null argument");
  const size_t CG = (size_t)cb->C * cb->G;
  CU_CHECK(cudaMemcpy(words, cb->d_state.get(), (size_t)CS_COUNT * CG * 4, cudaMemcpyDeviceToHost));
  CU_CHECK(cudaMemcpy(rows, cb->d_rows.get(), CG * MLB_BLOCK * 4, cudaMemcpyDeviceToHost));
  for (size_t s = 0; s < CG; ++s)  // an idle glide's row is its target (not kept in device memory)
    if ((int32_t)words[CS_REM * CG + s] < 0)
    {
      float tgt;
      memcpy(&tgt, &words[CS_TARGET * CG + s], 4);
      std::fill_n(rows + s * MLB_BLOCK, MLB_BLOCK, tgt);
    }
  return MLB_OK;
}

extern "C" int mlb_controllers_set_state(mlb_controllers* cb, const uint32_t* words, const float* rows)
{
  if (!cb || !words || !rows) return fail(MLB_ERR_INVALID, "null argument");
  const size_t CG = (size_t)cb->C * cb->G;
  CU_CHECK(cudaMemcpy(cb->d_state.get(), words, (size_t)CS_COUNT * CG * 4, cudaMemcpyHostToDevice));
  CU_CHECK(cudaMemcpy(cb->d_rows.get(), rows, CG * MLB_BLOCK * 4, cudaMemcpyHostToDevice));
  return MLB_OK;
}

extern "C" int mlb_controllers_set_voice_map(mlb_controllers* cb, const int32_t* voice_instrument, int n_voices)
{
  if (!cb) return fail(MLB_ERR_INVALID, "null controller bank");
  if (!voice_instrument)
  {
    cb->d_vmap.reset();
    cb->V = 0;
    return MLB_OK;
  }
  if (n_voices <= 0) return fail(MLB_ERR_INVALID, "n_voices must be positive (got %d)", n_voices);
  const int G = cb->G;
  std::vector<int32_t> tab((size_t)G + 2 + n_voices, 0);  // counting sort by instrument, the unmapped (-1) ones last
  for (int v = 0; v < n_voices; ++v)
  {
    const int g = voice_instrument[v];
    if (g < -1 || g >= G)
      return fail(MLB_ERR_INVALID, "voice %d: instrument %d is not -1 or one of the %d instruments", v, g, G);
    ++tab[(g < 0 ? G : g) + 1];
  }
  for (int g = 0; g <= G; ++g) tab[g + 1] += tab[g];
  std::vector<int32_t> fill(tab.begin(), tab.begin() + G + 1);
  for (int v = 0; v < n_voices; ++v)
  {
    const int g = voice_instrument[v] < 0 ? G : voice_instrument[v];
    tab[(size_t)G + 2 + fill[g]++] = v;
  }
  MLB_TRY(cb->d_vmap.alloc(tab.size() * 4, "voice map"));
  CU_CHECK(cudaMemcpy(cb->d_vmap.get(), tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
  cb->V = n_voices;
  return MLB_OK;
}

extern "C" int mlb_controllers_process_device(mlb_controllers* cb, const int32_t* offsets_dev,
                                              const mlb_controller_change* changes_dev, float* out_dev, int plane0,
                                              int n_planes, int n_blocks, void* stream)
{
  if (!cb || !offsets_dev || !out_dev) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive (got %d)", n_blocks);
  if (plane0 < 0 || n_planes < plane0 + cb->C)
    return fail(MLB_ERR_INVALID, "planes [%d, %d) of the %d controllers are not within the %d output planes", plane0,
                plane0 + cb->C, cb->C, n_planes);
  CtrlArgs a;
  a.offsets = offsets_dev, a.changes = changes_dev, a.ctrl = cb->d_ctrl.get();
  a.state = cb->d_state.get(), a.rows = cb->d_rows.get(), a.out = out_dev;
  a.vmap_off = cb->V ? cb->d_vmap.get() : nullptr;
  a.vmap_voice = cb->V ? cb->d_vmap.get() + cb->G + 2 : nullptr;
  a.G = cb->G, a.C = cb->C, a.N = cb->V ? cb->V : cb->G, a.T = n_blocks;
  a.plane0 = plane0, a.n_planes = n_planes;
  a.n_gblk = (cb->G + 31) / 32;
  a.per_f = cb->per_f, a.dy = cb->dy;
  const long long n_warps = (long long)a.C * a.n_gblk;
  controller_bank_kernel<<<(unsigned)((n_warps + kCtrlWarps - 1) / kCtrlWarps), 32 * kCtrlWarps, 0,
                           (cudaStream_t)stream>>>(a);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}

// offsets [T][G + 1] must index changes of n_changes entries, non-decreasing within each block
static int controllers_check_offsets(const mlb_controllers* cb, const int32_t* offsets, int n_changes, int n_blocks)
{
  for (int t = 0; t < n_blocks; ++t)
  {
    const int32_t* o = offsets + (size_t)t * (cb->G + 1);
    for (int g = 0; g < cb->G; ++g)
      if (o[g] < 0 || o[g] > o[g + 1] || o[g + 1] > n_changes)
        return fail(MLB_ERR_INVALID, "block %d, instrument %d: change range [%d, %d) is not within the %d changes", t,
                    g, o[g], o[g + 1], n_changes);
  }
  return MLB_OK;
}

extern "C" int mlb_controllers_process_host(mlb_controllers* cb, const int32_t* offsets_host,
                                            const mlb_controller_change* changes_host, int n_changes, float* out_host,
                                            int plane0, int n_planes, int n_blocks)
{
  if (!cb || !offsets_host || !out_host || (n_changes > 0 && !changes_host)) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive (got %d)", n_blocks);
  if (n_changes < 0) return fail(MLB_ERR_INVALID, "n_changes must not be negative (got %d)", n_changes);
  MLB_TRY(controllers_check_offsets(cb, offsets_host, n_changes, n_blocks));
  if (plane0 < 0 || n_planes < plane0 + cb->C)
    return fail(MLB_ERR_INVALID, "planes [%d, %d) of the %d controllers are not within the %d output planes", plane0,
                plane0 + cb->C, cb->C, n_planes);
  const size_t T = (size_t)n_blocks, N = cb->V ? cb->V : cb->G;
  const size_t off_bytes = T * (cb->G + 1) * 4, ch_bytes = (size_t)n_changes * sizeof(mlb_controller_change);
  const size_t out_bytes = T * n_planes * N * MLB_BLOCK * 4;
  MLB_TRY(cb->d_off.ensure(off_bytes, "staging"));
  if (n_changes) MLB_TRY(cb->d_ch.ensure(ch_bytes, "staging"));
  MLB_TRY(cb->d_out.ensure(out_bytes, "staging"));
  cudaStream_t s = cb->stream.get();
  const int rc = [&]() -> int
  {
    CU_CHECK(cudaMemcpyAsync(cb->d_off.get(), offsets_host, off_bytes, cudaMemcpyHostToDevice, s));
    if (n_changes) CU_CHECK(cudaMemcpyAsync(cb->d_ch.get(), changes_host, ch_bytes, cudaMemcpyHostToDevice, s));
    MLB_TRY(mlb_controllers_process_device(cb, cb->d_off.get(), cb->d_ch.get(), cb->d_out.get(), plane0, n_planes,
                                           n_blocks, s));
    // only the controller planes come down: the caller's other planes stay as they were
    const size_t plane = N * MLB_BLOCK * 4, pitch = (size_t)n_planes * plane;
    CU_CHECK(cudaMemcpy2DAsync(reinterpret_cast<char*>(out_host) + plane0 * plane, pitch,
                               reinterpret_cast<const char*>(cb->d_out.get()) + plane0 * plane, pitch, cb->C * plane, T,
                               cudaMemcpyDeviceToHost, s));
    return MLB_OK;
  }();
  return drain(rc, {s});
}

// Contract E with controller planes: the graph's input per block is the 8 Voice rows, then the C controller rows
// in the bank's list order.  Per time chunk on the pipeline of mlb_synth_process_host: records and offsets go up on
// s_h2d (all changes with the first chunk), the voice kernel, K11 and the graph run on the graph's stream, output rows
// come down on s_d2h.
extern "C" int mlb_synth_process_controllers_host(mlb_voices* vb, mlb_controllers* cb, mlb_graph* g,
                                                  const mlb_voice_events* events_host, const int32_t* ctrl_offsets_host,
                                                  const mlb_controller_change* ctrl_changes_host, float* out_host,
                                                  float* mix_host, int n_blocks)
{
  if (!cb || !ctrl_offsets_host) return fail(MLB_ERR_INVALID, "null argument");
  const int n_planes = MLB_VOICE_ROWS + cb->C;
  unsigned row_mask;
  MLB_TRY(synth_check(vb, g, events_host, n_blocks, out_host || mix_host, &row_mask, n_planes));
  if (cb->V != g->V)
    return fail(MLB_ERR_INVALID, "controller bank's voice map has %d voices, graph has %d (mlb_controllers_set_voice_map)",
                cb->V, g->V);
  if ((cb->protocol == 0) != ((vb->flags & MLB_VOICES_MIDI) != 0))
    return fail(MLB_ERR_INVALID, "controller bank protocol %s, voice bank %s MLB_VOICES_MIDI", cb->protocol ? "MPE" : "MIDI",
                (vb->flags & MLB_VOICES_MIDI) ? "with" : "without");
  int n_changes = 0;  // the changes the offsets index
  for (int t = 0; t < n_blocks; ++t) n_changes = std::max(n_changes, ctrl_offsets_host[(size_t)t * (cb->G + 1) + cb->G]);
  if (n_changes > 0 && !ctrl_changes_host) return fail(MLB_ERR_INVALID, "null controller changes");
  MLB_TRY(controllers_check_offsets(cb, ctrl_offsets_host, n_changes, n_blocks));
  MLB_TRY(ensure_init());
  const size_t V = (size_t)g->V, T = (size_t)n_blocks, n_out = g->outs.size(), G1 = (size_t)cb->G + 1;
  const int Tc = synth_chunk_blocks(g, n_blocks, n_planes);
  if (out_host) MLB_TRY(g->d_out.ensure(T * n_out * V * MLB_BLOCK * 4, "staging"));
  if (mix_host) MLB_TRY(g->d_mix.ensure(T * n_out * MLB_BLOCK * 4, "staging"));
  MLB_TRY(vb->d_ev.ensure(T * V * sizeof(mlb_voice_events), "staging"));
  MLB_TRY(vb->d_out.ensure((size_t)Tc * n_planes * V * MLB_BLOCK * 4, "staging"));
  MLB_TRY(cb->d_off.ensure(T * G1 * 4, "staging"));
  if (n_changes) MLB_TRY(cb->d_ch.ensure((size_t)n_changes * sizeof(mlb_controller_change), "staging"));
  const size_t row_floats = n_out * V * MLB_BLOCK;  // output rows per block
  const int rc = [&]() -> int
  {
    MLB_TRY(host_pipeline(
        g, n_blocks, Tc, true, out_host != nullptr,
        [&](int t0, int t1, cudaStream_t s)
        {
          cudaError_t e = cudaSuccess;
          if (t0 == 0 && n_changes)
            e = cudaMemcpyAsync(cb->d_ch.get(), ctrl_changes_host, (size_t)n_changes * sizeof(mlb_controller_change),
                                cudaMemcpyHostToDevice, s);
          if (e == cudaSuccess)
            e = cudaMemcpyAsync(cb->d_off.get() + t0 * G1, ctrl_offsets_host + t0 * G1, (t1 - t0) * G1 * 4,
                                cudaMemcpyHostToDevice, s);
          if (e == cudaSuccess)
            e = cudaMemcpyAsync(vb->d_ev.get() + t0 * V, events_host + t0 * V, (t1 - t0) * V * sizeof(mlb_voice_events),
                                cudaMemcpyHostToDevice, s);
          return e;
        },
        [&](int t0, int t1, cudaStream_t s) -> int
        {
          MLB_TRY(voices_launch(vb, vb->d_ev.get() + t0 * V, vb->d_out.get(), t1 - t0, row_mask, n_planes, s));
          MLB_TRY(mlb_controllers_process_device(cb, cb->d_off.get() + t0 * G1, cb->d_ch.get(), vb->d_out.get(),
                                                 MLB_VOICE_ROWS, n_planes, t1 - t0, s));
          return graph_process(g, vb->d_out.get(), n_planes, out_host ? g->d_out.get() + t0 * row_floats : nullptr,
                               mix_host ? g->d_mix.get() + t0 * n_out * MLB_BLOCK : nullptr, t1 - t0, s);
        },
        [&](int t0, int t1, cudaStream_t s)
        {
          return cudaMemcpyAsync(out_host + t0 * row_floats, g->d_out.get() + t0 * row_floats,
                                 (t1 - t0) * row_floats * 4, cudaMemcpyDeviceToHost, s);
        }));
    if (mix_host) MLB_TRY(mlb_graph_mix_wait(g, g->stream.get()));
    if (mix_host)
      CU_CHECK(cudaMemcpyAsync(mix_host, g->d_mix.get(), T * n_out * MLB_BLOCK * 4, cudaMemcpyDeviceToHost, g->stream.get()));
    return MLB_OK;
  }();
  return drain(rc, {g->s_h2d.get(), g->stream.get(), g->s_d2h.get()});
}

// ------------------------------------------------------------------------------------------
// Upsampler / Downsampler banks (K8, resample_kernel.cuh)

struct mlb_resampler
{
  // declared first, so released last: the buffers below are freed first, and cudaFree waits for the device
  LiveCount live;
  Stream stream;
  int dir = 0, oct = 0, V = 0;
  unsigned counter = 0;
  DevBuf<uint32_t> d_state;
  DevBuf<float> d_buf, d_in, d_out;
};

extern "C" int mlb_resampler_destroy(mlb_resampler* r)
{
  delete r;
  return MLB_OK;
}
extern "C" int mlb_resampler_clear(mlb_resampler* r)
{
  if (!r) return fail(MLB_ERR_INVALID, "null resampler");
  r->counter = 0;
  CU_CHECK(cudaMemset(r->d_state.get(), 0, r->d_state.bytes()));
  if (r->d_buf.get()) CU_CHECK(cudaMemset(r->d_buf.get(), 0, r->d_buf.bytes()));
  return MLB_OK;
}
extern "C" int mlb_resampler_create(int direction, int octaves, int n_voices, mlb_resampler** out)
{
  if (!out) return fail(MLB_ERR_INVALID, "out is null");
  *out = nullptr;
  if ((direction != MLB_RESAMPLE_UP && direction != MLB_RESAMPLE_DOWN) || octaves < 1 || octaves > 4 || n_voices <= 0)
    return fail(MLB_ERR_INVALID, "bad argument (direction %d, octaves %d, voices %d)", direction, octaves, n_voices);
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  std::unique_ptr<mlb_resampler> r(new mlb_resampler);
  r->live.arm();
  r->dir = direction, r->oct = octaves, r->V = n_voices;
  MLB_TRY(r->d_state.alloc((size_t)octaves * 9 * n_voices * 4, "resampler state"));
  if (direction == MLB_RESAMPLE_DOWN)
    MLB_TRY(r->d_buf.alloc((size_t)(2 * octaves + 1) * n_voices * MLB_BLOCK * 4, "resampler state"));
  MLB_TRY(r->stream.create(cudaStreamNonBlocking));
  MLB_TRY(mlb_resampler_clear(r.get()));
  *out = r.release();
  return MLB_OK;
}
static int resampler_out_blocks(const mlb_resampler* r, int n_in)
{
  if (r->dir == MLB_RESAMPLE_UP) return n_in << r->oct;
  return (int)(((long long)r->counter + n_in) >> r->oct);
}
extern "C" int mlb_resampler_process_device(mlb_resampler* r, const float* in_dev, float* out_dev, int n_blocks_in,
                                            int* n_blocks_out, void* stream)
{
  if (!r || !in_dev) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks_in <= 0) return fail(MLB_ERR_INVALID, "n_blocks_in must be positive");
  const int n_out = resampler_out_blocks(r, n_blocks_in);
  if (n_out > 0 && !out_dev) return fail(MLB_ERR_INVALID, "out is null");
  ResampleArgs a;
  a.in = in_dev, a.out = out_dev, a.state = r->d_state.get(), a.buf = r->d_buf.get();
  a.V = r->V, a.T = n_blocks_in, a.oct = r->oct, a.counter = r->counter;
  const int grid = (r->V + 127) / 128;
  if (r->dir == MLB_RESAMPLE_UP)
    upsample_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a);
  else
  {
    downsample_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a);
    r->counter = (r->counter + (unsigned)n_blocks_in) & ((1u << r->oct) - 1u);
  }
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  if (n_blocks_out) *n_blocks_out = n_out;
  return MLB_OK;
}
extern "C" int mlb_resampler_process_host(mlb_resampler* r, const float* in_host, float* out_host, int n_blocks_in,
                                          int* n_blocks_out)
{
  if (!r || !in_host) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks_in <= 0) return fail(MLB_ERR_INVALID, "n_blocks_in must be positive");
  const size_t row = (size_t)r->V * MLB_BLOCK * 4;
  const int n_out = resampler_out_blocks(r, n_blocks_in);
  if (n_out > 0 && !out_host) return fail(MLB_ERR_INVALID, "out is null");
  MLB_TRY(r->d_in.ensure((size_t)n_blocks_in * row, "staging"));
  MLB_TRY(r->d_out.ensure(std::max<size_t>(1, (size_t)n_out) * row, "staging"));
  cudaStream_t s = r->stream.get();
  const int rc = [&]() -> int
  {
    CU_CHECK(cudaMemcpyAsync(r->d_in.get(), in_host, (size_t)n_blocks_in * row, cudaMemcpyHostToDevice, s));
    MLB_TRY(mlb_resampler_process_device(r, r->d_in.get(), r->d_out.get(), n_blocks_in, n_blocks_out, s));
    if (n_out > 0) CU_CHECK(cudaMemcpyAsync(out_host, r->d_out.get(), (size_t)n_out * row, cudaMemcpyDeviceToHost, s));
    return MLB_OK;
  }();
  return drain(rc, {s});
}

// ------------------------------------------------------------------------------------------
// FDTD membrane banks (K9, fdtd_kernel.cuh)

struct mlb_fdtd
{
  // declared first, so released last: the buffers below are freed first, and cudaFree waits for the device
  LiveCount live;
  Stream stream;
  int V = 0, in_planes = 0, excite = 0, freq = 0;
  unsigned flags = 0;
  float sample_rate = 0.f;
  DevBuf<float> d_state;  // [V][2][16][16]
  DevBuf<float> d_in, d_out;
};

static size_t fdtd_state_bytes(const mlb_fdtd* f) { return (size_t)f->V * 2 * kFdtdCells * sizeof(float); }

extern "C" int mlb_fdtd_destroy(mlb_fdtd* f)
{
  delete f;
  return MLB_OK;
}
extern "C" int mlb_fdtd_clear(mlb_fdtd* f)
{
  if (!f) return fail(MLB_ERR_INVALID, "null FDTD bank");
  CU_CHECK(cudaMemset(f->d_state.get(), 0, fdtd_state_bytes(f)));
  CU_CHECK(cudaDeviceSynchronize());
  return MLB_OK;
}
extern "C" int mlb_fdtd_create(int n_instances, float sample_rate, int in_planes, int excite_plane, int freq_plane,
                               unsigned flags, mlb_fdtd** out)
{
  if (!out) return fail(MLB_ERR_INVALID, "out is null");
  *out = nullptr;
  if (n_instances <= 0) return fail(MLB_ERR_INVALID, "n_instances must be positive (got %d)", n_instances);
  if (!(sample_rate > 0.f) || !std::isfinite(sample_rate))
    return fail(MLB_ERR_INVALID, "sample_rate must be positive and finite (got %g)", (double)sample_rate);
  if (in_planes <= 0 || excite_plane < 0 || excite_plane >= in_planes || freq_plane < 0 || freq_plane >= in_planes)
    return fail(MLB_ERR_INVALID, "bad planes (in_planes %d, excite_plane %d, freq_plane %d)", in_planes,
                excite_plane, freq_plane);
  if (flags & ~MLB_FDTD_FTZ) return fail(MLB_ERR_INVALID, "unknown flags 0x%x", flags);
  int rc = ensure_init();
  if (rc != MLB_OK) return rc;
  std::unique_ptr<mlb_fdtd> f(new mlb_fdtd);
  f->live.arm();
  f->V = n_instances, f->in_planes = in_planes, f->excite = excite_plane, f->freq = freq_plane;
  f->flags = flags, f->sample_rate = sample_rate;
  MLB_TRY(f->d_state.alloc(fdtd_state_bytes(f.get()), "FDTD state"));
  MLB_TRY(f->stream.create(cudaStreamNonBlocking));
  MLB_TRY(mlb_fdtd_clear(f.get()));
  *out = f.release();
  return MLB_OK;
}
extern "C" int mlb_fdtd_get_state(mlb_fdtd* f, float* host)
{
  if (!f || !host) return fail(MLB_ERR_INVALID, "null argument");
  CU_CHECK(cudaDeviceSynchronize());
  CU_CHECK(cudaMemcpy(host, f->d_state.get(), fdtd_state_bytes(f), cudaMemcpyDeviceToHost));
  return MLB_OK;
}
extern "C" int mlb_fdtd_set_state(mlb_fdtd* f, const float* host)
{
  if (!f || !host) return fail(MLB_ERR_INVALID, "null argument");
  CU_CHECK(cudaDeviceSynchronize());
  CU_CHECK(cudaMemcpy(f->d_state.get(), host, fdtd_state_bytes(f), cudaMemcpyHostToDevice));
  return MLB_OK;
}
extern "C" int mlb_fdtd_process_device(mlb_fdtd* f, const float* in_dev, float* out_dev, int n_blocks, void* stream)
{
  if (!f || !in_dev || !out_dev) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive (got %d)", n_blocks);
  FdtdArgs a;
  a.in = in_dev, a.out = out_dev, a.state = f->d_state.get();
  a.V = f->V, a.T = n_blocks, a.in_planes = f->in_planes, a.excite_plane = f->excite, a.freq_plane = f->freq;
  // the example's constants (fdtd.cpp:23, 79, 89, 100-101, 118), rounded on the host as its compiler does
  a.k_size = sqrtf((float)(kFdtdN * kFdtdN) + (float)(kFdtdN * kFdtdN));
  a.k_tension = 3.0f / 5.0f;
  a.k_sixth = 1.f / 6.f;
  a.k_two_thirds = 2.f / 3.f;
  a.isr = 1.0f / f->sample_rate;
  a.sk = 1.0f / (1.0f + a.isr * 1.0f);
  const int grid = (f->V + kFdtdWarps - 1) / kFdtdWarps;
  if (f->flags & MLB_FDTD_FTZ)
    fdtd_kernel<true><<<grid, 32 * kFdtdWarps, 0, (cudaStream_t)stream>>>(a);
  else
    fdtd_kernel<false><<<grid, 32 * kFdtdWarps, 0, (cudaStream_t)stream>>>(a);
  ++g_launches;
  CU_CHECK(cudaGetLastError());
  return MLB_OK;
}
extern "C" int mlb_fdtd_process_host(mlb_fdtd* f, const float* in_host, float* out_host, int n_blocks)
{
  if (!f || !in_host || !out_host) return fail(MLB_ERR_INVALID, "null argument");
  if (n_blocks <= 0) return fail(MLB_ERR_INVALID, "n_blocks must be positive (got %d)", n_blocks);
  const size_t row = (size_t)f->V * MLB_BLOCK * sizeof(float);
  const size_t in_bytes = (size_t)n_blocks * f->in_planes * row, out_bytes = (size_t)n_blocks * 2 * row;
  MLB_TRY(f->d_in.ensure(in_bytes, "staging"));
  MLB_TRY(f->d_out.ensure(out_bytes, "staging"));
  cudaStream_t s = f->stream.get();
  const int rc = [&]() -> int
  {
    CU_CHECK(cudaMemcpyAsync(f->d_in.get(), in_host, in_bytes, cudaMemcpyHostToDevice, s));
    MLB_TRY(mlb_fdtd_process_device(f, f->d_in.get(), f->d_out.get(), n_blocks, s));
    CU_CHECK(cudaMemcpyAsync(out_host, f->d_out.get(), out_bytes, cudaMemcpyDeviceToHost, s));
    return MLB_OK;
  }();
  return drain(rc, {s});
}


// ------------------------------------------------------------------------------------------
// C face of mlb::VoiceRouter (host only)
#include "../../include/mlb200_events.hpp"

struct mlb_router
{
  mlb::VoiceRouter router;
  mlb_router(int polyphony, int protocol)
      : router(polyphony, protocol == 1 ? mlb::VoiceRouter::kMPE : mlb::VoiceRouter::kMIDI)
  {
  }
};
extern "C" mlb_router* mlb_router_create(int polyphony, int protocol)
{
  if (polyphony < 1 || (protocol != 0 && protocol != 1)) return nullptr;
  return new mlb_router(polyphony, protocol);
}
extern "C" void mlb_router_destroy(mlb_router* r) { delete r; }
extern "C" void mlb_router_set_unison(mlb_router* r, int on)
{
  if (r) r->router.setUnison(on != 0);
}
extern "C" void mlb_router_add_event(mlb_router* r, const mlb_event* e)
{
  if (!r || !e) return;
  mlb::Event ev;
  ev.type = e->type, ev.channel = e->channel, ev.sourceIdx = e->source_idx, ev.time = e->time;
  ev.value1 = e->value1, ev.value2 = e->value2;
  r->router.addEvent(ev);
}
extern "C" void mlb_router_clear_events(mlb_router* r)
{
  if (r) r->router.clearEvents();
}
extern "C" int mlb_router_unsupported_count(const mlb_router* r) { return r ? r->router.unsupportedEvents() : -1; }
extern "C" void mlb_router_set_mod_cc(mlb_router* r, int cc)
{
  if (r) r->router.setModCC(cc);
}
extern "C" int mlb_router_record_count(const mlb_router* r) { return r ? r->router.recordCount() : -1; }
extern "C" int mlb_router_process_vector(mlb_router* r, int start_time, mlb_voice_events* records)
{
  if (!r || !records) return -1;
  return r->router.processVector(start_time, records);
}
extern "C" int mlb_router_controller_changes(const mlb_router* r, mlb_controller_change* out, int cap)
{
  if (!r || (cap > 0 && !out)) return -1;
  const std::vector<mlb_controller_change>& c = r->router.controllerChanges();
  std::copy_n(c.begin(), std::min<size_t>(c.size(), (size_t)std::max(cap, 0)), out);
  return (int)c.size();
}
