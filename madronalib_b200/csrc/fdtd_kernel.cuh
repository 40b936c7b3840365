// fdtd_kernel.cuh -- K9: banks of 16 x 16 finite-difference (FDTD) membranes, the physical model of the
// reference's examples/audio-and-midi/fdtd.cpp (FDTDState + processFDTDModel, :26-154).
//
// One warp per instance; time is serial.  Lane l owns a 4-row x 2-column patch of the surface:
// rows 4*(l >> 3) .. +3, columns 2*(l & 7) .. +1.  A lane keeps both live surfaces (z^-1 and z^-2) as
// 6 x 4 register tiles: the 4 x 2 patch plus a one-cell halo.  Per sample the z^-1 halo is exchanged with
// 16 __shfl_sync (left / right columns first, then the up / down rows with their corners); the zero
// boundary of the reference's never-written padding is a +0 on the edge lanes.  The z^-2 halo is never
// exchanged again after the launch starts: the z^-2 surface of sample n+1 is the (already excited) z^-1
// surface of sample n, so its halo is the one exchanged one sample earlier.  The two tiles swap roles every
// sample (the sample loop is unrolled by two), so the reference's pointer rotation costs no register moves.
//
// Exactness: every operation is one separately rounded binary32 op in the reference's order and
// parenthesisation.  FTZ = true replaces each by its .ftz form (subnormal inputs and results become zeros
// of the same sign), which is what the example's UsingFlushDenormalsToZero (MXCSR FZ + DAZ) does on x86.
//
// Per block of 64 samples the warp designs the 64 coefficient sets (two samples per lane) into shared
// memory ahead of the sample loop; the excitation and frequency rows are prefetched a block ahead; the two
// pickups are staged in shared memory and leave as two full 256-byte rows.
#pragma once
#include "ops.cuh"

namespace mlb
{
constexpr int kFdtdN = MLB_FDTD_SIZE;          // 16 x 16 interior
constexpr int kFdtdCells = kFdtdN * kFdtdN;    // 256
constexpr int kFdtdWarps = 4;                  // instances per CTA

template <bool FTZ>
struct Ff
{
  static MLB_DEV float mul(float a, float b)
  {
    if (!FTZ) return __fmul_rn(a, b);
    float r;
    asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
  }
  static MLB_DEV float add(float a, float b)
  {
    if (!FTZ) return __fadd_rn(a, b);
    float r;
    asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
  }
  static MLB_DEV float sub(float a, float b)
  {
    if (!FTZ) return __fsub_rn(a, b);
    float r;
    asm("sub.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
  }
};

struct FdtdArgs
{
  const float* in;   // [T][in_planes][V][64]
  float* out;        // [T][2][V][64]: pickup L, pickup R
  float* state;      // [V][2][16][16]: z^-1 interior, then z^-2
  int V, T, in_planes, excite_plane, freq_plane;
  float k_size;      // sqrtf(16*16 + 16*16)
  float k_tension;   // 3.0f / 5.0f
  float k_sixth;     // 1.f / 6.f
  float k_two_thirds;// 2.f / 3.f
  float isr;         // 1.0f / sample_rate
  float sk;          // 1.0f / (1.0f + isr)
};

// One sample: excite u1, exchange its halo, write the new surface over u2's interior (u2 becomes the new u1).
template <bool FTZ>
MLB_DEV void fdtd_sample(float (&u1)[6][4], float (&u2)[6][4], const float4 k4, const float2 k2, bool exciter,
                         bool pickup, float* pickup_slot, int cg, int rg)
{
  using F = Ff<FTZ>;
  // processFDTDModel :127-129: *exciter += inputVec[i] * kInputGain (row 2, column 8 = lane 4, local (2, 0))
  if (exciter) u1[3][1] = F::add(u1[3][1], k2.y);
  // halo of z^-1: left / right columns (interior rows), then whole rows up / down (with the corners)
#pragma unroll
  for (int r = 1; r <= 4; ++r)
  {
    const float l = __shfl_up_sync(0xffffffffu, u1[r][2], 1);
    const float rr = __shfl_down_sync(0xffffffffu, u1[r][1], 1);
    u1[r][0] = cg == 0 ? 0.f : l;
    u1[r][3] = cg == 7 ? 0.f : rr;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c)
  {
    const float up = __shfl_up_sync(0xffffffffu, u1[4][c], 8);
    const float dn = __shfl_down_sync(0xffffffffu, u1[1][c], 8);
    u1[0][c] = rg == 0 ? 0.f : up;
    u1[5][c] = rg == 3 ? 0.f : dn;
  }
  // doFDTDStep2D :64-69 for the lane's 8 cells
  const float kc = k4.x, ke = k4.y, kk = k4.z, kc2 = k4.w, ke2 = k2.x;
  float nu[4][2];
#pragma unroll
  for (int r = 1; r <= 4; ++r)
#pragma unroll
    for (int c = 1; c <= 2; ++c)
    {
      float f = F::mul(kc, u1[r][c]);
      f = F::add(f, F::mul(ke, F::add(F::add(F::add(u1[r][c - 1], u1[r - 1][c]), u1[r][c + 1]), u1[r + 1][c])));
      f = F::add(f, F::mul(kk, F::add(F::add(F::add(u1[r - 1][c - 1], u1[r - 1][c + 1]), u1[r + 1][c - 1]),
                                      u1[r + 1][c + 1])));
      f = F::add(f, F::mul(kc2, u2[r][c]));
      f = F::add(f, F::mul(ke2, F::add(F::add(F::add(u2[r][c - 1], u2[r - 1][c]), u2[r][c + 1]), u2[r + 1][c])));
      nu[r - 1][c - 1] = f;
    }
#pragma unroll
  for (int r = 1; r <= 4; ++r)
#pragma unroll
    for (int c = 1; c <= 2; ++c) u2[r][c] = nu[r - 1][c - 1];
  // :136-143: pickups at row 9, columns 1 and 15 = lanes 16 and 23, local (1, 1)
  if (pickup) *pickup_slot = nu[1][1];
}

// The coefficient design of processFDTDModel :85-123 for one frequency sample, in the reference's order.
template <bool FTZ>
MLB_DEV void fdtd_coeffs(const FdtdArgs& a, float Fs, float4& k4, float& ke2_out)
{
  using F = Ff<FTZ>;
  const float c = F::mul(a.k_size, Fs);
  const float T = F::mul(a.k_tension, c);
  const float TT = F::mul(T, T);
  float kk = F::mul(TT, a.k_sixth);
  float ke = F::mul(TT, a.k_two_thirds);
  float kc = F::sub(2.f, F::mul(4.f, F::add(kk, ke)));
  const float ks1 = F::mul(F::mul(1.f, T), a.isr);   // s1 * T * isr, s1 = 1
  ke = F::add(ke, ks1);
  kc = F::add(kc, F::mul(-4.0f, ks1));
  float ke2 = F::mul(-1.0f, ks1);
  float kc2 = F::sub(F::add(F::mul(1.f, a.isr), F::mul(4.0f, ks1)), 1.0f);  // s0 * isr + 4 ks1 - 1, s0 = 1
  kc = F::mul(kc, a.sk);
  ke = F::mul(ke, a.sk);
  kk = F::mul(kk, a.sk);
  kc2 = F::mul(kc2, a.sk);
  ke2 = F::mul(ke2, a.sk);
  k4 = make_float4(kc, ke, kk, kc2);
  ke2_out = ke2;
}

template <bool FTZ>
__global__ void __launch_bounds__(32 * kFdtdWarps) fdtd_kernel(const FdtdArgs a)
{
  using F = Ff<FTZ>;
  __shared__ float4 s_k4[kFdtdWarps][MLB_BLOCK];   // kc, ke, kk, kc2 per sample
  __shared__ float2 s_k2[kFdtdWarps][MLB_BLOCK];   // ke2, excitation * kInputGain per sample
  __shared__ __align__(16) float s_out[kFdtdWarps][2 * MLB_BLOCK];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int v = blockIdx.x * kFdtdWarps + w;
  if (v >= a.V) return;  // whole warps only: the kernel synchronises warps, never the CTA
  const int cg = lane & 7, rg = lane >> 3;
  const size_t V = (size_t)a.V;

  // state [v][2][16][16]: each float2 load of the warp covers four 64-byte row pieces, every byte used
  float X[6][4], Y[6][4];
  const float* st = a.state + (size_t)v * 2 * kFdtdCells;
#pragma unroll
  for (int r = 0; r < 4; ++r)
  {
    const float2 p = *reinterpret_cast<const float2*>(st + (4 * rg + r) * kFdtdN + 2 * cg);
    const float2 q = *reinterpret_cast<const float2*>(st + kFdtdCells + (4 * rg + r) * kFdtdN + 2 * cg);
    X[r + 1][1] = p.x, X[r + 1][2] = p.y;
    Y[r + 1][1] = q.x, Y[r + 1][2] = q.y;
  }
  // the z^-2 halo once (edges only; its corners are never read)
#pragma unroll
  for (int r = 1; r <= 4; ++r)
  {
    const float l = __shfl_up_sync(0xffffffffu, Y[r][2], 1), rr = __shfl_down_sync(0xffffffffu, Y[r][1], 1);
    Y[r][0] = cg == 0 ? 0.f : l;
    Y[r][3] = cg == 7 ? 0.f : rr;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c)
  {
    const float up = __shfl_up_sync(0xffffffffu, Y[4][c], 8), dn = __shfl_down_sync(0xffffffffu, Y[1][c], 8);
    Y[0][c] = rg == 0 ? 0.f : up;
    Y[5][c] = rg == 3 ? 0.f : dn;
  }
  X[0][0] = X[0][3] = X[5][0] = X[5][3] = 0.f;  // (overwritten by the first exchange)
  Y[0][0] = Y[0][3] = Y[5][0] = Y[5][3] = 0.f;

  auto row_of = [&](int t, int plane) { return a.in + (((size_t)t * a.in_planes + plane) * V + v) * MLB_BLOCK; };
  float2 ex = reinterpret_cast<const float2*>(row_of(0, a.excite_plane))[lane];
  float2 fq = reinterpret_cast<const float2*>(row_of(0, a.freq_plane))[lane];
  const bool exciter = lane == 4, pickup = lane == 16 || lane == 23;
  float* pick = &s_out[w][lane == 23 ? MLB_BLOCK : 0];

#pragma unroll 1
  for (int t = 0; t < a.T; ++t)
  {
    const float2 ex_c = ex, fq_c = fq;
    if (t + 1 < a.T)
    {
      ex = reinterpret_cast<const float2*>(row_of(t + 1, a.excite_plane))[lane];
      fq = reinterpret_cast<const float2*>(row_of(t + 1, a.freq_plane))[lane];
    }
    __syncwarp();  // the previous block's readers of s_k4 / s_k2 / s_out are done
    {
      float4 k4;
      float ke2;
      fdtd_coeffs<FTZ>(a, fq_c.x, k4, ke2);
      s_k4[w][2 * lane] = k4;
      s_k2[w][2 * lane] = make_float2(ke2, F::mul(ex_c.x, 4.0f));  // kInputGain = 16 * 16 / 64
      fdtd_coeffs<FTZ>(a, fq_c.y, k4, ke2);
      s_k4[w][2 * lane + 1] = k4;
      s_k2[w][2 * lane + 1] = make_float2(ke2, F::mul(ex_c.y, 4.0f));
    }
    __syncwarp();
#pragma unroll 1
    for (int i = 0; i < MLB_BLOCK; i += 2)
    {
      fdtd_sample<FTZ>(X, Y, s_k4[w][i], s_k2[w][i], exciter, pickup, pick + i, cg, rg);
      fdtd_sample<FTZ>(Y, X, s_k4[w][i + 1], s_k2[w][i + 1], exciter, pickup, pick + i + 1, cg, rg);
    }
    __syncwarp();
    // rows L (lanes 0..15) and R (lanes 16..31), 256 B each
    const int row = lane >> 4;
    float4* dst = reinterpret_cast<float4*>(a.out + (((size_t)t * 2 + row) * V + v) * MLB_BLOCK);
    dst[lane & 15] = reinterpret_cast<const float4*>(s_out[w])[lane];
  }

  float* so = a.state + (size_t)v * 2 * kFdtdCells;
#pragma unroll
  for (int r = 0; r < 4; ++r)
  {
    *reinterpret_cast<float2*>(so + (4 * rg + r) * kFdtdN + 2 * cg) = make_float2(X[r + 1][1], X[r + 1][2]);
    *reinterpret_cast<float2*>(so + kFdtdCells + (4 * rg + r) * kFdtdN + 2 * cg) = make_float2(Y[r + 1][1], Y[r + 1][2]);
  }
}

}  // namespace mlb
