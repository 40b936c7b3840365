// mlb200.hpp -- C++17 host mirror of the reference's value/functor API over the C ABI (mlb200.h).
//
// Same spellings and value semantics as the reference where the host keeps data
// (reference: source/DSP/MLDSPOps.h:94-353 DSPVectorArray<ROWS>, :361 DSPVector,
// :523-533 load/store, :157 implicit float -> vector, :337-352 operator+ - * /), plus
// `mlb::DeviceBank`, the batched analogue of `Bank<T, ROWS>` (source/DSP/MLDSPFunctional.h:321-360)
// whose ROWS is chosen at run time and whose operator() runs on the GPU.
//
// Header only; link against libmlb200.so.  Elementwise operators on host DSPVectorArrays
// are computed on the GPU through mlb_map_host (there is no CPU arithmetic path in this
// project); use DeviceBank / graphs for anything performance relevant.
#pragma once
#include <array>
#include <cmath>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "mlb200.h"

constexpr size_t kFloatsPerDSPVectorBits = 6;  // reference MLDSPMath.h:8
constexpr size_t kFloatsPerDSPVector = 1 << kFloatsPerDSPVectorBits;
static_assert(kFloatsPerDSPVector == MLB_BLOCK, "block size");

namespace mlb
{
struct Error : std::runtime_error
{
  int code;
  Error(int c, const char* m) : std::runtime_error(m), code(c) {}
};
inline void check(int rc)
{
  if (rc != MLB_OK) throw Error(rc, mlb_last_error());
}

// ---- DSPVectorArray<ROWS>: ROWS x 64 f32, row-major, 16-byte aligned, value semantics ----
template <size_t ROWS>
class DSPVectorArray
{
  alignas(16) float data_[kFloatsPerDSPVector * ROWS];

 public:
  DSPVectorArray() { std::memset(data_, 0, sizeof(data_)); }  // zero fill, MLDSPOps.h:153
  DSPVectorArray(float k) { operator=(k); }                   // broadcast, MLDSPOps.h:157
  explicit DSPVectorArray(const float* p) { std::memcpy(data_, p, sizeof(data_)); }
  DSPVectorArray& operator=(float k)
  {
    for (float& f : data_) f = k;
    return *this;
  }
  float* getBuffer() { return data_; }
  const float* getConstBuffer() const { return data_; }
  float& operator[](size_t i) { return data_[i]; }
  float operator[](size_t i) const { return data_[i]; }
  DSPVectorArray<1>& row(int j) { return *reinterpret_cast<DSPVectorArray<1>*>(data_ + kFloatsPerDSPVector * j); }
  const DSPVectorArray<1>& constRow(int j) const
  {
    return *reinterpret_cast<const DSPVectorArray<1>*>(data_ + kFloatsPerDSPVector * j);
  }
  bool operator==(const DSPVectorArray& o) const
  {
    for (size_t i = 0; i < kFloatsPerDSPVector * ROWS; ++i)
      if (data_[i] != o.data_[i]) return false;
    return true;
  }

  friend DSPVectorArray map2(int op, const DSPVectorArray& a, const DSPVectorArray& b)
  {
    DSPVectorArray y;
    check(mlb_map_host(op, a.data_, b.data_, nullptr, y.data_, ROWS));
    return y;
  }
  friend DSPVectorArray operator+(const DSPVectorArray& a, const DSPVectorArray& b) { return map2(MLB_OP_ADD, a, b); }
  friend DSPVectorArray operator-(const DSPVectorArray& a, const DSPVectorArray& b) { return map2(MLB_OP_SUBTRACT, a, b); }
  friend DSPVectorArray operator*(const DSPVectorArray& a, const DSPVectorArray& b) { return map2(MLB_OP_MULTIPLY, a, b); }
  friend DSPVectorArray operator/(const DSPVectorArray& a, const DSPVectorArray& b) { return map2(MLB_OP_DIVIDE, a, b); }
  // MLDSPOps.h:312-331
  DSPVectorArray& operator+=(const DSPVectorArray& x) { return *this = map2(MLB_OP_ADD, *this, x); }
  DSPVectorArray& operator-=(const DSPVectorArray& x) { return *this = map2(MLB_OP_SUBTRACT, *this, x); }
  DSPVectorArray& operator*=(const DSPVectorArray& x) { return *this = map2(MLB_OP_MULTIPLY, *this, x); }
  DSPVectorArray& operator/=(const DSPVectorArray& x) { return *this = map2(MLB_OP_DIVIDE, *this, x); }
};
using DSPVector = DSPVectorArray<1>;

// ---- DSPVectorArrayInt<ROWS>: the same storage read as int32 (MLDSPOps.h:370-498) ----
template <size_t ROWS>
class DSPVectorArrayInt
{
  union
  {
    alignas(16) float asFloat[kFloatsPerDSPVector * ROWS];
    alignas(16) int32_t asInt[kFloatsPerDSPVector * ROWS];
  } data_;

 public:
  explicit DSPVectorArrayInt() { operator=(0); }
  explicit DSPVectorArrayInt(int32_t k) { operator=(k); }
  DSPVectorArrayInt& operator=(int32_t k)
  {
    for (int32_t& i : data_.asInt) i = k;
    return *this;
  }
  float* getBuffer() { return data_.asFloat; }
  const float* getConstBuffer() const { return data_.asFloat; }
  int32_t* getBufferInt() { return data_.asInt; }
  const int32_t* getConstBufferInt() const { return data_.asInt; }
  int32_t& operator[](int i) { return data_.asInt[i]; }
  int32_t operator[](int i) const { return data_.asInt[i]; }
  DSPVectorArrayInt<1>& row(int j) { return *reinterpret_cast<DSPVectorArrayInt<1>*>(data_.asInt + kFloatsPerDSPVector * j); }
  const DSPVectorArrayInt<1>& constRow(int j) const
  {
    return *reinterpret_cast<const DSPVectorArrayInt<1>*>(data_.asInt + kFloatsPerDSPVector * j);
  }
  bool operator==(const DSPVectorArrayInt& o) const { return std::memcmp(data_.asInt, o.data_.asInt, sizeof(data_.asInt)) == 0; }
  friend DSPVectorArrayInt operator+(const DSPVectorArrayInt& a, const DSPVectorArrayInt& b)
  {
    DSPVectorArrayInt y;
    check(mlb_map_host(MLB_OP_ADD_INT32, a.getConstBuffer(), b.getConstBuffer(), nullptr, y.getBuffer(), ROWS));
    return y;
  }
  friend DSPVectorArrayInt operator-(const DSPVectorArrayInt& a, const DSPVectorArrayInt& b)
  {
    DSPVectorArrayInt y;
    check(mlb_map_host(MLB_OP_SUBTRACT_INT32, a.getConstBuffer(), b.getConstBuffer(), nullptr, y.getBuffer(), ROWS));
    return y;
  }
};
using DSPVectorInt = DSPVectorArrayInt<1>;

template <size_t ROWS>
inline void load(DSPVectorArray<ROWS>& dst, const float* src) { std::memcpy(dst.getBuffer(), src, sizeof(float) * kFloatsPerDSPVector * ROWS); }
template <size_t ROWS>
inline void store(const DSPVectorArray<ROWS>& src, float* dst) { std::memcpy(dst, src.getConstBuffer(), sizeof(float) * kFloatsPerDSPVector * ROWS); }
// the aligned forms (MLDSPOps.h:536-562) move the same bytes; alignment only selects the SSE instruction there
template <size_t ROWS>
inline void loadAligned(DSPVectorArray<ROWS>& dst, const float* src) { load(dst, src); }
template <size_t ROWS>
inline void storeAligned(const DSPVectorArray<ROWS>& src, float* dst) { store(src, dst); }

#define MLB_DEFINE_OP1(NAME, OP)                                            \
  template <size_t ROWS>                                                    \
  inline DSPVectorArray<ROWS> NAME(const DSPVectorArray<ROWS>& x)           \
  {                                                                         \
    DSPVectorArray<ROWS> y;                                                 \
    check(mlb_map_host(OP, x.getConstBuffer(), nullptr, nullptr, y.getBuffer(), ROWS)); \
    return y;                                                               \
  }
MLB_DEFINE_OP1(sqrt, MLB_OP_SQRT)
MLB_DEFINE_OP1(abs, MLB_OP_ABS)
MLB_DEFINE_OP1(sign, MLB_OP_SIGN)
MLB_DEFINE_OP1(signBit, MLB_OP_SIGNBIT)
MLB_DEFINE_OP1(sin, MLB_OP_SIN)
MLB_DEFINE_OP1(cos, MLB_OP_COS)
MLB_DEFINE_OP1(log, MLB_OP_LOG)
MLB_DEFINE_OP1(exp, MLB_OP_EXP)
MLB_DEFINE_OP1(log2, MLB_OP_LOG2)
MLB_DEFINE_OP1(exp2, MLB_OP_EXP2)
MLB_DEFINE_OP1(sinApprox, MLB_OP_SIN_APPROX)
MLB_DEFINE_OP1(cosApprox, MLB_OP_COS_APPROX)
MLB_DEFINE_OP1(expApprox, MLB_OP_EXP_APPROX)
MLB_DEFINE_OP1(logApprox, MLB_OP_LOG_APPROX)
MLB_DEFINE_OP1(fractionalPart, MLB_OP_FRACTIONAL_PART)
#undef MLB_DEFINE_OP1

#define MLB_DEFINE_OP2(NAME, OP)                                                              \
  template <size_t ROWS>                                                                      \
  inline DSPVectorArray<ROWS> NAME(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b) \
  {                                                                                           \
    DSPVectorArray<ROWS> y;                                                                   \
    check(mlb_map_host(OP, a.getConstBuffer(), b.getConstBuffer(), nullptr, y.getBuffer(), ROWS)); \
    return y;                                                                                 \
  }
MLB_DEFINE_OP2(add, MLB_OP_ADD)
MLB_DEFINE_OP2(subtract, MLB_OP_SUBTRACT)
MLB_DEFINE_OP2(multiply, MLB_OP_MULTIPLY)
MLB_DEFINE_OP2(divide, MLB_OP_DIVIDE)
MLB_DEFINE_OP2(pow, MLB_OP_POW)
MLB_DEFINE_OP2(min, MLB_OP_MIN)
MLB_DEFINE_OP2(max, MLB_OP_MAX)
#undef MLB_DEFINE_OP2

template <size_t ROWS>
inline DSPVectorArray<ROWS> lerp(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b,
                                 const DSPVectorArray<ROWS>& m)
{
  DSPVectorArray<ROWS> y;
  check(mlb_map_host(MLB_OP_LERP, a.getConstBuffer(), b.getConstBuffer(), m.getConstBuffer(), y.getBuffer(), ROWS));
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> clamp(const DSPVectorArray<ROWS>& x, const DSPVectorArray<ROWS>& lo,
                                  const DSPVectorArray<ROWS>& hi)
{
  DSPVectorArray<ROWS> y;
  check(mlb_map_host(MLB_OP_CLAMP, x.getConstBuffer(), lo.getConstBuffer(), hi.getConstBuffer(), y.getBuffer(), ROWS));
  return y;
}

// the remaining unary / binary / ternary float ops of MLDSPOps.h:584-649,744-748
#define MLB_DEFINE_OP1B(NAME, OP)                                           \
  template <size_t ROWS>                                                    \
  inline DSPVectorArray<ROWS> NAME(const DSPVectorArray<ROWS>& x)           \
  {                                                                         \
    DSPVectorArray<ROWS> y;                                                 \
    check(mlb_map_host(OP, x.getConstBuffer(), nullptr, nullptr, y.getBuffer(), ROWS)); \
    return y;                                                               \
  }
MLB_DEFINE_OP1B(sqrtApprox, MLB_OP_SQRT_APPROX)
MLB_DEFINE_OP1B(log2Approx, MLB_OP_LOG2_APPROX)
MLB_DEFINE_OP1B(exp2Approx, MLB_OP_EXP2_APPROX)
#undef MLB_DEFINE_OP1B
template <size_t ROWS>
inline DSPVectorArray<ROWS> divideApprox(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b)
{
  DSPVectorArray<ROWS> y;
  check(mlb_map_host(MLB_OP_DIVIDE_APPROX, a.getConstBuffer(), b.getConstBuffer(), nullptr, y.getBuffer(), ROWS));
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> powApprox(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b)
{
  DSPVectorArray<ROWS> y;
  check(mlb_map_host(MLB_OP_POW_APPROX, a.getConstBuffer(), b.getConstBuffer(), nullptr, y.getBuffer(), ROWS));
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> inverseLerp(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b,
                                        const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<ROWS> y;
  check(mlb_map_host(MLB_OP_INVERSE_LERP, a.getConstBuffer(), b.getConstBuffer(), x.getConstBuffer(), y.getBuffer(), ROWS));
  return y;
}
template <size_t ROWS>
inline DSPVectorArrayInt<ROWS> within(const DSPVectorArray<ROWS>& x, const DSPVectorArray<ROWS>& lo,
                                      const DSPVectorArray<ROWS>& hi)
{
  DSPVectorArrayInt<ROWS> y;
  check(mlb_map_host(MLB_OP_WITHIN, x.getConstBuffer(), lo.getConstBuffer(), hi.getConstBuffer(), y.getBuffer(), ROWS));
  return y;
}

// ---- row manipulation: pure data movement, done on the host (MLDSPOps.h:1057-1383) ----
template <size_t ROWS, size_t N>
inline DSPVectorArray<ROWS * N> repeatRows(const DSPVectorArray<N>& x)
{
  DSPVectorArray<ROWS * N> y;
  for (size_t j = 0, k = 0; j < ROWS * N; ++j, k = (k + 1 < N ? k + 1 : 0)) y.row((int)j) = x.constRow((int)k);
  return y;
}
template <size_t ROWS, size_t N>
inline DSPVectorArray<ROWS> stretchRows(const DSPVectorArray<N>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j)  // k = roundf(j * (N - 1) / (ROWS - 1)), MLDSPOps.h:1078
    y.row((int)j) = x.constRow(ROWS > 1 ? (int)roundf(((float)j * ((float)N - 1.f)) / ((float)ROWS - 1.f)) : 0);
  return y;
}
template <size_t ROWS, size_t N>
inline DSPVectorArray<ROWS> zeroPadRows(const DSPVectorArray<N>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < (ROWS < N ? ROWS : N); ++j) y.row((int)j) = x.constRow((int)j);
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> shiftRows(const DSPVectorArray<ROWS>& x, int rowsToShift)
{
  DSPVectorArray<ROWS> y;
  for (int j = 0; j < (int)ROWS; ++j)
  {
    const int k = j - rowsToShift;
    if (k >= 0 && k < (int)ROWS) y.row(j) = x.constRow(k);
  }
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> rotateRows(const DSPVectorArray<ROWS>& x, int rowsToRotate)
{
  DSPVectorArray<ROWS> y;
  for (int j = 0; j < (int)ROWS; ++j)
  {
    int k = (j - rowsToRotate) % (int)ROWS;  // row 0 comes from modulo(-rowsToRotate, ROWS), MLDSPOps.h:1132
    if (k < 0) k += (int)ROWS;
    y.row(j) = x.constRow(k);
  }
  return y;
}
template <size_t ROWSA, size_t ROWSB>
inline DSPVectorArray<ROWSA + ROWSB> concatRows(const DSPVectorArray<ROWSA>& a, const DSPVectorArray<ROWSB>& b)
{
  DSPVectorArray<ROWSA + ROWSB> y;
  for (size_t j = 0; j < ROWSA; ++j) y.row((int)j) = a.constRow((int)j);
  for (size_t j = 0; j < ROWSB; ++j) y.row((int)(ROWSA + j)) = b.constRow((int)j);
  return y;
}
template <size_t A, size_t B, size_t C>
inline DSPVectorArray<A + B + C> concatRows(const DSPVectorArray<A>& a, const DSPVectorArray<B>& b, const DSPVectorArray<C>& c)
{
  return concatRows(concatRows(a, b), c);
}
template <size_t A, size_t B, size_t C, size_t D>
inline DSPVectorArray<A + B + C + D> concatRows(const DSPVectorArray<A>& a, const DSPVectorArray<B>& b,
                                                const DSPVectorArray<C>& c, const DSPVectorArray<D>& d)
{
  return concatRows(concatRows(a, b, c), d);
}
// shuffleRows: a0 b0 a1 b1 ... then the rest of the longer argument (MLDSPOps.h:1281-1307)
template <size_t ROWSA, size_t ROWSB>
inline DSPVectorArray<ROWSA + ROWSB> shuffleRows(const DSPVectorArray<ROWSA> a, const DSPVectorArray<ROWSB> b)
{
  DSPVectorArray<ROWSA + ROWSB> y;
  size_t ja = 0, jb = 0, jy = 0;
  while (ja < ROWSA || jb < ROWSB)
  {
    if (ja < ROWSA) y.row((int)jy++) = a.constRow((int)ja++);
    if (jb < ROWSB) y.row((int)jy++) = b.constRow((int)jb++);
  }
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<(ROWS + 1) / 2> evenRows(const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<(ROWS + 1) / 2> y;
  for (size_t j = 0; j < (ROWS + 1) / 2; ++j) y.row((int)j) = x.constRow((int)(j * 2));
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS / 2> oddRows(const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<ROWS / 2> y;
  for (size_t j = 0; j < ROWS / 2; ++j) y.row((int)j) = x.constRow((int)(j * 2 + 1));
  return y;
}
template <size_t A, size_t B, size_t ROWS>
inline DSPVectorArray<B - A> separateRows(const DSPVectorArray<ROWS>& x)
{
  static_assert(B <= ROWS && A < B, "separateRows: row range");
  DSPVectorArray<B - A> y;
  for (size_t j = A; j < B; ++j) y.row((int)(j - A)) = x.constRow((int)j);
  return y;
}
// index generators: exact small integers (MLDSPOps.h:965-966,1365-1388)
template <size_t ROWS = 1>
inline DSPVectorArray<ROWS> columnIndex()
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j)
    for (size_t i = 0; i < kFloatsPerDSPVector; ++i) y[j * kFloatsPerDSPVector + i] = (float)i;
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> rowIndex()
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = DSPVector((float)j);
  return y;
}
inline DSPVectorInt columnIndexInt()
{
  DSPVectorInt y;
  for (size_t i = 0; i < kFloatsPerDSPVector; ++i) y[(int)i] = (int32_t)i;
  return y;
}
// ranges: the scalar interval is host scalar arithmetic as in the reference, the row is built on the GPU
inline DSPVector rangeOpen(float start, float end)  // MLDSPOps.h:970-974
{
  const float interval = (end - start) / (kFloatsPerDSPVector);
  return columnIndex() * DSPVector(interval) + DSPVector(start);
}
inline DSPVector rangeClosed(float start, float end)  // :978-982
{
  const float interval = (end - start) / (kFloatsPerDSPVector - 1.f);
  return columnIndex() * DSPVector(interval) + DSPVector(start);
}
inline DSPVector interpolateDSPVectorLinear(float start, float end)  // :986-990
{
  const float interval = (end - start) / (kFloatsPerDSPVector);
  return columnIndex() * DSPVector(interval) + DSPVector(start + interval);
}
// addRows: rows summed left to right from zero (MLDSPOps.h:1349-1359), every add on the GPU
template <size_t ROWS>
inline DSPVector addRows(const DSPVectorArray<ROWS>& x)
{
  DSPVector vy(0.f);
  for (size_t j = 0; j < ROWS; ++j) vy = add(vy, x.constRow((int)j));
  return vy;
}

// "*1" forms: the second operand is ONE row applied to every row of the first (DEFINE_OP2_MS, MLDSPOps.h:655-687)
#define MLB_DEFINE_OP2_MS(NAME, OP)                                                            \
  template <size_t ROWS>                                                                       \
  inline DSPVectorArray<ROWS> NAME(const DSPVectorArray<ROWS>& a, const DSPVectorArray<1>& b)  \
  {                                                                                            \
    DSPVectorArray<ROWS> y;                                                                    \
    const DSPVectorArray<ROWS> bb = repeatRows<ROWS, 1>(b);                                    \
    check(mlb_map_host(OP, a.getConstBuffer(), bb.getConstBuffer(), nullptr, y.getBuffer(), ROWS)); \
    return y;                                                                                  \
  }
MLB_DEFINE_OP2_MS(add1, MLB_OP_ADD)
MLB_DEFINE_OP2_MS(subtract1, MLB_OP_SUBTRACT)
MLB_DEFINE_OP2_MS(multiply1, MLB_OP_MULTIPLY)
MLB_DEFINE_OP2_MS(divide1, MLB_OP_DIVIDE)
MLB_DEFINE_OP2_MS(divideApprox1, MLB_OP_DIVIDE_APPROX)
MLB_DEFINE_OP2_MS(pow1, MLB_OP_POW)
MLB_DEFINE_OP2_MS(powApprox1, MLB_OP_POW_APPROX)
MLB_DEFINE_OP2_MS(min1, MLB_OP_MIN)
MLB_DEFINE_OP2_MS(max1, MLB_OP_MAX)
#undef MLB_DEFINE_OP2_MS

// int <-> float conversions, comparisons -> masks, select, int add/sub (MLDSPOps.h:692-714,779-917)
#define MLB_DEFINE_F2I(NAME, OP)                                                     \
  template <size_t ROWS>                                                             \
  inline DSPVectorArrayInt<ROWS> NAME(const DSPVectorArray<ROWS>& x)                 \
  {                                                                                  \
    DSPVectorArrayInt<ROWS> y;                                                       \
    check(mlb_map_host(OP, x.getConstBuffer(), nullptr, nullptr, y.getBuffer(), ROWS)); \
    return y;                                                                        \
  }
MLB_DEFINE_F2I(roundFloatToInt, MLB_OP_ROUND_F2I)
MLB_DEFINE_F2I(truncateFloatToInt, MLB_OP_TRUNC_F2I)
#undef MLB_DEFINE_F2I
#define MLB_DEFINE_I2F(NAME, OP)                                                     \
  template <size_t ROWS>                                                             \
  inline DSPVectorArray<ROWS> NAME(const DSPVectorArrayInt<ROWS>& x)                 \
  {                                                                                  \
    DSPVectorArray<ROWS> y;                                                          \
    check(mlb_map_host(OP, x.getConstBuffer(), nullptr, nullptr, y.getBuffer(), ROWS)); \
    return y;                                                                        \
  }
MLB_DEFINE_I2F(intToFloat, MLB_OP_INT_TO_FLOAT)
MLB_DEFINE_I2F(unsignedIntToFloat, MLB_OP_UNSIGNED_TO_FLOAT)
#undef MLB_DEFINE_I2F
#define MLB_DEFINE_FF2I(NAME, OP)                                                                   \
  template <size_t ROWS>                                                                            \
  inline DSPVectorArrayInt<ROWS> NAME(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b) \
  {                                                                                                 \
    DSPVectorArrayInt<ROWS> y;                                                                      \
    check(mlb_map_host(OP, a.getConstBuffer(), b.getConstBuffer(), nullptr, y.getBuffer(), ROWS));  \
    return y;                                                                                       \
  }
MLB_DEFINE_FF2I(equal, MLB_OP_EQUAL)
MLB_DEFINE_FF2I(notEqual, MLB_OP_NOT_EQUAL)
MLB_DEFINE_FF2I(greaterThan, MLB_OP_GREATER_THAN)
MLB_DEFINE_FF2I(greaterThanOrEqual, MLB_OP_GREATER_EQUAL)
MLB_DEFINE_FF2I(lessThan, MLB_OP_LESS_THAN)
MLB_DEFINE_FF2I(lessThanOrEqual, MLB_OP_LESS_EQUAL)
#undef MLB_DEFINE_FF2I
template <size_t ROWS>  // bitwise select(resultIfTrue, resultIfFalse, conditionMask)
inline DSPVectorArray<ROWS> select(const DSPVectorArray<ROWS>& a, const DSPVectorArray<ROWS>& b, const DSPVectorArrayInt<ROWS>& m)
{
  DSPVectorArray<ROWS> y;
  check(mlb_map_host(MLB_OP_SELECT, a.getConstBuffer(), b.getConstBuffer(), m.getConstBuffer(), y.getBuffer(), ROWS));
  return y;
}
template <size_t ROWS>
inline DSPVectorArrayInt<ROWS> select(const DSPVectorArrayInt<ROWS>& a, const DSPVectorArrayInt<ROWS>& b,
                                      const DSPVectorArrayInt<ROWS>& m)
{
  DSPVectorArrayInt<ROWS> y;
  check(mlb_map_host(MLB_OP_SELECT, a.getConstBuffer(), b.getConstBuffer(), m.getConstBuffer(), y.getBuffer(), ROWS));
  return y;
}
template <size_t ROWS>
inline DSPVectorArrayInt<ROWS> addInt32(const DSPVectorArrayInt<ROWS>& a, const DSPVectorArrayInt<ROWS>& b) { return a + b; }
template <size_t ROWS>
inline DSPVectorArrayInt<ROWS> subtractInt32(const DSPVectorArrayInt<ROWS>& a, const DSPVectorArrayInt<ROWS>& b) { return a - b; }

// ---- map: the higher-order helpers of MLDSPFunctional.h:23-100.  The argument is an arbitrary host function,
// so these are plain host loops by nature (element forms) or one call per row (row forms; the row function itself
// may well be made of the GPU-backed operators above). ----
template <size_t ROWS>
inline DSPVectorArray<ROWS> map(std::function<float()> f, const DSPVectorArray<ROWS>& /*shape only*/)
{
  DSPVectorArray<ROWS> y;
  for (size_t n = 0; n < kFloatsPerDSPVector * ROWS; ++n) y[n] = f();
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> map(std::function<float(float)> f, const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t n = 0; n < kFloatsPerDSPVector * ROWS; ++n) y[n] = f(x[n]);
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> map(std::function<float(int)> f, const DSPVectorArrayInt<ROWS>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t n = 0; n < kFloatsPerDSPVector * ROWS; ++n) y[n] = f(x[(int)n]);
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> map(std::function<DSPVector(const DSPVector)> f, const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = f(x.constRow((int)j));
  return y;
}
template <size_t ROWS>
inline DSPVectorArray<ROWS> map(std::function<DSPVector(const DSPVector, int)> f, const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = f(x.constRow((int)j), (int)j);
  return y;
}
// the reference's sixth overload hands the row INDEX to a (DSPVector, DSPVector) function: the index arrives
// broadcast, as DSPVector(float(j)) (MLDSPFunctional.h:90-100)
template <size_t ROWS>
inline DSPVectorArray<ROWS> map(std::function<DSPVector(const DSPVector, const DSPVector)> f, const DSPVectorArray<ROWS>& x)
{
  DSPVectorArray<ROWS> y;
  for (size_t j = 0; j < ROWS; ++j) y.row((int)j) = f(x.constRow((int)j), DSPVector((float)j));
  return y;
}

// ---- Graph: a fixed DAG of functors, built in the reference's functional style ----
class Graph
{
  std::vector<mlb_node> nodes_;
  std::vector<int32_t> outs_;

  int add(int op, int a = -1, int b = -1, int c = -1, int iarg = 0)
  {
    mlb_node n;
    n.op = op;
    for (int k = 0; k < MLB_MAX_INS; ++k) n.in[k] = -1;
    n.in[0] = a, n.in[1] = b, n.in[2] = c;
    n.iarg = iarg;
    nodes_.push_back(n);
    return (int)nodes_.size() - 1;
  }

 public:
  using Sig = int;  // a node's output row
  Sig input(int plane = 0) { return add(MLB_OP_INPUT, -1, -1, -1, plane); }
  Sig param() { return add(MLB_OP_PARAM); }  // per-voice float, broadcast like DSPVector(float)
  Sig noise() { return add(MLB_OP_NOISE); }
  Sig phasor(Sig f) { return add(MLB_OP_PHASOR, f); }
  Sig sine(Sig f) { return add(MLB_OP_SINE, f); }
  Sig saw(Sig f) { return add(MLB_OP_SAW, f); }
  Sig pulse(Sig f, Sig w) { return add(MLB_OP_PULSE, f, w); }
  Sig lopass(Sig x) { return add(MLB_OP_LOPASS, x); }
  Sig hipass(Sig x) { return add(MLB_OP_HIPASS, x); }
  Sig bandpass(Sig x) { return add(MLB_OP_BANDPASS, x); }
  Sig loShelf(Sig x) { return add(MLB_OP_LOSHELF, x); }
  Sig hiShelf(Sig x) { return add(MLB_OP_HISHELF, x); }
  Sig bell(Sig x) { return add(MLB_OP_BELL, x); }
  Sig onePole(Sig x) { return add(MLB_OP_ONEPOLE, x); }
  Sig dcBlocker(Sig x) { return add(MLB_OP_DCBLOCKER, x); }
  Sig fdn8(Sig x) { return add(MLB_OP_FDN8, x); }
  Sig fdn8Right(Sig fdn) { return add(MLB_OP_FDN8_R, fdn); }
  // the rest of the L2 functor set (MLDSPGens.h / MLDSPFilters.h), see MLB_OP_TABLE for state and coefficients
  Sig adsr(Sig gate) { return add(MLB_OP_ADSR, gate); }
  Sig peak(Sig x) { return add(MLB_OP_PEAK, x); }
  Sig rms(Sig x) { return add(MLB_OP_RMS, x); }
  Sig allpass1(Sig x) { return add(MLB_OP_ALLPASS1, x); }
  Sig linearGlide(Sig target) { return add(MLB_OP_GLIDE, target); }
  Sig integerDelay(Sig x) { return add(MLB_OP_INTEGER_DELAY, x); }
  Sig fractionalDelay(Sig x) { return add(MLB_OP_FRACTIONAL_DELAY, x); }
  Sig pitchbendableDelay(Sig x, Sig delayInSamples) { return add(MLB_OP_PITCHBEND_DELAY, x, delayInSamples); }
  Sig allpassPitchbendable(Sig x, Sig delayInSamples) { return add(MLB_OP_ALLPASS_PB, x, delayInSamples); }
  Sig halfBandUp(Sig x) { return add(MLB_OP_HALFBAND_UP, x); }          // upsampleFirstHalf
  Sig halfBandUpSecond(Sig up) { return add(MLB_OP_HALFBAND_UP_2, up); } // upsampleSecondHalf of the same filter
  Sig halfBandDown(Sig x1, Sig x2) { return add(MLB_OP_HALFBAND_DOWN, x1, x2); }
  // a DSPVector member kept between processVector calls: read now, write at the end of the vector
  Sig feedbackRead() { return add(MLB_OP_FEEDBACK_READ); }
  Sig feedbackWrite(Sig reader, Sig x) { return add(MLB_OP_FEEDBACK_WRITE, x, -1, -1, reader); }
  // the functor of node `first` called once more in the same vector, on other inputs (MLB_AGAIN in mlb200.h): it shares
  // that node's state and coefficients -- e.g. the functors of a process function that Upsample2xFunction runs twice
  Sig again(Sig first, Sig a = -1, Sig b = -1, Sig c = -1) { return add(nodes_[(size_t)first].op, a, b, c, MLB_AGAIN(first)); }
  Sig op1(int op, Sig x) { return add(op, x); }
  Sig op2(int op, Sig a, Sig b) { return add(op, a, b); }
  Sig op3(int op, Sig a, Sig b, Sig c) { return add(op, a, b, c); }
  Sig multiply(Sig a, Sig b) { return add(MLB_OP_MULTIPLY, a, b); }
  Sig add2(Sig a, Sig b) { return add(MLB_OP_ADD, a, b); }
  void output(Sig s) { outs_.push_back(s); }

  const std::vector<mlb_node>& nodes() const { return nodes_; }
  const std::vector<int32_t>& outs() const { return outs_; }
};

// ---- DeviceBank: `rows` voices of one graph, resident on the GPU ----
class DeviceBank
{
  mlb_graph* g_ = nullptr;
  int rows_ = 0;
  mlb_layout layout_{};
  std::vector<int32_t> st_off_, co_off_;
  std::vector<float> coef_;
  std::vector<uint32_t> state_;
  int n_out_ = 0;

 public:
  DeviceBank(const Graph& graph, int rows, unsigned flags = MLB_GRAPH_EXACT) : rows_(rows)
  {
    const auto& n = graph.nodes();
    st_off_.resize(n.size());
    co_off_.resize(n.size());
    check(mlb_graph_layout(n.data(), (int)n.size(), &layout_, st_off_.data(), co_off_.data()));
    check(mlb_graph_create(n.data(), (int)n.size(), graph.outs().data(), (int)graph.outs().size(), rows, flags, &g_));
    coef_.assign((size_t)layout_.n_coef_words * rows, 0.f);
    state_.assign((size_t)layout_.n_state_words * rows, 0u);
    n_out_ = (int)graph.outs().size();
  }
  ~DeviceBank() { mlb_graph_destroy(g_); }
  DeviceBank(const DeviceBank&) = delete;
  DeviceBank& operator=(const DeviceBank&) = delete;

  int rows() const { return rows_; }
  const char* kernelName() const { return mlb_graph_kernel_name(g_); }
  mlb_graph* handle() const { return g_; }

  // like assigning `bank[row].coeffs = T::makeCoeffs(...)` in the reference
  void setCoeffs(int node, int row, const float* c, int n)
  {
    for (int k = 0; k < n; ++k) coef_[(size_t)(co_off_[node] + k) * rows_ + row] = c[k];
  }
  void setParam(int node, int row, float v) { setCoeffs(node, row, &v, 1); }
  void setStateWord(int node, int slot, int row, uint32_t w) { state_[(size_t)(st_off_[node] + slot) * rows_ + row] = w; }
  void commit()  // upload coefficients and state
  {
    check(mlb_graph_set_coefs(g_, coef_.data()));
    check(mlb_graph_set_state(g_, state_.data()));
  }
  void readState()
  {
    check(mlb_graph_get_state(g_, state_.data()));
  }
  uint32_t stateWord(int node, int slot, int row) const { return state_[(size_t)(st_off_[node] + slot) * rows_ + row]; }
  void clear() { check(mlb_graph_clear_delays(g_)); }

  // n_blocks successive Bank::operator() calls: in [T][n_in][rows][64], out [T][n_out][rows][64]
  void process(const float* in, float* out, float* mix, int n_blocks) { check(mlb_graph_process_host(g_, in, out, mix, n_blocks)); }

  // one block, reference-shaped: DSPVectorArray<ROWS> in -> DSPVectorArray<ROWS> out
  template <size_t ROWS>
  DSPVectorArray<ROWS> operator()(const DSPVectorArray<ROWS>& x)
  {
    if ((int)ROWS != rows_ || n_out_ != 1) throw Error(MLB_ERR_INVALID, "DeviceBank: shape mismatch");
    DSPVectorArray<ROWS> y;
    process(x.getConstBuffer(), y.getBuffer(), nullptr, 1);
    return y;
  }
};

// ---- VoiceBank: EventsToSignals::Voice x V on the GPU (mlb_voices_*; routing: mlb200_events.hpp) ----
class VoiceBank
{
  mlb_voices* vb_ = nullptr;
  int n_ = 0;

 public:
  VoiceBank(int nVoices, float sampleRate, const int32_t* voiceIndex, const float* pitchGlideSeconds,
            const float* driftAmount, const float* pitchBendSemitones, unsigned flags = 0)
      : n_(nVoices)
  {
    check(mlb_voices_create(nVoices, sampleRate, voiceIndex, pitchGlideSeconds, driftAmount, pitchBendSemitones, flags, &vb_));
  }
  ~VoiceBank() { mlb_voices_destroy(vb_); }
  VoiceBank(const VoiceBank&) = delete;
  VoiceBank& operator=(const VoiceBank&) = delete;
  int voices() const { return n_; }
  mlb_voices* handle() const { return vb_; }
  void setMainVoices(const int32_t* mainVoice) { check(mlb_voices_set_main_voices(vb_, mainVoice)); }
  // events [nBlocks][voices]; out [nBlocks][MLB_VOICE_ROWS][voices][64]
  void process(const mlb_voice_events* events, float* out, int nBlocks, unsigned rowMask = 0xFFu)
  {
    check(mlb_voices_process_host(vb_, events, out, nBlocks, rowMask));
  }
};

// Events -> signals -> voice DSP in one call (mlb_synth_process_host): what EventsToSignals::processVector
// followed by Synth::processVector does per vector (MLEventsToSignals.cpp:383-470, MLSynth.h:36-60), for
// nBlocks vectors of the whole bank.  The graph's input(r) is Voice row r (kPitch = 0, kGate = 1, ...);
// events [nBlocks][rows]; out [nBlocks][n_out][rows][64] or null; mix [nBlocks][n_out][64] or null.
inline void processEvents(VoiceBank& voices, DeviceBank& bank, const mlb_voice_events* events, float* out, float* mix,
                          int nBlocks)
{
  check(mlb_synth_process_host(voices.handle(), bank.handle(), events, out, mix, nBlocks));
}

// ---- Buses: per-instrument output buses over a voice bank on the GPU (mlb_buses_*) ----
// What one Synth::processVector (MLSynth.h:36-60) does per instrument: bus g = the strict left-to-right sum of the
// voice rows [first[g], first[g] + count[g]), starting from +0.
class Buses
{
  mlb_buses* b_ = nullptr;
  int voices_ = 0, n_ = 0;

 public:
  Buses(int nVoices, int nBuses, const int32_t* firstVoice, const int32_t* voiceCount)
      : voices_(nVoices), n_(nBuses)
  {
    check(mlb_buses_create(nVoices, nBuses, firstVoice, voiceCount, &b_));
  }
  ~Buses() { mlb_buses_destroy(b_); }
  Buses(const Buses&) = delete;
  Buses& operator=(const Buses&) = delete;
  int voices() const { return voices_; }
  int buses() const { return n_; }
  mlb_buses* handle() const { return b_; }
  // device buffers, asynchronous on `stream`: rows [nBlocks][nPlanes][voices][64] -> bus [nBlocks][nPlanes][buses][64]
  void sumDevice(const float* rows, float* bus, int nPlanes, int nBlocks, void* stream = nullptr)
  {
    check(mlb_buses_sum_device(b_, rows, bus, nPlanes, nBlocks, stream));
  }
};

// processEvents with per-instrument output (mlb_synth_process_buses_host): events [nBlocks][voices] in,
// bus [nBlocks][n_out][buses][64] out; the voice rows stay on the device.
inline void processEventsToBuses(VoiceBank& voices, DeviceBank& bank, Buses& buses, const mlb_voice_events* events,
                                 float* bus, int nBlocks)
{
  check(mlb_synth_process_buses_host(voices.handle(), bank.handle(), buses.handle(), events, bus, nBlocks));
}

// ---- ControllerBank: the smoothed MIDI controllers of G instruments (mlb_controllers_*), what
// AudioContext::getInputController(n) returns, for the requested controller numbers only ----
class ControllerBank
{
  mlb_controllers* c_ = nullptr;
  int instruments_ = 0, controllers_ = 0;

 public:
  // protocol 0 MIDI, 1 MPE; controllers: numbers 0..128, no repeats
  ControllerBank(int nInstruments, float sampleRate, int protocol, const int32_t* controllers, int nControllers)
      : instruments_(nInstruments), controllers_(nControllers)
  {
    check(mlb_controllers_create(nInstruments, sampleRate, protocol, controllers, nControllers, &c_));
  }
  ~ControllerBank() { mlb_controllers_destroy(c_); }
  ControllerBank(const ControllerBank&) = delete;
  ControllerBank& operator=(const ControllerBank&) = delete;
  int instruments() const { return instruments_; }
  int controllers() const { return controllers_; }
  mlb_controllers* handle() const { return c_; }
  void clear() { check(mlb_controllers_clear(c_)); }
  // voiceInstrument[nVoices]: each voice's instrument or -1; nullptr goes back to instrument rows
  void setVoiceMap(const int32_t* voiceInstrument, int nVoices) { check(mlb_controllers_set_voice_map(c_, voiceInstrument, nVoices)); }
  // device buffers, asynchronous on `stream`: offsets [nBlocks][instruments + 1] into changes ->
  // out [nBlocks][nPlanes][instruments or voices][64], controller k in plane plane0 + k
  void processDevice(const int32_t* offsets, const mlb_controller_change* changes, float* out, int plane0, int nPlanes,
                     int nBlocks, void* stream = nullptr)
  {
    check(mlb_controllers_process_device(c_, offsets, changes, out, plane0, nPlanes, nBlocks, stream));
  }
};

// processEvents with controller planes (mlb_synth_process_controllers_host): the graph's INPUT planes are the 8 Voice
// rows, then the controllers' rows in list order; records and change lists in, the graph's rows / mix out.
inline void processEventsWithControllers(VoiceBank& voices, ControllerBank& controllers, DeviceBank& bank,
                                         const mlb_voice_events* events, const int32_t* offsets,
                                         const mlb_controller_change* changes, float* out, float* mix, int nBlocks)
{
  check(mlb_synth_process_controllers_host(voices.handle(), controllers.handle(), bank.handle(), events, offsets,
                                           changes, out, mix, nBlocks));
}

// ---- Resampler: Upsampler(octaves) / Downsampler(octaves) x V on the GPU (mlb_resampler_*) ----
class Resampler
{
  mlb_resampler* r_ = nullptr;

 public:
  Resampler(int direction, int octaves, int nVoices) { check(mlb_resampler_create(direction, octaves, nVoices, &r_)); }
  ~Resampler() { mlb_resampler_destroy(r_); }
  Resampler(const Resampler&) = delete;
  Resampler& operator=(const Resampler&) = delete;
  void clear() { check(mlb_resampler_clear(r_)); }
  // in [nBlocksIn][voices][64] -> out; returns the number of output blocks
  int process(const float* in, float* out, int nBlocksIn)
  {
    int n = 0;
    check(mlb_resampler_process_host(r_, in, out, nBlocksIn, &n));
    return n;
  }
};

// ---- FDTDBank: V x the FDTD membrane of examples/audio-and-midi/fdtd.cpp on the GPU (mlb_fdtd_*) ----
// What FDTDState + processFDTDModel(input, freq, &state) is per instance.
class FDTDBank
{
  mlb_fdtd* f_ = nullptr;
  int n_ = 0, planes_ = 0;

 public:
  FDTDBank(int nInstances, float sampleRate = 48000.f, int inPlanes = 2, int excitePlane = 0, int freqPlane = 1,
           unsigned flags = 0)
      : n_(nInstances), planes_(inPlanes)
  {
    check(mlb_fdtd_create(nInstances, sampleRate, inPlanes, excitePlane, freqPlane, flags, &f_));
  }
  ~FDTDBank() { mlb_fdtd_destroy(f_); }
  FDTDBank(const FDTDBank&) = delete;
  FDTDBank& operator=(const FDTDBank&) = delete;
  int instances() const { return n_; }
  int inputPlanes() const { return planes_; }
  mlb_fdtd* handle() const { return f_; }
  void clear() { check(mlb_fdtd_clear(f_)); }
  // [instances][2][16][16]: z^-1 surface, then z^-2
  void getState(float* host) { check(mlb_fdtd_get_state(f_, host)); }
  void setState(const float* host) { check(mlb_fdtd_set_state(f_, host)); }
  // host buffers: in [nBlocks][inPlanes][instances][64] -> out [nBlocks][2][instances][64]
  void process(const float* in, float* out, int nBlocks) { check(mlb_fdtd_process_host(f_, in, out, nBlocks)); }
  // device buffers, asynchronous on `stream` (a cudaStream_t)
  void processDevice(const float* in, float* out, int nBlocks, void* stream = nullptr)
  {
    check(mlb_fdtd_process_device(f_, in, out, nBlocks, stream));
  }
};

}  // namespace mlb
