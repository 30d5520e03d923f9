// cell.cuh — scalar <value, valid> cells and the AQL functor set with SQL 3-valued logic.
//
// Semantics restated from the reference (not its code): every operand is a <value, valid>
// pair; comparison / arithmetic / bitwise functors yield (0, false) when any operand is
// NULL; OR lets TRUE dominate NULL; IsNull/IsNotNull are always valid; Noop passes the raw
// stored value AND validity through unchanged (reference query/functor.hpp:30-380,
// dispatch :663-698 and :924-970, float specialisation :1037-1076).  The C++ implicit
// tuple conversions the reference relies on are made explicit here as `cvt`:
//   operands  I -> T   where T = common_type(I1, I2)   (query/utils.hpp:83-94)
//   result    R -> O   where O = element type of the sink (scratch / dimension / measure)
#pragma once
#include <stdint.h>

#include "aresdb_b200/aql_abi.h"
#include "murmur.cuh"

namespace aresb {

// Value classes of a 32-bit cell (what the reference's iterators yield: bool, int32_t,
// uint32_t, float — query/binder.hpp:209-264) plus the two wide root-only classes.
enum ValClass : uint8_t { VC_BOOL = 0, VC_I32 = 1, VC_U32 = 2, VC_F32 = 3, VC_I64 = 4, VC_F64 = 5,
                          VC_I8 = 6, VC_U8 = 7, VC_I16 = 8, VC_U16 = 9, VC_UUID = 10, VC_NONE = 255 };

struct Cell {
  uint64_t v;   // raw bits of the value in its class (32-bit classes use the low word)
  bool valid;
};

ARES_HD float asF32(uint64_t v) {
#ifdef __CUDA_ARCH__
  return __uint_as_float((uint32_t)v);
#else
  union { uint32_t u; float f; } x; x.u = (uint32_t)v; return x.f;
#endif
}
ARES_HD uint64_t fromF32(float f) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(f);
#else
  union { uint32_t u; float f; } x; x.f = f; return x.u;
#endif
}
ARES_HD double asF64(uint64_t v) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)v);
#else
  union { uint64_t u; double f; } x; x.u = v; return x.f;
#endif
}
ARES_HD uint64_t fromF64(double f) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(f);
#else
  union { uint64_t u; double f; } x; x.f = f; return x.u;
#endif
}

// C++ implicit conversion `static_cast<To>(From value)` on raw bits.
ARES_HD uint64_t cvt(uint64_t v, ValClass from, ValClass to) {
  if (from == to) return v;
  // Bring the source to one of: signed 64 (s), unsigned 64 (u) or double (d).
  bool isF = false, isS = false;
  int64_t s = 0; uint64_t u = 0; double d = 0;
  switch (from) {
    case VC_BOOL: u = (v & 0xff) ? 1 : 0; break;
    case VC_I32: s = (int32_t)(uint32_t)v; isS = true; break;
    case VC_U32: u = (uint32_t)v; break;
    case VC_F32: d = asF32(v); isF = true; break;
    case VC_I64: s = (int64_t)v; isS = true; break;
    case VC_F64: d = asF64(v); isF = true; break;
    case VC_I8: s = (int8_t)(uint8_t)v; isS = true; break;
    case VC_U8: u = (uint8_t)v; break;
    case VC_I16: s = (int16_t)(uint16_t)v; isS = true; break;
    case VC_U16: u = (uint16_t)v; break;
    default: u = v; break;
  }
  switch (to) {
    case VC_BOOL: return isF ? (d != 0.0) : (isS ? (s != 0) : (u != 0));
    case VC_F32: return fromF32(isF ? (float)d : (isS ? (float)s : (float)u));
    case VC_F64: return fromF64(isF ? d : (isS ? (double)s : (double)u));
    case VC_I64: return isF ? (uint64_t)(int64_t)d : (isS ? (uint64_t)s : u);
    case VC_I32: return (uint32_t)(isF ? (int32_t)d : (isS ? (int32_t)s : (int32_t)u));
    case VC_U32: return (uint32_t)(isF ? (uint32_t)d : (isS ? (uint32_t)s : (uint32_t)u));
    // narrow integer sinks: float goes through int32 first (x86 cvttss2si then truncate)
    case VC_I8: case VC_U8: return (uint8_t)(isF ? (int32_t)d : (isS ? (int32_t)s : (int32_t)u));
    case VC_I16: case VC_U16: return (uint16_t)(isF ? (int32_t)d : (isS ? (int32_t)s : (int32_t)u));
    default: return v;
  }
}

// common_type of two 32-bit operand classes (reference query/utils.hpp:83-94): float if
// either is float, else int32 if either is signed, else uint32 (bool counts as unsigned).
ARES_HD ValClass commonClass(ValClass a, ValClass b) {
  if (a == VC_F32 || b == VC_F32) return VC_F32;
  if (a == VC_I64 || b == VC_I64) return VC_I64;
  if (a == VC_I32 || b == VC_I32) return VC_I32;
  return VC_U32;
}

// ---- calendar math (reference query/functor.cu:67-161, itself a restatement of Go's
// time.absDate; proleptic Gregorian, seconds since the Unix epoch, ts >= 0) -------------
enum TimeBucket : uint8_t { TB_YEAR, TB_QUARTER, TB_MONTH, TB_DAY_OF_MONTH, TB_DAY_OF_YEAR,
                            TB_MONTH_OF_YEAR, TB_QUARTER_OF_YEAR };

ARES_HD uint32_t daysBeforeMonth(int month, bool leap) {
  // cumulative days before month index (0 = January); table folded into arithmetic-free
  // constants so that no __constant__ upload is needed (BootstrapDevice becomes a no-op).
  const uint16_t t[13] = {0, 31, 59, 90, 120, 151, 181, 212, 243, 273, 304, 334, 365};
  uint32_t d = t[month];
  if (leap && month >= 2) d++;
  return d;
}

ARES_HD uint32_t resolveTimeBucket(int64_t ts, TimeBucket tb) {
  const int64_t kAbsZero = -62135596800LL;  // 0001-01-01T00:00:00Z
  const int kDay = 86400, k400 = 146097, k100 = 36524, k4 = 1461;
  ts -= kAbsZero;
  uint32_t days = (uint32_t)(ts / kDay);
  int64_t n = days / k400;
  uint16_t year = (uint16_t)(400 * n);
  int64_t start = n * k400 * (int64_t)kDay;
  days -= (uint32_t)(k400 * n);
  n = days / k100; n -= n >> 2;
  year += (uint16_t)(100 * n); start += n * k100 * (int64_t)kDay; days -= (uint32_t)(k100 * n);
  n = days / k4;
  year += (uint16_t)(4 * n); start += n * k4 * (int64_t)kDay; days -= (uint32_t)(k4 * n);
  n = days / 365; n -= n >> 2;
  year += (uint16_t)n; days -= (uint32_t)(365 * n); start += n * 365 * (int64_t)kDay;
  start += kAbsZero;
  if (tb == TB_YEAR) return (uint32_t)start;
  if (tb == TB_DAY_OF_YEAR) return days;
  uint16_t y1 = (uint16_t)(year + 1);
  bool leap = (y1 % 4 == 0) && (y1 % 100 != 0 || y1 % 400 == 0);
  uint8_t month = (uint8_t)(days / 31);
  if (days >= daysBeforeMonth(month + 1, leap)) month++;
  if (tb == TB_MONTH || tb == TB_DAY_OF_MONTH) {
    uint32_t dbm = daysBeforeMonth(month, leap);
    if (tb == TB_MONTH) return (uint32_t)(start + (int64_t)dbm * kDay);
    return days - dbm;
  }
  if (tb == TB_MONTH_OF_YEAR) return month;
  int quarter = month / 3;
  if (tb == TB_QUARTER_OF_YEAR) return (uint32_t)quarter;
  return (uint32_t)(start + (int64_t)daysBeforeMonth(quarter * 3, leap) * kDay);
}

// Monday 00:00 UTC of the week containing ts (reference query/functor.cu:207-212).
ARES_HD uint32_t weekStart(uint32_t ts) {
  const uint32_t fourDays = 4u * 86400u, week = 7u * 86400u;
  if (ts < fourDays) return 0;
  return ts - (ts - fourDays) % week;
}

// HLL register value of a 64-bit hash: reg = low 14 bits, rho = number of consecutive zero
// bits starting at bit 14; value = rho << 16 | reg (reference query/functor.hpp:445-466).
// The reference computes the probe mask as the *int* expression 1 << (rho + 14): for
// rho + 14 >= 32 a CUDA device shift yields 0 (so the scan runs to rho = 50), whereas the
// x86 HOST build wraps the shift count mod 32 and re-tests low bits.  We reproduce the
// DEVICE behaviour (the north star); `hostShift` selects the x86 variant so the oracle
// restatement can be validated against the reference's HOST build.
ARES_HD uint32_t hllValueOfHash(uint64_t hashed, bool hostShift = false) {
  uint32_t group = (uint32_t)(hashed & 0x3FFF);
#ifdef __CUDA_ARCH__
  if (!hostShift) {
    // CUDA semantics of the reference's int shift, closed form of the loop below: the lowest set bit among bits 14..31
    // decides; none set: the loop runs to bit 64 (rho = 50)
    // (branch-free: clz(brev(x)) is 32 for x == 0, and 32 + 18 = 50)
    const uint32_t x = (uint32_t)(hashed >> 14) & 0x3FFFFu;
    const uint32_t c = (uint32_t)__clz((int)__brev(x));
    const uint32_t r = c + (c >> 5) * 18u;
    return (r << 16) | group;
  }
#endif
  uint32_t rho = 0;
  while (true) {
    uint32_t sh = rho + 14;
    uint32_t bit;
    if (sh < 31) bit = (uint32_t)(hashed & (1u << sh));
    else if (sh == 31) bit = (uint32_t)(hashed & 0xFFFFFFFF80000000ULL);  // sign-extended int
    else bit = hostShift ? (uint32_t)(hashed & (uint64_t)(int64_t)(int32_t)(1u << (sh & 31))) : 0u;
    if (sh < 64 && bit == 0) rho++; else break;
  }
  return (rho << 16) | group;
}

ARES_HD uint64_t hllHash32(uint32_t value, int bytes) {
  uint64_t w[4] = {value, 0, 0, 0};
  return murmur3_128_lo(w, bytes, 0);
}

// ---- unary functors -------------------------------------------------------------------
// `ic` is the operand class I; the result class (before conversion to the sink) is
// returned through *rc.  Mirrors UnaryFunctor<O, I>::operator() including its "unknown
// functor behaves like Noop" default and the reduced float specialisation.
ARES_HD Cell evalUnary(int fn, Cell a, ValClass ic, ValClass *rc) {
  Cell r; r.v = 0; r.valid = false;
  const bool isFloat = (ic == VC_F32);
  switch (fn) {
    case Not:
      *rc = VC_BOOL;
      if (!a.valid) return r;
      r.v = cvt(a.v, ic, VC_BOOL) ? 0 : 1; r.valid = true; return r;
    case IsNull: *rc = VC_BOOL; r.v = a.valid ? 0 : 1; r.valid = true; return r;
    case IsNotNull: *rc = VC_BOOL; r.v = a.valid ? 1 : 0; r.valid = true; return r;
    case Negate:
      *rc = ic;
      if (!a.valid) return r;
      r.valid = true;
      if (isFloat) r.v = fromF32(-asF32(a.v));
      else if (ic == VC_BOOL) r.v = (a.v & 0xff) ? 1 : 0;          // -(true) = -1 -> true
      else r.v = (uint32_t)(0u - (uint32_t)a.v);
      return r;
    case BitwiseNot:
      if (isFloat) break;  // float specialisation: falls to Noop
      *rc = ic;
      if (!a.valid) return r;
      r.valid = true;
      if (ic == VC_BOOL) r.v = 1;                                   // ~0 = -1, ~1 = -2: both true
      else r.v = (uint32_t)~(uint32_t)a.v;
      return r;
    case GetWeekStart: case GetMonthStart: case GetQuarterStart: case GetYearStart:
    case GetDayOfMonth: case GetDayOfYear: case GetMonthOfYear: case GetQuarterOfYear: {
      if (isFloat) break;
      *rc = VC_U32;
      if (!a.valid) return r;
      uint32_t ts = (uint32_t)cvt(a.v, ic, VC_U32);
      r.valid = true;
      switch (fn) {
        case GetWeekStart: r.v = weekStart(ts); break;
        case GetMonthStart: r.v = resolveTimeBucket(ts, TB_MONTH); break;
        case GetQuarterStart: r.v = resolveTimeBucket(ts, TB_QUARTER); break;
        case GetYearStart: r.v = resolveTimeBucket(ts, TB_YEAR); break;
        case GetDayOfMonth: r.v = resolveTimeBucket(ts, TB_DAY_OF_MONTH); break;
        case GetDayOfYear: r.v = resolveTimeBucket(ts, TB_DAY_OF_YEAR); break;
        case GetMonthOfYear: r.v = resolveTimeBucket(ts, TB_MONTH_OF_YEAR); break;
        default: r.v = resolveTimeBucket(ts, TB_QUARTER_OF_YEAR); break;
      }
      return r;
    }
    case GetHLLValue: {
      if (isFloat) break;
      *rc = VC_U32;
      if (!a.valid) return r;
      r.valid = true;
      // hashes sizeof(I) bytes of the value: 1 for bool, 4 for (u)int32
      uint64_t h = (ic == VC_BOOL) ? hllHash32((uint32_t)((a.v & 0xff) ? 1 : 0), 1)
                                   : hllHash32((uint32_t)a.v, 4);
      r.v = hllValueOfHash(h);
      return r;
    }
    default: break;
  }
  // Noop and every functor the class does not implement: identity on <value, valid>.
  *rc = ic;
  return a;
}

// ---- binary functors ------------------------------------------------------------------
// Float32 Plus / Minus / Multiply / Divide, each rounded once to nearest-even: what the reference's per-node calls (every
// functor writes a float vector) and x86 compute.  On the device the _rn intrinsics keep the compiler from contracting
// `a * b` and a following `+ c` / `- c` of the same row into one FFMA (NVRTC compiles with --fmad=true).
ARES_HD float f32Arith(int fn, float x, float y) {
#ifdef __CUDA_ARCH__
  return fn == Plus ? __fadd_rn(x, y) : fn == Minus ? __fsub_rn(x, y) : fn == Multiply ? __fmul_rn(x, y) : __fdiv_rn(x, y);
#else
  return fn == Plus ? x + y : fn == Minus ? x - y : fn == Multiply ? x * y : x / y;
#endif
}

// Both operands are already converted to the common class `tc` (VC_I32, VC_U32 or VC_F32).
ARES_HD Cell evalBinary(int fn, Cell a, Cell b, ValClass tc, ValClass *rc) {
  Cell r; r.v = 0; r.valid = false;
  const bool isFloat = (tc == VC_F32);
  if (fn == And) {
    *rc = VC_BOOL;
    if (!a.valid || !b.valid) return r;
    r.valid = true; r.v = (cvt(a.v, tc, VC_BOOL) && cvt(b.v, tc, VC_BOOL)) ? 1 : 0; return r;
  }
  if (fn == Or) {
    *rc = VC_BOOL;
    bool av = cvt(a.v, tc, VC_BOOL) != 0, bv = cvt(b.v, tc, VC_BOOL) != 0;
    if ((av && a.valid) || (bv && b.valid)) { r.v = 1; r.valid = true; return r; }
    if (!a.valid || !b.valid) return r;
    r.valid = true; return r;
  }
  if (fn >= Equal && fn <= GreaterThanOrEqual) {
    *rc = VC_BOOL;
    if (!a.valid || !b.valid) return r;
    r.valid = true;
    bool res;
    if (isFloat) {
      float x = asF32(a.v), y = asF32(b.v);
      res = fn == Equal ? x == y : fn == NotEqual ? x != y : fn == LessThan ? x < y
          : fn == LessThanOrEqual ? x <= y : fn == GreaterThan ? x > y : x >= y;
    } else if (tc == VC_I32) {
      int32_t x = (int32_t)(uint32_t)a.v, y = (int32_t)(uint32_t)b.v;
      res = fn == Equal ? x == y : fn == NotEqual ? x != y : fn == LessThan ? x < y
          : fn == LessThanOrEqual ? x <= y : fn == GreaterThan ? x > y : x >= y;
    } else {
      uint32_t x = (uint32_t)a.v, y = (uint32_t)b.v;
      res = fn == Equal ? x == y : fn == NotEqual ? x != y : fn == LessThan ? x < y
          : fn == LessThanOrEqual ? x <= y : fn == GreaterThan ? x > y : x >= y;
    }
    r.v = res ? 1 : 0;
    return r;
  }
  const bool arithmetic = (fn >= Plus && fn <= Divide);
  const bool intOnly = (fn == Mod || (fn >= BitwiseAnd && fn <= Floor));
  if (arithmetic || (intOnly && !isFloat)) {
    *rc = tc;
    if (!a.valid || !b.valid) return r;
    r.valid = true;
    if (isFloat) {
      r.v = fromF32(f32Arith(fn, asF32(a.v), asF32(b.v)));
    } else if (tc == VC_I32) {
      int32_t x = (int32_t)(uint32_t)a.v, y = (int32_t)(uint32_t)b.v; uint32_t z;
      switch (fn) {
        case Plus: z = (uint32_t)x + (uint32_t)y; break;
        case Minus: z = (uint32_t)x - (uint32_t)y; break;
        case Multiply: z = (uint32_t)x * (uint32_t)y; break;
        case Divide: z = y == 0 ? 0xFFFFFFFFu : (y == -1 ? (uint32_t)0 - (uint32_t)x : (uint32_t)(x / y)); break;
        case Mod: z = (y == 0 || y == -1) ? (y == 0 ? (uint32_t)x : 0u) : (uint32_t)(x % y); break;
        case BitwiseAnd: z = (uint32_t)x & (uint32_t)y; break;
        case BitwiseOr: z = (uint32_t)x | (uint32_t)y; break;
        case BitwiseXor: z = (uint32_t)x ^ (uint32_t)y; break;
        default: /* Floor: a - a % b */
          z = (y == 0 || y == -1) ? (y == 0 ? 0u : (uint32_t)x) : (uint32_t)(x - x % y); break;
      }
      r.v = z;
    } else {
      uint32_t x = (uint32_t)a.v, y = (uint32_t)b.v, z;
      switch (fn) {
        case Plus: z = x + y; break;
        case Minus: z = x - y; break;
        case Multiply: z = x * y; break;
        case Divide: z = y == 0 ? 0xFFFFFFFFu : x / y; break;
        case Mod: z = y == 0 ? x : x % y; break;
        case BitwiseAnd: z = x & y; break;
        case BitwiseOr: z = x | y; break;
        case BitwiseXor: z = x ^ y; break;
        default: z = y == 0 ? 0u : x - x % y; break;
      }
      r.v = z;
    }
    return r;
  }
  // anything else (incl. Mod/bitwise/Floor on floats): "return t1"
  *rc = tc;
  return a;
}

// SUM measures of an RLE batch count `count` times: value * count in the sink's arithmetic
// (reference query/iterator.hpp:626-645, 704-709).  The float products are rounded on their own: never contracted with
// the accumulation that follows.
ARES_HD uint64_t mulCount(uint64_t v, ValClass oc, uint32_t count) {
  switch (oc) {
    case VC_I32: case VC_U32: return (uint32_t)((uint32_t)v * count);
    case VC_F32: return fromF32(f32Arith(Multiply, asF32(v), (float)count));
    case VC_I64: return (uint64_t)((int64_t)v * (int64_t)(uint64_t)count);
#ifdef __CUDA_ARCH__
    default: return fromF64(__dmul_rn(asF64(v), (double)count));
#else
    default: return fromF64(asF64(v) * (double)count);
#endif
  }
}

// Identity element of an aggregate in the sink's value class
// (reference query/utils.hpp:169-184: note MAX_FLOAT uses FLT_MIN, the smallest positive
// normal, not -FLT_MAX; reproduced as is).
ARES_HD uint64_t aggIdentity(int aggFunc, ValClass oc) {
  double d = 0; int64_t s = 0; bool isS = false, isD = false; uint64_t u = 0;
  switch (aggFunc) {
    case AGGR_MIN_UNSIGNED: u = 0xFFFFFFFFull; break;
    case AGGR_MIN_SIGNED: s = 2147483647; isS = true; break;
    case AGGR_MIN_FLOAT: d = 3.402823466e+38; isD = true; break;   // FLT_MAX
    case AGGR_MAX_SIGNED: s = -2147483647 - 1; isS = true; break;
    case AGGR_MAX_FLOAT: d = 1.175494351e-38; isD = true; break;   // FLT_MIN
    default: break;
  }
  // static_cast<Value>(constant)
  if (isD) {
    float f = (float)d;
    return cvt(fromF32(f), VC_F32, oc);
  }
  if (isS) return cvt((uint64_t)s, VC_I64, oc);
  return cvt(u, VC_I64, oc);
}

}  // namespace aresb
