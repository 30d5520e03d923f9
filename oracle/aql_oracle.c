/*
 * aql_oracle.c — TEST INFRASTRUCTURE.  A plain-C, single-threaded restatement of the
 * reference's AQL batch-execution hot path, exporting the reference's own C entry points
 * (same names, same by-value structs) so that the parity tests can drive it, the reference's
 * HOST build (oracle/_ref) and the B200 engine through one set of bindings.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library.  The product (aresdb_b200/) never does.
 *
 * Parity is PINNED: tests/test_golden_vectors.py checks this file against every known-answer
 * vector of the reference's native unit tests for the path, and tests/test_node_parity.py, tests/test_pipeline_parity.py
 * checks it against the reference's own HOST build on seeded random inputs.
 *
 * Each function cites the reference code whose behaviour it restates (paths relative to the
 * reference repository root).  "Memory" is host memory; `cudaStream` / `device` are ignored.
 */
#include <math.h>
#include <stdbool.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "aresdb_b200/aql_abi.h"

/* 0: x86 HOST semantics of the reference build (validated against oracle/_ref);
 * 1: CUDA DEVICE semantics where the two differ (only the shift in GetHLLValue does).
 * The north star is the DEVICE path, so GPU parity tests run the oracle in mode 1. */
static int g_device_semantics = 0;
void OracleSetDeviceSemantics(int on) { g_device_semantics = on; }

static CGoCallResHandle ok(int64_t res) {
  CGoCallResHandle h = {(void *)(intptr_t)res, NULL};
  return h;
}
static CGoCallResHandle fail(const char *msg) {
  CGoCallResHandle h = {NULL, strdup(msg)};
  return h;
}

/* ------------------------------------------------------------------------------------------
 * MurmurHash3 — query/utils.cu:113-155 (x86_32) and :157-241 (x64_128), canonical byte-wise form
 * ---------------------------------------------------------------------------------------- */
static uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t fmix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
}

uint32_t oracle_murmur3_32(const uint8_t *key, int bytes, uint32_t seed) {
  uint32_t h1 = seed;
  int nblocks = bytes / 4;
  for (int i = 0; i < nblocks; i++) {
    uint32_t k1;
    memcpy(&k1, key + 4 * i, 4);
    k1 *= 0xcc9e2d51u; k1 = (k1 << 15) | (k1 >> 17); k1 *= 0x1b873593u;
    h1 ^= k1; h1 = (h1 << 13) | (h1 >> 19); h1 = h1 * 5 + 0xe6546b64u;
  }
  const uint8_t *tail = key + 4 * nblocks;
  uint32_t k1 = 0;
  switch (bytes & 3) {
    case 3: k1 ^= (uint32_t)tail[2] << 16; /* fallthrough */
    case 2: k1 ^= (uint32_t)tail[1] << 8;  /* fallthrough */
    case 1: k1 ^= (uint32_t)tail[0];
      k1 *= 0xcc9e2d51u; k1 = (k1 << 15) | (k1 >> 17); k1 *= 0x1b873593u; h1 ^= k1;
  }
  h1 ^= (uint32_t)bytes;
  h1 ^= h1 >> 16; h1 *= 0x85ebca6bu; h1 ^= h1 >> 13; h1 *= 0xc2b2ae35u; h1 ^= h1 >> 16;
  return h1;
}

void oracle_murmur3_128(const uint8_t *key, int len, uint32_t seed, uint64_t out[2]) {
  const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
  uint64_t h1 = seed, h2 = seed;
  int nblocks = len / 16;
  for (int i = 0; i < nblocks; i++) {
    uint64_t k1, k2;
    memcpy(&k1, key + 16 * i, 8);
    memcpy(&k2, key + 16 * i + 8, 8);
    k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
    h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
    k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
    h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
  }
  const uint8_t *tail = key + 16 * nblocks;
  uint64_t k1 = 0, k2 = 0;
  int t = len & 15;
  for (int i = t - 1; i >= 8; i--) k2 ^= (uint64_t)tail[i] << (8 * (i - 8));
  if (t > 8) { k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2; }
  for (int i = (t > 8 ? 8 : t) - 1; i >= 0; i--) k1 ^= (uint64_t)tail[i] << (8 * i);
  if (t > 0) { k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1; }
  h1 ^= (uint64_t)len; h2 ^= (uint64_t)len;
  h1 += h2; h2 += h1;
  h1 = fmix64(h1); h2 = fmix64(h2);
  h1 += h2; h2 += h1;
  out[0] = h1; out[1] = h2;
}

/* ------------------------------------------------------------------------------------------
 * <value, valid> cells.  The reference's iterators yield bool / int32 / uint32 / float (and
 * int64 / UUID at expression roots): query/binder.hpp:209-264.  C casts below are the same
 * conversions the C++ tuple converting-constructors perform implicitly.
 * ---------------------------------------------------------------------------------------- */
typedef enum { K_BOOL, K_I32, K_U32, K_F32, K_I64, K_F64, K_I8, K_U8, K_I16, K_U16, K_UUID } kind_t;

typedef struct {
  kind_t k;
  bool valid;
  union { bool b; int32_t i; uint32_t u; float f; int64_t l; double d; } v;
  UUIDT uuid;
} cell_t;

static cell_t cell_cast(cell_t c, kind_t to) {
  if (c.k == to) return c;
  cell_t r = c;
  r.k = to;
#define FROM(expr)                                                                    \
  switch (to) {                                                                       \
    case K_BOOL: r.v.b = (bool)(expr); break;                                         \
    case K_I32: r.v.i = (int32_t)(expr); break;                                       \
    case K_U32: r.v.u = (uint32_t)(expr); break;                                      \
    case K_F32: r.v.f = (float)(expr); break;                                         \
    case K_I64: r.v.l = (int64_t)(expr); break;                                       \
    case K_F64: r.v.d = (double)(expr); break;                                        \
    case K_I8: r.v.l = 0; r.v.i = (int8_t)(expr); break;                              \
    case K_U8: r.v.l = 0; r.v.u = (uint8_t)(expr); break;                             \
    case K_I16: r.v.l = 0; r.v.i = (int16_t)(expr); break;                            \
    case K_U16: r.v.l = 0; r.v.u = (uint16_t)(expr); break;                           \
    default: break;                                                                   \
  }
  switch (c.k) {
    case K_BOOL: FROM(c.v.b) break;
    case K_I32: case K_I8: case K_I16: FROM(c.v.i) break;
    case K_U32: case K_U8: case K_U16: FROM(c.v.u) break;
    case K_F32: FROM(c.v.f) break;
    case K_I64: FROM(c.v.l) break;
    case K_F64: FROM(c.v.d) break;
    default: break;
  }
#undef FROM
  return r;
}

/* common_type — query/utils.hpp:83-94 */
static kind_t common_kind(kind_t a, kind_t b) {
  if (a == K_F32 || b == K_F32) return K_F32;
  if (a == K_I64 || b == K_I64) return K_I64;
  if (a == K_I32 || b == K_I32) return K_I32;
  return K_U32; /* bool is unsigned */
}

/* ------------------------------------------------------------------------------------------
 * Column decode — VectorPartyIterator, query/iterator.hpp:62-289
 * ---------------------------------------------------------------------------------------- */
static bool bit_at(const uint8_t *p, uint32_t bit) { return (p[bit / 8] >> (bit % 8)) & 1; }

static kind_t column_kind(enum DataType dt) {
  switch (dt) {
    case Bool: return K_BOOL;
    case Int8: case Int16: case Int32: return K_I32;
    case Uint8: case Uint16: case Uint32: return K_U32;
    case Float32: return K_F32;
    case Int64: return K_I64;
    case UUID: return K_UUID;
    default: return (kind_t)-1;
  }
}

static cell_t read_vp(const VectorPartySlice *vp, uint32_t idx, const uint32_t *baseCounts,
                      uint32_t startCount) {
  cell_t c;
  memset(&c, 0, sizeof(c));
  c.k = column_kind(vp->DataType);
  if (vp->BasePtr == NULL) { /* mode 0: constant default, query/binder.hpp:196-214 */
    c.valid = vp->DefaultValue.HasDefault;
    switch (c.k) {
      case K_BOOL: c.v.b = vp->DefaultValue.Value.BoolVal; break;
      case K_I32: c.v.i = vp->DefaultValue.Value.Int32Val; break;
      case K_U32: c.v.u = vp->DefaultValue.Value.Uint32Val; break;
      case K_F32: c.v.f = vp->DefaultValue.Value.FloatVal; break;
      case K_I64: c.v.l = vp->DefaultValue.Value.Int64Val; break;
      default: c.uuid = vp->DefaultValue.Value.UUIDVal; break;
    }
    return c;
  }
  int mode = vp->ValuesOffset == 0 ? 1 : (vp->NullsOffset == 0 ? 2 : 3);
  uint32_t p = idx;
  if (mode == 3) { /* position of the run containing the row, :217-278 */
    uint32_t row = baseCounts ? baseCounts[idx] : startCount + idx;
    const uint32_t *counts = (const uint32_t *)vp->BasePtr;
    uint32_t lo = 0, hi = vp->Length;
    while (lo < hi) {
      uint32_t mid = lo + (hi - lo) / 2;
      if (counts[mid] > row) hi = mid; else lo = mid + 1;
    }
    p = lo == 0 ? 0 : lo - 1;
  }
  const uint8_t *vals = vp->BasePtr + vp->ValuesOffset;
  switch (vp->DataType) {
    case Bool: c.v.b = bit_at(vals, p + vp->StartingIndex); break;
    case Int8: c.v.i = ((const int8_t *)vals)[p]; break;
    case Uint8: c.v.u = vals[p]; break;
    case Int16: c.v.i = ((const int16_t *)vals)[p]; break;
    case Uint16: c.v.u = ((const uint16_t *)vals)[p]; break;
    case Int32: c.v.i = ((const int32_t *)vals)[p]; break;
    case Uint32: c.v.u = ((const uint32_t *)vals)[p]; break;
    case Float32: c.v.f = ((const float *)vals)[p]; break;
    case Int64: c.v.l = ((const int64_t *)vals)[p]; break;
    default: c.uuid = ((const UUIDT *)vals)[p]; break;
  }
  c.valid = mode >= 2 ? bit_at(vp->BasePtr + vp->NullsOffset, p + vp->StartingIndex) : true;
  return c; /* raw value is returned even when NULL (:204-208) */
}

/* element i of an InputVector — query/binder.hpp:80-264, query/iterator.hpp:465-537 */
static int read_input(const InputVector *in, uint32_t i, const uint32_t *index,
                      const uint32_t *baseCounts, uint32_t startCount, cell_t *out) {
  memset(out, 0, sizeof(*out));
  switch (in->Type) {
    case ConstantInput:
      out->valid = in->Vector.Constant.IsValid;
      if (in->Vector.Constant.DataType == ConstInt) { out->k = K_I32; out->v.i = in->Vector.Constant.Value.IntVal; }
      else if (in->Vector.Constant.DataType == ConstFloat) { out->k = K_F32; out->v.f = in->Vector.Constant.Value.FloatVal; }
      else return -1;
      return 0;
    case ScratchSpaceInput: {
      const ScratchSpaceVector *s = &in->Vector.ScratchSpace;
      switch (s->DataType) {
        case Int32: out->k = K_I32; out->v.i = ((const int32_t *)s->Values)[i]; break;
        case Uint32: out->k = K_U32; out->v.u = ((const uint32_t *)s->Values)[i]; break;
        case Float32: out->k = K_F32; out->v.f = ((const float *)s->Values)[i]; break;
        case UUID: out->k = K_UUID; out->uuid = ((const UUIDT *)s->Values)[i]; break;
        default: return -1;
      }
      out->valid = ((const bool *)s->Values)[s->NullsOffset + i];
      return 0;
    }
    case VectorPartyInput: {
      if ((int)column_kind(in->Vector.VP.DataType) < 0) return -1;
      *out = read_vp(&in->Vector.VP, index ? index[i] : i, baseCounts, startCount);
      return 0;
    }
    case ForeignColumnInput: {
      /* RecordIDJoinIterator::dereference — query/iterator.hpp:916-930: positional over the RecordID vector; the batch
       * is batchID - BaseBatchID, bounds-checked against the last batch's record count; mode-0 batches yield the
       * column default (prepareForeignTableIterators, query/binder.hpp:163-176); then the timezone table (:889-905). */
      const ForeignColumnVector *f = &in->Vector.ForeignVP;
      kind_t k = column_kind(f->DataType);
      if ((int)k < 0) return -1;
      RecordID rid = f->RecordIDs[i];
      out->k = k;
      out->valid = false;
      /* (a batch outside [0, NumBatches) and a negative enum are NULL and offset 0 here, where the reference reads out
       * of bounds; the engine does the same, join.cuh foreignLoad) */
      const int32_t b = rid.batchID - f->BaseBatchID;
      if (rid.batchID && (b < f->NumBatches - 1 || rid.index < (uint32_t)f->NumRecordsInLastBatch) && b >= 0 && b < f->NumBatches) {
        VectorPartySlice vp = f->Batches[b];
        vp.DataType = f->DataType;
        if (vp.BasePtr == NULL) vp.DefaultValue = f->DefaultValue;
        *out = read_vp(&vp, rid.index, NULL, 0);
        if (f->TimezoneLookup && f->Batches[b].BasePtr != NULL && k != K_UUID && k != K_I64) {   /* mode 0: not mapped */
          int e = k == K_F32 ? (int)out->v.f : k == K_BOOL ? (int)out->v.b : (int)out->v.u;
          int16_t off = e >= 0 && e < f->TimezoneLookupSize ? f->TimezoneLookup[e] : 0;
          if (k == K_F32) out->v.f = (float)off; else if (k == K_BOOL) out->v.b = off != 0; else out->v.u = (uint32_t)(int32_t)off;
        }
      }
      return 0;
    }
    default: return -1;
  }
}

/* ------------------------------------------------------------------------------------------
 * Calendar — query/functor.cu:67-161 and :207-212
 * ---------------------------------------------------------------------------------------- */
enum { TB_YEAR, TB_QUARTER, TB_MONTH, TB_DOM, TB_DOY, TB_MOY, TB_QOY };
static const uint16_t kDaysBefore[13] = {0, 31, 59, 90, 120, 151, 181, 212, 243, 273, 304, 334, 365};

static uint16_t days_before_month(uint8_t month, bool leap) {
  uint16_t d = kDaysBefore[month];
  if (leap && month >= 2) d++;
  return d;
}

uint32_t oracle_time_bucket(int64_t ts, int tb) {
  const int64_t abs0 = -62135596800LL;
  ts -= abs0;
  uint32_t days = (uint32_t)(ts / 86400);
  int64_t n = days / 146097;
  uint16_t year = (uint16_t)(400 * n);
  int64_t start = n * 146097 * 86400LL;
  days -= 146097 * n;
  n = days / 36524; n -= n >> 2;
  year += 100 * n; start += n * 36524 * 86400LL; days -= 36524 * n;
  n = days / 1461;
  year += 4 * n; start += n * 1461 * 86400LL; days -= 1461 * n;
  n = days / 365; n -= n >> 2;
  year += n; days -= 365 * n; start += n * 365 * 86400LL;
  start += abs0;
  if (tb == TB_YEAR) return (uint32_t)start;
  if (tb == TB_DOY) return days;
  uint16_t y = year + 1;
  bool leap = y % 4 == 0 && (y % 100 != 0 || y % 400 == 0);
  uint8_t month = days / 31;
  if (days >= days_before_month(month + 1, leap)) month++;
  if (tb == TB_MONTH || tb == TB_DOM) {
    uint32_t dbm = days_before_month(month, leap);
    return tb == TB_MONTH ? (uint32_t)(start + (int64_t)dbm * 86400) : days - dbm;
  }
  if (tb == TB_MOY) return month;
  int quarter = month / 3;
  if (tb == TB_QOY) return quarter;
  return (uint32_t)(start + (int64_t)days_before_month(quarter * 3, leap) * 86400);
}

static uint32_t week_start(uint32_t ts) {
  if (ts < 4 * 86400u) return 0;
  return ts - (ts - 4 * 86400u) % (7 * 86400u);
}

/* GetHLLValueFunctor — query/functor.hpp:431-466.  `1 << (rho + HLL_BITS)` is an int shift:
 * x86 wraps the count mod 32 (HOST), CUDA yields 0 for counts >= 32 (DEVICE). */
uint32_t oracle_hll_value(uint64_t hashed, int device_semantics) {
  uint32_t group = (uint32_t)(hashed & ((1 << HLL_BITS) - 1));
  uint32_t rho = 0;
  for (;;) {
    uint32_t sh = rho + HLL_BITS;
    int32_t one = device_semantics ? (sh >= 32 ? 0 : (int32_t)(1u << sh)) : (int32_t)(1u << (sh & 31));
    uint32_t h = (uint32_t)(hashed & (uint64_t)(int64_t)one);
    if (sh < 64 && h == 0) rho++; else break;
  }
  return rho << 16 | group;
}

/* ------------------------------------------------------------------------------------------
 * Functors — query/functor.hpp:30-380 (scalar ops), :663-698 / :756-785 (unary dispatch),
 * :924-970 / :1037-1076 (binary dispatch)
 * ---------------------------------------------------------------------------------------- */
static cell_t null_of(kind_t k) { cell_t c; memset(&c, 0, sizeof(c)); c.k = k; return c; }
static cell_t bool_of(bool b) { cell_t c = null_of(K_BOOL); c.v.b = b; c.valid = true; return c; }

static cell_t apply_unary(int fn, cell_t a) {
  const kind_t I = a.k;
  if (I == K_UUID) { /* UnaryFunctor<O, UUIDT>: only GetHLLValue, hll_hash = p1 ^ p2 (:439-442) */
    if (fn == GetHLLValue) {
      cell_t r = null_of(K_U32);
      if (a.valid) { r.valid = true; r.v.u = oracle_hll_value(a.uuid.p1 ^ a.uuid.p2, g_device_semantics); }
      return r;
    }
    return a; /* caller maps UUID->UUID to a copy and everything else to NULL */
  }
  const bool is_float = I == K_F32;
  switch (fn) {
    case Not: if (!a.valid) return null_of(K_BOOL); return bool_of(!cell_cast(a, K_BOOL).v.b);
    case IsNull: return bool_of(!a.valid);
    case IsNotNull: return bool_of(a.valid);
    case Negate: {
      cell_t r = null_of(I);
      if (!a.valid) return r;
      r.valid = true;
      switch (I) {
        case K_BOOL: r.v.b = (bool)(-(int)a.v.b); break;
        case K_I32: r.v.i = (int32_t)(0u - (uint32_t)a.v.i); break;
        case K_U32: r.v.u = 0u - a.v.u; break;
        case K_F32: r.v.f = -a.v.f; break;
        default: r.v.l = (int64_t)(0ull - (uint64_t)a.v.l); break;
      }
      return r;
    }
    case BitwiseNot: {
      if (is_float) break;
      cell_t r = null_of(I);
      if (!a.valid) return r;
      r.valid = true;
      switch (I) {
        case K_BOOL: r.v.b = (bool)(~(int)a.v.b); break;
        case K_I32: r.v.i = ~a.v.i; break;
        case K_U32: r.v.u = ~a.v.u; break;
        default: r.v.l = ~a.v.l; break;
      }
      return r;
    }
    case GetWeekStart: case GetMonthStart: case GetQuarterStart: case GetYearStart:
    case GetDayOfMonth: case GetDayOfYear: case GetMonthOfYear: case GetQuarterOfYear: {
      if (is_float) break;
      cell_t r = null_of(K_U32);
      if (!a.valid) return r;
      uint32_t ts = cell_cast(a, K_U32).v.u;
      r.valid = true;
      switch (fn) {
        case GetWeekStart: r.v.u = week_start(ts); break;
        case GetMonthStart: r.v.u = oracle_time_bucket(ts, TB_MONTH); break;
        case GetQuarterStart: r.v.u = oracle_time_bucket(ts, TB_QUARTER); break;
        case GetYearStart: r.v.u = oracle_time_bucket(ts, TB_YEAR); break;
        case GetDayOfMonth: r.v.u = oracle_time_bucket(ts, TB_DOM); break;
        case GetDayOfYear: r.v.u = oracle_time_bucket(ts, TB_DOY); break;
        case GetMonthOfYear: r.v.u = oracle_time_bucket(ts, TB_MOY); break;
        default: r.v.u = oracle_time_bucket(ts, TB_QOY); break;
      }
      return r;
    }
    case GetHLLValue: {
      if (is_float) break;
      cell_t r = null_of(K_U32);
      if (!a.valid) return r;
      uint64_t out[2];
      uint8_t bytes[8];
      int len;
      if (I == K_BOOL) { bytes[0] = a.v.b; len = 1; }
      else if (I == K_I64) { memcpy(bytes, &a.v.l, 8); len = 8; }
      else { memcpy(bytes, &a.v.u, 4); len = 4; }
      oracle_murmur3_128(bytes, len, 0, out);
      r.valid = true;
      r.v.u = oracle_hll_value(out[0], g_device_semantics);
      return r;
    }
    default: break;
  }
  return a; /* Noop and anything the class does not implement */
}

static cell_t apply_binary(int fn, cell_t a, cell_t b) {
  /* both operands already share the common kind T */
  const kind_t T = a.k;
  const bool is_float = T == K_F32;
  if (fn == And) {
    if (!a.valid || !b.valid) return null_of(K_BOOL);
    return bool_of(cell_cast(a, K_BOOL).v.b && cell_cast(b, K_BOOL).v.b);
  }
  if (fn == Or) {
    bool av = cell_cast(a, K_BOOL).v.b, bv = cell_cast(b, K_BOOL).v.b;
    if ((av && a.valid) || (bv && b.valid)) return bool_of(true);
    if (!a.valid || !b.valid) return null_of(K_BOOL);
    return bool_of(false);
  }
  if (fn >= Equal && fn <= GreaterThanOrEqual) {
    if (!a.valid || !b.valid) return null_of(K_BOOL);
#define CMP(x, y) (fn == Equal ? (x) == (y) : fn == NotEqual ? (x) != (y) : fn == LessThan ? (x) < (y) \
                 : fn == LessThanOrEqual ? (x) <= (y) : fn == GreaterThan ? (x) > (y) : (x) >= (y))
    if (is_float) return bool_of(CMP(a.v.f, b.v.f));
    if (T == K_I32) return bool_of(CMP(a.v.i, b.v.i));
    return bool_of(CMP(a.v.u, b.v.u));
#undef CMP
  }
  bool arithmetic = fn >= Plus && fn <= Divide;
  bool int_only = fn == Mod || (fn >= BitwiseAnd && fn <= Floor);
  if (arithmetic || (int_only && !is_float)) {
    cell_t r = null_of(T);
    if (!a.valid || !b.valid) return r;
    r.valid = true;
    if (is_float) {
      float x = a.v.f, y = b.v.f;
      r.v.f = fn == Plus ? x + y : fn == Minus ? x - y : fn == Multiply ? x * y : x / y;
    } else if (T == K_I32) {
      int32_t x = a.v.i, y = b.v.i;
      switch (fn) {
        case Plus: r.v.i = (int32_t)((uint32_t)x + (uint32_t)y); break;
        case Minus: r.v.i = (int32_t)((uint32_t)x - (uint32_t)y); break;
        case Multiply: r.v.i = (int32_t)((uint32_t)x * (uint32_t)y); break;
        case Divide: r.v.i = y == 0 ? -1 : (y == -1 ? (int32_t)(0u - (uint32_t)x) : x / y); break;
        case Mod: r.v.i = y == 0 ? x : (y == -1 ? 0 : x % y); break;
        case BitwiseAnd: r.v.i = x & y; break;
        case BitwiseOr: r.v.i = x | y; break;
        case BitwiseXor: r.v.i = x ^ y; break;
        default: r.v.i = y == 0 ? 0 : (y == -1 ? x : x - x % y); break; /* Floor = a - a % b (:337-351) */
      }
    } else {
      uint32_t x = a.v.u, y = b.v.u;
      switch (fn) {
        case Plus: r.v.u = x + y; break;
        case Minus: r.v.u = x - y; break;
        case Multiply: r.v.u = x * y; break;
        case Divide: r.v.u = y == 0 ? 0xFFFFFFFFu : x / y; break;
        case Mod: r.v.u = y == 0 ? x : x % y; break;
        case BitwiseAnd: r.v.u = x & y; break;
        case BitwiseOr: r.v.u = x | y; break;
        case BitwiseXor: r.v.u = x ^ y; break;
        default: r.v.u = y == 0 ? 0 : x - x % y; break;
      }
    }
    return r;
  }
  return a;
}

/* evaluates one AST node for row i; returns <0 on unsupported input */
static int eval_node(const InputVector *ins, int nin, int fn, uint32_t i, const uint32_t *index,
                     const uint32_t *baseCounts, uint32_t startCount, cell_t *out) {
  cell_t a, b;
  if (read_input(&ins[0], i, index, baseCounts, startCount, &a) < 0) return -1;
  if (nin == 1) { *out = apply_unary(fn, a); return 0; }
  if (read_input(&ins[1], i, index, baseCounts, startCount, &b) < 0) return -1;
  if (a.k == K_I64 || b.k == K_I64 || a.k == K_UUID || b.k == K_UUID) return -2;
  kind_t T = common_kind(a.k, b.k);
  *out = apply_binary(fn, cell_cast(a, T), cell_cast(b, T));
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * Sinks — scratch query/scratch_space_transform.cu:20-39, dimension
 * query/dimension_transform.cu:25-83, measure query/measure_transform.cu:20-40 +
 * MeasureOutputIterator / MeasureProxy query/iterator.hpp:616-727
 * ---------------------------------------------------------------------------------------- */
static kind_t sink_kind(enum DataType dt, bool dim) {
  switch (dt) {
    case Bool: return dim ? K_BOOL : (kind_t)-1;
    case Int8: return dim ? K_I8 : (kind_t)-1;
    case Uint8: return dim ? K_U8 : (kind_t)-1;
    case Int16: return dim ? K_I16 : (kind_t)-1;
    case Uint16: return dim ? K_U16 : (kind_t)-1;
    case Int32: return K_I32;
    case Uint32: return K_U32;
    case Float32: return K_F32;
    case Int64: return K_I64;
    case Float64: return dim ? (kind_t)-1 : K_F64;
    case UUID: return K_UUID;
    default: return (kind_t)-1;
  }
}

static void store_cell(uint8_t *p, cell_t c) {
  switch (c.k) {
    case K_BOOL: *p = c.v.b; break;
    case K_I8: case K_U8: *p = (uint8_t)c.v.u; break;
    case K_I16: case K_U16: { uint16_t x = (uint16_t)c.v.u; memcpy(p, &x, 2); break; }
    case K_I32: case K_U32: case K_F32: memcpy(p, &c.v.u, 4); break;
    case K_I64: case K_F64: memcpy(p, &c.v.l, 8); break;
    default: memcpy(p, &c.uuid, 16); break;
  }
}
static int kind_width(kind_t k) {
  switch (k) {
    case K_BOOL: case K_I8: case K_U8: return 1;
    case K_I16: case K_U16: return 2;
    case K_I32: case K_U32: case K_F32: return 4;
    case K_I64: case K_F64: return 8;
    default: return 16;
  }
}

/* get_identity_value<Value> — query/utils.hpp:169-184 (MAX_FLOAT really is FLT_MIN there) */
static cell_t identity_of(enum AggregateFunction f, kind_t k) {
  cell_t c = null_of(K_I64);
  c.valid = true;
  switch (f) {
    case AGGR_MIN_UNSIGNED: c.v.l = 4294967295LL; break;
    case AGGR_MIN_SIGNED: c.v.l = 2147483647LL; break;
    case AGGR_MIN_FLOAT: c.k = K_F32; c.v.f = 3.402823466e+38F; break;
    case AGGR_MAX_SIGNED: c.v.l = -2147483648LL; break;
    case AGGR_MAX_FLOAT: c.k = K_F32; c.v.f = 1.175494351e-38F; break;
    default: c.v.l = 0; break;
  }
  return cell_cast(c, k);
}

static CGoCallResHandle transform(const InputVector *ins, int nin, OutputVector out, uint32_t *index,
                                  int n, uint32_t *baseCounts, uint32_t startCount, int fn) {
  bool dim = out.Type == DimensionOutput, meas = out.Type == MeasureOutput;
  enum DataType dt = dim ? out.Vector.Dimension.DataType
                         : meas ? out.Vector.Measure.DataType : out.Vector.ScratchSpace.DataType;
  kind_t O = sink_kind(dt, dim);
  if ((int)O < 0 || (!dim && !meas && O == K_F64) || (meas && O == K_UUID))
    return fail("Unsupported data type for output");
  uint8_t *values = dim ? out.Vector.Dimension.DimValues
                        : meas ? (uint8_t *)out.Vector.Measure.Values : out.Vector.ScratchSpace.Values;
  uint8_t *nulls = dim ? out.Vector.Dimension.DimNulls
                       : meas ? NULL : out.Vector.ScratchSpace.Values + out.Vector.ScratchSpace.NullsOffset;
  enum AggregateFunction agg = meas ? out.Vector.Measure.AggFunc : 0;
  bool is_avg = agg == AGGR_AVG_FLOAT;
  bool skip_count = !((agg >= AGGR_SUM_UNSIGNED && agg <= AGGR_SUM_FLOAT) || is_avg);
  int w = kind_width(O);
  for (int i = 0; i < n; i++) {
    cell_t r;
    int rc = eval_node(ins, nin, fn, (uint32_t)i, index, baseCounts, startCount, &r);
    if (rc == -2) return fail("int64/UUID data types are only supported in UnaryTransform");
    if (rc < 0) return fail("Unsupported input vector for the oracle");
    if (r.k == K_UUID || O == K_UUID) {
      if (!(r.k == K_UUID && O == K_UUID)) { bool v = false; r = null_of(O); r.valid = v; }
    } else {
      bool v = r.valid;
      r = cell_cast(r, O);
      r.valid = v;
    }
    if (!meas) {
      store_cell(values + (size_t)i * w, r);
      nulls[i] = r.valid;
      continue;
    }
    uint8_t *o = values + (size_t)i * w;
    if (!r.valid) { store_cell(o, identity_of(agg, O)); continue; }
    uint32_t count = 1;
    if (!skip_count && baseCounts != NULL) count = baseCounts[index[i] + 1] - baseCounts[index[i]];
    if (is_avg) { /* assignAvg, iterator.hpp:636-645 */
      float f = cell_cast(r, K_F32).v.f;
      memcpy(o, &f, 4);
      memcpy(o + 4, &count, 4);
      continue;
    }
    switch (O) { /* *outputIter = value * count in Value arithmetic */
      case K_I32: r.v.i = (int32_t)((uint32_t)r.v.i * count); break;
      case K_U32: r.v.u = r.v.u * count; break;
      case K_F32: r.v.f = r.v.f * count; break;
      case K_I64: r.v.l = r.v.l * count; break;
      default: r.v.d = r.v.d * count; break;
    }
    store_cell(o, r);
  }
  return ok(n);
}

/* FilterContext::executeRemoveIf — query/filter.cu:208-253: predicate = value part of the
 * functor result as bool; stable in-place compaction of index (+ RecordID vectors). */
static CGoCallResHandle filter(const InputVector *ins, int nin, uint32_t *index, uint8_t *pred, int n,
                               RecordID **recs, int nrec, uint32_t *baseCounts, uint32_t startCount,
                               int fn) {
  for (int i = 0; i < n; i++) {
    cell_t r;
    int rc = eval_node(ins, nin, fn, (uint32_t)i, index, baseCounts, startCount, &r);
    if (rc < 0) return fail("Unsupported input vector for the oracle");
    pred[i] = r.k == K_UUID ? 0 : cell_cast(r, K_BOOL).v.b;
  }
  int m = 0;
  for (int i = 0; i < n; i++) {
    if (!pred[i]) continue;
    index[m] = index[i];
    for (int f = 0; f < nrec; f++) recs[f][m] = recs[f][i];
    m++;
  }
  return ok(m);
}

CGoCallResHandle InitIndexVector(uint32_t *indexVector, uint32_t start, int n, void *s, int d) {
  (void)s; (void)d;
  for (int i = 0; i < n; i++) indexVector[i] = start + (uint32_t)i; /* query/algorithm.cu:22-41 */
  return ok(0);
}
CGoCallResHandle UnaryTransform(InputVector input, OutputVector output, uint32_t *indexVector, int n,
                                uint32_t *baseCounts, uint32_t startCount, enum UnaryFunctorType fn,
                                void *s, int d) {
  (void)s; (void)d;
  return transform(&input, 1, output, indexVector, n, baseCounts, startCount, (int)fn);
}
CGoCallResHandle BinaryTransform(InputVector lhs, InputVector rhs, OutputVector output,
                                 uint32_t *indexVector, int n, uint32_t *baseCounts, uint32_t startCount,
                                 enum BinaryFunctorType fn, void *s, int d) {
  (void)s; (void)d;
  InputVector ins[2] = {lhs, rhs};
  return transform(ins, 2, output, indexVector, n, baseCounts, startCount, (int)fn);
}
CGoCallResHandle UnaryFilter(InputVector input, uint32_t *indexVector, uint8_t *pred, int n,
                             RecordID **recs, int nrec, uint32_t *baseCounts, uint32_t startCount,
                             enum UnaryFunctorType fn, void *s, int d) {
  (void)s; (void)d;
  return filter(&input, 1, indexVector, pred, n, recs, nrec, baseCounts, startCount, (int)fn);
}
CGoCallResHandle BinaryFilter(InputVector lhs, InputVector rhs, uint32_t *indexVector, uint8_t *pred,
                              int n, RecordID **recs, int nrec, uint32_t *baseCounts,
                              uint32_t startCount, enum BinaryFunctorType fn, void *s, int d) {
  (void)s; (void)d;
  InputVector ins[2] = {lhs, rhs};
  return filter(ins, 2, indexVector, pred, n, recs, nrec, baseCounts, startCount, (int)fn);
}

/* ------------------------------------------------------------------------------------------
 * Dimension rows — DimensionHashIterator query/iterator.hpp:934-1025: pack the dims of row
 * `idx` in layout order (16,8,4,2,1-byte columns) followed by one validity byte per dim into a
 * zero-initialised 32-byte buffer; hash rowBytes bytes with seed 0.
 * ---------------------------------------------------------------------------------------- */
static int pack_row(const uint8_t *dimValues, const uint8_t nd[NUM_DIM_WIDTH], int capacity,
                    uint32_t idx, uint8_t row[MAX_DIMENSION_BYTES]) {
  memset(row, 0, MAX_DIMENSION_BYTES);
  int total = 0, valueBytes = 0;
  for (int i = 0; i < NUM_DIM_WIDTH; i++) { total += nd[i]; valueBytes += nd[i] * (1 << (NUM_DIM_WIDTH - 1 - i)); }
  const uint8_t *col = dimValues;
  const uint8_t *nullCol = dimValues + (size_t)valueBytes * capacity;
  int o = 0, n = 0;
  for (int i = 0; i < NUM_DIM_WIDTH; i++) {
    int w = 1 << (NUM_DIM_WIDTH - 1 - i);
    for (int j = 0; j < nd[i]; j++) {
      memcpy(row + o, col + (size_t)idx * w, w);
      o += w;
      col += (size_t)w * capacity;
      row[valueBytes + n] = nullCol[idx];
      nullCol += capacity;
      n++;
    }
  }
  return valueBytes + total;
}

/* TEST SEAM (tests/test_hash_collisions.py): ARESDB_B200_TEST_HASH64_MASK=<hex> ANDs the 64-bit group-identity hash
 * of a dimension row, so that the reference's merge rule for colliding hashes (sort_reduce.cu:140-157: equal
 * consecutive hashes are ONE run, the first row of the stable order supplies the dims) can be exercised; the engine
 * has the same seam.  Unset (always, outside that test): the full hash. */
static uint64_t test_hash64_mask(void) {
  static int init = 0;
  static uint64_t mask = ~0ull;
  if (!init) {
    const char *e = getenv("ARESDB_B200_TEST_HASH64_MASK");
    if (e && *e) mask = strtoull(e, NULL, 16);
    init = 1;
  }
  return mask;
}

static uint64_t row_hash64(const DimensionVector *k, uint32_t idx) {
  uint8_t row[MAX_DIMENSION_BYTES];
  uint64_t out[2];
  int len = pack_row(k->DimValues, k->NumDimsPerDimWidth, k->VectorCapacity, idx, row);
  oracle_murmur3_128(row, len, 0, out);
  return out[0] & test_hash64_mask();
}

/* copies every dim column + validity column of input row `from` to output row `to`
 * (DimensionColumnPermutateIterator -> DimensionColumnOutputIterator, iterator.hpp:1042-1167) */
static void copy_dim_row(const uint8_t *in, uint8_t *out, const uint8_t nd[NUM_DIM_WIDTH], int inCap,
                         int outCap, uint32_t from, uint32_t to) {
  size_t io = 0, oo = 0;
  int total = 0;
  for (int i = 0; i < NUM_DIM_WIDTH; i++) {
    int w = 1 << (NUM_DIM_WIDTH - 1 - i);
    for (int j = 0; j < nd[i]; j++) {
      memcpy(out + oo + (size_t)to * w, in + io + (size_t)from * w, w);
      io += (size_t)w * inCap;
      oo += (size_t)w * outCap;
      total++;
    }
  }
  for (int j = 0; j < total; j++) {
    out[oo + to] = in[io + from];
    io += inCap;
    oo += outCap;
  }
}

typedef struct { uint64_t key; uint32_t idx; uint32_t val; } sort_rec;

static void merge_sort(sort_rec *a, sort_rec *tmp, int n) { /* stable, ascending key */
  if (n < 2) return;
  int h = n / 2;
  merge_sort(a, tmp, h);
  merge_sort(a + h, tmp, n - h);
  int i = 0, j = h, k = 0;
  while (i < h && j < n) tmp[k++] = a[j].key < a[i].key ? a[j++] : a[i++];
  while (i < h) tmp[k++] = a[i++];
  while (j < n) tmp[k++] = a[j++];
  memcpy(a, tmp, sizeof(sort_rec) * n);
}

/* ares::sort — query/sort_reduce.cu:118-133 */
CGoCallResHandle Sort(DimensionVector keys, int length, void *s, int d) {
  (void)s; (void)d;
  if (length <= 0) return ok(0);
  sort_rec *a = malloc(sizeof(sort_rec) * length), *t = malloc(sizeof(sort_rec) * length);
  for (int i = 0; i < length; i++) {
    a[i].idx = keys.IndexVector[i];
    a[i].key = row_hash64(&keys, a[i].idx);
    a[i].val = 0;
  }
  merge_sort(a, t, length);
  for (int i = 0; i < length; i++) { keys.HashValues[i] = a[i].key; keys.IndexVector[i] = a[i].idx; }
  free(a); free(t);
  return ok(0);
}

/* RollingAvgFunctor — query/functor.hpp:1414-1436 */
static uint64_t rolling_avg(uint64_t lhs, uint64_t rhs) {
  uint32_t lc = (uint32_t)(lhs >> 32), rc = (uint32_t)(rhs >> 32), total = lc + rc;
  if (total == 0) return 0;
  float lf, rf;
  uint32_t lb = (uint32_t)lhs, rb = (uint32_t)rhs;
  memcpy(&lf, &lb, 4); memcpy(&rf, &rb, 4);
  float res = lf / total * lc + rf / total * rc;
  uint32_t bits;
  memcpy(&bits, &res, 4);
  return ((uint64_t)total << 32) | bits;
}

/* combine two measure values (bindValueAndAggFunc op table, query/sort_reduce.cu:160-217) */
static int combine(uint8_t *acc, const uint8_t *x, int valueBytes, enum AggregateFunction f) {
#define OP(T, expr) { T a, b; memcpy(&a, acc, sizeof(T)); memcpy(&b, x, sizeof(T)); a = (expr); memcpy(acc, &a, sizeof(T)); return 0; }
  switch (f) {
    case AGGR_SUM_UNSIGNED: if (valueBytes == 4) OP(uint32_t, a + b) else OP(uint64_t, a + b)
    case AGGR_SUM_SIGNED: if (valueBytes == 4) OP(uint32_t, a + b) else OP(uint64_t, a + b)
    case AGGR_SUM_FLOAT: if (valueBytes == 4) OP(float, a + b) else OP(double, a + b)
    case AGGR_MIN_UNSIGNED: OP(uint32_t, b < a ? b : a)
    case AGGR_MIN_SIGNED: OP(int32_t, b < a ? b : a)
    case AGGR_MIN_FLOAT: OP(float, b < a ? b : a)
    case AGGR_MAX_UNSIGNED: OP(uint32_t, a < b ? b : a)
    case AGGR_MAX_SIGNED: OP(int32_t, a < b ? b : a)
    case AGGR_MAX_FLOAT: OP(float, a < b ? b : a)
    case AGGR_AVG_FLOAT: OP(uint64_t, rolling_avg(a, b))
    default: return -1;
  }
#undef OP
}

static int agg_value_bytes(enum AggregateFunction f, int valueBytes) {
  if (f == AGGR_AVG_FLOAT) return 8;
  if (f >= AGGR_SUM_UNSIGNED && f <= AGGR_SUM_FLOAT) return valueBytes == 4 ? 4 : 8;
  return 4;
}

/* ares::reduce — query/sort_reduce.cu:135-249: sequential left fold over runs of equal hashes,
 * first index of the run kept, measure read through the index (permutation iterator). */
CGoCallResHandle Reduce(DimensionVector in, uint8_t *inValues, DimensionVector out, uint8_t *outValues,
                        int valueBytes, int length, enum AggregateFunction f, void *s, int d) {
  (void)s; (void)d;
  int vb = agg_value_bytes(f, valueBytes);
  int g = 0;
  for (int i = 0; i < length;) {
    int j = i;
    uint8_t acc[8];
    memcpy(acc, inValues + (size_t)in.IndexVector[i] * vb, vb);
    for (j = i + 1; j < length && in.HashValues[j] == in.HashValues[i]; j++)
      if (combine(acc, inValues + (size_t)in.IndexVector[j] * vb, vb, f) < 0)
        return fail("Unsupported aggregation function type");
    out.IndexVector[g] = in.IndexVector[i];
    memcpy(outValues + (size_t)g * vb, acc, vb);
    g++;
    i = j;
  }
  for (int r = 0; r < g; r++)
    copy_dim_row(in.DimValues, out.DimValues, in.NumDimsPerDimWidth, in.VectorCapacity, in.VectorCapacity,
                 out.IndexVector[r], (uint32_t)r);
  return ok(g);
}

/* ares::hash_reduction — query/hash_reduction.cu:183-391 with the HOST map
 * (query/concurrent_unordered_map.hpp:127-134): group identity = murmur3_32 of the packed row,
 * first row seen represents the group, values folded in row order starting FROM ZERO (the HOST
 * map default-constructs the slot; identical to the identity for the SUM family the Go side
 * restricts this path to, query/aql_context.go:426-434).  Output order: first appearance. */
CGoCallResHandle HashReduce(DimensionVector in, uint8_t *inValues, DimensionVector out,
                            uint8_t *outValues, int valueBytes, int length,
                            enum AggregateFunction f, void *s, int d) {
  (void)s; (void)d;
  if (length <= 0) return ok(0);
  int vb = agg_value_bytes(f, valueBytes);
  int cap = 1;
  while (cap < 2 * length) cap <<= 1;
  int32_t *slotGroup = malloc(sizeof(int32_t) * cap);
  uint32_t *slotHash = malloc(sizeof(uint32_t) * cap);
  for (int i = 0; i < cap; i++) slotGroup[i] = -1;
  int g = 0;
  for (int i = 0; i < length; i++) {
    uint8_t row[MAX_DIMENSION_BYTES];
    int len = pack_row(in.DimValues, in.NumDimsPerDimWidth, in.VectorCapacity, (uint32_t)i, row);
    uint32_t h = oracle_murmur3_32(row, len, 0);
    uint32_t p = h & (uint32_t)(cap - 1);
    while (slotGroup[p] >= 0 && slotHash[p] != h) p = (p + 1) & (uint32_t)(cap - 1);
    if (slotGroup[p] < 0) {
      slotGroup[p] = g;
      slotHash[p] = h;
      copy_dim_row(in.DimValues, out.DimValues, in.NumDimsPerDimWidth, in.VectorCapacity,
                   in.VectorCapacity, (uint32_t)i, (uint32_t)g);
      memset(outValues + (size_t)g * vb, 0, vb);
      g++;
    }
    if (combine(outValues + (size_t)slotGroup[p] * vb, inValues + (size_t)i * vb, vb, f) < 0) {
      free(slotGroup); free(slotHash);
      return fail("Unsupported aggregation function type");
    }
  }
  free(slotGroup); free(slotHash);
  return ok(g);
}

/* ------------------------------------------------------------------------------------------
 * HyperLogLog — query/hll.cu:62-290 (steps numbered as in ares::hyperloglog, :255-290)
 * ---------------------------------------------------------------------------------------- */
CGoCallResHandle HyperLogLog(DimensionVector prev, DimensionVector cur, uint32_t *prevValues,
                             uint32_t *curValues, int prevResultSize, int curBatchSize,
                             bool isLastBatch, uint8_t **hllVectorPtr, size_t *hllVectorSizePtr,
                             uint16_t **hllDimRegIDCountPtr, void *s, int d) {
  (void)s; (void)d;
  /* 1. sortCurrentBatch (:70-88): key = (dim hash & ~0xFFFF) | reg id, stable sort of (idx, value).
   *    Batch dim values live in prev.DimValues, addressed through cur.IndexVector. */
  int n = curBatchSize;
  sort_rec *a = malloc(sizeof(sort_rec) * (n + 1)), *t = malloc(sizeof(sort_rec) * (n + 1));
  DimensionVector hashSrc = prev;
  hashSrc.VectorCapacity = cur.VectorCapacity;
  for (int i = 0; i < NUM_DIM_WIDTH; i++) hashSrc.NumDimsPerDimWidth[i] = cur.NumDimsPerDimWidth[i];
  for (int i = 0; i < n; i++) {
    a[i].idx = cur.IndexVector[i];
    a[i].val = curValues[i];
    a[i].key = (row_hash64(&hashSrc, a[i].idx) & 0xFFFFFFFFFFFF0000ULL) | (curValues[i] & 0x3FFF);
  }
  merge_sort(a, t, n);
  /* 2. reduceCurrentBatch (:211-231): per key keep the first idx and the max value; results are
   *    appended after the carried rows of prev. */
  int m = 0;
  for (int i = 0; i < n;) {
    int j = i + 1;
    uint32_t best = a[i].val;
    for (; j < n && a[j].key == a[i].key; j++) if (a[j].val > best) best = a[j].val;
    prev.HashValues[prevResultSize + m] = a[i].key;
    prev.IndexVector[prevResultSize + m] = a[i].idx;
    prevValues[prevResultSize + m] = best;
    m++;
    i = j;
  }
  free(a); free(t);
  /* 3. merge (:191-209): stable merge of carried and current by (hash asc, value desc); ties
   *    take the carried element first. */
  int i = 0, j = prevResultSize, e1 = prevResultSize, e2 = prevResultSize + m, k = 0;
  while (i < e1 || j < e2) {
    bool takeSecond;
    if (i >= e1) takeSecond = true;
    else if (j >= e2) takeSecond = false;
    else {
      uint64_t h1 = prev.HashValues[i], h2 = prev.HashValues[j];
      uint32_t v1 = prevValues[i], v2 = prevValues[j];
      /* second precedes first iff comp(second, first) */
      takeSecond = h2 == h1 ? v2 > v1 : h2 < h1;
    }
    int src = takeSecond ? j++ : i++;
    cur.HashValues[k] = prev.HashValues[src];
    curValues[k] = prevValues[src];
    cur.IndexVector[k] = prev.IndexVector[src];
    k++;
  }
  int resSize = prevResultSize + m;
  if (isLastBatch && resSize > 0) {
    /* 4. makeHLLVector (:233-254) + createAndCopyHLLVector (:108-166) */
    uint32_t *dimOrdinal = malloc(sizeof(uint32_t) * resSize);
    int dims = 0;
    for (int r = 0; r < resSize; r++) {
      bool head = r == 0 || ((cur.HashValues[r] >> 16) ^ (cur.HashValues[r - 1] >> 16)) != 0;
      if (head) cur.IndexVector[dims++] = cur.IndexVector[r];
      dimOrdinal[r] = (uint32_t)dims; /* 1-based */
    }
    uint16_t *regCount = malloc(sizeof(uint16_t) * (dims ? dims : 1));
    memset(regCount, 0, sizeof(uint16_t) * (dims ? dims : 1));
    for (int r = 0; r < resSize; r++) {
      bool regHead = r == 0 || cur.HashValues[r] != cur.HashValues[r - 1];
      if (regHead) regCount[dimOrdinal[r] - 1]++;
    }
    uint64_t *offsets = malloc(sizeof(uint64_t) * (dims + 1));
    offsets[0] = 0;
    for (int g = 0; g < dims; g++)
      offsets[g + 1] = offsets[g] + (regCount[g] < HLL_DENSE_THRESHOLD ? (uint64_t)regCount[g] * 4 : HLL_DENSE_SIZE);
    size_t total = offsets[dims];
    uint8_t *hll = malloc(total ? total : 1);
    memset(hll, 0, total);
    int within = 0;
    for (int r = 0; r < resSize; r++) {
      bool regHead = r == 0 || cur.HashValues[r] != cur.HashValues[r - 1];
      bool dimHead = r == 0 || dimOrdinal[r] != dimOrdinal[r - 1];
      if (dimHead) within = 0;
      if (!regHead) continue;
      uint32_t g = dimOrdinal[r] - 1, v = curValues[r];
      uint16_t reg = (uint16_t)(v & 0x3FFF);
      uint8_t rho = (uint8_t)(((v >> 16) & 0xFF) + 1); /* CopyHLLFunctor, functor.hpp:1351-1374 */
      if (regCount[g] < HLL_DENSE_THRESHOLD) {
        uint32_t w = (uint32_t)rho << 16 | reg;
        memcpy(hll + offsets[g] + (size_t)within * 4, &w, 4);
      } else {
        hll[offsets[g] + reg] = rho;
      }
      within++;
    }
    *hllVectorPtr = hll;
    *hllVectorSizePtr = total;
    *hllDimRegIDCountPtr = regCount;
    free(offsets); free(dimOrdinal);
    resSize = dims;
  }
  /* 5. copyDim (:169-187) */
  for (int r = 0; r < resSize; r++)
    copy_dim_row(prev.DimValues, cur.DimValues, prev.NumDimsPerDimWidth, prev.VectorCapacity,
                 prev.VectorCapacity, cur.IndexVector[r], (uint32_t)r);
  return ok(resSize);
}

/* ------------------------------------------------------------------------------------------
 * HashLookup — query/hash_lookup.cu:70-157, HashLookupFunctor query/functor.hpp:1173-1266
 * ---------------------------------------------------------------------------------------- */
CGoCallResHandle HashLookup(InputVector input, RecordID *output, uint32_t *indexVector, int n, uint32_t *baseCounts,
                            uint32_t startCount, CuckooHashIndex h, void *s, int d) {
  (void)s; (void)d;
  const int cellBytes = 8 + h.keyBytes + 1;
  const int bucketBytes = HASH_BUCKET_SIZE * cellBytes;
  const int offSig = HASH_BUCKET_SIZE * 8, offKey = offSig + HASH_BUCKET_SIZE;
  uint8_t *stash = h.buckets + (size_t)bucketBytes * h.numBuckets;
  for (int i = 0; i < n; i++) {
    cell_t c;
    RecordID none = {0, 0};
    output[i] = none;
    if (read_input(&input, (uint32_t)i, indexVector, baseCounts, startCount, &c) < 0) return fail("HashLookup: unsupported input");
    if (!c.valid) continue;
    uint8_t key[16];
    memset(key, 0, sizeof(key));
    if (c.k == K_UUID) memcpy(key, &c.uuid, 16); else if (c.k == K_I64) memcpy(key, &c.v.l, 8);
    else if (c.k == K_BOOL) key[0] = c.v.b; else memcpy(key, &c.v.u, 4);
    bool found = false;
    for (int t = 0; t < h.numHashes && !found; t++) {
      uint32_t hv = oracle_murmur3_32(key, h.keyBytes, h.seeds[t]);
      uint8_t *bucket = h.buckets + (size_t)(hv % (uint32_t)h.numBuckets) * bucketBytes;
      uint8_t sig = (uint8_t)(hv >> 24);
      if (sig < 1) sig = 1;
      for (int j = 0; j < HASH_BUCKET_SIZE && !found; j++)
        if (bucket[offSig + j] == sig && memcmp(bucket + offKey + j * h.keyBytes, key, h.keyBytes) == 0) {
          memcpy(&output[i], bucket + 8 * j, 8);
          found = true;
        }
    }
    for (int j = 0; j < HASH_STASH_SIZE && !found; j++)
      if (stash[offSig + j] != 0 && memcmp(stash + offKey + j * h.keyBytes, key, h.keyBytes) == 0) {
        memcpy(&output[i], stash + 8 * j, 8);
        found = true;
      }
  }
  return ok(n);
}

CGoCallResHandle BootstrapDevice(void) { return ok(0); }
