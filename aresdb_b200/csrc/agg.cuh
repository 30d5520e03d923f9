// agg.cuh — the aggregate combine rules on raw 4/8-byte measure words (reference op table:
// bindValueAndAggFunc, query/sort_reduce.cu:160-217; RollingAvgFunctor query/functor.hpp:1414-1436).
#pragma once
#include "cell.cuh"
#ifndef __CUDACC_RTC__
#include "common.cuh"
#endif

namespace aresb {

enum AggOp : uint8_t {
  OP_SUM_I32, OP_SUM_F32, OP_SUM_I64, OP_SUM_F64,
  OP_MIN_U32, OP_MIN_I32, OP_MIN_F32, OP_MAX_U32, OP_MAX_I32, OP_MAX_F32, OP_AVG, OP_INVALID
};

#ifndef __CUDACC_RTC__
// (aggFunc, valueBytes) -> op and the effective element width the reference uses.
inline AggOp aggOpOf(int aggFunc, int valueBytes, int *width) {
  int w = 4;
  AggOp op = OP_INVALID;
  switch (aggFunc) {
    case AGGR_SUM_UNSIGNED: case AGGR_SUM_SIGNED: op = valueBytes == 4 ? OP_SUM_I32 : OP_SUM_I64; w = valueBytes == 4 ? 4 : 8; break;
    case AGGR_SUM_FLOAT: op = valueBytes == 4 ? OP_SUM_F32 : OP_SUM_F64; w = valueBytes == 4 ? 4 : 8; break;
    case AGGR_MIN_UNSIGNED: op = OP_MIN_U32; break;
    case AGGR_MIN_SIGNED: op = OP_MIN_I32; break;
    case AGGR_MIN_FLOAT: op = OP_MIN_F32; break;
    case AGGR_MAX_UNSIGNED: op = OP_MAX_U32; break;
    case AGGR_MAX_SIGNED: op = OP_MAX_I32; break;
    case AGGR_MAX_FLOAT: op = OP_MAX_F32; break;
    case AGGR_AVG_FLOAT: op = OP_AVG; w = 8; break;
    default: throw EngineError("Unsupported aggregation function type");
  }
  if (width) *width = w;
  return op;
}
#endif  // !__CUDACC_RTC__

#ifdef __CUDACC__
__device__ __forceinline__ uint64_t rollingAvg(uint64_t lhs, uint64_t rhs) {
  uint32_t lc = (uint32_t)(lhs >> 32), rc = (uint32_t)(rhs >> 32), total = lc + rc;
  if (total == 0) return 0;
  // divide first, as the reference does (avoids overflow of the weighted sum)
  float res = __fadd_rn(__fmul_rn(__fdiv_rn(__uint_as_float((uint32_t)lhs), (float)total), (float)lc),
                        __fmul_rn(__fdiv_rn(__uint_as_float((uint32_t)rhs), (float)total), (float)rc));
  return ((uint64_t)total << 32) | __float_as_uint(res);
}

// Float MIN / MAX keep a NaN once one is folded in: the value of a group whose rows are NaN is NaN, as the reference's
// Reduce gives it, whatever neutral element the accumulator started from (an ordered compare alone never lets a NaN in).
__device__ __forceinline__ uint64_t aggCombine(AggOp op, uint64_t a, uint64_t b) {
  switch (op) {
    case OP_SUM_I32: return (uint32_t)((uint32_t)a + (uint32_t)b);
    case OP_SUM_F32: return __float_as_uint(__fadd_rn(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b)));
    case OP_SUM_I64: return a + b;
    case OP_SUM_F64: return (uint64_t)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
    case OP_MIN_U32: return (uint32_t)b < (uint32_t)a ? (uint32_t)b : (uint32_t)a;
    case OP_MIN_I32: return (int32_t)(uint32_t)b < (int32_t)(uint32_t)a ? (uint32_t)b : (uint32_t)a;
    case OP_MIN_F32: {
      const float x = __uint_as_float((uint32_t)a), y = __uint_as_float((uint32_t)b);
      return (y < x || (y != y && x == x)) ? (uint32_t)b : (uint32_t)a;
    }
    case OP_MAX_U32: return (uint32_t)a < (uint32_t)b ? (uint32_t)b : (uint32_t)a;
    case OP_MAX_I32: return (int32_t)(uint32_t)a < (int32_t)(uint32_t)b ? (uint32_t)b : (uint32_t)a;
    case OP_MAX_F32: {
      const float x = __uint_as_float((uint32_t)a), y = __uint_as_float((uint32_t)b);
      return (x < y || (y != y && x == x)) ? (uint32_t)b : (uint32_t)a;
    }
    default: return rollingAvg(a, b);
  }
}

__device__ __forceinline__ uint64_t loadMeasure(const uint8_t *p, size_t i, int width) {
  return width == 4 ? (uint64_t)reinterpret_cast<const uint32_t *>(p)[i] : reinterpret_cast<const uint64_t *>(p)[i];
}
__device__ __forceinline__ void storeMeasure(uint8_t *p, size_t i, int width, uint64_t v) {
  if (width == 4) reinterpret_cast<uint32_t *>(p)[i] = (uint32_t)v;
  else reinterpret_cast<uint64_t *>(p)[i] = v;
}

// Atomic fold of v into *addr (global memory).  Float min/max and AVG use CAS loops.
__device__ __forceinline__ void aggAtomic(AggOp op, void *addr, uint64_t v) {
  switch (op) {
    case OP_SUM_I32: atomicAdd(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); break;
    case OP_SUM_F32: atomicAdd(reinterpret_cast<float *>(addr), __uint_as_float((uint32_t)v)); break;
    case OP_SUM_I64: atomicAdd(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)v); break;
    case OP_SUM_F64: atomicAdd(reinterpret_cast<double *>(addr), __longlong_as_double((long long)v)); break;
    case OP_MIN_U32: atomicMin(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); break;
    case OP_MIN_I32: atomicMin(reinterpret_cast<int *>(addr), (int)(uint32_t)v); break;
    case OP_MAX_U32: atomicMax(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); break;
    case OP_MAX_I32: atomicMax(reinterpret_cast<int *>(addr), (int)(uint32_t)v); break;
    case OP_MIN_F32: case OP_MAX_F32: {
      unsigned int *a = reinterpret_cast<unsigned int *>(addr);
      unsigned int old = *a, assumed;
      do {
        assumed = old;
        unsigned int want = (unsigned int)aggCombine(op, assumed, v);
        if (want == assumed) break;
        old = atomicCAS(a, assumed, want);
      } while (old != assumed);
      break;
    }
    default: {
      unsigned long long *a = reinterpret_cast<unsigned long long *>(addr);
      unsigned long long old = *a, assumed;
      do {
        assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)aggCombine(op, assumed, v));
      } while (old != assumed);
      break;
    }
  }
}
#endif

}  // namespace aresb
