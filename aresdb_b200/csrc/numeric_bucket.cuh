// numeric_bucket.cuh — the numeric bucketizer (PLAN_FN_NUMERIC_BUCKET, batch_plan.h): a value's bucket ordinal in the
// width, log-base or manual-partition form.  Pasted into the NVRTC kernel text (build.py: JIT_PRELUDE_FILES) and included
// by the host, which states the width form with the same function (jitAnalyzeDense).  NVRTC-clean: no host headers.
#pragma once
#include "cell.cuh"

namespace aresb {

constexpr int kJitMaxBuckets = 4;                 // = ARES_MAX_PLAN_BUCKETIZERS
constexpr uint32_t kBucketSmemBytes = 2048;       // shared memory a partition table takes in the kernel (255 doubles)
enum BucketKind : uint8_t { BK_WIDTH = 1, BK_LOG = 2, BK_PARTITIONS = 3 };   // = PlanBucketizerKind

// One bucketizer of a plan, as the kernel reads it (JitParams::bk).  Every number is runtime data: another width, base or
// table runs the same kernel.
struct JitBucket {
  const double *bounds;   // log table t[0..n-1] / partitions p[0..n-1], device memory
  double param;           // w (width form)
  float invLog2;          // 1 / log2(b) (log form: the first guess of the ordinal)
  int32_t logMin;         // exponent of t[0]
  uint32_t n;
  uint32_t pad;
};

constexpr double kMaxFinite = 1.7976931348623157e308;

// fl(a * b): one IEEE double multiply, never contracted into a fused multiply-add, on either side
ARES_HD double bucketMul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  volatile double r = a * b;
  return r;
#endif
}

// Width form: the k with fl(k * w) <= x < fl((k + 1) * w), for a finite x and a finite w > 0.  floor(x / w) is within one
// step of it (the quotient is correctly rounded and below 2^31 in magnitude wherever k fits Int32); the two products settle
// it.  false: k does not fit Int32.
ARES_HD bool widthOrdinal(double x, double w, int32_t &out) {
  double k = floor(x / w);
  if (bucketMul(k, w) > x) k -= 1.0;
  else if (bucketMul(k + 1.0, w) <= x) k += 1.0;
  if (!(k >= -2147483648.0 && k <= 2147483647.0)) return false;
  out = (int32_t)k;
  return true;
}

// Log form, first guess of j with t[j] <= x < t[j + 1] for x > 0 (clamped to the table; settled against it by the caller)
ARES_HD int32_t logGuess(double x, float invLog2, int32_t logMin, uint32_t n) {
  int32_t g = (int32_t)floorf(log2f((float)x) * invLog2) - logMin;
  const int32_t last = (int32_t)n - 2;
  return g < 0 ? 0 : g > last ? last : g;
}

#ifdef __CUDACC__
// The bucket ordinal of operand `a` (class ic): Int32 (width), Uint16 (log) or Uint8 (partitions).  NULL, NaN and the
// values the form leaves out give NULL.  `table`: the form's bounds (partitions: the CTA's shared-memory copy).
template <int KIND>
__device__ __forceinline__ Cell numericBucket(Cell a, ValClass ic, const JitBucket &B, const double *table) {
  Cell r; r.v = 0; r.valid = false;
  if (!a.valid) return r;
  const double x = asF64(cvt(a.v, ic, VC_F64));
  if (x != x) return r;
  if (KIND == BK_WIDTH) {
    int32_t k;
    if (!(x >= -kMaxFinite && x <= kMaxFinite) || !widthOrdinal(x, B.param, k)) return r;
    r.v = (uint32_t)k;
  } else if (KIND == BK_LOG) {
    if (!(x > 0.0 && x <= kMaxFinite)) return r;
    int32_t j = logGuess(x, B.invLog2, B.logMin, B.n);
    const int32_t last = (int32_t)B.n - 2;
    while (j > 0 && __ldg(table + j) > x) j--;
    while (j < last && __ldg(table + j + 1) <= x) j++;
    if (__ldg(table + j) > x || !(x < __ldg(table + j + 1))) return r;   // outside the table
    r.v = (uint32_t)j;
  } else {
    uint32_t lo = 0;   // number of partitions <= x (upper bound; n <= 255)
#pragma unroll
    for (uint32_t s = 128; s; s >>= 1)
      if (lo + s <= B.n && table[lo + s - 1] <= x) lo += s;
    r.v = lo;
  }
  r.valid = true;
  return r;
}
#endif

}  // namespace aresb
