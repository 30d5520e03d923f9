// jit_kernel_head.cuh — first half of the NVRTC-specialised fused kernel's source text: the quad
// loaders (the runtime parameter block JitParams precedes them: jit_params.cuh).  Compiled ONLY by
// NVRTC (see jit.cu); the generated
// rowEval() for one plan shape is pasted between this file and jit_kernel_tail.cuh, after a
// block of #defines / constexpr tables describing the shape (tile size, stage layout, key words,
// aggregate op).  Everything shape-dependent is a compile-time constant; only pointers, literal
// operands and row counts are runtime values, so one compiled kernel serves every batch and every
// query with the same structure.
namespace aresb {

// rows 4q .. 4q+3 of a staged value column of W bytes per value
template <int W, bool SIGNED>
__device__ __forceinline__ void ldq(const uint8_t *vals, uint32_t q, uint32_t (&v)[4]) {
  if (W == 4) {
    uint4 x = *reinterpret_cast<const uint4 *>(vals + 16 * q);
    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
  } else if (W == 2) {
    uint2 x = *reinterpret_cast<const uint2 *>(vals + 8 * q);
    if (SIGNED) {
      v[0] = (uint32_t)(int32_t)(int16_t)(x.x & 0xffff); v[1] = (uint32_t)((int32_t)x.x >> 16);
      v[2] = (uint32_t)(int32_t)(int16_t)(x.y & 0xffff); v[3] = (uint32_t)((int32_t)x.y >> 16);
    } else {
      v[0] = x.x & 0xffff; v[1] = x.x >> 16; v[2] = x.y & 0xffff; v[3] = x.y >> 16;
    }
  } else {
    uint32_t x = *reinterpret_cast<const uint32_t *>(vals + 4 * q);
#pragma unroll
    for (int r = 0; r < 4; r++)
      v[r] = SIGNED ? (uint32_t)(int32_t)(int8_t)((x >> (8 * r)) & 0xff) : ((x >> (8 * r)) & 0xff);
  }
}

// 4 consecutive bits (rows 4q..4q+3) of a bit-packed vector whose row 0 sits at bit START_BIT
template <int START_BIT>
__device__ __forceinline__ uint32_t ldbits(const uint8_t *bits, uint32_t q) {
  if (START_BIT == 0) return (bits[q >> 1] >> ((q & 1) * 4)) & 0xF;
  const uint32_t bit = 4 * q + START_BIT;
  const uint32_t w = bits[bit >> 3] | ((uint32_t)bits[(bit >> 3) + 1] << 8);
  return w >> (bit & 7);  // callers test bits 0..3
}

// rows 4q .. 4q+3 of a run-length encoded column, decoded from its RUNS (the column is never expanded): the row numbers of
// the quad's index positions are increasing, and the run of every position of tile `tile` lies in
// [tileRun[tile], tileRun[tile + 1]] — usually one or two runs — so the quad's first row is found by a search over that
// window and the next three by stepping forward.  Neighbouring threads read the same few counts / values (broadcast hits).
template <int W, bool SIGNED>
__device__ __forceinline__ void ldrle(const RleColumn &R, uint32_t tile, const uint32_t (&rows)[4], uint32_t (&v)[4], uint32_t &validNibble) {
  uint32_t lo = R.tileRun[tile], hi = R.tileRun[tile + 1];
  while (lo < hi) {   // last run in [lo, hi] that starts at or before rows[0]
    const uint32_t mid = lo + ((hi - lo + 1) >> 1);
    if (R.counts[mid] <= rows[0]) lo = mid; else hi = mid - 1;
  }
  uint32_t p = lo;
  const uint32_t last = R.length - 1;
  validNibble = 0;
#pragma unroll
  for (int r = 0; r < 4; r++) {
    while (p < last && R.counts[p + 1] <= rows[r]) p++;
    if (W == 0) v[r] = (R.values[(p + R.startBit) >> 3] >> ((p + R.startBit) & 7)) & 1u;
    else if (W == 1) v[r] = SIGNED ? (uint32_t)(int32_t)reinterpret_cast<const int8_t *>(R.values)[p] : R.values[p];
    else if (W == 2) v[r] = SIGNED ? (uint32_t)(int32_t)reinterpret_cast<const int16_t *>(R.values)[p] : reinterpret_cast<const uint16_t *>(R.values)[p];
    else v[r] = reinterpret_cast<const uint32_t *>(R.values)[p];
    validNibble |= ((R.nulls[(p + R.startBit) >> 3] >> ((p + R.startBit) & 7)) & 1u) << r;
  }
}

// x / d for a runtime-constant divisor as the high word of a 64x32-bit product (Lemire's fastdiv):
// M = floor((2^64 - 1) / d) + 1; exact for every 32-bit x and d >= 2 (for d = 1, M wraps to 0).  Two IMAD.WIDE.
__device__ __forceinline__ uint32_t fastDivU32(uint32_t x, unsigned long long M) {
  const uint32_t carry = __umulhi((uint32_t)M, x);
  const unsigned long long hi = (unsigned long long)(uint32_t)(M >> 32) * x + carry;
  return (uint32_t)(hi >> 32);
}
// Quotient / remainder / floor-to-multiple with C semantics (truncation, sign follows the dividend)
// for a signed or unsigned 32-bit x and a positive literal d.  WHAT: 0 = x / d, 1 = x % d, 2 = x - x % d.
template <int WHAT, bool SIGNED>
__device__ __forceinline__ uint32_t fastDivOp(uint32_t x, uint32_t d, unsigned long long M) {
  const bool neg = SIGNED && (int32_t)x < 0;
  const uint32_t ux = neg ? 0u - x : x;
  const uint32_t q = fastDivU32(ux, M);
  const uint32_t res = WHAT == 0 ? q : WHAT == 1 ? ux - q * d : q * d;
  return neg ? 0u - res : res;
}

__device__ __forceinline__ bool bitOf(const uint8_t *p, uint32_t bit) { return (p[bit >> 3] >> (bit & 7)) & 1; }

}  // namespace aresb
