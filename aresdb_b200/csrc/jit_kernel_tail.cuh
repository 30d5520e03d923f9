// jit_kernel_tail.cuh — second half of the NVRTC-specialised fused kernel: the persistent
// tile loop (TMA-staged ring of JIT_STAGES buffers), aggregation of the surviving rows into the
// CTA-private shared table, and the flush into the global table.  The shape macros
// (JIT_TILE_ROWS, JIT_STAGE_BYTES, JIT_SMEM_SLOTS, JIT_KW, JIT_AGG_OP, JIT_HASH_BITS,
// JIT_ROW_BYTES, JIT_THREADS, JIT_NUM_PARTS + kPartSmemOff/kPartBytes/kPartTileStride) and
// rowEval() precede this text.  JIT_NMEAS > 1: the plan's measure roots feed that many states (direct-indexed form), and
// the shape describes each measure's form in kMeas* tables (kMeasOp, kMeasAcc, kMeasFlags, kMeasCheck, kMeasSmemOff).
// A plan with one measure takes them from its own JIT_AGG_OP / JIT_DENSE_* macros, here; the global slot array
// (JIT_DENSE 2) has no flags.
#ifndef JIT_NMEAS
#define JIT_NMEAS 1
#define JIT_MEAS_REST(v, w)
#define JIT_MEAS_REST1(v)
namespace aresb {
__device__ constexpr int kMeasOp[1] = {JIT_AGG_OP};
__device__ constexpr int kMeasAcc[1] = {JIT_DENSE_ACC};
__device__ constexpr bool kMeasFlags[1] = {JIT_DENSE != 2 && JIT_DENSE_FLAGS};
__device__ constexpr bool kMeasCheck[1] = {JIT_DENSE_CHECK};
__device__ constexpr uint32_t kMeasSmemOff[1] = {0};
}  // namespace aresb
#endif
// Plans with member filters (PLAN_SINK_MEASURE_FILTER) define JIT_LIVE_ARG(x) as `, x`: their evaluators then report in
// live[M] the rows alive for measure M.  Without, every measure takes every alive row (live[M] stays 0xF).
#ifndef JIT_LIVE_ARG
#define JIT_LIVE_ARG(x)
#endif
// Plans whose measures differ in their dimensions (PLAN_SINK_MEMBER_DIMENSION) define JIT_MDIMS 1 and the per-measure
// tables kMeasCap (slots of the measure's region) and kMeasDims (its dimensions, bit k = dense dimension k): rowEval then
// gives each measure its own slot (dslot[M]), rowEvalGeneric the dimension values instead of a packed key, and
// memberPack<M> packs measure M's row.
#ifndef JIT_MDIMS
#define JIT_MDIMS 0
#endif
#if JIT_MDIMS
#define JIT_NSLOT JIT_NMEAS
#define JIT_DSLOT(d) d
#define JIT_DIM_ARG(dv, dvb) , dv, dvb
#else
#define JIT_NSLOT 1
#define JIT_DSLOT(d) d[0]
#define JIT_DIM_ARG(dv, dvb)
#endif
namespace aresb {

__device__ __forceinline__ void jitIssueTile(const JitParams &P, uint32_t tile, uint8_t *stage, uint64_t *bar) {
  mbarExpectTx(bar, JIT_STAGE_TX_BYTES);
#pragma unroll
  for (int p = 0; p < JIT_NUM_PARTS; p++)
    tmaLoad1D(stage + kPartSmemOff[p], P.partSrc[p] + (size_t)tile * kPartTileStride[p], kPartBytes[p], bar);
}

// Group identity of a packed dimension row: the row itself, or the reference's hash of it.
__device__ __forceinline__ unsigned long long jitKeyOfRow(const uint64_t (&key)[JIT_KW]) {
  if (JIT_KW == 1) return key[0];
  uint64_t w[4] = {key[0], key[JIT_KW > 1 ? 1 : 0], key[JIT_KW > 2 ? 2 : 0], key[JIT_KW > 3 ? 3 : 0]};
  return JIT_HASH_BITS == 64 ? murmur3_128_lo(w, JIT_ROW_BYTES, 0) : (unsigned long long)murmur3_32(w, JIT_ROW_BYTES, 0);
}
__device__ __forceinline__ unsigned long long jitKeyOf(const uint64_t (&key)[4][JIT_KW], const uint64_t (&meas)[4], int r) {
  unsigned long long k = jitKeyOfRow(key[r]);
  if (JIT_HLL == 1) k = (k & 0xFFFFFFFFFFFF0000ull) | (meas[r] & 0x3FFFu);  // the reference's HLL key
  return k;
}

#if JIT_DENSE
// ---- direct-indexed aggregation (zone map known for every dimension, see jit.cu) --------------------
// A row is evaluated once (filters, dimensions, slot); measure M's value goes to its own accumulators: region
// kMeasSmemOff[M] of the table area (three 32-bit piece counters per slot, or a flag byte per slot followed by 8-byte
// accumulators), the CTA's slice of its state's ctaAcc, and — for rows the fast path cannot finish — its state's group
// table.  Each measure keeps the form its single-measure plan takes (kMeasAcc / kMeasFlags / kMeasCheck, chosen by the
// host).  Where the accumulators of a measure's slots live (kMeasAcc):
//   1  shared memory (native ATOMS): 4-byte aggregates other than float min / max;
//   2  the others: row positions 0-1 of a quad go to shared memory (a CAS loop), 2-3 to the CTA's private slice of
//      global memory (fire-and-forget RED), so that neither the SM's shared-memory atomic path nor its global-atomic
//      path carries the whole stream; the flush adds the two halves;
//   4  exact integer accumulation of a bounded float sum (three 32-bit counters per slot).
// STEP(M) for every measure M (indexes past JIT_NMEAS fold to 0 in code that never runs)
#define JIT_EACH_MEASURE(STEP) { STEP(0) if (JIT_NMEAS > 1) { STEP((JIT_NMEAS > 1 ? 1 : 0)) } if (JIT_NMEAS > 2) { STEP((JIT_NMEAS > 2 ? 2 : 0)) } if (JIT_NMEAS > 3) { STEP((JIT_NMEAS > 3 ? 3 : 0)) } }
constexpr uint32_t kDenseCap = JIT_SMEM_SLOTS;   // a multiple of 16; JIT_TABLE_BYTES >= 9 * kDenseCap
// Unit of the fast path's slot offsets (dslot, repOff): bytes for the integer form of a one-measure plan, whose strides
// are pre-multiplied by the 12-byte slot (JitParams::dStrideB: one multiply-add per dimension per row and nothing else);
// slots otherwise (measures of several forms share the slot index).
constexpr uint32_t kSlotUnit = JIT_NMEAS == 1 && kMeasAcc[0] == 4 ? 12u : 1u;

// predicated single-instruction updates (no branch, no reconvergence point around them)
__device__ __forceinline__ void stsFlag(uint32_t addr, bool p) {
  asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p st.shared.u8 [%1], %2; }" ::"r"((uint32_t)p), "r"(addr), "r"(1u) : "memory");
}
template <int OP>
__device__ __forceinline__ void redGlobalPred(unsigned long long *a, uint64_t v, bool p) {
  const uint32_t pp = p;
  if (OP == OP_SUM_F64) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.add.f64 [%1], %2; }" ::"r"(pp), "l"(a), "d"(__longlong_as_double((long long)v)) : "memory");
  else if (OP == OP_SUM_I64) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.add.u64 [%1], %2; }" ::"r"(pp), "l"(a), "l"(v) : "memory");
  else if (OP == OP_SUM_I32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.add.u32 [%1], %2; }" ::"r"(pp), "l"(a), "r"((uint32_t)v) : "memory");
  else if (OP == OP_SUM_F32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.add.f32 [%1], %2; }" ::"r"(pp), "l"(a), "f"(__uint_as_float((uint32_t)v)) : "memory");
  else if (OP == OP_MIN_U32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.min.u32 [%1], %2; }" ::"r"(pp), "l"(a), "r"((uint32_t)v) : "memory");
  else if (OP == OP_MAX_U32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.max.u32 [%1], %2; }" ::"r"(pp), "l"(a), "r"((uint32_t)v) : "memory");
  else if (OP == OP_MIN_I32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.min.s32 [%1], %2; }" ::"r"(pp), "l"(a), "r"((uint32_t)v) : "memory");
  else if (OP == OP_MAX_I32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.max.s32 [%1], %2; }" ::"r"(pp), "l"(a), "r"((uint32_t)v) : "memory");
  else if (p) aggAtomic((AggOp)OP, a, v);   // float min / max, AVG: CAS loops
}
template <int OP>
__device__ __forceinline__ void redSharedPred(uint32_t addr, unsigned long long *generic, uint64_t v, bool p) {
  const uint32_t pp = p;
  if (OP == OP_SUM_I32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.shared.add.u32 [%1], %2; }" ::"r"(pp), "r"(addr), "r"((uint32_t)v) : "memory");
  else if (OP == OP_SUM_F32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.shared.add.f32 [%1], %2; }" ::"r"(pp), "r"(addr), "f"(__uint_as_float((uint32_t)v)) : "memory");
  else if (OP == OP_MIN_U32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.shared.min.u32 [%1], %2; }" ::"r"(pp), "r"(addr), "r"((uint32_t)v) : "memory");
  else if (OP == OP_MAX_U32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.shared.max.u32 [%1], %2; }" ::"r"(pp), "r"(addr), "r"((uint32_t)v) : "memory");
  else if (OP == OP_MIN_I32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.shared.min.s32 [%1], %2; }" ::"r"(pp), "r"(addr), "r"((uint32_t)v) : "memory");
  else if (OP == OP_MAX_I32) asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.shared.max.s32 [%1], %2; }" ::"r"(pp), "r"(addr), "r"((uint32_t)v) : "memory");
  else if (OP == OP_SUM_F64) {
    if (p) {   // 64-bit shared-memory adds are compare-and-swap loops on this hardware either way; keep ours minimal
      unsigned long long old, assumed;
      asm volatile("ld.shared.u64 %0, [%1];" : "=l"(old) : "r"(addr) : "memory");
      do {
        assumed = old;
        const unsigned long long want = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)assumed) + __longlong_as_double((long long)v));
        asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "r"(addr), "l"(assumed), "l"(want) : "memory");
      } while (old != assumed);
    }
  } else if (OP == OP_SUM_I64) {
    if (p) asm volatile("red.shared.add.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
  } else if (p) smemAtomic((AggOp)OP, generic, v);
}

__device__ __forceinline__ uint8_t *denseSmemBase() {
  extern __shared__ __align__(128) uint8_t denseSmem0[];
  return denseSmem0 + 128;
}

// Dense-register HLL, rows the map could not serve (`unknown`: inside the zone map, slot not resolved yet) or that lie
// outside the zone map: the group's directory slot is found the general way; resolved slots are entered into the map.
static __device__ __noinline__ void denseHllColdRows(const uint8_t *stage, uint32_t q, uint32_t row0, const JitParams &P, uint32_t nvalid,
                                                     uint32_t inRange, uint32_t unknown, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3) {
#if JIT_HLL == 2
  uint64_t key[4][JIT_KW], meas[4];
  const uint32_t slot[4] = {s0, s1, s2, s3};
  uint32_t alive = rowEvalGeneric(stage, q, row0, P, key, meas);
  alive &= (1u << nvalid) - 1u;
  volatile uint32_t *map = reinterpret_cast<volatile uint32_t *>(denseSmemBase());
#pragma unroll
  for (int r = 0; r < 4; r++) {
    if (!((alive >> r) & 1u)) continue;
    const bool in = (inRange >> r) & 1u;
    if (in && !((unknown >> r) & 1u)) continue;            // folded on the fast path
    const uint32_t ds = hllDenseLocate(P.G, nullptr, jitKeyOf(key, meas, r), JIT_KW == 1 ? nullptr : key[r]);
    if (ds == 0xFFFFFFFFu) continue;
    if (in) map[slot[r]] = ds;
    atomicMax(&P.G.regs[(size_t)ds * kHllRegisters + ((uint32_t)meas[r] & (kHllRegisters - 1))], (uint32_t)meas[r] + 1u);
  }
#endif
}

template <int M>
__device__ __forceinline__ unsigned long long *measSlice(const JitParams &P) { return P.ms[M].ctaAcc + (size_t)blockIdx.x * JIT_SMEM_SLOTS; }
// slots of measure M's region, its dimensions, and the slots its CTA-private copies span
template <int M>
__device__ __forceinline__ uint32_t measCap() {
#if JIT_MDIMS
  return kMeasCap[M];
#else
  return kDenseCap;
#endif
}
template <int M>
__device__ __forceinline__ uint32_t measDims() {
#if JIT_MDIMS
  return kMeasDims[M];
#else
  return 0xFFu;
#endif
}
template <int M>
__device__ __forceinline__ uint32_t measSlots(const JitParams &P, uint32_t denseSlots) {
  return JIT_MDIMS ? P.mRepStride[M] * P.mReps[M] : denseSlots;
}
// a quad's slots: one set (shared dimensions) or one per measure (JIT_MDIMS)
struct JitSlots { uint32_t v[JIT_NSLOT][4]; };

// Quads the fast path could not finish — out of line, rare.  The fast path only says WHICH rows were inside the zone map
// (inRange) and at which slots; everything else is recomputed here with full generality (rowEvalGeneric: alive mask,
// packed key, converted measure), so that the fast path keeps no masks, keys or doubles alive:
//   * alive rows outside the ranges (or a NULL whose stored value is not the canonical zero): the global hash table, keyed
//     like every other path (new groups park in the spill list while the table is at its growth threshold);
//   * rows inside whose value would leave a flag-less slot at its neutral element: the hash table as well;
//   * integer form: rows inside whose value is off the 2^-S grid: added in double on the CTA's L2 slice at `slot`
//     (-0.0, which would leave that half at its neutral element: the hash table).
template <int M>
__device__ __forceinline__ void coldMeasure(const JitParams &P, uint32_t alive, uint32_t inRange, const uint64_t (&key)[4][JIT_KW],
                                            const uint64_t (&meas)[4], const uint32_t (&slot)[4]) {
  constexpr int OP = kMeasOp[M];
  unsigned long long *tAcc = measSlice<M>(P);
#pragma unroll
  for (int r = 0; r < 4; r++) {
    if (!((alive >> r) & 1u)) continue;
    if ((inRange >> r) & 1u) {
      if (kMeasAcc[M] == 4) {
        const float x = (float)__longlong_as_double((long long)meas[r]);   // the measure is a float32 widened exactly
        const float y = x * P.ms[M].fxScale;
        const bool onGrid = x > 0.0f && y < 4294967296.0f && __uint2float_rn(__float2uint_rz(y)) == y;
        if (onGrid) continue;                                   // the fast path added its pieces
        if (meas[r] != 0x8000000000000000ull) { aggAtomic((AggOp)OP, tAcc + slot[r], meas[r]); continue; }
      } else {
        // flagged slots take every value; otherwise the fast path handled every value but the neutral element
        if (kMeasFlags[M] || !kMeasCheck[M] || meas[r] != P.ms[M].accNeutral) continue;
      }
    }
    globalUpdate<M>(P.ms[M].G, (AggOp)OP, jitKeyOfRow(key[r]), JIT_KW == 1 ? nullptr : key[r], meas[r], /*spillWhenStopped=*/true);
  }
}

// the rows some measure's fast path could not finish, evaluated again with full generality; `s`: the quad's slots, in slots
static __device__ __noinline__ void denseColdQuad(const uint8_t *stage, uint32_t q, uint32_t row0, const JitParams &P, uint32_t nvalid,
                                                  uint32_t inRange, const JitSlots s) {
  uint64_t key[4][JIT_KW], mv[JIT_NMEAS][4];
  uint32_t live[JIT_NMEAS];
#pragma unroll
  for (int m = 0; m < JIT_NMEAS; m++) live[m] = 0xFu;
#if JIT_MDIMS
  uint32_t dv[4][JIT_ND], dvb[4];
#endif
  uint32_t alive = rowEvalGeneric(stage, q, row0, P, key, mv[0] JIT_MEAS_REST1(mv) JIT_DIM_ARG(dv, dvb) JIT_LIVE_ARG(live));
  alive &= (1u << nvalid) - 1u;
  // (a cold row claims a group only in the tables of the measures it is alive for, keyed by their own dimensions)
#if JIT_MDIMS
#define JIT_STEP(M) {                                                  \
    uint64_t mkey[4][JIT_KW];                                          \
    _Pragma("unroll") for (int r = 0; r < 4; r++) memberPack<M>(dv[r], dvb[r], mkey[r]); \
    coldMeasure<M>(P, alive & live[M], inRange, mkey, mv[M], s.v[JIT_MDIMS ? M : 0]); }
#else
#define JIT_STEP(M) coldMeasure<M>(P, alive & live[M], inRange, key, mv[M], s.v[0]);
#endif
  JIT_EACH_MEASURE(JIT_STEP)
#undef JIT_STEP
}

// `live`: the rows of the quad alive for measure M (bit r); `fastAny` holds the rows alive for some measure inside the
// zone map; `s`: the slots, in kSlotUnit.  true: some row needs the cold path.
template <int M>
__device__ __forceinline__ bool denseMeasure(uint32_t tableAddr, const JitParams &P, const bool (&fastAny)[4], uint32_t live,
                                             const uint32_t (&s)[4], const uint64_t (&meas)[4], const uint32_t (&mraw)[4]) {
  constexpr int OP = kMeasOp[M];
  const uint32_t base = tableAddr + kMeasSmemOff[M];
  bool cold = false;
  bool fast[4];
#pragma unroll
  for (int r = 0; r < 4; r++) fast[r] = fastAny[r] && ((live >> r) & 1u) != 0;
  if (kMeasAcc[M] == 4) {
    // Exact integer accumulation of a float sum (jitAnalyzeDense): a slot is three 32-bit counters for the 11 / 11 / 10
    // bit pieces of x * 2^S, updated with fire-and-forget adds (nothing returns, nothing spins), and carries no flag —
    // it was reached iff a counter is non-zero or its double half on the L2 slice left the neutral element.  A row is
    // taken row by row — decide, then add — so that only one row's predicates are alive at a time: x > 0 on the grid
    // (y = x * 2^S is an integer below 2^32: float -> u32 -> float gives y back) adds its three pieces.  Everything else
    // in range (zeros, NULL -> +0.0, negative, off the grid, beyond the announced maximum, NaN, -0.0) is rare and is
    // finished by the cold path.
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const float x = __uint_as_float(mraw[r]);
      const float y = x * P.ms[M].fxScale;
      const uint32_t ix = __float2uint_rz(y);
      const bool onGrid = fast[r] && x > 0.0f && y < 4294967296.0f && __uint2float_rn(ix) == y;
      cold = cold || (fast[r] && !onGrid);
      if (onGrid) {   // one branch around the three adds
        const uint32_t a = base + 12u / kSlotUnit * s[r];
        asm volatile("red.shared.add.u32 [%0], %1;\n\tred.shared.add.u32 [%0+4], %2;\n\tred.shared.add.u32 [%0+8], %3;"
                     ::"r"(a), "r"(ix & 0x7FFu), "r"((ix >> 11) & 0x7FFu), "r"(ix >> 22) : "memory");
      }
    }
  } else {
    bool go[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      // no flags: a row that would leave its slot at the neutral element goes down the hash path instead
      go[r] = fast[r] && (kMeasFlags[M] || !kMeasCheck[M] || meas[r] != P.ms[M].accNeutral);
      cold = cold || (fast[r] && !go[r]);
    }
    if (kMeasFlags[M]) {
#pragma unroll
      for (int r = 0; r < 4; r++) stsFlag(base + s[r], go[r]);
    }
    unsigned long long *tAcc = measSlice<M>(P);
    unsigned long long *generic = reinterpret_cast<unsigned long long *>(denseSmemBase() + kMeasSmemOff[M] + measCap<M>());
    // (issuing the compare-and-swap loops of the shared-memory rows interleaved instead of one after the other was
    // measured and changed nothing: 0.376 vs 0.372 ms on cfg3)
    constexpr int kToShared = kMeasAcc[M] == 1 ? 4 : 2;   // row positions 0 .. kToShared-1
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (r < kToShared) redSharedPred<OP>(base + measCap<M>() + 8u * s[r], generic + s[r], meas[r], go[r]);
      else redGlobalPred<OP>(tAcc + s[r], meas[r], go[r]);
    }
  }
  return cold;
}

// `repOff`: this lane's copy of the slots (few slots are replicated per lane), in kSlotUnit — loop invariant, computed once.
__device__ __forceinline__ void jitAggregateDense(uint32_t tableAddr, const JitParams &P, const uint8_t *stage, uint32_t q, uint32_t row0,
                                                  uint32_t nvalid, uint32_t repOff, const bool (&fast)[4], bool cold,
                                                  const uint32_t (&dslot)[JIT_NSLOT][4], const uint64_t (&mv)[JIT_NMEAS][4],
                                                  const uint32_t (&mr)[JIT_NMEAS][4], const uint32_t (&live)[JIT_NMEAS]) {
  // slots: dslot + this lane's copy (JIT_MDIMS: each measure's copy follows its own slot count)
  JitSlots s;
#pragma unroll
  for (int m = 0; m < JIT_NSLOT; m++) {
    const uint32_t off = JIT_MDIMS ? (threadIdx.x & (P.mReps[m] - 1u)) * P.mRepStride[m] : repOff;
#pragma unroll
    for (int r = 0; r < 4; r++) s.v[m][r] = dslot[m][r] + off;
  }
  if (JIT_HLL == 2) {
    // Dense-register HLL addressed by the zone map: the table region is a map slot -> directory slot of the group (whose
    // 16384 registers live at regs + 16384 * that).  A known slot costs one shared-memory load and one fire-and-forget
    // RED.MAX; an unknown one (first row of the group in this CTA) goes through denseHllColdRows, which fills the map.
    // (the four map entries are read back to back — plain loads: a stale "unknown" only sends the row to the cold path,
    // which resolves the slot again — and only then the four updates are issued)
    const uint32_t *map = reinterpret_cast<const uint32_t *>(denseSmemBase());
    asm volatile("" ::: "memory");
    uint32_t ds[4];
#pragma unroll
    for (int r = 0; r < 4; r++) ds[r] = map[fast[r] ? s.v[0][r] : 0u];
    // (register index in 32 bits — the dense directory has at most 2^18 groups —, the update a PREDICATED red: no branch
    // around it, and the four addresses are ready before the first one is issued)
    uint32_t *reg[4];
#pragma unroll
    for (int r = 0; r < 4; r++) reg[r] = P.G.regs + ((ds[r] << 14) | ((uint32_t)mv[0][r] & (kHllRegisters - 1)));
    static_assert(kHllRegisters == 1u << 14, "register index packing");
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const bool known = fast[r] && ds[r] != 0xFFFFFFFFu;
      cold = cold || (fast[r] && !known);
      asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p red.global.max.u32 [%1], %2; }"
                   ::"r"((uint32_t)known), "l"(reg[r]), "r"((uint32_t)mv[0][r] + 1u) : "memory");
    }
    if (cold) {
      const uint32_t unknown = (fast[0] && ds[0] == 0xFFFFFFFFu ? 1u : 0u) | (fast[1] && ds[1] == 0xFFFFFFFFu ? 2u : 0u) |
                               (fast[2] && ds[2] == 0xFFFFFFFFu ? 4u : 0u) | (fast[3] && ds[3] == 0xFFFFFFFFu ? 8u : 0u);
      const uint32_t inRange = (fast[0] ? 1u : 0u) | (fast[1] ? 2u : 0u) | (fast[2] ? 4u : 0u) | (fast[3] ? 8u : 0u);
      // rows already folded through the map must not be folded again: hand over only unknown-slot and out-of-range rows
      denseHllColdRows(stage, q, row0, P, nvalid, inRange, unknown, s.v[0][0], s.v[0][1], s.v[0][2], s.v[0][3]);
    }
    return;
  }
  if (JIT_DENSE == 2) {
    // One accumulator array for the whole grid (more slots than a CTA holds).  No flags: a slot was reached iff it
    // differs from the aggregate's neutral element, so a row whose value would leave it there (-0.0 for float sums,
    // the extreme for min / max) goes down the hash path instead; the host only selects this form for aggregates
    // that cannot return to the neutral element otherwise.
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const bool f = fast[r] && (!JIT_DENSE_CHECK || mv[0][r] != P.accNeutral);
      cold = cold || (fast[r] && !f);
      redGlobalPred<JIT_AGG_OP>(P.gAcc + s.v[0][r], mv[0][r], f);
    }
  } else {
#define JIT_STEP(M) cold = denseMeasure<M>(tableAddr, P, fast, live[M], s.v[JIT_MDIMS ? M : 0], mv[M], mr[M]) || cold;
    JIT_EACH_MEASURE(JIT_STEP)
#undef JIT_STEP
  }
  if (cold) {
    const uint32_t inRange = (fast[0] ? 1u : 0u) | (fast[1] ? 2u : 0u) | (fast[2] ? 4u : 0u) | (fast[3] ? 8u : 0u);
#pragma unroll
    for (int m = 0; m < JIT_NSLOT; m++) {
#pragma unroll
      for (int r = 0; r < 4; r++) s.v[m][r] /= kSlotUnit;
    }
    denseColdQuad(stage, q, row0, P, nvalid, inRange, s);
  }
}

template <int M>
__device__ __forceinline__ void denseInitMeasure(const JitParams &P, uint32_t denseSlots) {
  uint8_t *base = denseSmemBase() + kMeasSmemOff[M];
  unsigned long long *tAcc = measSlice<M>(P);
  const uint32_t n = measSlots<M>(P, denseSlots);
  for (uint32_t i = threadIdx.x; i < n; i += JIT_THREADS) {
    if (kMeasFlags[M]) base[i] = 0;   // (flags only in the 9-byte form)
    if (kMeasAcc[M] != 1) tAcc[i] = P.ms[M].accNeutral;
    if (kMeasAcc[M] == 4) {
      uint32_t *c = reinterpret_cast<uint32_t *>(base) + 3u * i;
      c[0] = 0; c[1] = 0; c[2] = 0;
    } else {
      reinterpret_cast<unsigned long long *>(base + measCap<M>())[i] = P.ms[M].accNeutral;
    }
  }
}
__device__ __forceinline__ void denseInit(const JitParams &P, uint32_t denseSlots) {
#define JIT_STEP(M) denseInitMeasure<M>(P, denseSlots);
  JIT_EACH_MEASURE(JIT_STEP)
#undef JIT_STEP
}

// the CTA's slots of measure M into its state's group table: the slot index decodes to the dimension values
template <int M>
__device__ __forceinline__ void denseFlushMeasure(const JitParams &P, uint32_t denseSlots) {
  constexpr int OP = kMeasOp[M];
  const uint8_t *base = denseSmemBase() + kMeasSmemOff[M];
  unsigned long long *tAcc = measSlice<M>(P);
  const unsigned long long neutral = P.ms[M].accNeutral;
  const uint32_t n = measSlots<M>(P, denseSlots);
  for (uint32_t i = threadIdx.x; i < n; i += JIT_THREADS) {
    unsigned long long accS = neutral;
    if (kMeasAcc[M] == 4) {
      // pieces -> integer -> double: only positive values were added, so 0 = no such row (adding the neutral element
      // below is then a no-op); 2^-S is a power of two and the integer is exact below 2^53
      const uint32_t *c = reinterpret_cast<const uint32_t *>(base) + 3u * i;
      const unsigned long long v = (unsigned long long)c[0] + ((unsigned long long)c[1] << 11) + ((unsigned long long)c[2] << 22);
      if (v != 0) accS = (unsigned long long)__double_as_longlong(__ull2double_rn(v) * P.ms[M].fxInv);
    } else {
      accS = reinterpret_cast<const unsigned long long *>(base + measCap<M>())[i];
    }
    const unsigned long long accG = kMeasAcc[M] != 1 ? __ldcg(&tAcc[i]) : neutral;
    if (kMeasFlags[M] ? !base[i] : (accS == neutral && accG == neutral)) continue;
    // (JIT_MDIMS: measure M's slot decodes over its own dimensions and strides; padding slots between copies are never
    // reached)
    uint32_t rem = i % (JIT_MDIMS ? P.mRepStride[M] : P.dRepStride), dvr[JIT_ND], vb = 0;
#pragma unroll
    for (int k = JIT_ND - 1; k >= 0; k--) {
      dvr[k] = 0u;
      if (!((measDims<M>() >> k) & 1u)) continue;
      const uint32_t stride = JIT_MDIMS ? P.mStride[M][k] : P.dStride[k];
      const uint32_t ix = rem / stride;
      rem -= ix * stride;
      const bool valid = ix != P.dCnt[k];
      dvr[k] = valid ? (P.dLo[k] + ix) * P.dStep[k] : 0u;
      vb |= (valid ? 1u : 0u) << k;
    }
    uint64_t key[JIT_KW];
#if JIT_MDIMS
    memberPack<M>(dvr, vb, key);
#else
    densePack(dvr, vb, key);
#endif
    const unsigned long long k = jitKeyOfRow(key);
    // (the host does not wait for these kernels: when the table is at its growth threshold new groups are parked)
    if (kMeasAcc[M] != 1) globalUpdate<M>(P.ms[M].G, (AggOp)OP, k, JIT_KW == 1 ? nullptr : key, accG, true);
    globalUpdate<M>(P.ms[M].G, (AggOp)OP, k, JIT_KW == 1 ? nullptr : key, accS, true);
  }
}
__device__ __forceinline__ void denseFlush(const JitParams &P, uint32_t denseSlots) {
#define JIT_STEP(M) denseFlushMeasure<M>(P, denseSlots);
  JIT_EACH_MEASURE(JIT_STEP)
#undef JIT_STEP
}
#endif

// Folds the surviving rows of one quad.  Normal mode: the CTA's shared table first, the global table
// for rows it cannot take (counted in *misses).  Bypass mode (the batch has far more groups than the
// shared table holds, so looking there is wasted work): straight to the L2-resident global table,
// with the four home-slot key loads issued back to back so that their latencies overlap.  The mode
// is compiled in (JIT_BYPASS) only when AggSpec.ExpectedGroups announces such a batch, or for HLL.
__device__ __forceinline__ void jitAggregate(const SmemTable &T, const JitParams &P, uint32_t alive,
                                             const uint64_t (&key)[4][JIT_KW], const uint64_t (&meas)[4], bool allowClaim,
                                             bool bypass, uint32_t *misses) {
  constexpr AggOp op = (AggOp)JIT_AGG_OP;
  if (JIT_HLL == 2) {  // dense registers: the shared table mirrors the directory of groups
    // locate the four registers, read them back to back (the latencies overlap), then raise only those that grow
    uint32_t *reg[4];
    uint32_t cur[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      reg[r] = nullptr;
      if (!((alive >> r) & 1)) continue;
      const uint32_t slot = hllDenseLocate(P.G, JIT_SMEM_SLOTS == JIT_DENSE_SLOTS ? T.keys : nullptr, jitKeyOf(key, meas, r),
                                           JIT_KW == 1 ? nullptr : key[r]);
      if (slot != 0xFFFFFFFFu) reg[r] = &P.G.regs[(size_t)slot * kHllRegisters + ((uint32_t)meas[r] & (kHllRegisters - 1))];
    }
#pragma unroll
    for (int r = 0; r < 4; r++) cur[r] = reg[r] ? __ldcg(reg[r]) : 0xFFFFFFFFu;
#pragma unroll
    for (int r = 0; r < 4; r++)
      if (cur[r] < (uint32_t)meas[r] + 1u) atomicMax(reg[r], (uint32_t)meas[r] + 1u);
    return;
  }
  if (JIT_BYPASS && bypass) {
    unsigned long long k[4], seen[4];
    uint32_t slot[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (!((alive >> r) & 1)) continue;
      k[r] = jitKeyOf(key, meas, r);
      slot[r] = globalHome(P.G, k[r]);
      asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(seen[r]) : "l"(P.G.keys + slot[r]));
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
      if (!((alive >> r) & 1)) continue;
      if (seen[r] == k[r]) aggAtomic(op, &P.G.acc[slot[r]], meas[r]);
      else globalUpdate(P.G, op, k[r], JIT_KW == 1 ? nullptr : key[r], meas[r]);
    }
    return;
  }
#pragma unroll
  for (int r = 0; r < 4; r++) {
    if (!((alive >> r) & 1)) continue;
    const unsigned long long k = jitKeyOf(key, meas, r);
    const uint64_t *roww = JIT_KW == 1 ? nullptr : key[r];
    if (!smemUpdate(T, P.G, op, k, roww, meas[r], allowClaim)) {
      if (JIT_BYPASS) atomicAdd(misses, 1u);
      globalUpdate(P.G, op, k, roww, meas[r]);
    }
  }
}

extern "C" __global__ void __launch_bounds__(JIT_THREADS, 1) aresFusedJit(const __grid_constant__ JitParams P) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem);        // full[JIT_STAGES]: bytes of a tile have landed
  uint64_t *empty = bars + kMaxStages;                        // empty[JIT_STAGES]: every warp is done with the stage
  uint32_t *claims = reinterpret_cast<uint32_t *>(smem + 64);   // occupied slots of the shared table
  uint32_t *misses = claims + 1;                                // rows the shared table turned away
  unsigned long long *tKeys = reinterpret_cast<unsigned long long *>(smem + 128);
  // keys of the CTA's table in shared memory (latency-critical, read-mostly); accumulators in an
  // L2-resident private slice of global memory, updated with fire-and-forget RED
  unsigned long long *tAcc = P.ctaAcc + (size_t)blockIdx.x * JIT_SMEM_SLOTS;
  uint8_t *stages = smem + 128 + JIT_TABLE_BYTES;

  SmemTable T;
  T.keys = tKeys; T.acc = tAcc; T.claims = claims; T.mask = JIT_SMEM_SLOTS - 1;
#if JIT_DENSE
  // no keys: the slot index IS the group; the table area holds each measure's accumulators (and "reached" flags)
  uint32_t tableAddr = smemAddr(tKeys);
  asm volatile("" : "+r"(tableAddr));   // keep it in a register: the compiler otherwise rebuilds the window address per store
  const uint32_t denseSlots = JIT_DENSE == 2 ? 0u : P.dRepStride * P.dReps;   // <= kDenseCap (host); 2: nothing CTA-private
  const uint32_t repOff = JIT_DENSE == 2 ? (blockIdx.x & (P.dReps - 1u)) * P.dRepStride
                                         : (threadIdx.x & (P.dReps - 1u)) * P.dRepStride * kSlotUnit;   // this lane's copy of the slots
  for (uint32_t i = threadIdx.x; JIT_HLL == 2 && i < denseSlots; i += JIT_THREADS) reinterpret_cast<uint32_t *>(tKeys)[i] = 0xFFFFFFFFu;
  if (JIT_HLL != 2) denseInit(P, denseSlots);
#else
  for (uint32_t i = threadIdx.x; i < JIT_SMEM_SLOTS; i += JIT_THREADS) {
    tKeys[i] = kEmptyKey;
    if (JIT_HLL != 2) tAcc[i] = P.accNeutral;
  }
#endif
  if (threadIdx.x == 0) {
    *claims = 0;
    *misses = 0;
    for (int s = 0; s < JIT_STAGES; s++) {
      mbarInit(&bars[s], 1);
      mbarInit(&empty[s], JIT_THREADS / 32 - 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
#ifdef JIT_BUCKETS
  jitStageBuckets(P);   // partition tables of the plan's numeric bucketizers
#endif
  __syncthreads();

  // Warp specialisation: the last warp is the TMA producer (one lane issues the bulk copies as soon
  // as a stage is released), the other JIT_THREADS/32 - 1 warps consume; a tile holds exactly one quad
  // per consumer thread (JIT_TILE_ROWS = 128 x consumer warps).  No CTA-wide barrier in the loop.
  constexpr uint32_t kConsumerThreads = JIT_THREADS - 32;
  static_assert(JIT_TILE_ROWS == kConsumerThreads * 4, "one quad per consumer thread");
  const uint32_t first = blockIdx.x, step = gridDim.x;
  // Growth of the group table (AggState: capacity doubles when half full).  The claim that crosses DevTable::growAt
  // raises the STOP flag; a consumer warp that sees it before a tile stops folding rows ("drains": it keeps the ring
  // protocol alive but touches nothing), and records how many tile iterations it has folded.  The host then grows the
  // table and launches the kernel again with `resume`: every warp skips the iterations it already folded.  Nothing is
  // lost and nothing is counted twice; the unit is one warp's 128 rows of one tile.
  // (Direct-indexed kernels never drain — the host does not wait for them: their out-of-range rows and their flush park
  // new groups in DevTable::spill while the table is at its threshold.)
  constexpr bool kCanDrain = JIT_DENSE == 0;
  const uint32_t progIdx = blockIdx.x * kProgressWarps + (threadIdx.x >> 5);
  uint32_t myStart = 0;
  if (kCanDrain && P.resume) myStart = P.G.progress[progIdx];
  bool draining = false;
  uint32_t foldedUntil = 0xFFFFFFFFu;   // iterations folded when the warp stopped (0xFFFFFFFF: all)
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      uint32_t it = 0;
      for (uint32_t t = first; t < P.numFullTiles; t += step, it++) {
        const uint32_t s = it % JIT_STAGES;
        if (it >= JIT_STAGES) mbarWait(&empty[s], ((it / JIT_STAGES) - 1) & 1);
        jitIssueTile(P, t, stages + (size_t)s * JIT_STAGE_BYTES, &bars[s]);
      }
    }
  } else {
    uint32_t it = 0;
    for (uint32_t t = first; t < P.numFullTiles; t += step, it++) {
      const uint32_t s = it % JIT_STAGES, parity = (it / JIT_STAGES) & 1;
      // (read before the wait: the L2 round trip overlaps with it; a slightly older value only delays the stop by a tile)
      const uint32_t stopFlag = kCanDrain ? __ldcg(&P.G.counters[3]) : 0u;   // (L2, not system scope)
      mbarWait(&bars[s], parity);
      if (!draining && it >= myStart && stopFlag != 0u) {
        draining = true;
        foldedUntil = it;
      }
      if (draining || it < myStart) {   // nothing to fold: release the stage and move on
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbarArrive(&empty[s]);
        continue;
      }
      const uint8_t *stage = stages + (size_t)s * JIT_STAGE_BYTES;
      // (direct-indexed forms have no shared key table: no volatile read of its fill per tile)
      const bool allowClaim = JIT_DENSE != 0 || *reinterpret_cast<volatile uint32_t *>(claims) < (JIT_SMEM_SLOTS / 4) * 3;
      // the shared table is full and has turned away several times its size in rows: stop consulting it
      const bool bypass = JIT_BYPASS && !allowClaim && *reinterpret_cast<volatile uint32_t *>(misses) > 4u * JIT_SMEM_SLOTS;
      {
        const uint32_t q = threadIdx.x;
#if JIT_DENSE
        uint32_t dslot[JIT_NSLOT][4];
        bool fast[4], anySlow;
        uint64_t mv[JIT_NMEAS][4];
        uint32_t mr[JIT_NMEAS][4], live[JIT_NMEAS];
#pragma unroll
        for (int m = 0; m < JIT_NMEAS; m++) live[m] = 0xFu;
        if (rowEval(stage, q, t * JIT_TILE_ROWS + q * 4, P, 4u, fast, anySlow, JIT_DSLOT(dslot), mv[0], mr[0] JIT_MEAS_REST(mv, mr) JIT_LIVE_ARG(live)))
          jitAggregateDense(tableAddr, P, stage, q, t * JIT_TILE_ROWS + q * 4, 4u, repOff, fast, anySlow, dslot, mv, mr, live);
        (void)allowClaim; (void)bypass;
#else
        uint64_t meas[4], key[4][JIT_KW];
        const uint32_t alive = rowEval(stage, q, t * JIT_TILE_ROWS + q * 4, P, key, meas);
        jitAggregate(T, P, alive, key, meas, allowClaim, bypass, misses);
#endif
      }
      __syncwarp();
      if ((threadIdx.x & 31) == 0) mbarArrive(&empty[s]);
    }
  }
  if (kCanDrain && threadIdx.x < kConsumerThreads && (threadIdx.x & 31) == 0) P.G.progress[progIdx] = foldedUntil;
  // ---- tail: the rows after the last full tile (< JIT_TILE_ROWS + 128) are copied into stage 0 by
  // the threads themselves, byte-exact (nothing beyond a column's last byte is touched), and go
  // through the same rowEval.  One CTA does it; rows past the end are masked dead.  (A stopped run leaves the tail to
  // the resumed one: DevTable::progress[kProgressTail] records that it has been folded.)
  volatile uint32_t &sDoTail = *reinterpret_cast<volatile uint32_t *>(smem + 72);   // header word (no static shared memory:
                                                                                     // the dynamic part takes the CTA's whole budget)
  if (threadIdx.x == 0) {
    if (kCanDrain && !P.resume && blockIdx.x == gridDim.x - 1) P.G.progress[kProgressTail] = 0u;   // a fresh batch
    sDoTail = blockIdx.x == gridDim.x - 1 &&
              (!kCanDrain || (*reinterpret_cast<volatile uint32_t *>(&P.G.counters[3]) == 0u && !(P.resume && P.G.progress[kProgressTail] != 0u)));
  }
  __syncthreads();
  if (sDoTail) {
    if (kCanDrain && threadIdx.x == 0) P.G.progress[kProgressTail] = 1u;
    uint32_t done = P.numFullTiles * JIT_TILE_ROWS;
    while (done < P.numRows) {
      __syncthreads();  // every warp has left the ring / the previous tail tile
      const uint32_t rows = P.numRows - done < JIT_TILE_ROWS ? P.numRows - done : JIT_TILE_ROWS;
#pragma unroll
      for (int p = 0; p < JIT_NUM_PARTS; p++) {
        // bytes of this part that exist for `rows` rows: values rows*width; bit-packed parts cover
        // bits [startBit, startBit + rows)
        const uint32_t per = kPartTileStride[p];                       // bytes per full tile
        // (kPartIsBits 2: the base counts, one 4-byte element more than rows)
        const uint32_t valid = kPartIsBits[p] == 2 ? (rows + 1) * 4
                             : kPartIsBits[p] ? (rows + kPartStartBit[p] + 7) / 8 : (uint32_t)((size_t)per * rows / JIT_TILE_ROWS);
        const uint8_t *src = P.partSrc[p] + (size_t)(done / JIT_TILE_ROWS) * per;
        uint8_t *dst = stages + kPartSmemOff[p];
        for (uint32_t i = threadIdx.x; i < kPartBytes[p]; i += JIT_THREADS) dst[i] = i < valid ? src[i] : (uint8_t)0;
      }
      __syncthreads();
      for (uint32_t q = threadIdx.x; q * 4 < rows; q += JIT_THREADS) {
        const uint32_t nvalid = rows - q * 4 < 4 ? rows - q * 4 : 4;
#if JIT_DENSE
        uint32_t dslot[JIT_NSLOT][4];
        bool fast[4], anySlow;
        uint64_t mv[JIT_NMEAS][4];
        uint32_t mr[JIT_NMEAS][4], live[JIT_NMEAS];
#pragma unroll
        for (int m = 0; m < JIT_NMEAS; m++) live[m] = 0xFu;
        if (rowEval(stages, q, done + q * 4, P, nvalid, fast, anySlow, JIT_DSLOT(dslot), mv[0], mr[0] JIT_MEAS_REST(mv, mr) JIT_LIVE_ARG(live)))
          jitAggregateDense(tableAddr, P, stages, q, done + q * 4, nvalid, repOff, fast, anySlow, dslot, mv, mr, live);
#else
        uint64_t meas[4], key[4][JIT_KW];
        uint32_t alive = rowEval(stages, q, done + q * 4, P, key, meas);
        alive &= (1u << nvalid) - 1u;
        jitAggregate(T, P, alive, key, meas, true, false, misses);
#endif
      }
      done += rows;
    }
  }
  __syncthreads();
  if (JIT_HLL == 2) return;  // nothing CTA-private to fold: registers are updated in place
#if JIT_DENSE == 2
  return;   // denseFoldKernel (batch_plan.cu) folds the shared array after the batch
#elif JIT_DENSE
  denseFlush(P, denseSlots);
  return;
#endif
  // (the CTA's table is folded whatever the state of the global one: groups it cannot take right now are parked)
  for (uint32_t i = threadIdx.x; i < JIT_SMEM_SLOTS; i += JIT_THREADS) {
    unsigned long long k = tKeys[i];
    if (k != kEmptyKey) globalUpdate(P.G, (AggOp)JIT_AGG_OP, k, nullptr, __ldcg(&tAcc[i]), /*spillWhenStopped=*/true);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *P.G.occPublish = *reinterpret_cast<volatile uint32_t *>(&P.G.counters[0]);
}

}  // namespace aresb
