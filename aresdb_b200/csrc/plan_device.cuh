// plan_device.cuh — the device form of a BatchPlan: what compilePlan() (batch_plan.cu) produces and
// the NVRTC generator (jit.cu) specialises the fused kernel for.
#pragma once
#include "column.cuh"
#include "fused_device.cuh"
#include "jit_params.cuh"
#include "join.cuh"

namespace aresb {

constexpr int kSmemBudget = 232448;           // 227 KB: the most dynamic shared memory a CTA may opt into on sm_90
constexpr int kJitThreads = 1024;
constexpr int kMaxGridCtas = 160;             // persistent grid: one CTA per SM (132 on H100 SXM)
static_assert(kMaxPlanInsts == ARES_MAX_PLAN_INSTS && kMaxForeignTables == ARES_MAX_FOREIGN_TABLES &&
              kMaxForeignCols == ARES_MAX_FOREIGN_COLUMNS, "jit_params.cuh restates the plan bounds of batch_plan.h");

enum KeyMode : uint8_t { KEY_PACKED = 0, KEY_HASHED = 1 };
enum OperandKind : uint8_t { OPK_NONE = 0, OPK_COLUMN = 1, OPK_CONST = 2, OPK_STACK = 3, OPK_FOREIGN = 4 };

struct DevColumn {
  InputDesc in;            // how to read it straight from global memory (any mode)
  uint32_t smemValues;     // byte offsets inside one stage
  uint32_t smemNulls;
  uint32_t tileValueBytes; // bytes of one full tile
  uint32_t tileNullBytes;
  uint8_t width;           // bytes per value, 0 for bit-packed bool
  uint8_t staged;          // values staged
  uint8_t hasNulls;        // mode 2 bitmap staged
  uint8_t used;            // some instruction reads the column (unreferenced columns of the batch cost nothing)
  uint32_t rangeLo, rangeHi;  // zone map of the batch (BatchPlan.Ranges): valid values lie in [rangeLo, rangeHi]
  uint8_t rangeKnown;
  uint8_t rle;             // run-length encoded (mode 3) column decoded in the kernel from its runs — never expanded, never staged
  uint8_t expand;          // run-length encoded column read as a plain copy: `in` describes the copy (base set when it is made)
  uint8_t pad[1];
  const uint32_t *tileRun; // rle: run that holds the first index position of every tile (+ one entry for the last position)
};

struct DevInst {
  uint32_t aconst, bconst;
  uint8_t nops, fn, sink, sinkArg;
  uint8_t akind, acol, aclass, avalid;
  uint8_t bkind, bcol, bclass, bvalid;
  uint8_t tclass;   // class the functor runs in
  uint8_t rclass;   // class of the functor result
  uint8_t oclass;   // class of the sink element
  uint8_t wide;     // 1: 8/16-byte column copied verbatim into a dimension
  uint8_t rowOff, width, nullOff;
  int8_t magic;       // slot in JitParams::magic of a fast division (isFastDiv), -1: none
  int8_t asrc, bsrc;  // instruction that pushed the value a stack operand pops, -1: not a stack operand
  uint8_t bucket;     // PLAN_FN_NUMERIC_BUCKET: index into DevPlan::buckets
};

// One measure root of a plan: what the single-measure plan of its state decided (compilePlan + layoutStages on that plan),
// so that each measure of a plan that feeds several states (DevPlan::nmeas > 1) takes the accumulation form it would take
// alone.  A single-measure plan describes its own measure in meas[0].
struct DevMeasure {
  DevTable G;                    // the state's group table and CTA slices (filled just before the launch)
  unsigned long long *ctaAcc;
  uint64_t measureIdentity, accNeutral;
  int8_t inst;                   // the measure root in the shared plan
  int8_t fxShift;
  uint8_t aggOp, measWidth, skipCount, neutralSafe, denseFx, pad;
  // member dimensions (DevPlan::memberDims): the state's dimensions among the plan's (bit j = dense dimension j), where
  // each sits in the state's row (byte offset of the value, of the validity byte; by member dimension root), its slots
  // (prod of (count + 1) over its dimensions) and the slots of its region in the CTA (>= total, set by layoutStages)
  uint8_t dims;
  uint8_t rowOff[kJitMaxDenseDims], nullOff[kJitMaxDenseDims];
  uint32_t total, slots;
};

struct DevPlan {
  DevColumn cols[kMaxPlanCols];
  DevInst insts[ARES_MAX_PLAN_INSTS];
  const uint32_t *baseCounts;
  unsigned long long *ctaAcc;   // [grid][smemSlots] accumulator slices (global, L2-resident)
  uint32_t startCount;
  uint32_t numRows;
  uint32_t tileRows;
  uint32_t numFullTiles;   // staged tiles; the tail (fewer than tileRows + 128 rows) is copied by the kernel itself
  uint32_t stageBytes;
  uint32_t smemSlots;      // shared table slots (power of two)
  uint32_t numStages;      // depth of the TMA ring (2..kMaxStages)
  uint32_t denseSlots;     // dense HLL mode: slots of the group directory (0 otherwise)
  uint32_t smemBc;         // staged base counts (RLE batches, SUM / AVG): byte offset inside a stage, tileBcBytes bytes
  uint32_t tileBcBytes;    // (tileRows + 4) * 4, or 0 when the base counts are not staged
  int32_t ncols, ninsts, lastFilter;
  uint64_t measureIdentity;  // NULL measure -> this (sink class bits)
  uint64_t accNeutral;       // neutral element of the combine op
  uint8_t keyMode, rowBytes, valueBytes, hashBits;
  uint8_t aggOp, measWidth, measClass, skipCount;
  uint8_t hasMeasure, hll, bypassOk;
  // direct-indexed aggregation (jitAnalyzeDense; denseNd == 0: hash table).  Dimension k is produced by instruction
  // denseInst[k]; its slot index is (quotient or value) - denseLo[k], below denseCnt[k]; index denseCnt[k] = NULL.
  uint8_t denseNd;
  uint8_t denseInst[8], denseViaQuot[8], denseNullCanon[8];
  uint32_t denseLo[8], denseCnt[8], denseStep[8];
  // quotient dimensions whose dividend range is small (span * step <= 2^32): index = umulhi(x - denseBase, 2^32 / step + 1),
  // in range iff x - denseBase < denseSpan (one subtraction, one multiply, one compare per row)
  uint8_t denseSpan32[8];
  uint32_t denseBase[8], denseSpan[8];
  uint32_t denseTotal;     // slots of one copy = prod (denseCnt[k] + 1)
  uint32_t tableBytes;     // shared memory between the header and the first stage (keys, or flags + accumulators)
  // more slots than a CTA holds: ONE array of accumulators in global memory (L2-resident) shared by all CTAs, folded
  // into the group table by denseFoldKernel after the batch; a slot was reached iff it differs from accNeutral
  unsigned long long *denseAcc;
  uint8_t denseGlobal;
  uint8_t denseGlobalReps;   // copies of the global slot array (power of two; CTA b uses copy b mod reps): spreads the L2 atomics
  uint8_t neutralSafe;     // no sequence of row values can bring a reached accumulator back to accNeutral (set by compilePlan)
  uint8_t denseFx;         // float sum accumulated as exact integers in the CTA's slots (three 32-bit pieces each), see jitAnalyzeDense
  int8_t fxShift;          // S: a row adds x * 2^S
  uint8_t numForeignTables, numForeignCols;
  uint8_t joinCol[kMaxForeignTables];       // main-table column matched with table t's primary key
  uint8_t foreignTableOf[kMaxForeignCols];  // table of foreign column k (operand kind OPK_FOREIGN, acol / bcol = k)
  uint8_t foreignClass[kMaxForeignCols];    // ValClass a read of foreign column k yields
  uint8_t pad2[1];
  const DevJoin *join;     // device copy of the tables' indexes and the foreign columns' batches
  uint32_t resume;         // 1: relaunch of the same batch after the group table grew (DevTable::progress holds the resume points)
  uint8_t nmeas;           // > 1: measure roots feeding that many states (direct-indexed form only); meas[] describes them
  uint8_t memberDims;      // PLAN_SINK_MEMBER_DIMENSION roots of the plan (0: plain dimension roots; the states differ in theirs)
  DevMeasure meas[kJitMaxMeasures];
  // numeric bucketizers (BatchPlan.Bucketizers): kind, the kernel's descriptor, and for partition tables their
  // kBucketSmemBytes slot in the shared memory after the stages (bucketSmem bytes in all, staged once per CTA)
  uint8_t nbuckets;
  uint8_t bucketKind[kJitMaxBuckets], bucketSlot[kJitMaxBuckets];
  uint32_t bucketSmem;
  JitBucket buckets[kJitMaxBuckets];
};

// Calls f(j) for instruction i and every instruction whose pushed value it consumes, directly or through others.
template <class F>
void forSubexpression(const DevPlan &P, int i, const F &f) {
  f(i);
  if (P.insts[i].asrc >= 0) forSubexpression(P, P.insts[i].asrc, f);
  if (P.insts[i].bsrc >= 0) forSubexpression(P, P.insts[i].bsrc, f);
}

// Div / Mod / Floor of an integer class by a literal: strength-reduced with a magic multiplier (DevInst::magic)
inline bool isFastDiv(const DevInst &I) {
  return I.nops == 2 && (I.fn == Mod || I.fn == Floor || I.fn == Divide) && I.bkind == OPK_CONST &&
         (I.tclass == VC_I32 || I.tclass == VC_U32) && (I.bclass == VC_I32 || I.bclass == VC_U32);
}

// count(*) and other sums of a positive literal: the sum never returns to 0 (below 2^32 rows), so a slot is reached iff
// it is non-zero
inline bool positiveLiteralSum(const DevInst &I, uint8_t aggOp) {
  return I.sink == PLAN_SINK_MEASURE && !I.wide && (aggOp == OP_SUM_I32 || aggOp == OP_SUM_I64) && I.nops == 1 && I.fn == Noop &&
         I.akind == OPK_CONST && I.avalid && (I.aclass == VC_I32 || I.aclass == VC_U32) && (int32_t)I.aconst > 0;
}

// Bytes of one direct-indexed slot in the CTA: three 32-bit piece counters (exact-integer float sum, `fx`) or a "reached"
// flag and an 8-byte accumulator; HLL: one 32-bit map entry (slot -> the group's registers)
inline uint32_t denseSlotBytes(bool fx, bool hll = false) { return hll ? 4u : fx ? 12u : 9u; }

// Measure m's region of the table area of a multi-measure plan (the regions follow the 128-byte header in measure order):
// its slots (member dimensions: its own, else the plan's), 128-byte aligned
inline uint32_t measureRegionBytes(const DevPlan &P, int m) {
  return ((P.memberDims ? P.meas[m].slots : P.smemSlots) * denseSlotBytes(P.meas[m].denseFx) + 127u) / 128u * 128u;
}

constexpr uint32_t kDenseMaxSlots = 8192;   // = slots of a CTA's accumulator slice in AggState::ctaAcc
constexpr uint32_t kFxMaxRowsPerCta = 1u << 21;   // each 32-bit piece accumulator takes 2^21 adds of an 11-bit piece
constexpr uint32_t kGlobalDenseMaxSlots = 1u << 21;   // 16 MB of accumulators per state, allocated on first use

// jit.cu: the fused kernel specialised for the plan's shape.  jitLaunch runs a batch on it and throws EngineError when
// the kernel cannot be built (libnvrtc missing, the shape's compile failed: reported again for every batch of that
// shape without compiling it twice); jitCompileOnly generates and compiles it without a GPU (AresJitDryRun).
void jitAnalyzeDense(DevPlan &P);
size_t jitCompileOnly(const DevPlan &P, std::string *sourceOut);
void jitLaunch(const DevPlan &P, const DevTable &G, size_t smemBytes, int grid, cudaStream_t s);

}  // namespace aresb
