// jit_params.cuh — the runtime parameter block of the NVRTC-specialised fused kernel and the limits it is sized by.
// Included by the host (jit.cu fills the block) and pasted into the kernel's source text (build.py: JIT_PRELUDE_FILES),
// so both sides see one definition.  NVRTC-clean: no host headers.
#pragma once
#include "fused_device.cuh"
#include "join.cuh"
#include "numeric_bucket.cuh"

namespace aresb {

// bounds of a plan (batch_plan.h: ARES_MAX_PLAN_INSTS, ARES_MAX_FOREIGN_TABLES / COLUMNS; checked on the host)
constexpr int kMaxPlanCols = 16;
constexpr int kMaxPlanInsts = 64;
constexpr int kMaxForeignTables = 4;
constexpr int kMaxForeignCols = 8;

// Joined dimension tables of a plan, in device memory for the duration of the batch's kernel (uploaded by executePlan).
struct DevJoin {
  CuckooDesc tables[kMaxForeignTables];
  ForeignDesc cols[kMaxForeignCols];
};

constexpr int kJitMaxParts = 2 * kMaxPlanCols + 1;                  // values + null bitmap per column, and the base counts
constexpr int kJitMaxConsts = 2 * kMaxPlanInsts + kMaxPlanCols;     // two literal operands per instruction, mode-0 columns
constexpr int kJitMaxWide = 8;
constexpr int kJitMaxMagic = 16;
constexpr int kJitMaxDenseDims = 8;
constexpr int kJitMaxRle = 4;
constexpr int kJitMaxMeasures = 4;   // measure roots of one plan, each feeding its own AggState (ExecuteBatchPlanMulti)
// A mode-3 column read by the kernel straight from its runs: cumulative counts (length + 1 entries), null bitmap and
// values of the RUNS, and the per-tile run hint computed by rleTileRunsKernel.
struct RleColumn {
  const uint32_t *counts;
  const uint8_t *nulls, *values;
  const uint32_t *tileRun;
  uint32_t length, startBit;
};

// One measure of a direct-indexed plan (JIT_NMEAS of them): the group table and CTA slices of the state it feeds, and the
// constants of its form.
struct JitMeasure {
  DevTable G;
  unsigned long long *ctaAcc;
  unsigned long long measureIdentity, accNeutral;
  double fxInv;                           // integer form (kMeasAcc 4): 2^-S
  float fxScale;                          //                            2^S (a float sum's rows are added as integers x * 2^S)
  uint32_t pad;
};

struct JitParams {
  const uint8_t *partSrc[kJitMaxParts];   // global base address of every staged part
  const uint8_t *wideValues[kJitMaxWide]; // 8/16-byte dimension columns read straight from global
  const uint8_t *wideNulls[kJitMaxWide];
  uint32_t consts[kJitMaxConsts];         // literal operands / mode-0 defaults (raw 32-bit cells)
  unsigned long long magic[kJitMaxMagic]; // 2^64/d + 1 for literal divisors d >= 2 (0: use the generic path)
  unsigned long long measureIdentity;
  unsigned long long accNeutral;
  DevTable G;
  unsigned long long *ctaAcc;             // [grid][JIT_SMEM_SLOTS] accumulator slices in global memory
  uint32_t numFullTiles;
  uint32_t numRows;                       // rows of the batch (tail = numRows - numFullTiles * JIT_TILE_ROWS)
  // direct-indexed aggregation (JIT_DENSE): dimension k of a row has index (value or quotient) - dLo[k], valid when
  // below dCnt[k]; index dCnt[k] is the dimension's NULL; slot = sum_k index_k * dStride[k]; value = (dLo + index) * dStep
  uint32_t dLo[kJitMaxDenseDims], dCnt[kJitMaxDenseDims], dStride[kJitMaxDenseDims], dStep[kJitMaxDenseDims];
  uint32_t dBase[kJitMaxDenseDims], dSpan[kJitMaxDenseDims], dMagic32[kJitMaxDenseDims];   // span division (see plan_device.cuh)
  uint32_t dStrideB[kJitMaxDenseDims];   // dStride in the unit the fast path addresses slots in (bytes for the integer form: x 12)
  uint32_t dTotal, dReps, dRepStride;     // slots of one copy; lane-private copies (power of two), dRepStride slots apart
  unsigned long long *gAcc;               // JIT_DENSE == 2: the state's global accumulator array (dTotal slots in use)
  const DevJoin *join;                    // joined dimension tables (join.cuh), null without joins
  uint32_t resume;                        // 1: second launch of the same batch after the table grew (progress[] says where)
  uint32_t startCount;                    // row number of index position 0 when the batch has no base counts
  RleColumn rle[kJitMaxRle];              // run-length encoded columns decoded in place (see ldrle)
  JitMeasure ms[kJitMaxMeasures];         // direct-indexed CTA slots: measure m's state and form (ms[0]: the plan's own)
  // JIT_MDIMS (the measures differ in their dimensions): measure m's slot = sum_k index_k * mStride[m][k] (0 for a
  // dimension m does not have); lane-private copies of its slots, mRepStride[m] slots apart
  uint32_t mStride[kJitMaxMeasures][kJitMaxDenseDims];
  uint32_t mReps[kJitMaxMeasures], mRepStride[kJitMaxMeasures];
  JitBucket bk[kJitMaxBuckets];           // the plan's numeric bucketizers (BatchPlan.Bucketizers)
};
// (with every measure's group table in it: the block stays far below the 32 KB kernel-parameter limit of sm_90)
static_assert(sizeof(JitParams) <= 4096, "the kernel's parameter block is limited to 4 KB");

}  // namespace aresb
