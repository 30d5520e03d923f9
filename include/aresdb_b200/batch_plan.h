/*
 * batch_plan.h — ADDITIVE whole-batch API of the B200 engine (no counterpart symbol in the
 * reference; SURVEY.md §0.1-0.2 / §8b explain why it must exist).
 *
 * The reference executes one cgo call (= 1-2 Thrust launches, a 5 B/row scratch vector and a
 * stream sync for every filter) per AST node: query/time_series_aggregate.go:493-593.  Here
 * the Go batch executor (query/aql_batchexecutor.go:102-273: preExec + filter + project +
 * reduce) hands the WHOLE batch to one call.  The plan is the same post-order walk
 * processExpression() performs, flattened: every PlanInst is exactly one non-leaf AST node
 * with the meaning of the legacy Unary/Binary Transform/Filter call it replaces — leaf
 * operands (VarRef columns, literals) are referenced in place, sub-expression operands come
 * from an evaluation stack that lives in registers instead of scratch vectors, and the root
 * of each expression is routed to a filter / dimension / measure sink.
 *
 * Aggregation state lives across batches in an AggState (a device hash table keyed by the
 * packed dimension row), replacing the "carry previous results in the input buffers and
 * re-sort / re-insert them every batch" protocol (query/aql_processor.go:743-776,
 * query/time_series_aggregate.go:683-716).  AggStateFinalize emits exactly what the last
 * Reduce / HashReduce of the reference would have left in the output DimensionVector and
 * measure vector: groups identified by the murmur3 hash of the packed row (64-bit low word
 * for ARES_REDUCE_SORT, 32-bit for ARES_REDUCE_HASH), ascending-hash order for SORT.
 */
#ifndef ARESDB_B200_BATCH_PLAN_H_
#define ARESDB_B200_BATCH_PLAN_H_

#include "aql_abi.h"

enum {
  ARES_MAX_PLAN_COLUMNS = MAX_COLUMNS_OF_A_TABLE,
  ARES_MAX_PLAN_INSTS = 64,
  ARES_PLAN_STACK_DEPTH = 4,
  ARES_MAX_FOREIGN_TABLES = 4,
  ARES_MAX_FOREIGN_COLUMNS = 8
};

enum PlanOperandKind {
  PLAN_OPERAND_NONE = 0,
  PLAN_OPERAND_COLUMN = 1, /* BatchPlan.Columns[Column]: what makeVectorPartySliceInput passes   */
  PLAN_OPERAND_CONST = 2,  /* what makeConstantInput passes (ConstInt / ConstFloat + IsValid)   */
  PLAN_OPERAND_STACK = 3,  /* result of an earlier PLAN_SINK_STACK instruction (LIFO)            */
  PLAN_OPERAND_FOREIGN = 4 /* BatchPlan.ForeignColumns[Column]: what makeForeignColumnInput passes — a column of a
                            * joined dimension table, read at the RecordID the join finds for the row       */
};

typedef struct {
  uint8_t Kind;       /* enum PlanOperandKind */
  uint8_t Column;     /* PLAN_OPERAND_COLUMN: index into BatchPlan.Columns */
  uint8_t ConstType;  /* PLAN_OPERAND_CONST: ConstInt or ConstFloat */
  uint8_t ConstValid; /* PLAN_OPERAND_CONST: ConstantVector.IsValid */
  union {
    int32_t IntVal;
    float FloatVal;
  } Const;
} PlanOperand;

enum PlanSink {
  PLAN_SINK_STACK = 0,     /* non-root node: ScratchSpaceOutput of DataType SinkDataType       */
  PLAN_SINK_FILTER = 1,    /* root of a filter: row survives iff bool(value) (filterAction)      */
  PLAN_SINK_DIMENSION = 2, /* root of dimension #SinkArg (layout order), DimensionOutput         */
  PLAN_SINK_MEASURE = 3,   /* root of the measure, MeasureOutput of SinkDataType / AggSpec.AggFunc; ExecuteBatchPlanMulti:
                            * one root per state, SinkArg = the ordinal of the state it feeds */
  PLAN_SINK_MEASURE_FILTER = 4, /* ExecuteBatchPlanMulti only: root of a filter that applies to state SinkArg alone (a
                                 * member filter, see ExecuteBatchPlanMulti) */
  PLAN_SINK_MEMBER_DIMENSION = 5 /* ExecuteBatchPlanMulti only: root of a dimension of the states whose bits are set in
                                  * SinkArg (bit k = state k); its ordinal in state k's layout is its position among the
                                  * member dimension roots with bit k (a member dimension, see ExecuteBatchPlanMulti) */
};

/* Plan-only unary functor (no UnaryFunctorType has this value): the numeric bucketizer BatchPlan.Bucketizers[Bucket]
 * applied to the operand.  The instruction is a dimension root (PLAN_SINK_DIMENSION or PLAN_SINK_MEMBER_DIMENSION) whose
 * SinkDataType is the ordinal type of the bucketizer's kind; its operand is a Bool, 1-, 2-, 4-byte integer or Float32
 * value, compared as an exact double.  A NULL or NaN operand gives a NULL dimension. */
enum { PLAN_FN_NUMERIC_BUCKET = 200 };

enum PlanBucketizerKind {
  PLAN_BUCKET_WIDTH = 1,      /* Param = w (finite, > 0): Int32 ordinal k with fl(k*w) <= x < fl((k+1)*w); +-inf and
                               * ordinals outside Int32: NULL */
  PLAN_BUCKET_LOG = 2,        /* Param = b (finite, > 1), Bounds = t[0..NumBounds-1] strictly increasing (t[j] = b^(LogMin+j)):
                               * Uint16 ordinal j with t[j] <= x < t[j+1]; x <= 0, +inf and x outside the table: NULL */
  PLAN_BUCKET_PARTITIONS = 3  /* Bounds = p[0..NumBounds-1] (1..255, finite, strictly increasing): Uint8 ordinal = the
                               * number of p[i] <= x (-inf: 0, +inf: NumBounds) */
};

typedef struct {
  uint8_t Kind;          /* enum PlanBucketizerKind */
  uint8_t Reserved[3];
  int32_t LogMin;        /* PLAN_BUCKET_LOG: exponent of t[0] */
  double Param;          /* w or b */
  const double *Bounds;  /* device memory, valid until the batch's kernel has run (PLAN_BUCKET_LOG / PARTITIONS) */
  uint32_t NumBounds;    /* PLAN_BUCKET_LOG: 2..65537; PLAN_BUCKET_PARTITIONS: 1..255 */
  uint32_t Reserved2;
} PlanBucketizer;

enum { ARES_MAX_PLAN_BUCKETIZERS = 4 };

typedef struct {
  uint8_t NumOperands;  /* 1: Functor is a UnaryFunctorType (or PLAN_FN_NUMERIC_BUCKET); 2: a BinaryFunctorType */
  uint8_t Functor;
  uint8_t Sink;         /* enum PlanSink */
  uint8_t SinkArg;      /* dimension ordinal for PLAN_SINK_DIMENSION; state ordinal for PLAN_SINK_MEASURE and
                         * PLAN_SINK_MEASURE_FILTER (Multi); mask of states for PLAN_SINK_MEMBER_DIMENSION (Multi) */
  uint8_t SinkDataType; /* enum DataType of the sink element */
  uint8_t Bucket;       /* PLAN_FN_NUMERIC_BUCKET: index into BatchPlan.Bucketizers (0 otherwise) */
  uint8_t Reserved[2];
  PlanOperand A;
  PlanOperand B;
} PlanInst;

/* Optional zone-map entry of one column of one batch: every VALID (non-NULL) value of the column in this
 * batch lies in [Min, Max] as a non-negative integer below 2^31 (Bool / Uint8 / Uint16 / Uint32 columns and
 * non-negative signed ones; for a Float32 column whose valid values are all >= 0: the IEEE bit patterns of the
 * smallest and largest value, which order like the values — a float SUM then accumulates the rows that lie on
 * the 2^-S grid the maximum allows as exact integers).  The reference keeps exactly this for the time column of live batches
 * (LiveVectorParty.GetMinMaxValue, memstore/common/vector_party.go:184-186, used for batch skipping in
 * query/aql_processor.go:1509) and knows it by construction for archive batches (batch ID = day) and for
 * enum columns (dictionary size).  It is a HINT: when every dimension of the query has a small known range
 * the fused kernel addresses its CTA-private accumulators directly by (dimension value - Min) instead of
 * probing a hash table; every row is checked against the range and rows outside it take the hash path, so a
 * stale or wrong entry costs speed, never correctness.  Known = 0: no information. */
typedef struct {
  uint8_t Known;
  uint8_t Reserved[3];
  uint32_t Min;
  uint32_t Max;
} ColumnRange;

/* Dimension-table joins on the fused path (what BatchExecutorImpl.join() prepares per batch with HashLookup,
 * query/aql_batchexecutor.go:115-147, and what makeForeignColumnInput passes per expression leaf).  The lookup is a gather
 * stage INSIDE the fused kernel: the RecordID of a surviving row is found by probing the dimension table's cuckoo index
 * with the row's join-column value when the first instruction that reads the table is reached, and the foreign column is
 * read at it; no RecordID vector is materialised.  Join keys are 1- / 2- / 4-byte main-table columns. */
typedef struct {
  int32_t JoinColumn;    /* index into BatchPlan.Columns: the main-table column matched with the table's primary key */
  CuckooHashIndex Index; /* the dimension table's primary-key index (device memory)                                  */
} PlanForeignTable;

typedef struct {
  int32_t Table;              /* index into BatchPlan.ForeignTables                                                  */
  ForeignColumnVector Column; /* as makeForeignColumnInput fills it; RecordIDs is ignored; Batches points to HOST memory
                               * valid for the duration of the call (at most 8 batches); TimezoneLookup to device memory */
} PlanForeignColumn;

/* One batch of one table shard: column slices already resident on the device. */
typedef struct {
  VectorPartySlice Columns[ARES_MAX_PLAN_COLUMNS];
  int32_t NumColumns; /* at most 16 per call: list the columns the query reads (what transferBatch copies), not the table */
  PlanInst Insts[ARES_MAX_PLAN_INSTS];
  int32_t NumInsts;
  /* Index space of the batch = rows of the first column (as in the reference).  BaseCounts
   * is that column's cumulative count vector for RLE (archive, sorted) batches, or NULL;
   * StartCount is the row number of index 0 when BaseCounts is NULL
   * (oopkBatchContext.baseCountD / startRow, query/aql_context.go:151-235). */
  uint32_t *BaseCounts;
  uint32_t StartCount;
  uint32_t NumRows;
  ColumnRange Ranges[ARES_MAX_PLAN_COLUMNS]; /* zone map per entry of Columns (all zero: none) */
  PlanForeignTable ForeignTables[ARES_MAX_FOREIGN_TABLES];
  int32_t NumForeignTables;
  PlanForeignColumn ForeignColumns[ARES_MAX_FOREIGN_COLUMNS];
  int32_t NumForeignColumns;
  PlanBucketizer Bucketizers[ARES_MAX_PLAN_BUCKETIZERS]; /* numeric bucketizers of PLAN_FN_NUMERIC_BUCKET instructions */
  int32_t NumBucketizers;
} BatchPlan;

enum AresReduceMode {
  ARES_REDUCE_SORT = 0, /* semantics of Sort + Reduce (64-bit hash identity, hash-ascending output) */
  ARES_REDUCE_HASH = 1  /* semantics of HashReduce (32-bit hash identity, unordered output)        */
};

typedef struct {
  uint8_t NumDimsPerDimWidth[NUM_DIM_WIDTH]; /* as DimensionVector */
  uint8_t Reserved[3];
  int32_t AggFunc;         /* enum AggregateFunction: SUM/MIN/MAX families, AGGR_AVG_FLOAT (8-byte (float average, count)
                            * pairs combined with the reference's rolling average), or AGGR_HLL (measure = Uint32
                            * rho << 16 | reg values; group identity and results as HyperLogLog's,
                            * query/hll.cu:21-290; read the result with AggStateFinalizeHLL) */
  int32_t MeasureDataType; /* enum DataType of one measure element: Int32/Uint32/Float32/Int64/Float64 */
  int32_t ReduceMode;      /* enum AresReduceMode */
  uint32_t ExpectedGroups; /* capacity hint: the group table holds max(2^21, 2 x ExpectedGroups) slots; exceeding it
                            * is reported as an error by AggStateGroupCount / AggStateFinalize, never silently */
} AggSpec;

#ifdef __cplusplus
extern "C" {
#endif

/* res = opaque state handle.  Allocates the group table on `device`. */
CGoCallResHandle AggStateCreate(AggSpec spec, void *cudaStream, int device);

/* Fused preExec+filter+project+reduce of one batch into `state`.  Asynchronous on
 * cudaStream: nothing is returned to the host, nothing is synchronised (res = 0).  A state is used from
 * one stream at a time (the batches of a query follow each other, as in the reference); different states
 * run concurrently on different streams / devices. */
CGoCallResHandle ExecuteBatchPlan(void *state, const BatchPlan *plan, void *cudaStream, int device);

/* Several aggregates over the same rows in one pass: the plan carries numStates (1..4) PLAN_SINK_MEASURE roots, root
 * SinkArg = k feeding states[k]; filters, dimensions and joins are shared.  Every state is an ordinary AggState
 * (AggStateCreate; finalized, reset, exported and merged as usual); they must agree in NumDimsPerDimWidth and
 * ReduceMode, and none may be AGGR_HLL.  When the batch's zone map lets every measure's own single-measure plan take the
 * CTA's direct-indexed slots and they all fit a CTA together, one kernel evaluates each row once and feeds every state;
 * otherwise each state runs its single-measure plan (what ExecuteBatchPlan would launch).  Results are the same either
 * way.  numStates == 1 is ExecuteBatchPlan.  Asynchronous like ExecuteBatchPlan.
 *
 * Member filters: the states may also differ in their filters.  A PLAN_SINK_MEASURE_FILTER root applies to state
 * SinkArg only; a row feeds state k iff it passes every PLAN_SINK_FILTER root and every PLAN_SINK_MEASURE_FILTER root
 * with SinkArg == k.  Filters every state carries are PLAN_SINK_FILTER roots and are evaluated once per row.  Member
 * filter roots follow the last PLAN_SINK_FILTER root and precede the first PLAN_SINK_DIMENSION root.  Rejected with an
 * error string: a member filter in a plan given to ExecuteBatchPlan, a SinkArg outside 0..numStates-1, and member
 * filter roots out of that order.  In the one-kernel form a row's dimensions are computed when it is alive for some
 * state, and each state's accumulators see only the rows alive for it; in the per-state form state k runs its
 * single-measure plan, which keeps state k's member filters as ordinary filters and drops the other states' member
 * filters.  numStates == 1 is ExecuteBatchPlan of the plan with its member filters turned into filters.
 *
 * Member dimensions: the states may also differ in their dimensions.  Such a plan has no PLAN_SINK_DIMENSION root;
 * instead every dimension of the union of the states' dimensions is one PLAN_SINK_MEMBER_DIMENSION root whose SinkArg
 * is the mask of the states that group by it, so that a dimension several states share is evaluated once.  State k's
 * dimensions are the roots with bit k, in plan order, and their widths must be the layout its NumDimsPerDimWidth
 * describes (16, 8, 4, 2, 1 bytes); the states may then differ in NumDimsPerDimWidth.  Member dimension roots follow
 * the member filter roots and precede the measure roots.  Rejected with an error string: a member dimension in a plan
 * given to ExecuteBatchPlan, a zero mask, a mask bit >= numStates, a plan with both kinds of dimension roots, roots out
 * of that order, and widths that differ from a state's layout.  The form is chosen per batch, in this order:
 *   1. one kernel for all states: every state's own plan takes the CTA's direct-indexed slots, their regions (each
 *      sized by its own slot count) fit a CTA together, and the states agree in key form (rows of at most 8 bytes, or
 *      rows of the same length); a row's index in every union dimension is computed once, and each state's slot is
 *      derived from the indexes of its own dimensions;
 *   2. otherwise each set of states with identical dimensions runs the plan of that set (its measure and member
 *      filter roots, its dimensions as PLAN_SINK_DIMENSION roots), the sets in the order of their first state, each
 *      taking its form as above: one kernel for the set, or one kernel per state of the set;
 *   3. when no such set takes a direct-indexed form, that is one kernel per state.
 * Every state gets exactly the result it gets alone.  A caller builds the union from the states' dimension
 * expressions, compared structurally together with their output type: each state's dimensions must appear in the
 * union in its own layout order, which is possible unless two states order two dimensions of the same width
 * differently (such states belong in separate calls). */
CGoCallResHandle ExecuteBatchPlanMulti(void *const *states, int numStates, const BatchPlan *plan, void *cudaStream, int device);

/* Folds already-reduced rows (a DimensionVector block + measure vector, e.g. the carried
 * result of the legacy protocol, or the all-gathered results of other GPUs) into `state`
 * with the aggregate's combine rule (broker/result_merge.go:80-105 semantics). */
CGoCallResHandle AggStateMerge(void *state, DimensionVector inputKeys, uint8_t *inputValues,
                               int length, void *cudaStream, int device);

/* res = number of occupied group slots (>= number of output groups); synchronises. */
CGoCallResHandle AggStateGroupCount(void *state, void *cudaStream, int device);

/* Writes the groups into outputKeys (capacity outputKeys.VectorCapacity; DimValues required,
 * HashValues / IndexVector filled when non-NULL) and outputValues; res = number of groups.
 * Synchronises cudaStream.  The state stays valid (it can be finalized again or reset). */
CGoCallResHandle AggStateFinalize(void *state, DimensionVector outputKeys, uint8_t *outputValues,
                                  void *cudaStream, int device);

/* Exchange form of AggStateFinalize: the occupied table slots as (dim row, partial measure) pairs in
 * no particular order and without merging equal hashes — what another state's AggStateMerge consumes.
 * Cheaper than AggStateFinalize (no sort); res = number of rows (== AggStateGroupCount). Synchronises. */
CGoCallResHandle AggStateExport(void *state, DimensionVector outputKeys, uint8_t *outputValues,
                                void *cudaStream, int device);

/* The queries of one request, several states per launch (1..16 distinct states; AGGR_HLL states are refused — they keep
 * the exact protocol).  Every call below rejects null arrays, a numStates outside 1..16, a state given twice and an HLL
 * state with an error.  A single query is a request of one state (one-element arrays).
 *
 * AggStatesFinalize: AggStateFinalize of states[k] into (outputKeys[k], outputValues[k]); groups[k] = its group count.
 * States that announce at most 32768 groups are finalized by ONE launch (one cluster each) and ONE synchronise; the
 * others, and those that turn out to need it (parked rows, more than 32768 groups), complete through AggStateFinalize's
 * other paths within the same call, so every state gets its complete result.  When a state fails (e.g. "exchange part
 * truncated") the others are still finalized: its groups[k] is -1 and the error lists every failed state as a line
 * "state k: <message>".  outputKeys[k] must have states[k]'s NumDimsPerDimWidth.
 *
 * The exchange step of a sharded request, without host involvement: every rank exports its states as fixed-capacity
 * parts, the parts of all ranks reach every rank, and every rank folds them into its receiving states, whose next
 * AggStatesFinalize completes the request.  Nothing is synchronised and the row counts stay on the device.
 *
 * AggStatesExportPartsToPeers: ONE launch exports every state into its sub-part of this rank's slot — sub-part k at
 * partOffset[k] inside the slot: a 16-byte header [uint32 rows, uint32 status, uint32 claimed, pad], the DimensionVector
 * block of capRows rows at dimOffset[k] and the measures at valuesOffset[k], both relative to the sub-part — in
 * peerSlots[myRank], copies every sub-part into peerSlots[r] of every peer r with 16-byte stores, and then stores `epoch`
 * into state k's flag for this rank on every peer (release, system scope): peerFlags[r] + 16 * k, where peerFlags[r] =
 * the address of flags[0][myRank] on rank r (a rank's flags are uint32 flags[state][16 ranks]).  peerSlots[r] is the
 * address of THIS rank's slot inside rank r's receive buffer: the host maps every rank's receive buffer into every
 * process (peer memory on one NVLink / NVSwitch node: CUDA IPC / fabric handles — torch symmetric memory does it).
 * peerFlags == NULL: the local export only (peerSlots[myRank]; the slots then travel by a collective all-gather).
 * capRows in [1, 32768]; slotBytes and every offset are multiples of 16, and each sub-part lies inside the slot without
 * overlapping another; numPeers in 1..16, 0 <= myRank < numPeers.  A state with more rows than capRows marks its
 * sub-part (status != 0, no rows): the receiving state's next finalize fails with "exchange part truncated", and that
 * state's step is repeated with AggStateGroupCount / AggStateExport / AggStateMerge (exact sizes).
 *
 * AggStatesMergeParts: ONE launch folds, for every state k, sub-part k of each of the numParts slots (slot p at
 * slots + p * slotStride, as an all-gather or the peers' exports leave them) into states[k], reading the row counts from
 * the sub-part headers.  flags != NULL: the CTAs of state k first wait until flags[16 * k + p] has reached `epoch` for
 * every p < numParts; a state never waits for another state's flags.  The wait is bounded (~2 s): a peer that does not
 * arrive makes that state's next finalize fail ("did not arrive") instead of hanging the GPU.  A truncated sub-part or a
 * late peer is reported by that state's next finalize only.  Use two flag blocks and receive buffers alternately by
 * epoch parity, with a growing epoch: a rank can be at most one exchange ahead of its peers.
 * All three are asynchronous except AggStatesFinalize, which synchronises. */
CGoCallResHandle AggStatesFinalize(void *const *states, int numStates, const DimensionVector *outputKeys, uint8_t *const *outputValues,
                                   int64_t *groups, void *cudaStream, int device);
CGoCallResHandle AggStatesExportPartsToPeers(void *const *states, int numStates, uint8_t *const *peerSlots, uint32_t *const *peerFlags,
                                             int numPeers, int myRank, size_t slotBytes, int capRows, const size_t *partOffset,
                                             const size_t *dimOffset, const size_t *valuesOffset, uint32_t epoch, void *cudaStream,
                                             int device);
CGoCallResHandle AggStatesMergeParts(void *const *states, int numStates, const uint8_t *slots, int numParts, size_t slotStride, int capRows,
                                     const size_t *partOffset, const size_t *dimOffset, const size_t *valuesOffset, const uint32_t *flags,
                                     uint32_t epoch, void *cudaStream, int device);

/* AGGR_HLL states: the final outputs of the reference's last-batch HyperLogLog call
 * (query/hll.cu:262-290, adopted by query/time_series_aggregate.go:661-681).  res = number of dimension
 * groups g.  *dimValuesPtr = a DimensionVector block of VectorCapacity g (groups in key order),
 * *hllDimRegIDCountPtr = g register counts, *hllVectorPtr / *hllVectorSizePtr = per group either
 * count x 4 bytes ((rho+1) << 16 | reg, count < 4096) or 16384 dense bytes.  All three are allocated
 * with deviceMalloc; the caller frees them with DeviceFree.  On such a state AggStateGroupCount
 * counts (group, register) entries and AggStateFinalize / AggStateMerge exchange the carried form
 * (one row per entry, Uint32 value) — which is how several GPUs combine HLL states.  Synchronises. */
CGoCallResHandle AggStateFinalizeHLL(void *state, uint8_t **dimValuesPtr, uint8_t **hllVectorPtr,
                                     size_t *hllVectorSizePtr, uint16_t **hllDimRegIDCountPtr,
                                     void *cudaStream, int device);

/* AGGR_HLL states: the distinct-count estimate of every group, computed on the device.  res = number of groups g: the
 * groups of AggStateFinalizeHLL, in its order, with its *dimValuesPtr block (VectorCapacity g).  *estimatesPtr = g
 * float64 values, each equal bit for bit to the reference's HLL.Compute (query/common/hll.go:735-775) of that group's
 * register vector: bias correction up to 5m, linear counting up to 15500, truncated toward zero.  The register vectors
 * stay on the device and are freed by the call.  Both outputs are allocated with deviceMalloc; the caller frees them
 * with DeviceFree.  A state that is not AGGR_HLL and a null output pointer are errors.  Synchronises. */
CGoCallResHandle AggStateFinalizeHLLEstimate(void *state, uint8_t **dimValuesPtr, double **estimatesPtr, void *cudaStream,
                                             int device);

/* Zone-map production: out[i] = min / max of the VALID values of columns[i] (at most 16 per call; Bool / 1- / 2- /
 * 4-byte integer and Float32 columns in modes 0-3; everything else, columns without a valid value, and columns whose
 * values the ColumnRange contract cannot describe — negative, >= 2^31, negative or non-finite floats — get Known = 0).
 * One kernel over all columns, called once when a batch becomes device resident; the result is what BatchPlan.Ranges
 * takes.  The reference keeps this pair only for live Uint32 vector parties (memstore/live_vector_party.go:74-75).
 * res = number of columns scanned.  Synchronises cudaStream. */
CGoCallResHandle ComputeColumnRanges(const VectorPartySlice *columns, int numColumns, ColumnRange *out,
                                     void *cudaStream, int device);

/* Empties the table, keeping its memory. */
CGoCallResHandle AggStateReset(void *state, void *cudaStream, int device);

CGoCallResHandle AggStateDestroy(void *state, int device);

/* Diagnostics: engine kernels launched by this process so far (bench.py reports the delta over the
 * timed region as `gpu_launches`). */
unsigned long long AresKernelLaunchCount();

#ifdef __cplusplus
}
#endif

#endif /* ARESDB_B200_BATCH_PLAN_H_ */
