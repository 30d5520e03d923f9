"""Aggregate-query description and its translation into the two call forms of the hot path.

An `AggQuery` carries what AQLQueryContext.OOPK carries after compilation (reference
query/aql_context.go:151-235, query/aql_compiler.go:1139-1370): the main-table common filters,
the dimension expressions with their output widths sorted into layout order
(sortDimensionColumns), and the single measure with its aggregate function and byte width
(count -> SUM_UNSIGNED of the literal 1 in 4 bytes; sum -> 8-byte accumulators).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import cabi as A
from . import expr as E


@dataclass
class Measure:
    kind: str                 # "count" | "sum" | "min" | "max" | "avg" | "hll" | "countdistincthll"
    expr: E.Expr | None = None


@dataclass
class Join:
    """One joined dimension table: `table` (joins.DimensionTable, resident in the executor's memory space) matched on its
    primary key by main-table column `on`; `timezone_table` optionally maps an enum column to a timezone offset."""
    table: object
    on: E.Col
    timezone_ptr: int | None = None
    timezone_size: int = 0


class AggQuery:
    def __init__(self, filters, dimensions, measure: Measure, reduce_mode: int = A.ARES_REDUCE_SORT, joins=None, time_filters=None):
        self.joins = list(joins or [])
        resolved = [E.resolve(f) for f in filters]
        # the query's time filter (AQL timeFilter: `col >= from`, `col < to`) is kept apart from the common filters: it runs
        # in the batch's custom-filter step, and archive batches strictly inside the range skip it
        # (OOPK.TimeFilters; archiveBatchCustomFilterExecutor, reference query/aql_processor.go:627-638)
        timed = [E.resolve(f) for f in (time_filters or [])]
        if any(E.uses_foreign(f) for f in timed):
            raise ValueError("time filters read the main table")
        # main-table filters run before the join, filters that read a joined table after it
        # (MainTableCommonFilters / ForeignTableCommonFilters, reference query/aql_batchexecutor.go:100-147)
        main = [f for f in resolved if not E.uses_foreign(f)]
        self.filters = main + timed + [f for f in resolved if E.uses_foreign(f)]
        self.time_filter_range = (len(main), len(main) + len(timed))     # positions in self.filters
        self.time_column = 0          # fact tables: column 0 is the time column
        self.num_main_filters = len(main) + len(timed)
        self.dimensions = [E.resolve(d) for d in dimensions]
        self.reduce_mode = reduce_mode
        # ---- dimensions: widest first, stable (reference query/aql_compiler.go:1341-1370) ----------
        self.dim_types = [E.dimension_data_type(d) for d in self.dimensions]
        widths = [max(A.DATA_TYPE_BYTES[t], 1) for t in self.dim_types]
        self.dim_order = sorted(range(len(widths)), key=lambda i: -widths[i])  # layout position -> query dim
        self.num_dims_per_width = [sum(1 for w in widths if w == W) for W in A.DIM_WIDTHS]
        self.layout_widths = [widths[i] for i in self.dim_order]
        if sum(widths) + len(widths) > A.MAX_DIMENSION_BYTES:
            raise ValueError("dimension row exceeds MAX_DIMENSION_BYTES")
        # ---- measure (reference query/aql_compiler.go:1139-1250) -------------------------------------
        self.measure_kind = measure.kind
        if measure.kind == "count":
            self.measure = E.Lit(1, E.Type.Unsigned)
            self.agg_func, self.measure_bytes = A.AGGR_SUM_UNSIGNED, 4
        elif measure.kind in ("hll", "countdistincthll"):
            # hll(col): col already holds rho << 16 | reg; countdistincthll(col) computes it on the fly
            # (reference query/context/query_context_helper.go:540-575, aql_compiler.go:1243)
            col = E.resolve(measure.expr)
            if not isinstance(col, E.Col):
                raise ValueError(f"expect 1 argument to be a column for {measure.kind}")
            if measure.kind == "hll" and col.data_type != A.Uint32:
                raise ValueError("expect 1 argument to be a valid hll column")
            self.measure = col if measure.kind == "hll" else E.resolve(E.Unary(A.GetHLLValue, col))
            self.agg_func, self.measure_bytes = A.AGGR_HLL, 4
        elif measure.kind == "avg":
            # 4 bytes for the average and 4 for the count; always the float aggregate (aql_compiler.go:1212-1216)
            self.measure = E.resolve(measure.expr)
            if self.measure.type not in (E.Type.Unsigned, E.Type.Signed, E.Type.Float):
                raise ValueError("unsupported input type for avg")
            self.agg_func, self.measure_bytes = A.AGGR_AVG_FLOAT, 8
        else:
            self.measure = E.resolve(measure.expr)
            t = self.measure.type
            fam = {"sum": (A.AGGR_SUM_UNSIGNED, A.AGGR_SUM_SIGNED, A.AGGR_SUM_FLOAT),
                   "min": (A.AGGR_MIN_UNSIGNED, A.AGGR_MIN_SIGNED, A.AGGR_MIN_FLOAT),
                   "max": (A.AGGR_MAX_UNSIGNED, A.AGGR_MAX_SIGNED, A.AGGR_MAX_FLOAT)}[measure.kind]
            if t not in (E.Type.Unsigned, E.Type.Signed, E.Type.Float):
                raise ValueError(f"unsupported input type for {measure.kind}")
            self.agg_func = fam[{E.Type.Unsigned: 0, E.Type.Signed: 1, E.Type.Float: 2}[t]]
            self.measure_bytes = 8 if measure.kind == "sum" else 4
        self.measure_data_type = A.Uint32 if self.agg_func == A.AGGR_HLL else \
            self._output_data_type(self.measure.type, self.measure_bytes)

    @property
    def is_hll(self) -> bool:
        return self.agg_func == A.AGGR_HLL

    @staticmethod
    def _output_data_type(t: E.Type, width: int) -> int:
        """getOutputDataType — reference query/time_series_aggregate.go:337-363."""
        if width == 4:
            return A.Float32 if t == E.Type.Float else (A.Uint32 if t == E.Type.Unsigned else A.Int32)
        return A.Float64 if t == E.Type.Float else A.Int64

    @property
    def row_bytes(self) -> int:
        return sum(self.layout_widths) + len(self.layout_widths)

    def agg_spec(self, expected_groups: int = 0) -> A.AggSpec:
        spec = A.AggSpec()
        for i in range(A.NUM_DIM_WIDTH):
            spec.NumDimsPerDimWidth[i] = self.num_dims_per_width[i]
        spec.AggFunc = self.agg_func
        spec.MeasureDataType = self.measure_data_type
        spec.ReduceMode = self.reduce_mode
        spec.ExpectedGroups = expected_groups
        return spec

    # ---- fused plan ------------------------------------------------------------------------------
    def cutoff_filter(self, cutoff: int) -> E.Expr:
        """`time column >= cutoff`: what a LIVE batch of a fact table evaluates besides the query's own filters — rows older
        than the shard's archiving cutoff are served by the archive batches (createCutoffTimeFilter, reference
        query/aql_processor.go:543-552; the time column of a fact table is column 0)."""
        return E.resolve(E.Binary(A.GreaterThanOrEqual, E.Col(self.time_column, A.Uint32, "time"), E.Lit(int(cutoff), E.Type.Unsigned)))

    def plan_instructions(self, time_filters: bool = True, cutoff: int = 0, measures: list | None = None) -> list[A.PlanInst]:
        """Post-order flattening of every expression: one PlanInst per non-leaf AST node (what
        processExpression turns into one cgo call, reference query/time_series_aggregate.go:493-593).
        `time_filters=False`: the plan of an archive batch strictly inside the query's time range.
        `measures`: queries sharing this query's dimensions, time filter, joins and reduce mode (shared_scan_key); the
        plan ends with their measure roots, root k (SinkArg k) feeding the k-th state of ExecuteBatchPlanMulti.  The
        filters every one of them carries come first, in this query's order; each query's other filters follow as member
        filter roots (PLAN_SINK_MEASURE_FILTER, SinkArg k), before the dimensions.  When their dimensions differ, the plan
        carries the union of them (member_dimensions) as member dimension roots (PLAN_SINK_MEMBER_DIMENSION, SinkArg = the
        mask of the queries that group by the dimension)."""
        members = [self] if measures is None else measures
        insts: list[A.PlanInst] = []
        self.foreign_columns = []   # distinct (table, column, timezone) leaves in first-use order = BatchPlan.ForeignColumns
        self.bucketizers = []       # distinct numeric bucketizers in first-use order = BatchPlan.Bucketizers

        def operand(e: E.Expr) -> A.PlanOperand:
            o = A.PlanOperand()
            if isinstance(e, E.ForeignCol):
                key = (e.table, e.index, e.timezone)
                if key not in self.foreign_columns:
                    self.foreign_columns.append(key)
                o.Kind, o.Column = A.PLAN_OPERAND_FOREIGN, self.foreign_columns.index(key)
            elif isinstance(e, E.Col):
                o.Kind, o.Column = A.PLAN_OPERAND_COLUMN, e.index
            elif isinstance(e, E.Lit):
                o.Kind, o.ConstValid = A.PLAN_OPERAND_CONST, 1
                if e.type == E.Type.Float:
                    o.ConstType, o.Const.FloatVal = A.ConstFloat, float(e.value)
                else:
                    o.ConstType, o.Const.IntVal = A.ConstInt, int(e.value)
            else:
                emit(e, A.PLAN_SINK_STACK, 0, E.scratch_data_type(e.type))
                o.Kind = A.PLAN_OPERAND_STACK
            return o

        def emit(e: E.Expr, sink: int, sink_arg: int, sink_dt: int):
            pi = A.PlanInst()
            if isinstance(e, E.Bucket):
                if sink not in (A.PLAN_SINK_DIMENSION, A.PLAN_SINK_MEMBER_DIMENSION):
                    raise ValueError("a numeric bucketizer is a dimension")
                if e not in self.bucketizers:
                    self.bucketizers.append(e)
                if len(self.bucketizers) > A.ARES_MAX_PLAN_BUCKETIZERS:
                    raise ValueError(f"at most {A.ARES_MAX_PLAN_BUCKETIZERS} numeric bucketizers per plan")
                pi.NumOperands, pi.Functor, pi.A = 1, A.PLAN_FN_NUMERIC_BUCKET, operand(e.expr)
                pi.Bucket = self.bucketizers.index(e)
            elif isinstance(e, E.Binary):
                a = operand(e.lhs)
                b = operand(e.rhs)
                pi.NumOperands, pi.Functor, pi.A, pi.B = 2, e.op, a, b
            elif isinstance(e, E.Unary):
                pi.NumOperands, pi.Functor, pi.A = 1, e.op, operand(e.expr)
            else:  # a bare column / literal at the root: the Noop action
                pi.NumOperands, pi.Functor, pi.A = 1, A.Noop, operand(e)
            pi.Sink, pi.SinkArg, pi.SinkDataType = sink, sink_arg, sink_dt
            insts.append(pi)

        # (structural comparison: the instruction bytes of a foreign column depend on the plan it is in)
        common = [all(any(f == g for g in m.filters) for m in members) for f in self.filters]
        lo, hi = self.time_filter_range
        for i, f in enumerate(self.filters):
            if i == lo and cutoff > 0:          # the custom-filter step: cutoff filter first, then the time filters
                emit(self.cutoff_filter(cutoff), A.PLAN_SINK_FILTER, 0, A.Bool)
            if common[i] and (time_filters or not lo <= i < hi):
                emit(f, A.PLAN_SINK_FILTER, 0, A.Bool)
        if cutoff > 0 and lo >= len(self.filters):
            emit(self.cutoff_filter(cutoff), A.PLAN_SINK_FILTER, 0, A.Bool)
        shared = [f for f, c in zip(self.filters, common) if c]
        for k, q in enumerate(members):
            for f in q.filters:
                if not any(f == g for g in shared):
                    emit(f, A.PLAN_SINK_MEASURE_FILTER, k, A.Bool)
        union = member_dimensions(members)
        if union is None:
            for pos, qi in enumerate(self.dim_order):
                emit(self.dimensions[qi], A.PLAN_SINK_DIMENSION, pos, self.dim_types[qi])
        for e, dt, mask in union or ():
            emit(e, A.PLAN_SINK_MEMBER_DIMENSION, mask, dt)
        for k, q in enumerate(members):
            emit(q.measure, A.PLAN_SINK_MEASURE, k, q.measure_data_type)
        if len(insts) > A.ARES_MAX_PLAN_INSTS:
            raise ValueError("plan too long")
        return insts


    def shared_scan_key(self, member_filters: bool = False):
        """What queries must agree on to read the batches in one pass: the plan up to the measure root (filters in order,
        with their literals, and dimensions), the time-filter positions, the joins and the reduce mode.  None for HLL
        queries, which never share.  `member_filters`: the filters may differ (each query's own filters become member
        filters of the shared plan); the dimensions, the time filter, the joins and the reduce mode must not."""
        if self.is_hll:
            return None
        joins = tuple((id(j.table), j.on.index, j.timezone_ptr, j.timezone_size) for j in self.joins)
        if member_filters:
            lo, hi = self.time_filter_range
            # (expressions compare structurally: their repr is the key)
            dims = repr([(self.dimensions[qi], self.dim_types[qi]) for qi in self.dim_order])
            return dims, repr(self.filters[lo:hi]), joins, self.reduce_mode
        prefix = tuple(bytes(pi) for pi in self.plan_instructions(measures=[]))
        # (an instruction names its bucketizer by index: the specs themselves tell two widths apart)
        return prefix, repr([b.spec for b in self.bucketizers]), self.time_filter_range, joins, self.reduce_mode


def member_dimensions(queries: list):
    """The union of the dimensions of `queries` as (expression, output data type, mask of the queries that have it), or
    None when they all have the same dimensions.  Dimensions compare structurally, with their type; the union is ordered
    so that every query's dimensions appear in its own layout order (dim_order), each new dimension as early as that
    allows.  Raises ValueError when no such order exists (two queries order two dimensions of the same width
    differently)."""
    seqs = [[repr((q.dimensions[qi], q.dim_types[qi])) for qi in q.dim_order] for q in queries]
    if all(s == seqs[0] for s in seqs):
        return None
    info, order = {}, []
    for q, s in zip(queries, seqs):
        for key, qi in zip(s, q.dim_order):
            if key not in info:
                info[key] = (q.dimensions[qi], q.dim_types[qi])
                order.append(key)
    pos, out = [0] * len(seqs), []
    while len(out) < len(order):
        # a dimension comes next when it is the next one of every query that has it
        nxt = next((key for key in order if key not in out and
                    all(key not in s or (pos[k] < len(s) and s[pos[k]] == key) for k, s in enumerate(seqs))), None)
        if nxt is None:
            raise ValueError("the queries order their dimensions differently")
        out.append(nxt)
        for k, s in enumerate(seqs):
            if pos[k] < len(s) and s[pos[k]] == nxt:
                pos[k] += 1
    return [(*info[key], sum(1 << k for k, s in enumerate(seqs) if key in s)) for key in out]


class QueryResult:
    """Groups of an aggregate query, decoded from the output DimensionVector block + measures."""

    def __init__(self, query: AggQuery, block: np.ndarray, capacity: int, measures_raw: np.ndarray, groups: int):
        self.query, self.groups = query, groups
        np_meas = {A.Int32: np.int32, A.Uint32: np.uint32, A.Float32: np.float32, A.Int64: np.int64,
                   A.Float64: np.float64}[query.measure_data_type]
        if query.agg_func == A.AGGR_SUM_UNSIGNED and query.measure_bytes == 8:
            np_meas = np.uint64
        self.measures = measures_raw[:groups * query.measure_bytes].view(np_meas).copy()
        self.counts = None
        if query.agg_func == A.AGGR_AVG_FLOAT:   # packed (float average, uint32 count); the average is what is reported
            pairs = measures_raw[:groups * 8].view(np.uint32).reshape(groups, 2)
            self.measures, self.counts = pairs[:, 0].copy().view(np.float32), pairs[:, 1].copy()
        self.dim_values: list[np.ndarray] = [None] * len(query.dimensions)
        self.dim_valid: list[np.ndarray] = [None] * len(query.dimensions)
        n = len(query.layout_widths)
        pos = 0
        value_offs = []
        for w in query.layout_widths:
            value_offs.append(pos)
            pos += w * capacity
        raw_cols = []
        for p, qi in enumerate(query.dim_order):
            w = query.layout_widths[p]
            vals = block[value_offs[p]:value_offs[p] + w * groups].reshape(groups, w).copy()
            valid = block[pos + p * capacity: pos + p * capacity + groups].copy()
            raw_cols.append((vals, valid))
            self.dim_values[qi] = vals
            self.dim_valid[qi] = valid
        self._raw_cols = raw_cols
        self._rows = None

    def packed_rows(self) -> np.ndarray:
        """uint8[groups, row_bytes]: the packed dimension rows in layout order (values, then validity bytes)."""
        if not self._raw_cols:
            return np.zeros((self.groups, 0), np.uint8)
        return np.concatenate([v for v, _ in self._raw_cols] + [vd.reshape(-1, 1) for _, vd in self._raw_cols], axis=1)

    @property
    def rows(self) -> list:
        """The reference's group identity: one bytes object per group (built on first use)."""
        if self._rows is None:
            self._rows = [r.tobytes() for r in self.packed_rows()]
        return self._rows

    def as_dict(self) -> dict:
        """packed dim row (bytes) -> measure value."""
        return {r: self.measures[i].item() for i, r in enumerate(self.rows)}

    def decoded_dims(self):
        """Per query dimension: python values (None for NULL)."""
        out = []
        for qi, dt in enumerate(self.query.dim_types):
            npdt = {A.Bool: np.uint8, A.Int8: np.int8, A.Uint8: np.uint8, A.Int16: np.int16, A.Uint16: np.uint16,
                    A.Int32: np.int32, A.Uint32: np.uint32, A.Float32: np.float32, A.Int64: np.int64}.get(dt)
            vals = self.dim_values[qi]
            if npdt is None:
                col = [bytes(v) for v in vals]
            else:
                col = vals.reshape(-1).view(npdt).tolist()
            out.append([c if v else None for c, v in zip(col, self.dim_valid[qi])])
        return out


class HLLEstimates(QueryResult):
    """The distinct-count estimates of an hll query: the groups of its HLLResult, in the same order, with one float64
    estimate each in `measures` (HLL.Compute on the device, AggStateFinalizeHLLEstimate).  postprocess.nested_result
    formats it."""

    def __init__(self, query: AggQuery, groups: int, block: np.ndarray, capacity: int, estimates: np.ndarray):
        super().__init__(query, block, capacity, np.zeros(groups * query.measure_bytes, np.uint8), groups)
        self.measures = estimates


HLL_REGISTERS = 1 << 14          # p = 14 (reference query/common/hll.go:786)
HLL_DENSE_THRESHOLD = HLL_REGISTERS // 4


class HLLResult:
    """Output of an hll query: one register set per dimension group.

    `regs` is the library's register vector: for every group, in output order, either
    `count` 4-byte little-endian entries `(rho+1) << 16 | reg` (count < 4096) or 16384 bytes of
    `rho+1` per register (reference query/functor.hpp:1351-1374); `counts[g]` = number of non-zero
    registers of group g.  `block` is the DimensionVector block holding the groups' dim rows."""

    def __init__(self, query: AggQuery, groups: int, block: np.ndarray, capacity: int, regs: np.ndarray,
                 counts: np.ndarray):
        self.query, self.groups, self.regs, self.counts = query, groups, regs, counts
        self.dims = QueryResult(query, block, capacity, np.zeros(groups * query.measure_bytes, np.uint8), groups)

    def dense_registers(self) -> dict:
        """packed dim row (bytes) -> uint8[16384] of rho+1 (0 = register never hit)."""
        out, pos = {}, 0
        for g in range(self.groups):
            c = int(self.counts[g])
            dense = np.zeros(HLL_REGISTERS, np.uint8)
            if c < HLL_DENSE_THRESHOLD:
                e = self.regs[pos:pos + 4 * c].view(np.uint32)
                dense[e & 0xFFFF] = (e >> 16).astype(np.uint8)
                pos += 4 * c
            else:
                dense[:] = self.regs[pos:pos + HLL_REGISTERS]
                pos += HLL_REGISTERS
            out[self.dims.rows[g]] = dense
        if pos != self.regs.size:
            raise ValueError("register vector size does not match the per-group counts")
        return out
