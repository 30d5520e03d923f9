"""Host-side batch executors: the driver of the hot path, mirroring the reference's Go
`BatchExecutorImpl` (query/aql_batchexecutor.go:68-273) above the C ABI.

* `LegacyBatchExecutor` issues exactly the per-node call sequence of the reference
  (preExec -> filter -> project -> reduce -> postExec, with carried result vectors,
  query/aql_processor.go:718-776) against ANY library exporting the reference's symbols — the B200
  engine, or (in tests / the CPU baseline) a HOST-mode build running on host memory.
* `FusedBatchExecutor` is the B200-native form: one ExecuteBatchPlan call per batch into a
  device-resident AggState, one AggStateFinalize per query.
* `FusedRequestExecutor` runs the queries of one AQL request: queries that share dimensions, time filter and joins read
  each batch once (ExecuteBatchPlanMulti, one state per query; filters they do not all have are member filters).

Both take batches as lists of `VectorPartySlice`s that already live in the executor's memory space.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, field

import numpy as np

from . import cabi as A
from . import expr as E
from .memory import Buf
from .query import AggQuery, HLLEstimates, HLLResult, QueryResult, member_dimensions
from .skipping import should_skip_batch


@dataclass
class Batch:
    """One live/archive batch of a table shard: column slices in device (or host) memory."""
    columns: list            # list[cabi.VectorPartySlice], indexed by expr.Col.index
    num_rows: int
    base_counts: Buf | None = None   # cumulative counts of the first (RLE) column, or None
    start_count: int = 0
    keep: list = field(default_factory=list)  # owning buffers
    # zone map: {column index: (min, max)} of the VALID values of this batch (BatchPlan.Ranges; a hint the
    # fused kernel verifies per row — what LiveVectorParty.GetMinMaxValue / the archive day give the reference)
    ranges: dict | None = None


def dim_offsets(num_dims_per_width, capacity: int):
    """Value / validity byte offsets of every dim in a DimensionVector block
    (reference query/common/dimval.go:122-145)."""
    offs, widths, pos = [], [], 0
    for w, cnt in zip(A.DIM_WIDTHS, num_dims_per_width):
        for _ in range(cnt):
            offs.append(pos)
            widths.append(w)
            pos += w * capacity
    nulls = [pos + i * capacity for i in range(len(widths))]
    return offs, nulls, widths, pos + len(widths) * capacity


class _ResultBuffers:
    def __init__(self, space, query: AggQuery, capacity: int, zero: bool = True):
        """zero=True is what the reference's DeviceAllocate gives the per-node sequence (it reads carried rows back);
        AggStateFinalize writes every byte of the rows it returns, so the fused path skips the four fill launches."""
        self.capacity = capacity
        _, _, _, total = dim_offsets(query.num_dims_per_width, capacity)
        alloc = space.zeros if zero else space.empty
        self.dims = alloc(total)
        self.hash = alloc(8 * capacity)
        self.index = alloc(4 * capacity)
        self.measures = alloc(query.measure_bytes * capacity)

    def dimension_vector(self, query: AggQuery) -> A.DimensionVector:
        return A.make_dimension_vector(self.dims.ptr, self.hash.ptr, self.index.ptr, query.num_dims_per_width,
                                       self.capacity)


class LegacyBatchExecutor:
    """The reference's one-operator-per-kernel call sequence, batch after batch."""

    def __init__(self, lib: A.Library, space, query: AggQuery):
        if any(E.uses_bucket(d) for d in query.dimensions):
            raise ValueError("numeric bucketizers run on the fused path only: the per-node call sequence has no such functor")
        self.lib, self.space, self.q = lib, space, query
        self.result_size = 0
        self.out: _ResultBuffers | None = None   # results of the batches processed so far
        self.calls = 0                           # C-ABI calls issued (the reference's kernel-launch proxy)
        self.hll: HLLResult | None = None        # set by the last batch of an hll query

    # -- processExpression (reference query/time_series_aggregate.go:493-593) ----------------------
    def _call(self, name, *args):
        self.calls += 1
        return getattr(self.lib, name)(*args)

    def _eval(self, e: E.Expr, batch: Batch, ctx, action):
        """Post-order walk; `action(functor, inputs)` consumes the root, inner nodes go to scratch."""
        sp, lib, stream, dev = self.space, self.lib, self.space.stream, self.space.device
        if isinstance(e, E.Col):
            iv = A.vp_input(batch.columns[e.index])
            if action:
                action(A.Noop, [iv])
                return None
            return iv
        if isinstance(e, E.ForeignCol):
            from . import joins as J
            j = self.q.joins[e.table]
            iv, keep = J.foreign_input(j.table, e.index, ctx["record_ids"][e.table].ptr,
                                       j.timezone_ptr if e.timezone else None, j.timezone_size if e.timezone else 0)
            ctx["frames"].append(keep)   # the host array of batch slices lives until the call returns
            if action:
                action(A.Noop, [iv])
                return None
            return iv
        if isinstance(e, E.Lit):
            iv = A.const_input(e.value, True, is_float=e.type == E.Type.Float)
            if action:
                action(A.Noop, [iv])
                return None
            return iv
        if isinstance(e, E.Unary):
            inputs = [self._eval(e.expr, batch, ctx, None)]
        else:
            inputs = [self._eval(e.lhs, batch, ctx, None), self._eval(e.rhs, batch, ctx, None)]
        if action:
            action(e.op, inputs)
            return None
        dt = E.scratch_data_type(e.type)
        size = ctx["size"]
        frame = sp.zeros(5 * max(size, 1))         # allocateStackFrame: values[4B] + valid[1B] per row
        ctx["frames"].append(frame)
        ov = A.scratch_output(frame.ptr, 4 * size, dt)
        bc = batch.base_counts.ptr if batch.base_counts else None
        if size > 0:
            if len(inputs) == 1:
                self._call("UnaryTransform", inputs[0], ov, ctx["index"].ptr, size, bc, batch.start_count, e.op, stream, dev)
            else:
                self._call("BinaryTransform", inputs[0], inputs[1], ov, ctx["index"].ptr, size, bc, batch.start_count,
                           e.op, stream, dev)
        return A.scratch_input(frame.ptr, 4 * size, dt)

    def process_batch(self, batch: Batch, is_last: bool = False, time_filters: bool = True, cutoff: int = 0):
        """One batch through preExec -> filter -> project -> reduce -> postExec.  `is_last` only
        matters for hll queries (HyperLogLog builds the register vectors on the last batch,
        reference query/aql_batchexecutor.go:228-233)."""
        q, sp, stream, dev = self.q, self.space, self.space.stream, self.space.device
        bc = batch.base_counts.ptr if batch.base_counts else None
        size = batch.num_rows
        # preExec: prepareForFiltering + InitIndexVector (aql_batchexecutor.go:256)
        ctx = {"size": size, "index": sp.zeros(4 * max(size, 1)), "frames": [], "record_ids": [], "rec_ptrs": None}
        predicate = sp.zeros(max(size, 1))
        self._call("InitIndexVector", ctx["index"].ptr, 0, size, stream, dev)

        # filter (aql_batchexecutor.go:103; filterAction time_series_aggregate.go:369-396)
        def filter_action(fn, inputs):
            if ctx["size"] <= 0:
                return
            recs, nrec = ctx["rec_ptrs"], len(ctx["record_ids"])   # RecordID vectors are compacted with the index vector
            if len(inputs) == 1:
                ctx["size"] = self._call("UnaryFilter", inputs[0], ctx["index"].ptr, predicate.ptr, ctx["size"], recs, nrec,
                                         bc, batch.start_count, fn, stream, dev)
            else:
                ctx["size"] = self._call("BinaryFilter", inputs[0], inputs[1], ctx["index"].ptr, predicate.ptr,
                                         ctx["size"], recs, nrec, bc, batch.start_count, fn, stream, dev)

        lo, hi = q.time_filter_range
        main = list(enumerate(q.filters[:q.num_main_filters]))
        if cutoff > 0:                                # a live batch: the cutoff filter opens the custom-filter step
            main.insert(lo, (-1, q.cutoff_filter(cutoff)))
        for i, f in main:
            if not time_filters and lo <= i < hi:     # an archive batch strictly inside the time range (customFilterFunc)
                continue
            self._eval(f, batch, ctx, filter_action)
            ctx["frames"].clear()
        # join (aql_batchexecutor.go:115-147): one RecordID per surviving index position and joined table
        if q.joins:
            for j in q.joins:
                rec = sp.zeros(8 * max(ctx["size"], 1))
                ctx["record_ids"].append(rec)
                if ctx["size"] > 0:
                    self._call("HashLookup", A.vp_input(batch.columns[j.on.index]), rec.ptr, ctx["index"].ptr, ctx["size"], bc,
                               batch.start_count, j.table.hash_index(), stream, dev)
            ptrs = (C.c_void_p * len(q.joins))(*[r.ptr for r in ctx["record_ids"]])
            ctx["rec_ptr_array"] = ptrs
            ctx["rec_ptrs"] = C.cast(ptrs, C.c_void_p).value
            for f in q.filters[q.num_main_filters:]:
                self._eval(f, batch, ctx, filter_action)
                ctx["frames"].clear()
        size = ctx["size"]

        # project: prepareForDimAndMeasureEval (aql_processor.go:743-776) — input buffers hold the
        # carried results in rows [0, resultSize) followed by this batch's rows
        prev = self.result_size
        cap = max(prev + size, 1)
        inb = _ResultBuffers(sp, q, cap)
        outb = _ResultBuffers(sp, q, cap)
        if prev > 0:
            self._copy_results(self.out, inb, prev)
        offs, nulls, widths, _ = dim_offsets(q.num_dims_per_width, cap)
        for pos, qi in enumerate(q.dim_order):
            dexpr, dt, w = q.dimensions[qi], q.dim_types[qi], widths[pos]

            def dim_action(fn, inputs, pos=pos, dt=dt, w=w):
                if ctx["size"] <= 0:
                    return
                ov = A.dimension_output(inb.dims.at(offs[pos] + w * prev), inb.dims.at(nulls[pos] + prev), dt)
                if len(inputs) == 1:
                    self._call("UnaryTransform", inputs[0], ov, ctx["index"].ptr, ctx["size"], bc, batch.start_count, fn, stream, dev)
                else:
                    self._call("BinaryTransform", inputs[0], inputs[1], ov, ctx["index"].ptr, ctx["size"], bc,
                               batch.start_count, fn, stream, dev)

            self._eval(dexpr, batch, ctx, dim_action)
            ctx["frames"].clear()

        def measure_action(fn, inputs):
            if ctx["size"] <= 0:
                return
            # hll: this batch's values go to measureVectorD[1] from row 0 (time_series_aggregate.go:405-408)
            target = outb.measures.ptr if q.is_hll else inb.measures.at(prev * q.measure_bytes)
            ov = A.measure_output(target, q.measure_data_type, q.agg_func)
            if len(inputs) == 1:
                self._call("UnaryTransform", inputs[0], ov, ctx["index"].ptr, ctx["size"], bc, batch.start_count, fn, stream, dev)
            else:
                self._call("BinaryTransform", inputs[0], inputs[1], ov, ctx["index"].ptr, ctx["size"], bc,
                           batch.start_count, fn, stream, dev)

        self._eval(q.measure, batch, ctx, measure_action)
        ctx["frames"].clear()

        # reduce (aql_batchexecutor.go:219-253)
        length = prev + size
        kin, kout = inb.dimension_vector(q), outb.dimension_vector(q)
        if q.is_hll:
            self._call("InitIndexVector", inb.index.ptr, 0, prev, stream, dev)
            self._call("InitIndexVector", outb.index.ptr, prev, prev + size, stream, dev)
            vec, vec_size, counts = C.c_void_p(), C.c_size_t(), C.c_void_p()
            self.result_size = self._call("HyperLogLog", kin, kout, inb.measures.ptr, outb.measures.ptr, prev, size,
                                          bool(is_last), C.byref(vec), C.byref(vec_size), C.byref(counts), stream, dev)
            if is_last:
                self.hll = self._adopt_hll(outb, vec.value, vec_size.value, counts.value, self.result_size)
        elif length > 0:
            if q.reduce_mode == A.ARES_REDUCE_HASH:
                self.result_size = self._call("HashReduce", kin, inb.measures.ptr, kout, outb.measures.ptr,
                                              q.measure_bytes, length, q.agg_func, stream, dev)
            else:
                self._call("InitIndexVector", inb.index.ptr, 0, length, stream, dev)
                self._call("Sort", kin, length, stream, dev)
                self.result_size = self._call("Reduce", kin, inb.measures.ptr, kout, outb.measures.ptr, q.measure_bytes,
                                              length, q.agg_func, stream, dev)
        # postExec: swapResultBufferForNextBatch (aql_processor.go:718-723)
        self.out = outb

    def _adopt_hll(self, outb: _ResultBuffers, vec: int, vec_size: int, counts: int, num_dims: int):
        """Copies the two library-allocated outputs to the host and frees them (the Go side adopts
        them as devicePointers, reference query/time_series_aggregate.go:661-681)."""
        lib, sp = self.lib, self.space
        if num_dims <= 0 or not vec:
            return HLLResult(self.q, 0, np.zeros(0, np.uint8), 1, np.zeros(0, np.uint8), np.zeros(0, np.uint16))

        def read(ptr, nbytes):
            if not sp.is_cuda:
                return np.frombuffer(C.string_at(ptr, nbytes), dtype=np.uint8).copy()
            host = np.zeros(max(nbytes, 1), np.uint8)
            lib.AsyncCopyDeviceToHost(host.ctypes.data, ptr, nbytes, sp.stream, sp.device)
            lib.WaitForCudaStream(sp.stream, sp.device)
            return host[:nbytes]

        regs = read(vec, vec_size)
        cnt = read(counts, 2 * num_dims).view(np.uint16).copy()
        for p in (vec, counts):
            if sp.is_cuda:
                lib.DeviceFree(p, sp.device)
            else:
                C.CDLL(None).free(C.c_void_p(p))
        return HLLResult(self.q, num_dims, outb.dims.get(np.uint8), outb.capacity, regs, cnt)

    def _copy_results(self, src: _ResultBuffers, dst: _ResultBuffers, rows: int):
        q, sp = self.q, self.space
        so, sn, widths, _ = dim_offsets(q.num_dims_per_width, src.capacity)
        do, dn, _, _ = dim_offsets(q.num_dims_per_width, dst.capacity)
        for p, w in enumerate(widths):
            sp.copy(dst.dims, do[p], src.dims, so[p], w * rows)
            sp.copy(dst.dims, dn[p], src.dims, sn[p], rows)
        sp.copy(dst.measures, 0, src.measures, 0, q.measure_bytes * rows)
        if q.is_hll:  # the carried keys travel with the rows (aql_processor.go:763-768)
            sp.copy(dst.hash, 0, src.hash, 0, 8 * rows)

    def result(self) -> QueryResult:
        if self.out is None or self.result_size == 0:
            return QueryResult(self.q, np.zeros(0, np.uint8), 1, np.zeros(0, np.uint8), 0)
        return QueryResult(self.q, self.out.dims.get(np.uint8), self.out.capacity, self.out.measures.get(np.uint8),
                           self.result_size)


def compute_zone_map(lib: A.Library, space, columns: list) -> dict:
    """{column index: (min, max)} of the VALID values of a device-resident batch, computed by the engine
    (ComputeColumnRanges: one kernel over all columns) — what Batch.ranges / BatchPlan.Ranges take.  Called once when a
    batch becomes device resident, the way the memstore maintains LiveVectorParty min / max at ingestion
    (memstore/live_vector_party.go:74-75)."""
    n = len(columns)
    vps = (A.VectorPartySlice * n)(*columns)
    out = (A.ColumnRange * n)()
    lib.ComputeColumnRanges(vps, n, out, space.stream, space.device)
    return {i: (int(out[i].Min), int(out[i].Max)) for i in range(n) if out[i].Known}


class _PinnedLease:
    """One pinned host buffer on loan from the pool; returns itself when collected."""

    def __init__(self, pool, ptr: int, cap: int):
        self.pool, self.ptr, self.cap = pool, ptr, cap
        self.array = np.frombuffer((C.c_uint8 * cap).from_address(ptr), dtype=np.uint8)

    def __del__(self):
        try:
            self.pool.free.setdefault(self.cap, []).append(self.ptr)
        except Exception:
            pass


class _PinnedPool:
    """Pinned (HostAlloc) staging buffers by power-of-two size; buffers are reused, never freed (a few result-sized
    buffers per process)."""

    def __init__(self):
        self.free: dict = {}

    def acquire(self, lib, nbytes: int) -> _PinnedLease:
        cap = 1 << max(16, (max(nbytes, 1) - 1).bit_length())
        stack = self.free.get(cap)
        ptr = stack.pop() if stack else lib.HostAlloc(cap)
        return _PinnedLease(self, ptr, cap)


_PINNED = _PinnedPool()


class _BatchPlans:
    """The BatchPlan of a query's batches: instructions from `instructions(time_filters, cutoff)`, joined tables, and per
    batch the columns, row count and zone map."""

    def __init__(self, query: AggQuery, instructions):
        self.q, self._instructions = query, instructions
        self.insts = instructions(True, 0)
        self._plan = A.BatchPlan()
        self._plan.NumInsts = len(self.insts)
        for i, pi in enumerate(self.insts):
            self._plan.Insts[i] = pi
        self._plan_variants = {}
        # numeric bucketizers: parameters, and their bounds in the executor's memory space (uploaded by the front-end)
        self._plan.NumBucketizers = len(query.bucketizers)
        for j, b in enumerate(query.bucketizers):
            pb = self._plan.Bucketizers[j]
            pb.Kind = {"width": A.PLAN_BUCKET_WIDTH, "log": A.PLAN_BUCKET_LOG, "partitions": A.PLAN_BUCKET_PARTITIONS}[b.kind]
            if b.kind != "partitions":
                pb.Param = b.spec[1]
            if b.kind == "log":
                pb.LogMin = b.spec[2]
            if b.kind != "width":
                if not b.bounds_ptr:
                    raise ValueError("a numeric bucketizer's bounds are not in the executor's memory space (bounds_ptr)")
                pb.Bounds, pb.NumBounds = b.bounds_ptr, len(b.bounds)
        # joined dimension tables: the lookup + foreign-column reads are a gather stage of the fused kernel
        self._join_keep = []
        if query.joins:
            if len(query.joins) > A.ARES_MAX_FOREIGN_TABLES or len(query.foreign_columns) > A.ARES_MAX_FOREIGN_COLUMNS:
                raise ValueError("too many joined tables / foreign columns for one plan")
            self._plan.NumForeignTables = len(query.joins)
            for t, j in enumerate(query.joins):
                self._plan.ForeignTables[t].JoinColumn = j.on.index
                self._plan.ForeignTables[t].Index = j.table.hash_index()
            self._plan.NumForeignColumns = len(query.foreign_columns)
            for k, (t, col, tz) in enumerate(query.foreign_columns):
                j = query.joins[t]
                f, keep = j.table.foreign_column(col, None, j.timezone_ptr if tz else None, j.timezone_size if tz else 0)
                self._join_keep.append(keep)
                self._plan.ForeignColumns[k].Table = t
                self._plan.ForeignColumns[k].Column = f

    def _plan_variant(self, time_filters: bool, cutoff: int):
        """A plan with other custom filters than the query's full set: an archive batch strictly inside the time range
        leaves the time filters out, a live batch adds the cutoff filter.  Same columns, joins and sinks; a different plan
        SHAPE compiles its own specialised kernel, a different cutoff is only a different literal."""
        key = (time_filters, cutoff)
        p = self._plan_variants.get(key)
        if p is None:
            insts = self._instructions(time_filters, cutoff)
            p = A.BatchPlan()
            C.memmove(C.byref(p), C.byref(self._plan), C.sizeof(A.BatchPlan))   # foreign tables / columns as in the full plan
            p.NumInsts = len(insts)
            for i, pi in enumerate(insts):
                p.Insts[i] = pi
            if len(self._plan_variants) > 8:
                self._plan_variants.clear()
            self._plan_variants[key] = p
        return p

    def plan_for(self, batch: Batch, time_filters: bool, cutoff: int) -> A.BatchPlan:
        lo, hi = self.q.time_filter_range
        p = self._plan if (time_filters or lo == hi) and cutoff <= 0 else self._plan_variant(time_filters or lo == hi, max(cutoff, 0))
        p.NumColumns = len(batch.columns)
        for i, vp in enumerate(batch.columns):
            p.Columns[i] = vp
        p.BaseCounts = batch.base_counts.ptr if batch.base_counts else None
        p.StartCount = batch.start_count
        p.NumRows = batch.num_rows
        for i in range(len(batch.columns)):
            r = batch.ranges.get(i) if batch.ranges else None
            p.Ranges[i].Known = 0 if r is None else 1
            p.Ranges[i].Min, p.Ranges[i].Max = (0, 0) if r is None else (int(r[0]), int(r[1]))
        return p


class FusedBatchExecutor:
    """B200-native: one fused kernel per batch into a device-resident group table."""

    def __init__(self, lib: A.Library, space, query: AggQuery, expected_groups: int = 0):
        if not lib.has_plan_api:
            raise RuntimeError("this library does not export the whole-batch plan API")
        self.lib, self.space, self.q = lib, space, query
        self.plans = _BatchPlans(query, lambda tf, co: query.plan_instructions(time_filters=tf, cutoff=co))
        self.state = C.c_void_p(lib.AggStateCreate(query.agg_spec(expected_groups), space.stream, space.device))
        self.calls = 0
        self.skipped = 0   # batches whose zone map contradicts a filter (skipping.py): never launched
        self.expected_groups = expected_groups

    def process_batch(self, batch: Batch, stream=None, time_filters: bool = True, cutoff: int = 0):
        """`time_filters=False`: an archive batch that lies strictly inside the query's time range skips the time filter
        (archiveBatchCustomFilterExecutor evaluates it for the first and the last batch only, query/aql_processor.go:627-638).
        `cutoff` > 0: a live batch of a fact table also evaluates `time >= cutoff` (liveBatchCustomFilterExecutor :543-567)."""
        if should_skip_batch(self.q, batch.ranges):
            self.skipped += 1
            return
        p = self.plans.plan_for(batch, time_filters, cutoff)
        self.calls += 1
        self.lib.ExecuteBatchPlan(self.state, C.byref(p), self.space.stream if stream is None else stream,
                                  self.space.device)

    SMALL_RESULT = 32768   # kSmallFinalizeMax of the engine

    def merge(self, dim_vector: A.DimensionVector, measures_ptr: int, length: int):
        self.lib.AggStateMerge(self.state, dim_vector, measures_ptr, length, self.space.stream, self.space.device)

    def group_count(self) -> int:
        return self.lib.AggStateGroupCount(self.state, self.space.stream, self.space.device)

    def finalize_into(self, capacity: int | None = None):
        """Returns (groups, _ResultBuffers) with the result left in device memory."""
        # Results of up to SMALL_RESULT groups need no count first: AggStateFinalize is one launch + one synchronise
        # and reports a too-small output as an error, after which the exact count is asked for.
        guess = capacity is None and self.expected_groups <= self.SMALL_RESULT and not self.q.is_hll
        cap = self.SMALL_RESULT if guess else max(capacity if capacity is not None else self.group_count(), 1)
        for attempt in (0, 1):
            out = _ResultBuffers(self.space, self.q, cap, zero=not getattr(self.space, "is_cuda", False))
            try:
                g = self.lib.AggStateFinalize(self.state, out.dimension_vector(self.q), out.measures.ptr, self.space.stream,
                                              self.space.device)
                return g, out
            except A.AresError as e:
                if attempt or "capacity is smaller" not in str(e):
                    raise
                cap = max(self.group_count(), 1)

    def result(self) -> QueryResult:
        return query_result(self.q, *self.finalize_into())

    def hll_result(self) -> HLLResult:
        """hll queries: the register vectors of every dimension group (AggStateFinalizeHLL)."""
        lib, sp = self.lib, self.space
        dims, vec, counts, size = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_size_t()
        g = lib.AggStateFinalizeHLL(self.state, C.byref(dims), C.byref(vec), C.byref(size), C.byref(counts), sp.stream, sp.device)
        if g == 0:
            return HLLResult(self.q, 0, np.zeros(0, np.uint8), 1, np.zeros(0, np.uint8), np.zeros(0, np.uint16))

        # one pinned staging buffer for the three vectors (13 MB of register vectors for 808 groups: a pageable read-back
        # costs ~2 ms, a pinned one 0.3), three copies, ONE wait; the result owns the lease of the buffer
        nb, nr, nc = self.q.row_bytes * g, size.value, 2 * g
        o_r, o_c = (nb + 63) // 64 * 64, (nb + 63) // 64 * 64 + (nr + 63) // 64 * 64
        lease = _PINNED.acquire(lib, o_c + nc)
        for ptr, off, n in ((dims.value, 0, nb), (vec.value, o_r, nr), (counts.value, o_c, nc)):
            lib.AsyncCopyDeviceToHost(lease.ptr + off, ptr, n, sp.stream, sp.device)
        lib.WaitForCudaStream(sp.stream, sp.device)
        for p in (dims, vec, counts):
            lib.DeviceFree(p, sp.device)
        host = lease.array
        res = HLLResult(self.q, g, host[:nb], g, host[o_r:o_r + nr], host[o_c:o_c + nc].view(np.uint16))
        res._lease = lease   # back to the pool when the result is collected
        return res

    def hll_estimates(self) -> HLLEstimates:
        """hll queries: the groups of hll_result() with their distinct-count estimates (AggStateFinalizeHLLEstimate);
        the register vectors never leave the device."""
        lib, sp = self.lib, self.space
        dims, est = C.c_void_p(), C.c_void_p()
        g = lib.AggStateFinalizeHLLEstimate(self.state, C.byref(dims), C.byref(est), sp.stream, sp.device)
        if g == 0:
            return HLLEstimates(self.q, 0, np.zeros(0, np.uint8), 1, np.zeros(0, np.float64))
        nb, o_e = self.q.row_bytes * g, (self.q.row_bytes * g + 63) // 64 * 64
        lease = _PINNED.acquire(lib, o_e + 8 * g)
        for ptr, off, n in ((dims.value, 0, nb), (est.value, o_e, 8 * g)):
            lib.AsyncCopyDeviceToHost(lease.ptr + off, ptr, n, sp.stream, sp.device)
        lib.WaitForCudaStream(sp.stream, sp.device)
        for p in (dims, est):
            lib.DeviceFree(p, sp.device)
        host = lease.array   # (the result copies what it keeps: the buffer goes back to the pool with the lease)
        return HLLEstimates(self.q, g, host[:nb], g, host[o_e:o_e + 8 * g].view(np.float64).copy())

    def reset(self):
        self.lib.AggStateReset(self.state, self.space.stream, self.space.device)

    def close(self):
        if self.state:
            self.lib.AggStateDestroy(self.state, self.space.device)
            self.state = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def query_result(q: AggQuery, g: int, out: _ResultBuffers) -> QueryResult:
    """The QueryResult of `g` groups finalized into `out`."""
    if g == 0:
        return QueryResult(q, np.zeros(0, np.uint8), 1, np.zeros(0, np.uint8), 0)
    return QueryResult(q, out.dims.get(np.uint8), out.capacity, out.measures.get(np.uint8), g)


MAX_LAUNCH_STATES = 16   # states of one AggStatesFinalize / AggStatesExportPartsToPeers / AggStatesMergeParts call


def finalize_states(executors: list) -> list:
    """finalize_into of every executor (non-HLL queries) with one AggStatesFinalize per MAX_LAUNCH_STATES states: those
    that announce at most SMALL_RESULT groups share one launch and one synchronise.  Per executor: (groups,
    _ResultBuffers), or the AresError of a state whose finalize failed while the others completed."""
    done = []
    for i in range(0, len(executors), MAX_LAUNCH_STATES):
        done += _finalize_some(executors[i:i + MAX_LAUNCH_STATES])
    return done


def _finalize_some(exs: list) -> list:
    if not exs:
        return []
    lib, sp, n = exs[0].lib, exs[0].space, len(exs)
    bufs = []
    for ex in exs:   # (capacity as finalize_into's first attempt)
        cap = ex.SMALL_RESULT if ex.expected_groups <= ex.SMALL_RESULT else max(ex.group_count(), 1)
        bufs.append(_ResultBuffers(sp, ex.q, cap, zero=not getattr(sp, "is_cuda", False)))
    states = (C.c_void_p * n)(*[ex.state.value for ex in exs])
    keys = (A.DimensionVector * n)(*[b.dimension_vector(ex.q) for b, ex in zip(bufs, exs)])
    values = (C.c_void_p * n)(*[b.measures.ptr for b in bufs])
    groups = (C.c_int64 * n)(*([-2] * n))
    failed = {}
    try:
        lib.AggStatesFinalize(states, n, keys, values, groups, sp.stream, sp.device)
    except A.AresError as e:
        # per-state failures: one line "state k: <message>" each, groups[k] = -1; anything else failed the whole call
        for line in str(e).removeprefix("AggStatesFinalize: ").split("\n"):
            m = re.match(r"state (\d+): (.*)", line)
            if m is None or groups[int(m.group(1))] != -1:
                raise
            failed[int(m.group(1))] = A.AresError(m.group(2))
        if any(g == -2 for g in groups):
            raise
    done = []
    for k, ex in enumerate(exs):
        if k not in failed:
            done.append((groups[k], bufs[k]))
        elif "capacity is smaller" in str(failed[k]):
            done.append(ex.finalize_into(max(ex.group_count(), 1)))   # finalize_into's second attempt: the exact count
        else:
            done.append(failed[k])
    return done


MAX_SHARED_MEASURES = 4   # measure roots (states) of one ExecuteBatchPlanMulti plan


def shared_scan_groups(queries: list, member_filters: bool = False) -> list[list[int]]:
    """Indexes of `queries` grouped for one pass: queries with the same plan instructions except the measure root (same
    filters in the same order, time-filter range, dimensions), the same joins and reduce mode, and no HLL; at most
    MAX_SHARED_MEASURES per group, in request order.  Every other query is a group of its own.
    `member_filters`: queries whose filters differ group as well (same dimensions, time filter, joins and reduce mode);
    a query whose filters would make the group's plan longer than ARES_MAX_PLAN_INSTS starts a new group."""
    groups, open_group = [], {}
    for i, q in enumerate(queries):
        key = q.shared_scan_key(member_filters=member_filters)
        g = open_group.get(key) if key is not None else None
        if g is None or len(g) >= MAX_SHARED_MEASURES or (member_filters and not _plan_fits([queries[j] for j in g + [i]])):
            g = []
            groups.append(g)
            if key is not None:
                open_group[key] = g
        g.append(i)
    return groups


MAX_PASS_DIMENSIONS = 8   # union dimensions of one pass: what the kernel indexes directly (kJitMaxDenseDims)


def shared_scan_passes(queries: list, groups: list) -> list[list[int]]:
    """`groups` (shared_scan_groups with member filters) packed into passes over the batches: groups that agree in time
    filter, joins and reduce mode, with dimensions and without HLL, share a pass (their dimensions become member
    dimensions of its plan) while it has at most MAX_SHARED_MEASURES queries and MAX_PASS_DIMENSIONS dimensions, its plan
    fits the plan limits, and its queries order their dimensions consistently (query.member_dimensions).  Returns the
    indexes of each pass's queries, group by group, in request order."""
    passes, open_pass = [], {}
    for g in groups:
        q = queries[g[0]]
        key = q.shared_scan_key(member_filters=True)
        key = key[1:] if key is not None and q.dimensions else None
        p = open_pass.get(key) if key is not None else None
        if p is not None and _pass_fits([queries[i] for i in p + g]):
            p.extend(g)
            continue
        p = list(g)
        passes.append(p)
        if key is not None:
            open_pass[key] = p
    return passes


def _pass_fits(members: list) -> bool:
    if len(members) > MAX_SHARED_MEASURES:
        return False
    try:
        union = member_dimensions(members)
    except ValueError:
        return False
    return (union is None or len(union) <= MAX_PASS_DIMENSIONS) and _plan_fits(members)


def _plan_fits(members: list) -> bool:
    """The shared plan of `members` (with the cutoff filter of a live batch, its longest variant) stays within the plan
    limits."""
    lead = members[0]
    try:
        lead.plan_instructions(cutoff=1, measures=members)
    except ValueError:
        return False
    return len(lead.foreign_columns) <= A.ARES_MAX_FOREIGN_COLUMNS


class FusedRequestExecutor:
    """The queries of one AQL request (aql.compile_request): each keeps its own AggState and result.  `groups` are the
    compatible groups (shared_scan_groups with member filters: same dimensions, time filter, joins and reduce mode);
    `passes` packs groups that differ only in their dimensions (shared_scan_passes).  The queries of a pass read every
    batch once — one ExecuteBatchPlanMulti call whose plan carries the filters they all have, each query's own filters as
    member filters, their dimensions (as member dimensions when they differ), and one measure root per query.  The engine
    picks the form per batch: one kernel for all of them, one kernel per set of queries with the same dimensions, or each
    query's own kernel."""

    def __init__(self, lib: A.Library, space, queries: list, expected_groups: int | list = 0):
        """`expected_groups`: one hint for every query, or a list with one per query."""
        self.lib, self.space, self.queries = lib, space, list(queries)
        eg = list(expected_groups) if isinstance(expected_groups, (list, tuple)) else [expected_groups] * len(self.queries)
        self.executors = [FusedBatchExecutor(lib, space, q, g) for q, g in zip(self.queries, eg)]
        self.groups = shared_scan_groups(self.queries, member_filters=True)
        self.passes = shared_scan_passes(self.queries, self.groups)
        self._shared = {}   # (indexes of the queries that run a batch together) -> their _BatchPlans
        self.calls = 0

    def _plans(self, members: tuple) -> _BatchPlans:
        """The plans of the members of a pass that run a batch: the whole pass, or the members whose filters the
        batch's zone map does not contradict (built on first use, like the time-filter variants)."""
        p = self._shared.get(members)
        if p is None:
            lead, qs = self.queries[members[0]], [self.queries[i] for i in members]
            p = self._shared[members] = _BatchPlans(lead, lambda tf, co: lead.plan_instructions(time_filters=tf, cutoff=co,
                                                                                               measures=qs))
        return p

    def process_batch(self, batch: Batch, stream=None, time_filters: bool = True, cutoff: int = 0):
        """Same meaning as FusedBatchExecutor.process_batch, for every query of the request.  A query whose filters the
        batch's zone map contradicts skips the batch as it would alone; the other queries of its pass run it together."""
        for g in self.passes:
            if len(g) == 1:
                self.executors[g[0]].process_batch(batch, stream, time_filters, cutoff)
                continue
            run = []
            for i in g:
                if should_skip_batch(self.queries[i], batch.ranges):
                    self.executors[i].skipped += 1
                else:
                    run.append(i)
            if not run:
                continue
            if len(run) == 1:
                self.executors[run[0]].process_batch(batch, stream, time_filters, cutoff)
                continue
            p = self._plans(tuple(run)).plan_for(batch, time_filters, cutoff)
            states = (C.c_void_p * len(run))(*[self.executors[i].state.value for i in run])
            self.calls += 1
            self.lib.ExecuteBatchPlanMulti(states, len(run), C.byref(p), self.space.stream if stream is None else stream,
                                           self.space.device)

    def results(self, hll_estimates: bool = False) -> list:
        """One QueryResult per query, in request order.  The non-HLL queries are finalized together (one AggStatesFinalize
        launch and one synchronise for those that announce at most SMALL_RESULT groups).  `hll_estimates`: an HLL query
        gives its HLLEstimates (distinct counts computed on the device) instead of the QueryResult of its carried rows."""
        idx = [i for i, q in enumerate(self.queries) if not q.is_hll]
        done = dict(zip(idx, finalize_states([self.executors[i] for i in idx])))
        out = []
        for i, ex in enumerate(self.executors):
            if i not in done:
                out.append(ex.hll_estimates() if hll_estimates else ex.result())
            elif isinstance(done[i], Exception):
                raise done[i]
            else:
                out.append(query_result(ex.q, *done[i]))
        return out

    def reset(self):
        for ex in self.executors:
            ex.reset()

    def close(self):
        for ex in self.executors:
            ex.close()
