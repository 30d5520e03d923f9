"""The NVRTC generator (aresdb_b200/csrc/jit.cu) needs no GPU to be exercised: AresJitDryRun generates the
shape-specialised kernel of a plan and compiles it for sm_90a.  Every query of the pipeline parity suite must
be eligible and compile; the GPU suite then checks that what it computes is bit-identical to the reference."""
import ctypes as C

import pytest

from aresdb_b200 import expr as E
from aresdb_b200.query import AggQuery, Measure

from aresdb_b200 import cabi as A
from aresdb_b200 import columns, synth
import test_pipeline_parity as T


def _dry_run(lib, q, rows=100000, start_bit=0, expected_groups=0, base_counts=None, ranges=None):
    fn = lib.alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    p = A.BatchPlan()
    insts = q.plan_instructions()
    p.NumInsts = len(insts)
    for i, pi in enumerate(insts):
        p.Insts[i] = pi
    p.NumColumns = len(synth.COLUMN_TYPES)
    for i, dt in enumerate(synth.COLUMN_TYPES):  # fake, 64-byte aligned device addresses: nothing is dereferenced
        p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, rows, 0, 64 * 200, 2, start_bit)
    p.NumRows = rows
    if base_counts is not None:
        p.BaseCounts = base_counts
    for col, (lo, hi) in (ranges or {}).items():
        p.Ranges[col].Known, p.Ranges[col].Min, p.Ranges[col].Max = 1, lo, hi
    keep = []
    if getattr(q, "joins", None):   # joined dimension tables: fake device addresses, real host-side batch arrays
        p.NumForeignTables = len(q.joins)
        for t, j in enumerate(q.joins):
            p.ForeignTables[t].JoinColumn = j.on.index
            p.ForeignTables[t].Index = j.table.hash_index()
        p.NumForeignColumns = len(q.foreign_columns)
        for k, (t, col, tz) in enumerate(q.foreign_columns):
            f, arr = q.joins[t].table.foreign_column(col, None, 0x7E0000000000 if tz else None, 12 if tz else 0)
            keep.append(arr)
            p.ForeignColumns[k].Table, p.ForeignColumns[k].Column = t, f
    src = C.c_char_p()
    h = fn(q.agg_spec(expected_groups), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return int(h.res or 0), (src.value or b"").decode()


@pytest.mark.parametrize("name", list(T.queries()))
def test_every_pipeline_query_specialises(name):
    lib = A.load_engine()
    size, src = _dry_run(lib, T.queries()[name])
    assert size > 0, "plan was not eligible for specialisation"
    assert "rowEval" in src and "evalBinary" in src or "evalUnary" in src


def test_literals_are_runtime_parameters():
    """Two queries that differ only in their literal operands share one kernel (same generated text)."""
    from aresdb_b200 import expr as E
    from aresdb_b200.query import AggQuery, Measure
    lib = A.load_engine()
    q1 = AggQuery([E.ge(T.TS, E.Lit(1000)), E.gt(T.FARE, E.Lit(5.0))], [T.CITY], Measure("count"))
    q2 = AggQuery([E.ge(T.TS, E.Lit(2000)), E.gt(T.FARE, E.Lit(7.5))], [T.CITY], Measure("count"))
    assert _dry_run(lib, q1)[1] == _dry_run(lib, q2)[1]


def test_hll_queries_specialise_in_both_modes():
    """AGGR_HLL plans compile too.  Entry mode (many groups expected) keys the table by
    (dim-row hash & ~0xFFFF) | register; dense mode keeps one register array per dimension row and
    mirrors the directory of rows in shared memory."""
    import test_hll_pipeline as HP
    lib = A.load_engine()
    for name, q in HP.hll_queries().items():
        size, src = _dry_run(lib, q, expected_groups=100000)
        assert size > 0, name
        assert "#define JIT_HLL 1" in src and "#define JIT_KW 4" in src
        size, src = _dry_run(lib, q)
        assert size > 0, name
        assert "#define JIT_HLL 2" in src and "#define JIT_DENSE_SLOTS 8192" in src


def test_avg_queries_specialise():
    lib = A.load_engine()
    for name, q in T.avg_queries().items():
        size, src = _dry_run(lib, q)
        assert size > 0, name
        assert "<< 32) | (uint32_t)cvt" in src      # (float average, count) packing of the measure


def test_on_disk_cubin_cache(tmp_path, monkeypatch):
    """ARESDB_B200_JIT_CACHE_DIR: the second compile of the same shape is served from disk; an entry whose
    stored source differs (hash collision / stale build) is ignored."""
    import time
    monkeypatch.setenv("ARESDB_B200_JIT_CACHE_DIR", str(tmp_path))
    lib = A.load_engine()
    q = T.queries()["cfg3_sum"]
    t0 = time.perf_counter(); size1, _ = _dry_run(lib, q); t1 = time.perf_counter()
    size2, _ = _dry_run(lib, q); t2 = time.perf_counter()
    files = sorted(p.name for p in tmp_path.iterdir())
    assert len(files) == 2 and files[0].endswith(".cu") and files[1].endswith(".cubin")
    assert size1 == size2 > 0 and (t2 - t1) < 0.5 * (t1 - t0)
    src = tmp_path / files[0]
    src.write_bytes(src.read_bytes() + b"// tampered")
    size3, _ = _dry_run(lib, q)
    assert size3 == size1     # recompiled, not served from the mismatching entry


def test_mixed_column_modes_and_wide_dims_all_specialise():
    """Mode-0 / mode-1 columns, bool columns with a bit offset and 8- / 16-byte dimension columns."""
    lib = A.load_engine()
    fn = lib.alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    rows = 100000
    for name, q in T.mixed_queries().items():
        p = A.BatchPlan()
        insts = q.plan_instructions()
        p.NumInsts = len(insts)
        for i, pi in enumerate(insts):
            p.Insts[i] = pi
        base = 0x7F0000000000
        specs = [(A.Uint32, 1, 0), None, (A.Bool, 2, 3), (A.Float32, 2, 0), (A.Int64, 2, 0), (A.UUID, 2, 0)]
        p.NumColumns = len(specs)
        for i, sp in enumerate(specs):
            if sp is None:
                p.Columns[i] = columns.constant_column(A.Uint16, 7, True)
            else:
                dt, mode, sb = sp
                p.Columns[i] = columns.slice_of(base + i * (1 << 32), dt, rows, 0, 64 * 200, mode, sb)
        p.NumRows = rows
        src = C.c_char_p()
        h = fn(q.agg_spec(), C.byref(p), C.byref(src))
        assert not h.pStrErr, C.string_at(h.pStrErr).decode()
        # (uuid_dim reads only a 16-byte and a constant column: nothing is staged, the tile loop runs on empty stages)
        assert int(h.res or 0) > 0, f"{name} was not eligible for specialisation"


def test_rle_batches_stage_their_base_counts_aligned_or_not():
    """An archive batch (base counts given): SUM / COUNT / AVG kernels stage the cumulative counts and multiply
    by the run length; MIN / MAX ignore them.  Unaligned base counts are copied to an aligned buffer before the launch:
    the kernel is the same."""
    lib = A.load_engine()
    aligned, unaligned = 0x7E0000000000, 0x7E0000000004
    size, src = _dry_run(lib, T.queries()["cfg3_count"], base_counts=aligned)
    assert size > 0 and "runLen[r]" in src and "mulCount(" in src
    size, src = _dry_run(lib, T.avg_queries()["avg_fare_by_city"], base_counts=aligned)
    assert size > 0 and "(uint64_t)runLen[r] << 32" in src
    size, src = _dry_run(lib, T.queries()["min_city"], base_counts=aligned)
    assert size > 0 and "runLen" not in src
    size, src = _dry_run(lib, T.queries()["cfg3_count"], base_counts=aligned)
    assert _dry_run(lib, T.queries()["cfg3_count"], base_counts=unaligned) == (size, src)


DAY_RANGES = {synth.COL_REQUEST_AT: (synth.BASE_TS, synth.BASE_TS + 86399), synth.COL_CITY_ID: (0, 100),
              synth.COL_STATUS: (0, 3)}
FARE_RANGE = {synth.COL_FARE: (0, 0x42C80000)}   # [0.0, 100.0] as float bits


def test_float_sum_accumulates_integers_when_the_measure_is_bounded():
    """SUM(float column) in f64 with a zone map on the measure column: accumulator mode 4 (exact integers on the 2^-S
    grid, native 32-bit atomics); without it, or for expressions / other aggregates, the split CAS / RED form."""
    lib = A.load_engine()
    q = T.queries()["cfg3_sum"]
    both = {**DAY_RANGES, **FARE_RANGE}
    assert "#define JIT_DENSE_ACC 4" in _dry_run(lib, q, ranges=both)[1]
    assert "#define JIT_DENSE_ACC 2" in _dry_run(lib, q, ranges=DAY_RANGES)[1]
    doubled = AggQuery(q.filters, [E.floor(T.TS, E.Lit(3600)), T.CITY], Measure("sum", E.mul(T.FARE, E.Lit(2.0))))
    assert "#define JIT_DENSE_ACC 2" in _dry_run(lib, doubled, ranges=both)[1]
    assert "#define JIT_DENSE_ACC 1" in _dry_run(lib, T.queries()["cfg3_count"], ranges=both)[1]


def test_zone_map_selects_direct_indexed_aggregation():
    """With a zone map (BatchPlan.Ranges) that bounds every dimension the kernel is generated in its
    direct-indexed form: slots addressed by (value - min), no key table.  The ranges themselves are runtime
    parameters (another day, another city range: same kernel text); unknown or too wide ranges, HLL and
    high-cardinality plans keep the hash-table form."""
    lib = A.load_engine()
    q = T.queries()["cfg3_sum"]
    size, src = _dry_run(lib, q, ranges=DAY_RANGES)
    assert size > 0 and "#define JIT_DENSE 1" in src and "#define JIT_ND 2" in src and "densePack" in src
    other_day = dict(DAY_RANGES)
    other_day[synth.COL_REQUEST_AT] = (synth.BASE_TS + 5 * 86400, synth.BASE_TS + 6 * 86400 - 1)
    other_day[synth.COL_CITY_ID] = (1, 57)
    assert _dry_run(lib, q, ranges=other_day)[1] == src
    # no zone map / only one of the two dimensions bounded / range too wide for the CTA's slots
    assert "#define JIT_DENSE 0" in _dry_run(lib, q)[1]
    assert "#define JIT_DENSE 0" in _dry_run(lib, q, ranges={synth.COL_CITY_ID: (0, 100)})[1]
    # more slots than a CTA holds (25 hours x 65537 cities): ONE accumulator array in global memory for the whole grid
    wide = dict(DAY_RANGES)
    wide[synth.COL_CITY_ID] = (0, 65535)
    assert "#define JIT_DENSE 2" in _dry_run(lib, q, ranges=wide)[1]
    # ... which has no "reached" flags, so a sum of an integer column (may return to 0) keeps the hash table there,
    wide_int = AggQuery(q.filters, [E.floor(T.TS, E.Lit(3600)), T.CITY], Measure("sum", T.CITY))
    assert "#define JIT_DENSE 0" in _dry_run(lib, wide_int, ranges=wide)[1]
    assert "#define JIT_DENSE 2" in _dry_run(lib, AggQuery(q.filters, [E.floor(T.TS, E.Lit(3600)), T.CITY], Measure("count")), ranges=wide)[1]
    # and beyond 2^21 slots nothing is dense
    assert "#define JIT_DENSE 0" in _dry_run(lib, AggQuery([], [T.TS, T.CITY], Measure("count")), ranges=DAY_RANGES)[1]
    # every aggregate of the suite compiles in the dense form
    for name, qq in list(T.queries().items()) + list(T.avg_queries().items()):
        size, s2 = _dry_run(lib, qq, ranges=DAY_RANGES)
        assert size > 0, name


def test_join_queries_specialise():
    """Plans that read joined dimension tables (cuckoo probe + foreign-column gather inside the fused kernel) compile."""
    import harness as H
    import test_joins as TJ
    lib = A.load_engine()
    orc = H.get_backend("oracle")            # host memory stands in for the device buffers: nothing is dereferenced
    table, _ = TJ._dimension_table(orc)
    for name, q in TJ.join_queries(table, 0x7E0000000000, 12).items():
        size, src = _dry_run(lib, q)
        assert size > 0, name
        assert "cuckooLookup(P.join->tables[0]" in src and "foreignLoad(P.join->cols[" in src
