"""Every batch of ExecuteBatchPlan runs on the plan-shape specialised fused kernel: there is no second executor.  The
inputs that need care on the way in are covered here — batches without a full tile (all rows are the tail one CTA copies
and folds), plans that stage nothing, column parts and base counts off a 16-byte boundary (copied to an aligned buffer
before the launch), more RLE columns than the kernel decodes from their runs and 8-byte RLE columns (expanded), constant
8-byte dimensions, and plans at the bounds of the parameter block (33 staged parts, more than 64 literals).
CPU: AresJitDryRun generates and compiles the kernel of each.  GPU: the result equals the reference call sequence on
the oracle, and every batch was one launch of the specialised kernel."""
import ctypes as C
import types

import numpy as np
import pytest

import harness as H
import test_jit_codegen as J
import test_pipeline_parity as T
from aresdb_b200 import cabi as A, columns, expr as E, synth
from aresdb_b200.executor import Batch, FusedBatchExecutor, LegacyBatchExecutor
from aresdb_b200.query import AggQuery, Measure

FAKE = 0x7F0000000000   # dry runs: fake device addresses, nothing is dereferenced


def _dry_run_columns(lib, q, cols, rows, base_counts=None):
    fn = lib.alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    p = A.BatchPlan()
    insts = q.plan_instructions()
    p.NumInsts = len(insts)
    for i, pi in enumerate(insts):
        p.Insts[i] = pi
    p.NumColumns = len(cols)
    for i, vp in enumerate(cols):
        p.Columns[i] = vp
    p.NumRows = rows
    if base_counts is not None:
        p.BaseCounts = base_counts
    src = C.c_char_p()
    h = fn(q.agg_spec(), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return int(h.res or 0), (src.value or b"").decode()


# ---- plans ----------------------------------------------------------------------------------------------------------
UUID_COL = E.Col(0, A.UUID, "uuid")


def wide_columns_query():
    """16 Uint32 columns, each read by an instruction: values + null bitmaps + base counts = 33 staged parts."""
    cols = [E.Col(i, A.Uint32, f"c{i}") for i in range(16)]
    return AggQuery([E.ne(c, E.Lit(1000 + i)) for i, c in enumerate(cols[1:15])], [cols[0]], Measure("sum", cols[15]))


def many_literals_query():
    """91 literal operands in 63 instructions (a literal sum compared with a literal: two instructions, three literals)."""
    always = [E.lt(E.add(E.Lit(i), E.Lit(i + 1)), E.Lit(1000 + i)) for i in range(30)]
    return AggQuery(always + [E.ne(T.CITY, E.Lit(0))], [T.CITY], Measure("sum", T.FARE))


I64 = E.Col(4, A.Int64, "id64")


def const_int64_query():
    return AggQuery([E.ne(T.CITY, E.Lit(0))], [I64, T.CITY], Measure("sum", T.FARE))


# ---- CPU: these plans specialise ------------------------------------------------------------------------------------
def test_uuid_only_plan_specialises():
    """Nothing to stage: the tile loop runs on empty stages (mbarrier phases with zero bytes) and the kernel reads the
    16-byte column per row."""
    lib = A.load_engine()
    q = AggQuery([], [UUID_COL], Measure("count"))
    size, src = _dry_run_columns(lib, q, [columns.slice_of(FAKE, A.UUID, 100000, 0, 64 * 200, 2)], 100000)
    assert size > 0 and "#define JIT_NUM_PARTS 0" in src and "#define JIT_STAGE_BYTES 0" in src


@pytest.mark.parametrize("rows", [1, 127, 4095])
def test_batches_without_a_full_tile_specialise(rows):
    """The layout does not depend on the row count: a batch too short for a full tile gets the text of a large batch
    without a zone map (its zone map is ignored: the hash-table form) and shares its kernel."""
    lib = A.load_engine()
    q = T.queries()["cfg3_sum"]
    size, src = J._dry_run(lib, q, rows=rows, ranges=J.DAY_RANGES)
    assert size > 0 and "#define JIT_DENSE 0" in src
    assert src == J._dry_run(lib, q, rows=1000000)[1]


def test_sixteen_columns_with_nulls_and_base_counts_specialise():
    lib = A.load_engine()
    cols = [columns.slice_of(FAKE + i * (1 << 30), A.Uint32, 100000, 0, 64 * 200, 2) for i in range(16)]
    size, src = _dry_run_columns(lib, wide_columns_query(), cols, 100000, base_counts=0x7E0000000000)
    assert size > 0 and "#define JIT_NUM_PARTS 33" in src and "runLen[r]" in src


def test_plan_with_more_than_64_literals_specialises():
    lib = A.load_engine()
    q = many_literals_query()
    assert sum(pi.A.Kind == A.PLAN_OPERAND_CONST for pi in q.plan_instructions()) + \
        sum(pi.NumOperands == 2 and pi.B.Kind == A.PLAN_OPERAND_CONST for pi in q.plan_instructions()) > 64
    size, src = J._dry_run(lib, q)
    assert size > 0 and "P.consts[90]" in src


def test_rle_columns_of_a_min_plan_do_not_count_run_lengths():
    """Archive batch whose RLE columns are decoded from their runs: the staged base counts give the row numbers, and
    only SUM / COUNT / AVG multiply by the run lengths — a MIN does not."""
    lib = A.load_engine()
    cols = [columns.slice_of(FAKE + i * (1 << 30), dt, 6000, 64 * 100, 64 * 200, 3 if i in (1, 2) else 2)
            for i, dt in enumerate(synth.COLUMN_TYPES)]
    size, src = _dry_run_columns(lib, T.queries()["min_city"], cols, 6000, base_counts=0x7E0000000000)
    assert size > 0 and "ldrle<" in src and "rowNo[" in src and "runLen" not in src and "mulCount(" not in src
    size, src = _dry_run_columns(lib, T.queries()["cfg3_count"], cols, 6000, base_counts=0x7E0000000000)
    assert size > 0 and "ldrle<" in src and "runLen[r]" in src


def test_constant_int64_dimension_specialises():
    """A mode-0 8-byte dimension: its default value is emitted as constant words of the key."""
    lib = A.load_engine()
    cols = [columns.slice_of(FAKE + i * (1 << 30), dt, 100000, 0, 64 * 200, 2) for i, dt in enumerate(synth.COLUMN_TYPES)]
    cols.append(columns.constant_column(A.Int64, -(5 << 40), True))
    size, src = _dry_run_columns(lib, const_int64_query(), cols, 100000)
    assert size > 0 and f"0x{(-(5 << 40)) & (2 ** 64 - 1):016x}ull" in src


# ---- GPU: each input class against the oracle's reference sequence --------------------------------------------------
def _jit_launches(eng) -> int:
    out = (C.c_ulonglong * 2)()
    eng.lib.alg.AresJitStats(out)
    return int(out[1])


def _check(q, make_batches, ctx, avg=False):
    """make_batches(backend) -> list of Batch.  The fused result equals the reference sequence on the oracle, and every
    batch was exactly one launch of the specialised kernel."""
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    exp_ex = LegacyBatchExecutor(orc.lib, orc.space, q)
    for b in make_batches(orc):
        exp_ex.process_batch(b)
    exp = exp_ex.result()
    got_ex = FusedBatchExecutor(eng.lib, eng.space, q)
    batches = make_batches(eng)
    before = _jit_launches(eng)
    for b in batches:
        got_ex.process_batch(b)
    got = got_ex.result()
    got_ex.close()
    assert _jit_launches(eng) - before == len(batches), f"{ctx}: not every batch ran on the specialised kernel"
    assert exp.groups > 0, ctx
    T.assert_same_result(got, exp, ordered=q.reduce_mode == A.ARES_REDUCE_SORT, ctx=ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("value_align", [4, 2, 1])
def test_unaligned_columns_on_b200(value_align):
    """Null bitmaps and values of every column off a 16-byte boundary, and a bool column whose row 0 is bit 3."""
    hbs = [synth.generate_batch(d, n, num_cities=30, null_rate=0.05) for d, n in ((0, 30011), (1, 9000))]
    flags = [(hb.values[synth.COL_REQUEST_AT] // 7 % 2).astype(np.uint8) for hb in hbs]

    def make(be):
        out = []
        for hb, flag in zip(hbs, flags):
            cols, keep = [], []
            for dt, v, ok in zip(synth.COLUMN_TYPES, hb.values, hb.valid):
                buf, vp = columns.make_column(be.space, dt, v, valid=ok, value_align=value_align)
                cols.append(vp)
                keep.append(buf)
            buf, vp = columns.make_column(be.space, A.Bool, flag, valid=np.arange(flag.size) % 11 != 0, start_bit=3,
                                          value_align=value_align)
            cols.append(vp)
            keep.append(buf)
            out.append(Batch(cols, hb.num_rows, keep=keep))
        return out
    flag = E.Col(4, A.Bool, "flag")
    for name, q in (("flag", AggQuery([flag, E.ne(T.CITY, E.Lit(0))], [T.CITY, E.floor(T.TS, E.Lit(3600)), T.STATUS],
                                      Measure("sum", T.FARE))),
                    ("cfg3_count", T.queries()["cfg3_count"])):
        _check(q, make, f"align {value_align}/{name}")


def _archive(be, seed, runs, extra_rle, unaligned_bc=False):
    """Archive batch: index positions are runs of the batch's base counts; request_at and fare carry one value per index
    position, city is RLE over the base counts (read directly), `extra_rle` further columns (dtype, values per run) are
    RLE with their own, finer counts."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 9, runs)
    base = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    total = int(base[-1])
    cols, keep = [], []

    def add(dt, v, ok=None, counts=None):
        buf, vp = columns.make_column(be.space, dt, v, valid=ok, counts=counts)
        cols.append(vp)
        keep.append(buf)
    add(A.Uint32, (synth.BASE_TS + rng.integers(0, 86400, runs)).astype(np.uint32), rng.random(runs) > 0.02)
    add(A.Uint16, np.sort(rng.integers(1, 40, runs)).astype(np.uint16), None, base)
    add(A.Float32, (rng.integers(0, 6400, runs) / 64.0).astype(np.float32), rng.random(runs) > 0.02)
    for k, (dt, make_values) in enumerate(extra_rle):
        cuts = np.sort(rng.choice(np.arange(1, total), size=runs // (k + 2), replace=False))
        counts = np.concatenate([[0], cuts, [total]]).astype(np.uint32)
        n = len(counts) - 1
        add(dt, make_values(rng, n), rng.random(n) > 0.05, counts)
    if unaligned_bc:   # the same counts 4 bytes into a buffer: off the 16-byte boundary
        buf = be.put(np.concatenate([[7], base]).astype(np.uint32))
        keep.append(buf)
        bc = types.SimpleNamespace(ptr=buf.ptr + 4)
    else:
        bc = be.put(base)
    return Batch(cols, runs, base_counts=bc, start_count=0, keep=keep)


ARCHIVE_TS, ARCHIVE_CITY, ARCHIVE_FARE = E.Col(0, A.Uint32, "ts"), E.Col(1, A.Uint16, "city"), E.Col(2, A.Float32, "fare")


@pytest.mark.gpu
def test_unaligned_base_counts_on_b200():
    """SUM / COUNT multiply by run lengths read from base counts that start 4 bytes off a 16-byte boundary; city's
    counts are then no longer the batch's base counts (another address): it is decoded from its runs."""
    for q in (AggQuery([E.ne(ARCHIVE_CITY, E.Lit(3))], [ARCHIVE_CITY, E.floor(ARCHIVE_TS, E.Lit(3600))], Measure("sum", ARCHIVE_FARE)),
              AggQuery([], [ARCHIVE_CITY], Measure("count"))):
        _check(q, lambda be: [_archive(be, s, 20000, [], unaligned_bc=True) for s in (1, 2)], "unaligned base counts")


@pytest.mark.gpu
def test_six_rle_columns_with_an_int64_dimension_on_b200():
    """Six RLE columns with their own counts besides city: four are decoded from their runs, the fifth and the 8-byte
    one are expanded."""
    extra = [(A.Uint8, lambda r, n: r.integers(0, 4, n).astype(np.uint8)),
             (A.Uint16, lambda r, n: r.integers(0, 9, n).astype(np.uint16)),
             (A.Uint32, lambda r, n: r.integers(0, 1000, n).astype(np.uint32)),
             (A.Int16, lambda r, n: r.integers(-50, 50, n).astype(np.int16)),
             (A.Bool, lambda r, n: r.integers(0, 2, n).astype(np.uint8)),
             (A.Int64, lambda r, n: r.integers(-3, 3, n).astype(np.int64) * (1 << 40))]
    c = [E.Col(3 + k, dt, f"r{k}") for k, (dt, _) in enumerate(extra)]
    q = AggQuery([E.ne(c[0], E.Lit(2)), E.lt(c[2], E.Lit(900)), E.gt(c[3], E.Lit(-40)), c[4]], [c[5], c[1], ARCHIVE_CITY],
                 Measure("sum", ARCHIVE_FARE))
    _check(q, lambda be: [_archive(be, s, n, extra) for s, n in ((1, 30000), (2, 2000))], "six RLE columns")


@pytest.mark.gpu
def test_constant_int64_dimension_on_b200():
    def make(be):
        out = []
        for d, n in ((0, 20000), (1, 3001)):
            b = T.upload(be, synth.generate_batch(d, n, num_cities=25, null_rate=0.02))
            b.columns.append(columns.constant_column(A.Int64, -(5 << 40) + d, True))
            out.append(b)
        return out
    _check(const_int64_query(), make, "constant int64 dimension")


@pytest.mark.gpu
def test_thirty_three_part_plan_on_b200():
    """16 mode-2 columns and the base counts of an archive batch: every part the parameter block holds."""
    def make(be):
        out = []
        for seed, runs in ((1, 25000), (2, 6000)):
            rng = np.random.default_rng(seed)
            base = np.concatenate([[0], np.cumsum(rng.integers(1, 5, runs))]).astype(np.uint32)
            cols, keep = [], []
            for i in range(16):
                v = rng.integers(0, 20 if i == 0 else 1200, runs).astype(np.uint32)
                buf, vp = columns.make_column(be.space, A.Uint32, v, valid=rng.random(runs) > 0.01)
                cols.append(vp)
                keep.append(buf)
            out.append(Batch(cols, runs, base_counts=be.put(base), keep=keep))
        return out
    _check(wide_columns_query(), make, "33 parts")


@pytest.mark.gpu
def test_many_literals_on_b200():
    _check(many_literals_query(), lambda be: [T.upload(be, synth.generate_batch(d, 15000, num_cities=20)) for d in range(2)],
           "many literals")


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 3, 129, 1023, 4095])
def test_batches_without_a_full_tile_on_b200(rows):
    """All rows are the tail: one CTA copies them byte for byte and folds them.  With a zone map the hash-table form
    is kept (no direct-indexed launch)."""
    eng = H.get_backend("b200")
    hbs = [synth.generate_batch(d, rows, num_cities=6, null_rate=0.05) for d in range(2)]
    _check(T.queries()["no_dims_wide"], lambda be: [T.upload(be, hb) for hb in hbs], f"rows={rows}/wide rows")
    q = AggQuery([], [T.CITY, E.floor(T.TS, E.Lit(3600))], Measure("sum", T.FARE))
    before = T.dense_launches(eng)
    _check(q, lambda be: [T.upload(be, hb, ranges=synth.zone_map(hb)) for hb in hbs], f"rows={rows}/zone map")
    assert T.dense_launches(eng) == before
