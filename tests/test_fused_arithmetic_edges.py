"""Edge tables for the arithmetic the specialised fused kernel (csrc/jit.cu) rewrites instead of calling the shared
functors of cell.cuh:

  * division by an integer literal: a magic multiplier (fastDivU32 / fastDivOp) and, for a direct-indexed quotient
    dimension, the 32-bit span form (__umulhi(x - base, floor(2^32/d) + 1));
  * `1-byte column == literal` filters compared four bytes at a time (packedEq, the `dead` word);
  * SUM of a bounded Float32 column accumulated as integers on the 2^-S grid (JIT_DENSE_ACC 4).

Expected values come from a plain Python-integer restatement of evalBinary (C truncating division, remainder with
the dividend's sign, Floor = a - a % b, u32 wraparound, comparisons in the common class) and, for float sums, from
exact integer sums on the 2^-149 grid rounded once to double.  The CPU tests pin the restatement against the C
restatement of the per-node ABI (oracle) and the reference's HOST build (stored digests), and check with the
generator's dry run that every GPU case reaches the path it targets.  The GPU tests run the same tables through
FusedBatchExecutor and the per-node sequence on the engine.
"""
import ctypes as C
import struct
from fractions import Fraction

import numpy as np
import pytest

import harness as H
import parity_cases as P
import test_jit_codegen as J
from aresdb_b200 import cabi as A
from aresdb_b200 import columns, expr as E
from aresdb_b200.executor import Batch, FusedBatchExecutor, LegacyBatchExecutor
from aresdb_b200.query import AggQuery, Measure

M32 = 0xFFFFFFFF
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


# ---- restatement of evalBinary (cell.cuh) over 32-bit cells --------------------------------------------------------
def u32(x):
    return x & M32


def i32(x):
    x &= M32
    return x - 2 ** 32 if x >= 2 ** 31 else x


def c_div(a, b):
    """C truncating division."""
    q = abs(a) // abs(b)
    return -q if (a < 0) != (b < 0) else q


def c_mod(a, b):
    """C remainder: takes the dividend's sign."""
    return a - b * c_div(a, b)


def eval_binary(fn, a, b, signed):
    """Result bits of `a fn b` in the common class (I32 when `signed`, else U32); a, b are the operands' 32-bit cells.
    Divisors 0 and -1 give the engine's defined results (cell.cuh: evalBinary)."""
    if signed:
        x, y = i32(a), i32(b)
        if fn == A.Divide:
            return M32 if y == 0 else u32(-x) if y == -1 else u32(c_div(x, y))
        if fn == A.Mod:
            return u32(x) if y == 0 else 0 if y == -1 else u32(c_mod(x, y))
        if fn == A.Floor:
            return 0 if y == 0 else u32(x) if y == -1 else u32(x - c_mod(x, y))
    else:
        x, y = u32(a), u32(b)
        if fn == A.Divide:
            return M32 if y == 0 else x // y
        if fn == A.Mod:
            return x if y == 0 else x % y
        if fn == A.Floor:
            return 0 if y == 0 else x - x % y
    cmp = {A.Equal: x == y, A.NotEqual: x != y, A.LessThan: x < y, A.LessThanOrEqual: x <= y,
           A.GreaterThan: x > y, A.GreaterThanOrEqual: x >= y}
    return int(cmp[fn])


SIGNED_TYPES = (A.Int8, A.Int16, A.Int32)
INT_TYPES = [A.Int8, A.Uint8, A.Int16, A.Uint16, A.Int32, A.Uint32]
NP = {A.Int8: np.int8, A.Uint8: np.uint8, A.Int16: np.int16, A.Uint16: np.uint16, A.Int32: np.int32, A.Uint32: np.uint32}


def cell(dt, v):
    """32-bit cell of a stored value of column type `dt` (the loaders sign-extend Int8 / Int16)."""
    return u32(int(v))


# ---- edge tables -------------------------------------------------------------------------------------------------
DIVISORS = [1, 2, 3, 7, 60, 641, 3600, 65535, 65536, 86400, 2 ** 31 - 1]
U32_DIVISORS = [2 ** 31, 2 ** 31 + 1, 2 ** 32 - 1]           # negative as the int32 a literal is
GENERIC_DIVISORS = [0, -1, -3600]


def dividends(dt, d):
    """The dividends of one (column type, divisor) case that the column type can hold."""
    info = np.iinfo(NP[dt])
    ds = i32(d) if dt in SIGNED_TYPES else u32(d)
    cand = [0, 1, ds - 1, ds, ds + 1, info.min, info.max, info.min + 1, info.max - 1, 2 ** 31, 2 ** 32 - 1,
            INT_MIN, INT_MIN + 1, -1, -ds, -(ds + 1), 100, -100, 3599, 86399]
    out = []
    for v in cand:
        if info.min <= v <= info.max and v not in out:
            out.append(v)
    return out


def legal_for_c(x, d):
    """The reference / oracle compute in C: no division by zero, no INT_MIN / -1."""
    return i32(d) != 0 and not (i32(x) == INT_MIN and i32(d) == -1)


# ---- CPU: the restatement equals the oracle's BinaryTransform / BinaryFilter and the reference build ----------------
def _transform_outputs(be, dt, values, d, fn):
    """fn(column, literal d) into an Int32 scratch vector (the common class is I32: a literal is a ConstInt)."""
    n = len(values)
    spec = P.InputSpec("column", dt, np.asarray(values, NP[dt]), np.ones(n, bool), mode=2)
    out = P.run_transform(be, [spec, P.InputSpec("const", const=i32(d))], fn, ("scratch", A.Int32), n)
    return out["values"].view(np.uint32).tolist()


def _filter_outputs(be, dt, values, lit, fn):
    n = len(values)
    spec = P.InputSpec("column", dt, np.asarray(values, NP[dt]), np.ones(n, bool), mode=2)
    return P.run_filter(be, [spec, P.InputSpec("const", const=i32(lit))], fn, n)["index"].tolist()


PACKED_LITERALS = [-256, -129, -128, -1, 0, 1, 127, 128, 255, 256, 257, 2 ** 31 - 1, 2 ** 32 - 1]


def _cpu_cases(be):
    """Every (functor, column type, divisor) and (comparison, 1-byte type, literal) case the C ABI is defined on,
    with its outputs on backend `be`."""
    outs = []
    for fn in (A.Floor, A.Mod, A.Divide):
        for dt in INT_TYPES:
            for d in DIVISORS + U32_DIVISORS + GENERIC_DIVISORS:
                xs = [x for x in dividends(dt, d) if legal_for_c(x, d)]
                if xs:
                    outs.append(((fn, dt, d), xs, _transform_outputs(be, dt, xs, d, fn)))
    for dt in (A.Int8, A.Uint8):
        xs = list(range(-128, 128)) if dt == A.Int8 else list(range(256))
        for lit in PACKED_LITERALS:
            outs.append(((A.Equal, dt, lit), xs, _filter_outputs(be, dt, xs, lit, A.Equal)))
    return outs


def test_restatement_matches_oracle_and_reference():
    orc = H.get_backend("oracle")
    outs = _cpu_cases(orc)
    for (fn, dt, d), xs, got in outs:
        if fn == A.Equal:
            exp = [r for r, x in enumerate(xs) if eval_binary(fn, cell(dt, x), u32(d), True)]
        else:
            exp = [eval_binary(fn, cell(dt, x), u32(d), True) for x in xs]
        assert got == exp, f"fn={fn} type={dt} d={d}"
    mine = H.digest([o[2] for o in outs])
    H.assert_matches_reference("fused_edges/restatement", mine,
                               lambda: H.digest([o[2] for o in _cpu_cases(H.get_backend("ref"))]))


def test_restatement_defined_results():
    """The engine's own results where C is undefined (cell.cuh: evalBinary), and the unsigned class."""
    assert eval_binary(A.Divide, u32(INT_MIN), u32(-1), True) == u32(INT_MIN)
    assert eval_binary(A.Mod, u32(INT_MIN), u32(-1), True) == 0
    assert eval_binary(A.Floor, u32(INT_MIN), u32(-1), True) == u32(INT_MIN)
    assert eval_binary(A.Divide, 7, 0, True) == M32 and eval_binary(A.Divide, 7, 0, False) == M32
    assert eval_binary(A.Mod, u32(-7), 0, True) == u32(-7) and eval_binary(A.Mod, 7, 0, False) == 7
    assert eval_binary(A.Floor, 7, 0, True) == 0 and eval_binary(A.Floor, 7, 0, False) == 0
    assert eval_binary(A.Mod, u32(-7), 3, True) == u32(-1) and eval_binary(A.Floor, u32(-7), 3, True) == u32(-6)
    assert eval_binary(A.Mod, u32(-7), 3, False) == (2 ** 32 - 7) % 3
    assert eval_binary(A.Floor, 2 ** 32 - 1, 2 ** 32 - 1, False) == 2 ** 32 - 1


# ---- CPU: each GPU case reaches the path it targets ---------------------------------------------------------------
TAG = E.Col(0, A.Uint16, "tag")


def X(dt):
    return E.Col(1, dt, "x")


def _dry(q, dts, rows=100003, ranges=None, start_bit=0, modes=None):
    """AresJitDryRun of `q` over a batch of columns of types `dts` (fake device addresses)."""
    lib = A.load_engine()
    fn = lib.alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    p = A.BatchPlan()
    insts = q.plan_instructions()
    p.NumInsts = len(insts)
    for i, pi in enumerate(insts):
        p.Insts[i] = pi
    p.NumColumns = len(dts)
    for i, dt in enumerate(dts):
        mode = modes[i] if modes else 2
        p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, rows, 0, 64 * 200, mode, start_bit)
    p.NumRows = rows
    for col, (lo, hi) in (ranges or {}).items():
        p.Ranges[col].Known, p.Ranges[col].Min, p.Ranges[col].Max = 1, lo, hi
    src = C.c_char_p()
    h = fn(q.agg_spec(), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    assert int(h.res or 0) > 0, "plan was not eligible for specialisation"
    return (src.value or b"").decode()


def division_query(dt, d):
    """Dimension (Floor), stack operand of a filter (Mod) and 8-byte SUM measure (Mod) of one column by literal d."""
    x = X(dt)
    return AggQuery([E.ne(E.mod(x, E.Lit(i32(d))), E.Lit(12345))], [TAG, E.floor(x, E.Lit(i32(d)))],
                    Measure("sum", E.mod(x, E.Lit(i32(d)))))


def test_division_paths(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    for dt in INT_TYPES:
        src = _dry(division_query(dt, 3600), [A.Uint16, dt])
        assert src.count("fastDivU32(x[r], M)") == 3 and "#define JIT_DENSE 0" in src
        # divisor 1 (magic 2^64 / 1 + 1 would wrap to 0), 0, negative and u32-class literals take the functor
        for d in [1] + U32_DIVISORS + GENERIC_DIVISORS:
            src = _dry(division_query(dt, d), [A.Uint16, dt])
            assert "fastDivU32" not in src and src.count("evalBinary(") >= 3, (dt, d)
    # with a zone map: direct-indexed, the quotient dimension by the span form while span * d <= 2^32
    zm = {0: (0, 20), 1: (0, 2 ** 20 - 1)}
    src = _dry(division_query(A.Uint32, 2 ** 12), [A.Uint16, A.Uint32], ranges=zm)
    assert "#define JIT_DENSE 1" in src and "__umulhi(xr, P.dMagic32[" in src
    src = _dry(division_query(A.Uint32, 2 ** 16), [A.Uint16, A.Uint32], ranges={0: (0, 20), 1: (0, 2 ** 16 - 1)})
    assert "__umulhi(xr, P.dMagic32[" in src
    # span * d = 2^32 + d: the quotient dimension stays on fastDivU32
    src = _dry(division_query(A.Uint32, 2 ** 12), [A.Uint16, A.Uint32], ranges={0: (0, 20), 1: (0, 2 ** 20)})
    assert "#define JIT_DENSE 1" in src and "__umulhi(xr" not in src and "fastDivU32(x[r], M)" in src
    src = _dry(division_query(A.Uint32, 1), [A.Uint16, A.Uint32], ranges={0: (0, 20), 1: (0, 300)})
    assert "#define JIT_DENSE 1" in src and "__umulhi(xr" not in src and "fastDivU32" not in src
    # a negative Int32 dividend is divided by its raw bits: with d = 2^31 - 1 its quotient (1) would be inside the
    # zone map's quotients [0, 1], so that dimension is not indexed by quotient (here: no direct indexing at all)
    src = _dry(division_query(A.Int32, 2 ** 31 - 1), [A.Uint16, A.Int32], ranges={0: (0, 20), 1: (0, 2 ** 31 - 1)})
    assert "#define JIT_DENSE 0" in src
    src = _dry(division_query(A.Int32, 2 ** 31 - 1), [A.Uint16, A.Int32], ranges={0: (0, 20), 1: (0, 2 ** 31 - 2)})
    assert "#define JIT_DENSE 1" in src


def packed_query(dt, lit, lit_type):
    x = X(dt)
    return AggQuery([E.eq(x, E.Lit(i32(lit), lit_type))], [x], Measure("count"))


def mixed_filter_query(l1, l2):
    """Two packed filters, a hoisted non-packed filter and a non-hoisted one (an OR)."""
    s8, u8, w = E.Col(1, A.Int8, "s8"), E.Col(2, A.Uint8, "u8"), E.Col(3, A.Int16, "w")
    return AggQuery([E.eq(s8, E.Lit(i32(l1))), E.eq(u8, E.Lit(i32(l2))), E.ge(w, E.Lit(-100)),
                     E.or_(E.lt(w, E.Lit(0)), E.gt(u8, E.Lit(3)))], [s8, u8, TAG], Measure("count"))


def test_packed_equality_paths(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    for dt in (A.Int8, A.Uint8):
        for mode in (1, 2):
            for sb in (0, 5):
                src = _dry(packed_query(dt, 5, E.Type.Signed), [A.Uint16, dt], modes=[1, mode], start_bit=sb)
                assert "uint32_t pk0;" in src and "dead |= pk0;" in src, (dt, mode, sb)
                assert ("lit + 128u < 256u" in src) == (dt == A.Int8)
    src = _dry(mixed_filter_query(3, 4), [A.Uint16, A.Int8, A.Uint8, A.Int16])
    assert "dead |= pk0;" in src and "dead |= pk1;" in src and "pk2" not in src and "pk3" not in src
    # a 2-byte column is compared row by row
    src = _dry(packed_query(A.Int16, 5, E.Type.Signed), [A.Uint16, A.Int16])
    assert "pk0" not in src


GRP, FARE = E.Col(0, A.Uint8, "grp"), E.Col(1, A.Float32, "fare")
FLOAT_SUM = AggQuery([E.ge(FARE, E.Lit(-1e9))], [GRP], Measure("sum", FARE))


def f32_bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def bits_f32(b):
    return struct.unpack("<f", struct.pack("<I", b))[0]


def scale_of(max_bits):
    """S of the integer float-sum form for a zone-map maximum (jit.cu: jitAnalyzeDense)."""
    e = (max_bits >> 23) & 0xFF
    return max(-60, min(60, 60 if e == 0 else 31 - (e - 127)))


FLT_MAX_BITS = 0x7F7FFFFF
MAXIMA = [f32_bits(100.0), f32_bits(1.0), f32_bits(2.0 ** 31 - 128), f32_bits(2.0 ** 31), f32_bits(2.0 ** 32 - 256),
          f32_bits(2.0 ** 32), f32_bits(2.0 ** 40), FLT_MAX_BITS, 0x00400000, 0]


def test_float_sum_paths(monkeypatch):
    """The integer form is taken exactly when 2^S >= 1 (a maximum below 2^32): x * 2^S cannot underflow."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    assert [scale_of(m) for m in MAXIMA] == [25, 31, 1, 0, 0, -1, -9, -60, 60, 60]
    for m in MAXIMA:
        src = _dry(FLOAT_SUM, [A.Uint8, A.Float32], ranges={0: (0, 20), 1: (0, m)}, modes=[1, 2])
        assert "#define JIT_DENSE 1" in src
        assert ("#define JIT_DENSE_ACC 4" in src) == (scale_of(m) >= 0), hex(m)


# ---- GPU ----------------------------------------------------------------------------------------------------------
# Row counts: not multiples of 4, each ending in a partial tile; the first batch has more tiles than the H100 has SMs.
BATCH_ROWS = [132 * 8192 + 4099, 5003, 33331]


def _upload(be, cols, ranges=None):
    """cols: list of (data type, values, valid or None, start_bit)."""
    vps, keep = [], []
    n = len(cols[0][1])
    for dt, v, ok, sb in cols:
        buf, vp = columns.make_column(be.space, dt, v, valid=ok, start_bit=sb)
        vps.append(vp)
        keep.append(buf)
    return Batch(vps, n, keep=keep, ranges=ranges)


def _as_dict(res):
    dims = res.decoded_dims()
    return {tuple(d[g] for d in dims): res.measures[g].item() for g in range(res.groups)}


def _run(be, q, batches, fused=True):
    if fused:
        ex = FusedBatchExecutor(be.lib, be.space, q)
        for b in batches:
            ex.process_batch(b)
        r = ex.result()
        ex.close()
        return r
    ex = LegacyBatchExecutor(be.lib, be.space, q)
    for b in batches:
        ex.process_batch(b)
    return ex.result()


def _spread(rng, k, rows):
    """Row r holds edge value idx[r]: every value occurs, in every quad position, spread over the whole batch."""
    idx = np.arange(rows) % k
    return idx[rng.permutation(rows)] if rows > 4 * k else idx


def _decode_dim(dt, bits):
    v = bits & ((1 << (8 * max(A.DATA_TYPE_BYTES[dt], 1))) - 1)
    w = 8 * A.DATA_TYPE_BYTES[dt]
    return v - (1 << w) if dt in SIGNED_TYPES and v >= 1 << (w - 1) else v


def division_expected(dt, d, tables):
    """{(tag, floor(x, d)) : sum(x % d)} over the valid rows whose x % d != 12345 (tag = edge value index)."""
    q = division_query(dt, d)
    floor_dt = q.dim_types[1]
    signed_sum = q.agg_func == A.AGGR_SUM_SIGNED
    exp = {}
    for xs, valid in tables:
        for t, x in enumerate(xs):
            cnt = int(valid[t])
            if not cnt:
                continue
            c = cell(dt, x)
            m = eval_binary(A.Mod, c, u32(d), True)
            if not eval_binary(A.NotEqual, m, 12345, True):
                continue
            key = (t, _decode_dim(floor_dt, eval_binary(A.Floor, c, u32(d), True)))
            s = i32(m) * cnt   # SUM in Int64 of the I32 result, sign-extended (cell.cuh: cvt)
            exp[key] = exp.get(key, 0) + s
    if not signed_sum:
        exp = {k: v & (2 ** 64 - 1) for k, v in exp.items()}
    return exp


@pytest.mark.gpu
@pytest.mark.parametrize("dt", INT_TYPES)
def test_division_edges_on_gpu(dt):
    """Floor / Mod by literals through one plan shape per column type and divisor class; with and without a zone
    map (direct-indexed quotient dimension, rows outside it on the cold path)."""
    eng = H.get_backend("b200")
    rng = np.random.default_rng(11 + dt)
    for d in DIVISORS + U32_DIVISORS + GENERIC_DIVISORS:
        xs = dividends(dt, d)
        k = len(xs)
        batches, tables = [], []
        for rows in BATCH_ROWS:
            idx = _spread(rng, k, rows)
            vals = np.asarray(xs, NP[dt])[idx]
            valid = rng.random(rows) >= 0.1
            # garbage under NULL: a negative value in a signed column (the quad-level sign branch sees it)
            if dt in SIGNED_TYPES:
                vals[~valid] = np.iinfo(NP[dt]).min
            batches.append([(A.Uint16, idx.astype(np.uint16), None, 0), (dt, vals, valid, 0)])
            tables.append((xs, np.bincount(idx[valid], minlength=k)))
        exp = division_expected(dt, d, tables)
        q = division_query(dt, d)
        uploads = [_upload(eng, b) for b in batches]
        got = _run(eng, q, uploads)
        assert _as_dict(got) == exp, f"fused d={d}"
        assert _as_dict(_run(eng, q, uploads, fused=False)) == exp, f"per-node d={d}"
        # zone maps over the non-negative dividends (negative ones and, in the second, the lower half take the cold path)
        nonneg = [x for x in xs if 0 <= x < 2 ** 31]
        for zm in ({0: (0, k - 1), 1: (min(nonneg), max(nonneg))}, {0: (0, k - 1), 1: (max(nonneg) // 2 + 1, max(nonneg))}):
            got = _run(eng, q, [_upload(eng, b, zm) for b in batches])
            assert _as_dict(got) == exp, f"fused d={d} zone map {zm}"


SPAN_CASES = [  # (d, zone-map min, max): span * d exactly 2^32, just below it, a minimum that is not a multiple of d
    (2 ** 12, 0, 2 ** 20 - 1), (2 ** 16, 0, 2 ** 16 - 1), (3600, 7200, 7200 + 2 ** 32 // 3600 - 1), (3600, 1000, 90000),
    (3600, 1_726_963_201, 1_726_963_200 + 86399)]


@pytest.mark.gpu
def test_span_division_on_gpu():
    """The span form of a direct-indexed quotient dimension; exact, too narrow and stale zone maps."""
    eng = H.get_backend("b200")
    before = J.T.dense_launches(eng)
    launches = 0
    rng = np.random.default_rng(3)
    for d, lo, hi in SPAN_CASES:
        base = lo - lo % d
        xs = sorted({v for v in (lo, base, hi, lo - 1, hi + 1, 0, 2 ** 31 - 1, (lo + hi) // 2, hi - d, lo + d) if 0 <= v < 2 ** 32})
        k = len(xs)
        q = AggQuery([E.ne(E.mod(X(A.Uint32), E.Lit(d)), E.Lit(12345))], [TAG, E.floor(X(A.Uint32), E.Lit(d))],
                     Measure("sum", E.mod(X(A.Uint32), E.Lit(d))))
        assert "__umulhi(xr, P.dMagic32[" in _dry(q, [A.Uint16, A.Uint32], ranges={0: (0, k - 1), 1: (lo, hi)})
        batches, tables = [], []
        for rows in BATCH_ROWS[1:]:
            idx = _spread(rng, k, rows)
            valid = rng.random(rows) >= 0.05
            batches.append([(A.Uint16, idx.astype(np.uint16), None, 0), (A.Uint32, np.asarray(xs, np.uint32)[idx], valid, 0)])
            tables.append((xs, np.bincount(idx[valid], minlength=k)))
        exp = division_expected(A.Uint32, d, tables)
        for zm in ({0: (0, k - 1), 1: (lo, hi)}, {0: (0, k - 1), 1: (lo, lo + (hi - lo) // 2)},
                   {0: (0, k - 1), 1: (hi + 1, hi + 1 + (hi - lo))}):
            if zm[1][1] >= 2 ** 31:
                continue
            got = _run(eng, q, [_upload(eng, b, zm) for b in batches])
            assert _as_dict(got) == exp, f"d={d} zone map {zm}"
            launches += len(batches)
    assert J.T.dense_launches(eng) - before == launches


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [A.Int8, A.Uint8])
def test_packed_equality_on_gpu(dt):
    """Every byte value at each of the four positions of a quad, NULL rows whose stored byte is the literal's low
    byte, mode 1 and mode 2 columns, null bitmaps starting at bit 0 and 5."""
    eng = H.get_backend("b200")
    rng = np.random.default_rng(5)
    quad = np.arange(1024)
    pattern = ((quad // 4) + 64 * (quad % 4)) % 256      # value v at position p of quad (v - 64 p) mod 256
    for mode in (1, 2):
        for sb in (0, 5):
            batches, tables = [], []
            for rows in BATCH_ROWS[1:]:
                raw = pattern[np.arange(rows) % 1024].astype(np.uint8)
                valid = None if mode == 1 else rng.random(rows) >= 0.3
                batches.append([(A.Uint16, np.zeros(rows, np.uint16), None, 0), (dt, raw.view(NP[dt]), valid, sb)])
                tables.append((raw, valid))
            uploads = [_upload(eng, b) for b in batches]
            for lit in PACKED_LITERALS:
                for lt in (E.Type.Signed, E.Type.Unsigned):
                    q = packed_query(dt, lit, lt)
                    exp = {}
                    for raw, valid in tables:
                        vals = raw.view(NP[dt]).astype(np.int64)
                        ok = np.ones(len(raw), bool) if valid is None else valid
                        for v, c in zip(*np.unique(vals[ok], return_counts=True)):
                            if eval_binary(A.Equal, u32(int(v)), u32(lit), True):
                                exp[(int(v),)] = exp.get((int(v),), 0) + int(c)
                    assert _as_dict(_run(eng, q, uploads)) == exp, f"mode {mode} bit {sb} lit {lit}"
                assert _as_dict(_run(eng, q, uploads, fused=False)) == exp, f"per-node lit {lit}"


@pytest.mark.gpu
def test_mixed_filters_on_gpu():
    eng = H.get_backend("b200")
    rng = np.random.default_rng(9)
    batches, rowsets = [], []
    for rows in BATCH_ROWS:
        s8 = rng.integers(-128, 128, rows).astype(np.int8)
        u8 = rng.integers(0, 8, rows).astype(np.uint8)
        w = rng.integers(-300, 300, rows).astype(np.int16)
        tag = rng.integers(0, 3, rows).astype(np.uint16)
        vs, vu, vw = (rng.random(rows) >= 0.2 for _ in range(3))
        s8[~vs & (rng.random(rows) < 0.5)] = 3      # NULL rows holding the literal's byte
        batches.append([(A.Uint16, tag, None, 0), (A.Int8, s8, vs, 5), (A.Uint8, u8, vu, 0), (A.Int16, w, vw, 3)])
        rowsets.append((tag, s8, u8, w, vs, vu, vw))
    uploads = [_upload(eng, b) for b in batches]
    for l1, l2 in ((3, 4), (-128, 0), (127, 7), (-1, 255)):
        exp = {}
        for tag, s8, u8, w, vs, vu, vw in rowsets:
            alive = vs & vu & vw & (s8.astype(np.int64) == l1) & (u8.astype(np.int64) == l2) & (w >= -100) & ((w < 0) | (u8 > 3))
            for key in zip(s8[alive].tolist(), u8[alive].tolist(), tag[alive].tolist()):
                exp[key] = exp.get(key, 0) + 1
        q = mixed_filter_query(l1, l2)
        assert _as_dict(_run(eng, q, uploads)) == exp, (l1, l2)
        assert _as_dict(_run(eng, q, uploads, fused=False)) == exp, (l1, l2)


def float_groups(max_bits):
    """Per zone-map maximum: one value per group (the maximum, its next float up, 2^-S, the smallest normal and
    denormal values, off-grid values, +-0.0, a negative value, and values that x * 2^S would underflow under S < 0)."""
    m = bits_f32(max_bits)
    S = scale_of(max_bits)
    vals = [m, bits_f32(max_bits + 1), 2.0 ** -S, bits_f32(0x00800000), bits_f32(1), 1.5 * 2.0 ** -S, 0.0, -0.0, -1.5,
            1e-30, 3e-38, 0.75]
    return [float(np.float32(v)) for v in vals]


def exact_sum(values_counts):
    """Exact sum on the 2^-149 grid, rounded once to double; all -0.0 addends sum to -0.0."""
    total = Fraction(0)
    for v, c in values_counts:
        if np.isinf(v):
            return v
        total += Fraction(v) * c
    if total == 0:
        return -0.0 if all(struct.pack("<d", v)[7] & 0x80 or c == 0 for v, c in values_counts) else 0.0
    return float(total)


@pytest.mark.gpu
def test_float_sum_edges_on_gpu():
    """SUM(fare) with `fare >= -1e9` (the measure is non-NULL on surviving rows) for every zone-map maximum; each
    group holds one value repeated, so every partial sum is exact and the result is bit-exact."""
    eng = H.get_backend("b200")
    rng = np.random.default_rng(17)
    for mb in MAXIMA:
        vals = float_groups(mb)
        k = len(vals)
        batches, counts = [], np.zeros(k, np.int64)
        for rows in BATCH_ROWS:
            idx = _spread(rng, k, rows)
            fare = np.asarray(vals, np.float32)[idx]
            valid = rng.random(rows) >= 0.01
            batches.append([(A.Uint8, idx.astype(np.uint8), None, 0), (A.Float32, fare, valid, 0)])
            counts += np.bincount(idx[valid], minlength=k)
        exp = {(g,): exact_sum([(vals[g], int(counts[g]))]) for g in range(k) if counts[g]}
        zm = {0: (0, k - 1), 1: (0, mb)}
        before = J.T.dense_launches(eng)
        got = _as_dict(_run(eng, FLOAT_SUM, [_upload(eng, b, zm) for b in batches]))
        assert J.T.dense_launches(eng) - before == len(batches)
        pack = lambda dct: {kk: struct.pack("<d", v) for kk, v in dct.items()}
        assert pack(got) == pack(exp), f"max {hex(mb)}: " + str({kk: (got.get(kk), exp[kk]) for kk in exp if got.get(kk) != exp[kk]})
        legacy = _as_dict(_run(eng, FLOAT_SUM, [_upload(eng, b) for b in batches], fused=False))
        assert pack(legacy) == pack(exp), f"per-node max {hex(mb)}"
