"""The functor code every other expression goes through (csrc/cell.cuh: cvt, commonClass, evalUnary, evalBinary, which
the NVRTC generator instantiates once per plan instruction), at value edges, against the plain restatement of the
reference's functors in functor_restatement.py.

Edge tables: every column type (Bool, Int8 ... Uint32, Float32) at 0, +-1, its min and max, 127 / 128 / 255 / 256,
32767 / 32768 / 65535 / 65536, 2^31 - 1, 2^31, 2^32 - 1, -2^31; floats at +-0.0, the smallest denormal, FLT_MIN, FLT_MAX,
+-inf, NaN (two patterns), 0.1, 16777216, 16777217 (stored as 16777216), 2^31; NULL rows holding a stored value;
literals negative, >= 2^31 as int32, 0.1, -0.0 and 16777217.0.

CPU: the restatement equals the C restatement of the per-node ABI (oracle: UnaryTransform, BinaryTransform,
BinaryFilter) on every case C++ defines, and on those rows the oracle's outputs equal the digests recorded from the
reference's HOST build (tests/golden/functor_edges_reference.json, tests/golden/make_functor_edges_fixture.py); the
generator's dry run shows that each GPU case reaches the form it targets; the kernels of the Float32 chains contain no
FFMA.

GPU: each functor as a dimension root (every pairing of value classes commonClass tells apart, column and literal
operands), as a filter root (hoisted `column CMP literal` and not), as a member filter of a shared scan, as a stack
intermediate, as a measure root into sum / min / max (hash, global-slot and CTA-slot forms, and the cold path of rows
outside a narrow zone map); chains a*b + c, a*b - c, c - a*b, a*b + c*d, a/b + c over mode-0, mode-1 and mode-2 columns.  A Uint32 row-number column is the first dimension, so that every group is one row and the
other dimensions read out one expression result each; count(*) reads out which rows a filter keeps.  Every case is also
run through the per-node sequence on the engine and must be byte-identical (two Float64 NaNs count as equal).
"""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

import functor_restatement as R
import harness as H
import parity_cases as P
import test_jit_codegen as J
from aresdb_b200 import cabi as A
from aresdb_b200 import columns, expr as E
from aresdb_b200.executor import Batch, FusedBatchExecutor, FusedRequestExecutor, LegacyBatchExecutor
from aresdb_b200.query import AggQuery, Measure

M32 = R.M32
FIXTURE = Path(__file__).resolve().parent / "golden" / "functor_edges_reference.json"

# ---- edge tables -------------------------------------------------------------------------------------------------
INT_EDGES = [0, 1, -1, 127, 128, 255, 256, 32767, 32768, 65535, 65536, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, -2 ** 31,
             -128, -129, -32768, 3, -7]
NP = {A.Bool: np.uint8, A.Int8: np.int8, A.Uint8: np.uint8, A.Int16: np.int16, A.Uint16: np.uint16, A.Int32: np.int32,
      A.Uint32: np.uint32, A.Float32: np.float32}
FLOAT_BITS = [R.f32_bits(v) for v in (0.0, -0.0, 1.0, -1.0, 0.1, 3.0, -1.5, 16777216.0, 16777217.0, 2.0 ** 31, -2.0 ** 31,
                                      2.0 ** 32, 1e10)] + \
             [0x00000001, 0x00800000, 0x7F7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00123]
NAMES = {A.Bool: "bool", A.Int8: "i8", A.Uint8: "u8", A.Int16: "i16", A.Uint16: "u16", A.Int32: "i32", A.Uint32: "u32",
         A.Float32: "f32"}


def edges(dt):
    """Stored edge values of a column type (Float32: bit patterns)."""
    if dt == A.Bool:
        return [0, 1]
    if dt == A.Float32:
        return list(FLOAT_BITS)
    info = np.iinfo(NP[dt])
    return [v for v in INT_EDGES if info.min <= v <= info.max]


def stored_array(dt, vals):
    if dt == A.Float32:
        return np.asarray(vals, np.uint32).view(np.float32)
    return np.asarray(vals, np.int64).astype(NP[dt])


INT_LITERALS = [0, 1, -1, -7, 255, 65536, 2 ** 31 - 1, -2 ** 31, 2 ** 31, 2 ** 32 - 1]   # >= 2^31: the int32 it is
FLOAT_LITERALS = [0.1, -0.0, 16777217.0, 3.0, -1.5]


def lit_cell(v):
    """(bits, class) of a literal operand: ConstInt is int32, ConstFloat float (binder.hpp)."""
    return (R.f32_bits(v), R.F32) if isinstance(v, float) else (v & M32, R.I32)


# Pairings of operand classes that commonClass tells apart (bool counts as unsigned; a narrow column is its 32-bit class)
PAIRINGS = [(A.Float32, A.Float32), (A.Float32, A.Int16), (A.Uint8, A.Float32), (A.Int32, A.Uint32),
            (A.Uint32, A.Uint16), (A.Int8, A.Int32), (A.Bool, A.Bool), (A.Bool, A.Int8), (A.Uint32, A.Bool)]


def pair_table(da, db):
    """Rows of (a, a valid, b, b valid): every pair of edge values, valid; each value of one NULL against each of the
    other (the stored value under a NULL is an edge value too)."""
    rows = []
    for x in edges(da):
        for y in edges(db):
            rows.append((x, True, y, True))
    for k, x in enumerate(edges(da)):
        y = edges(db)[k % len(edges(db))]
        rows += [(x, False, y, True), (x, True, y, False), (x, False, y, False)]
    return rows


# ---- CPU: the restatement against the oracle -------------------------------------------------------------------
def _scratch_type(rc):
    return {R.BOOL: A.Int32, R.I32: A.Int32, R.U32: A.Uint32, R.F32: A.Float32}[rc]


def _spec(dt, vals, valid, mode=2, start_bit=0):
    return P.InputSpec("column", dt, stored_array(dt, vals), np.asarray(valid, bool), mode=mode, start_bit=start_bit)


def _column_cell(dt, v, ok):
    return (R.load(dt, v), ok)


def _expected_transform(fn, cells, classes, sink_cls):
    """Per row: (output bits, valid, defined) for a transform into a sink of class sink_cls."""
    out = []
    for row in cells:
        if len(row) == 1:
            (c, rc) = R.eval_unary(fn, row[0], classes[0], device=False)
        else:
            (c, rc) = R.binary(fn, row[0], classes[0], row[1], classes[1], device=False)
        # (which NaN an x86 operation returns depends on its operand order, which C compilers and numpy choose freely)
        nan = rc == R.F32 and fn in R.ARITH + (A.Negate,) and np.isnan(R.bits_f32(c[0]))
        out.append((R.cvt(c[0], rc, sink_cls), c[1], R.host_defined(c[0], rc, sink_cls) and not nan))
    return out


def cpu_cases():
    """(key, fn, input specs, sink, rows' cells, operand classes): every binary functor on every pairing (column and
    literal right operands) and every unary functor on every column type, into the scratch vector of its result and, for
    Noop / Negate / Plus, into dimensions of every type."""
    cases = []
    for da, db in PAIRINGS:
        rows = pair_table(da, db)
        a = _spec(da, [r[0] for r in rows], [r[1] for r in rows], start_bit=3)
        b = _spec(db, [r[2] for r in rows], [r[3] for r in rows])
        cells = [(_column_cell(da, r[0], r[1]), _column_cell(db, r[2], r[3])) for r in rows]
        classes = (R.operand_class(da), R.operand_class(db))
        for fn in P.BINARY_FNS:
            cases.append((f"bin/{NAMES[da]}/{NAMES[db]}/{fn}", fn, [a, b], cells, classes))
        # a literal right operand: one batch per literal
        for lit in INT_LITERALS[::3] + FLOAT_LITERALS[::2]:
            la = _spec(da, edges(da), [True] * len(edges(da)))
            lc, lcls = lit_cell(lit)
            lcells = [(_column_cell(da, v, True), (lc, True)) for v in edges(da)]
            for fn in (A.LessThan, A.Equal, A.Minus, A.Multiply, A.Divide, A.Mod, A.Or):
                cases.append((f"lit/{NAMES[da]}/{lit!r}/{fn}", fn, [la, P.InputSpec("const", const=lit)], lcells,
                              (R.operand_class(da), lcls)))
    for dt in P.COLUMN_TYPES:
        vals = edges(dt) * 2
        valid = [True] * len(edges(dt)) + [False] * len(edges(dt))
        spec = _spec(dt, vals, valid, start_bit=5)
        cells = [(_column_cell(dt, v, ok),) for v, ok in zip(vals, valid)]
        for fn in (A.Not, A.IsNull, A.IsNotNull, A.Negate, A.BitwiseNot, A.Noop):
            cases.append((f"un/{NAMES[dt]}/{fn}", fn, [spec], cells, (R.operand_class(dt),)))
        # mode 0: the default value, valid and not
        for dv in (True, False):
            d = edges(dt)[-1]
            m0 = P.InputSpec("column", dt, mode=0, default=(float(R.bits_f32(d)) if dt == A.Float32 else d), default_valid=dv)
            for fn in (A.Not, A.IsNull, A.Negate):
                cases.append((f"m0/{NAMES[dt]}/{dv}/{fn}", fn, [m0], [((R.load(dt, d) if dv else 0, dv),)] * 4,
                              (R.operand_class(dt),)))
    return cases


SINK_DIMS = [A.Bool, A.Int8, A.Uint8, A.Int16, A.Uint16, A.Int32, A.Uint32, A.Float32]


def run_case(be, case):
    """Outputs of one case on backend `be`: [(sink, values bytes, valid bytes or None)]."""
    key, fn, specs, cells, classes = case
    n = len(cells)
    if len(classes) == 1:
        _, rc = R.eval_unary(fn, (0, True), classes[0])
    else:
        _, rc = R.eval_binary(fn, (0, True), (0, True), R.common_class(*classes))
    sinks = [("scratch", _scratch_type(rc))]
    if fn in (A.Noop, A.Negate, A.Plus) or key.startswith("m0/"):
        sinks += [("dim", dt) for dt in SINK_DIMS]
    out = []
    for s in sinks:
        o = P.run_transform(be, specs, fn, s, n)
        out.append((s, o["values"], o.get("valid")))
    if len(specs) == 2:
        out.append((("filter",), P.run_filter(be, specs, fn, n)["index"], None))
    return rc, out


def defined_mask(case, rc, sink):
    key, fn, specs, cells, classes = case
    exp = _expected_transform(fn, cells, classes, R.sink_class(sink[1], sink[0] == "dim"))
    return exp, np.array([d for _, _, d in exp], bool)


def c_defined(case):
    """Rows whose result C++ defines in the reference's code: an integer Divide / Mod / Floor of valid operands by 0, or
    of INT_MIN by -1, is undefined (the x86 HOST build traps)."""
    key, fn, specs, cells, classes = case
    if len(classes) == 1 or fn not in (A.Divide, A.Mod, A.Floor):
        return np.ones(len(cells), bool)
    tc = R.common_class(*classes)
    if tc == R.F32:
        return np.ones(len(cells), bool)
    ok = []
    for (x, xo), (y, yo) in cells:
        xv, yv = R.value_of(R.cvt(x, classes[0], tc), tc), R.value_of(R.cvt(y, classes[1], tc), tc)
        ok.append(not (xo and yo and (yv == 0 or (tc == R.I32 and xv == R.INT_MIN and yv == -1))))
    return np.asarray(ok, bool)


def reference_case(case):
    """The case restricted to the rows C++ defines (what the reference's HOST build can run)."""
    key, fn, specs, cells, classes = case
    m = c_defined(case)
    if m.all():
        return case
    sub = []
    for s in specs:
        if s.kind == "column" and s.mode != 0:
            s = P.InputSpec("column", s.data_type, s.values[m], s.valid[m], mode=s.mode, start_bit=s.start_bit)
        sub.append(s)
    return key, fn, sub, [c for c, k in zip(cells, m) if k], classes


def case_outputs(be, case):
    """The outputs of a case on `be`, with the rows whose conversion into the sink C++ leaves undefined zeroed."""
    rc, out = run_case(be, case)
    res = []
    for s, vals, valid in out:
        if s[0] == "filter":
            res.append(vals)
            continue
        _, mask = defined_mask(case, rc, s)
        w = 4 if s[0] == "scratch" else max(A.DATA_TYPE_BYTES[s[1]], 1)
        v = vals.reshape(-1, w).copy()
        v[~mask] = 0
        res.append((v, valid))
    return res


def reference_digests(be):
    return {c[0]: H.digest(case_outputs(be, c)) for c in map(reference_case, cpu_cases())}


def test_oracle_matches_reference_digests():
    """Every case of cpu_cases(), on the rows C++ defines, gives the oracle the outputs the reference's HOST build gave
    (digests in tests/golden/functor_edges_reference.json); with oracle/_ref built, the build itself is run too."""
    stored = json.loads(FIXTURE.read_text())
    mine = reference_digests(H.get_backend("oracle"))
    assert sorted(stored) == sorted(mine)
    assert [k for k in mine if mine[k] != stored[k]] == []
    if H.reference_built():
        live = reference_digests(H.get_backend("ref"))
        assert [k for k in live if live[k] != stored[k]] == []


def test_restatement_rules():
    """The reference's NULL rules, the defined division results, the bool byte, the float fall-through and the two
    departures between the DEVICE and x86."""
    T, F, N = (1, True), (0, True), (0, False)
    b = R.BOOL
    assert R.eval_binary(A.And, N, F, R.U32)[0] == N and R.eval_binary(A.And, F, N, R.U32)[0] == N
    assert R.eval_binary(A.And, T, T, R.U32)[0] == T
    assert R.eval_binary(A.Or, N, T, R.U32)[0] == T and R.eval_binary(A.Or, T, N, R.U32)[0] == T
    assert R.eval_binary(A.Or, N, F, R.U32)[0] == N and R.eval_binary(A.Or, F, F, R.U32)[0] == F
    # TRUE dominates even when the true operand's cell sits beside a NULL one holding "true" garbage
    assert R.eval_binary(A.Or, (5, False), F, R.U32)[0] == N
    assert R.eval_unary(A.Not, N, b)[0] == N and R.eval_unary(A.IsNull, N, b)[0] == T
    # a bool is its byte: 0x100 is false, 0x101 true
    assert R.cvt(0x100, b, R.U32) == 0 and R.cvt(0x101, b, R.U32) == 1 and R.eval_unary(A.Not, (0x100, True), b)[0] == T
    assert R.eval_unary(A.Negate, (1, True), b) == ((1, True), b)
    assert R.eval_unary(A.BitwiseNot, (0, True), b) == ((1, True), b)
    # int32 literal against a uint32 value >= 2^31: the common class is int32
    assert R.common_class(R.U32, R.I32) == R.I32 and R.common_class(R.BOOL, R.BOOL) == R.U32
    assert R.binary(A.LessThan, (2 ** 31, True), R.U32, (0, True), R.I32)[0] == T
    assert R.binary(A.LessThan, (2 ** 31, True), R.U32, (0, True), R.U32)[0] == F
    # unsigned Minus wraps; Negate of INT_MIN is INT_MIN; x / 0 and INT_MIN / -1
    assert R.binary(A.Minus, (1, True), R.U32, (2, True), R.U32)[0] == (M32, True)
    assert R.eval_unary(A.Negate, (2 ** 31, True), R.I32)[0] == (2 ** 31, True)
    assert R.eval_binary(A.Divide, (7, True), (0, True), R.U32)[0] == (M32, True)
    assert R.eval_binary(A.Divide, (2 ** 31, True), (M32, True), R.I32)[0] == (2 ** 31, True)
    # Mod / bitwise / Floor on floats return the first operand, validity included
    for fn in R.INT_ONLY:
        assert R.eval_binary(fn, (R.f32_bits(2.5), False), (R.f32_bits(2.0), True), R.F32) == ((R.f32_bits(2.5), False), R.F32)
    # Float32: one rounding per functor.  fare = 0.1f: fare * 3 rounds to 0.3f exactly, so fare * 3 - 0.3f is 0; one
    # fused multiply-add would give -7.45e-9
    p, _ = R.binary(A.Multiply, (R.f32_bits(0.1), True), R.F32, (R.f32_bits(3.0), True), R.F32)
    d, _ = R.binary(A.Minus, p, R.F32, (R.f32_bits(0.3), True), R.F32)
    assert d == (0, True)
    assert np.float32(np.float64(np.float32(0.1)) * 3.0 - np.float64(np.float32(0.3))) != 0
    # departures: NaN results, out-of-range and NaN conversions
    nan = R.binary(A.Minus, (0x7F800000, True), R.F32, (0x7F800000, True), R.F32, device=True)[0]
    assert nan == (R.CANONICAL_NAN, True)
    assert R.binary(A.Minus, (0x7F800000, True), R.F32, (0x7F800000, True), R.F32, device=False)[0] == (0xFFC00000, True)
    assert R.eval_unary(A.Negate, (0x7FC00000, True), R.F32, device=False)[0] == (0xFFC00000, True)
    # float -> integer conversions C++ leaves undefined are not modelled; defined ones truncate
    assert R.cvt(R.f32_bits(1e10), R.F32, R.I32) is None and R.cvt(0x7FC00000, R.F32, R.U32) is None
    assert R.cvt(R.f32_bits(-1.5), R.F32, R.U32) is None and R.cvt(R.f32_bits(-0.5), R.F32, R.U32) == 0
    assert R.cvt(R.f32_bits(300.0), R.F32, R.U8) == 300 & 0xFF and R.cvt(R.f32_bits(-2.5), R.F32, R.I16) == 0xFFFE
    assert R.cvt(R.f32_bits(1e10), R.F32, R.I16) is None and R.cvt(R.f32_bits(2.0 ** 31), R.F32, R.U32) == 2 ** 31


def test_restatement_matches_oracle():
    orc = H.get_backend("oracle")
    cases = cpu_cases()
    bad = []
    for case in cases:
        key, fn, specs, cells, classes = case
        rc, out = run_case(orc, case)
        for s, vals, valid in out:
            if s[0] == "filter":
                want = [i for i, row in enumerate(cells)
                        if R.keep(*R.binary(fn, row[0], classes[0], row[1], classes[1], device=False))]
                if vals.tolist() != want:
                    bad.append((key, s))
                continue
            exp, mask = defined_mask(case, rc, s)
            w = 4 if s[0] == "scratch" else max(A.DATA_TYPE_BYTES[s[1]], 1)
            got = vals.reshape(-1, w)
            for i, (bits, ok, d) in enumerate(exp):
                if not d:
                    continue
                gb = int.from_bytes(got[i].tobytes(), "little")
                if gb != bits & ((1 << (8 * w)) - 1) or (valid is not None and bool(valid[i]) != ok):
                    bad.append((key, s, i, cells[i], hex(gb), hex(bits), ok))
                    break
    assert not bad, bad[:10]


# ---- GPU cases -----------------------------------------------------------------------------------------------------
ROWNO = E.Col(0, A.Uint32, "row")


def a_col(dt):
    return E.Col(1, dt, "a")


def b_col(dt):
    return E.Col(2, dt, "b")


BIN_OPS = [A.And, A.Or, A.Equal, A.NotEqual, A.LessThan, A.LessThanOrEqual, A.GreaterThan, A.GreaterThanOrEqual,
           A.Plus, A.Minus, A.Multiply, A.Divide, A.Mod, A.BitwiseAnd, A.BitwiseOr, A.BitwiseXor, A.Floor]
DIMS_PER_KERNEL = 5     # the row number (5 bytes with its validity byte) and five 4-byte results fill 32 bytes


def chunks(xs, k):
    return [xs[i:i + k] for i in range(0, len(xs), k)]


def binary_dim_queries(da, db):
    """Every binary functor on (a, b), and on (a, literal), as dimension roots; a Bool result keeps 1 byte."""
    exprs = [E.Binary(fn, a_col(da), b_col(db)) for fn in BIN_OPS]
    exprs += [E.Binary(fn, a_col(da), E.Lit(lit)) for fn, lit in
              [(A.LessThan, -1), (A.Equal, 2 ** 31), (A.Minus, 2 ** 32 - 1), (A.Plus, 0.1), (A.Multiply, 16777217.0),
               (A.GreaterThan, -0.0), (A.Mod, -7), (A.Floor, 0), (A.Divide, -1), (A.Or, 0)]]
    return [AggQuery([], [ROWNO] + list(c), Measure("count")) for c in chunks(exprs, DIMS_PER_KERNEL)]


def unary_dim_queries(dt):
    col = a_col(dt)
    exprs = [E.Unary(fn, col) for fn in (A.Not, A.IsNull, A.IsNotNull, A.Negate, A.BitwiseNot)] + [col]
    # a stack intermediate feeding another functor
    exprs += [E.Unary(A.Not, E.Unary(A.Negate, col)), E.Binary(A.Plus, E.Unary(A.Negate, col), E.Lit(1))]
    return [AggQuery([], [ROWNO] + list(c), Measure("count")) for c in chunks(exprs, DIMS_PER_KERNEL)]


# ---- evaluation of a resolved expression tree by the restatement ---------------------------------------------------
def eval_expr(e, row, dts):
    """(cell, class) of resolved expression `e` on one row: row[i] = (stored value, valid) of column i."""
    if isinstance(e, E.Col):
        v, ok = row[e.index]
        return (R.load(dts[e.index], v), ok), R.operand_class(dts[e.index])
    if isinstance(e, E.Lit):
        return ((R.f32_bits(e.value), True), R.F32) if e.type == E.Type.Float else ((int(e.value) & M32, True), R.I32)

    def operand(x):
        c, cls = eval_expr(x, row, dts)
        if isinstance(x, (E.Col, E.Lit)):
            return c, cls
        oc = R.sink_class(E.scratch_data_type(x.type), False)      # a stack temporary: the scratch type of its type
        v = R.cvt(c[0], cls, oc)
        assert v is not None, f"{x}: an undefined conversion feeds another functor"
        return (v, c[1]), oc
    if isinstance(e, E.Unary):
        a, ac = operand(e.expr)
        return R.eval_unary(e.op, a, ac)
    a, ac = operand(e.lhs)
    b, bc = operand(e.rhs)
    return R.binary(e.op, a, ac, b, bc)


def expected_dims(q, rows, dts):
    """{row number: tuple of (bits, valid) per dimension} for a query whose first dimension is the row number."""
    out = {}
    for r, row in enumerate(rows):
        vals = []
        for e, dt in zip(q.dimensions, q.dim_types):
            c, cls = eval_expr(e, row, dts)
            w = max(A.DATA_TYPE_BYTES[dt], 1)
            sc = R.sink_class(dt, True)
            # (a NaN or out-of-range float -> integer conversion: only its validity is pinned here; the fused and the
            # per-node results must still be the same bytes)
            bits = R.cvt(c[0], cls, sc) & ((1 << (8 * w)) - 1) if R.host_defined(c[0], cls, sc) else None
            vals.append((bits, c[1]))
        out[r] = tuple(vals)
    return out


def got_dims(res):
    """{row number: tuple of (bits, valid) per dimension} of a fused / per-node result."""
    out = {}
    for g in range(res.groups):
        vals = tuple((int.from_bytes(res.dim_values[qi][g].tobytes(), "little"), bool(res.dim_valid[qi][g]))
                     for qi in range(len(res.query.dimensions)))
        out[vals[0][0]] = vals
    return out


def diff(got, exp, q, limit=6):
    def same(g, w):
        return g is not None and w is not None and len(g) == len(w) and \
            all(gv == wv and (gb == wb or wb is None) for (gb, gv), (wb, wv) in zip(g, w))
    keys = sorted(set(got) | set(exp))
    bad = [(k, got.get(k), exp.get(k)) for k in keys if not same(got.get(k), exp.get(k))]
    return [f"row {k}: got {g} want {w} dims {q.dimensions}" for k, g, w in bad[:limit]] if bad else []


def dry(q, dts, modes, rows=4099, ranges=None):
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
    for i, (dt, mode) in enumerate(zip(dts, modes)):
        if mode == 0:
            p.Columns[i] = columns.constant_column(dt, 1)
        else:
            p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, rows, 0, 64 * 200, mode, 3)
    p.NumRows = rows
    for col, (lo, hi) in (ranges or {}).items():
        p.Ranges[col].Known, p.Ranges[col].Min, p.Ranges[col].Max = 1, lo, hi
    src = C.c_char_p()
    h = fn(q.agg_spec(), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    assert int(h.res or 0) > 0, "plan was not eligible for specialisation"
    return (src.value or b"").decode()


# ---- chains -------------------------------------------------------------------------------------------------------
FA, FB, FC, FD = (E.Col(i, A.Float32, n) for i, n in ((1, "a"), (2, "b"), (3, "c"), (4, "d")))
UA, UB = E.Col(5, A.Uint32, "ua"), E.Col(6, A.Int32, "ib")
CHAIN_DTS = [A.Uint32, A.Float32, A.Float32, A.Float32, A.Float32, A.Uint32, A.Int32]


def chain_exprs():
    mul = E.mul(FA, FB)
    return [E.add(mul, FC), E.Binary(A.Minus, mul, FC), E.Binary(A.Minus, FC, mul), E.add(mul, E.mul(FC, FD)),
            E.add(E.div(FA, FB), FC), E.Binary(A.Minus, E.mul(FA, E.Lit(3.0)), E.Lit(0.3)),
            E.Binary(A.Minus, UA, E.Lit(7)), E.Unary(A.Negate, UB), E.Binary(A.Minus, UA, UB),
            E.Unary(A.Not, FD), E.Unary(A.IsNull, FD)]


CHAIN_FLOATS = [0.1, 3.0, 0.3, -0.0, 0.0, 1e-45, 1.17549435e-38, 3.4028235e38, float("inf"), float("-inf"), 16777217.0,
                1.0 / 3.0, 7.0, -2.5, 1e-20, 2.0 ** 31]
CHAIN_INTS = [0, 1, 7, 2 ** 31, 2 ** 31 - 1, 2 ** 32 - 1, 6, 65536]


def chain_rows():
    """Column tuples and validity for the chain cases (c and d are mode-0 columns in some batches: their default)."""
    rng = np.random.default_rng(23)
    rows = []
    fl = [R.f32_bits(v) for v in CHAIN_FLOATS] + [0x7FC00000]
    for i, a in enumerate(fl):
        for j, b in enumerate(fl):
            c = fl[(i * 3 + j) % len(fl)]
            d = fl[(i + 5 * j) % len(fl)]
            ua, ib = CHAIN_INTS[(i + j) % 8], [0, -1, -2 ** 31, 2 ** 31 - 1, 5][(i * j) % 5] & M32
            rows.append([a, b, c, d, ua, ib])
    # the fare case: 0.1f * 3 - 0.3f
    rows.append([R.f32_bits(0.1), R.f32_bits(3.0), R.f32_bits(0.3), R.f32_bits(0.0), 0, 0])
    valid = rng.random((len(rows), 6)) >= 0.15
    return rows, valid


# ---- GPU helpers ---------------------------------------------------------------------------------------------------
def spread(table, copies=7):
    """The table repeated with its length made odd, so that every row lands in every position of a quad; the last copy
    is cut short (a partial tile)."""
    n = len(table) * copies + len(table) // 2 + 1
    return [table[i % len(table)] for i in range(n)]


def upload(be, dts, rows, valid_fn, modes, defaults=None, start_bits=None):
    """A Batch of columns dts (column 0: the row number); rows[r][i - 1] is column i's stored value."""
    n = len(rows)
    cols, keep = [], []
    for i, dt in enumerate(dts):
        if i == 0:
            buf, vp = columns.make_column(be.space, A.Uint32, np.arange(n, dtype=np.uint32))
        elif modes[i] == 0:
            d, dv = defaults[i]
            vp = columns.constant_column(dt, d, dv)
            buf = None
        else:
            vals = stored_array(dt, [r[i - 1] for r in rows])
            ok = None if modes[i] == 1 else np.asarray([valid_fn(r, i) for r in range(n)], bool)
            buf, vp = columns.make_column(be.space, dt, vals, valid=ok, start_bit=(start_bits or {}).get(i, 0))
        cols.append(vp)
        if buf is not None:
            keep.append(buf)
    return Batch(cols, n, keep=keep)


def run(be, q, batch, fused=True):
    ex = FusedBatchExecutor(be.lib, be.space, q) if fused else LegacyBatchExecutor(be.lib, be.space, q)
    ex.process_batch(batch)
    r = ex.result()
    if fused:
        ex.close()
    return r


def row_view(rows, valid_fn, modes, defaults, dts):
    """Per row: [(stored, valid)] per column as the restatement reads it (a mode-0 column is its default)."""
    out = []
    for r, row in enumerate(rows):
        cells = [(r, True)]
        for i in range(1, len(dts)):
            if modes[i] == 0:
                d, dv = defaults[i]
                cells.append(((R.f32_bits(d) if dts[i] == A.Float32 else d) if dv else 0, dv))
            else:
                cells.append((row[i - 1], True if modes[i] == 1 else valid_fn(r, i)))
        out.append(cells)
    return out


def check_dims(eng, q, batch, view, dts, ctx):
    got = run(eng, q, batch)
    assert not diff(got_dims(got), expected_dims(q, view, dts), q), (ctx, diff(got_dims(got), expected_dims(q, view, dts), q))
    per_node = run(eng, q, batch, fused=False)
    assert got_dims(per_node) == got_dims(got), (ctx, "per-node", diff(got_dims(got), got_dims(per_node), q))


def rows_kept(res):
    return sorted(int.from_bytes(res.dim_values[0][g].tobytes(), "little") for g in range(res.groups))


# ---- CPU: each GPU case reaches the form it targets, and the chains have no FFMA -----------------------------------
def test_gpu_cases_reach_their_forms(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    for da, db in PAIRINGS:
        for q in binary_dim_queries(da, db):
            src = dry(q, [A.Uint32, da, db], [1, 2, 2])
            # hash form, every dimension through the shared functors (no division or packed-equality rewrite here)
            assert "#define JIT_DENSE 0" in src and "fastDivU32(x[r]" not in src
            assert src.count("evalBinary(") == len(q.dimensions) - 1, q.dimensions
    for dt in P.COLUMN_TYPES:
        for q in unary_dim_queries(dt):
            assert "evalUnary(" in dry(q, [A.Uint32, dt], [1, 2])
    # filter roots: `column CMP literal` is hoisted (its validity folded into nbAll), a chain is not
    for q, hoisted in filter_queries():
        src = dry(q, CHAIN_DTS, [1, 2, 2, 2, 2, 2, 2])
        assert ("nbAll &= nb" in src) == hoisted, q.filters
    for qs in member_filter_groups():
        from test_shared_scan import dry_run_multi
        from test_aggregate_forms import _plan
        p = _plan(qs[0].plan_instructions(measures=qs), 4099, {0: (0, 4098)})
        p.NumColumns = len(CHAIN_DTS)
        for i, dt in enumerate(CHAIN_DTS):
            p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, 4099, 0, 64 * 200, 2, 0)
        _, src = dry_run_multi(A.load_engine(), qs, p)
        assert f"#define JIT_NMEAS {len(qs)}" in src and "am0[r]" in src and "#define JIT_DENSE 1" in src
    for modes in CHAIN_MODES:
        for q in chain_queries():
            src = dry(q, CHAIN_DTS, modes)
            assert "#define JIT_DENSE 0" in src and ("evalBinary(" in src or "evalUnary(" in src)
            n = CHAIN_BATCH_ROWS
            for zm in ((0, n - 1), NARROW):
                src = dry(q, CHAIN_DTS, modes, rows=n, ranges={0: zm})
                want = measure_form(q, zm)
                assert f"#define JIT_DENSE {want}\n" in src, (q.measure_kind, q.measure, zm)


CHAIN_MODES = [[1, 1, 1, 1, 1, 1, 1], [1, 2, 2, 2, 2, 2, 2], [1, 1, 1, 0, 0, 1, 1]]
NARROW = (0, 999)           # a zone map that leaves most rows of a chain batch to the cold path
CHAIN_BATCH_ROWS = 9136     # rows of a chain batch (spread of the chain table, 31 copies)


def measure_form(q, zone_map):
    """JIT_DENSE of a chain query under a zone map of the row number.  A dimension root over a functor is bounded only
    when its result is a Bool (Not, IsNull): other such dimensions keep the hash table (0).  Otherwise 1 (CTA slots)
    under the narrow zone map; under the exact one 2 (global slots: more slots than a CTA holds), or 0 for an integer
    SUM, which keeps the hash table."""
    if any(dt != A.Bool for dt in q.dim_types[1:]):
        return 0
    if zone_map == NARROW:
        return 1
    return 0 if q.measure_kind == "sum" and q.agg_func != A.AGGR_SUM_FLOAT else 2


def chain_queries():
    ex = chain_exprs()
    qs = [AggQuery([], [ROWNO] + list(c), Measure("count")) for c in chunks(ex, DIMS_PER_KERNEL)]
    # measure roots: sums (Float64 / Int64), min / max (Float32 / Int32 / Uint32)
    mul = E.mul(FA, FB)
    for kind, e in [("sum", E.Binary(A.Minus, mul, FC)), ("sum", E.add(mul, E.mul(FC, FD))), ("min", E.add(mul, FC)),
                    ("max", E.Binary(A.Minus, FC, mul)), ("sum", E.Binary(A.Minus, UA, UB)), ("max", E.Unary(A.Negate, UB)),
                    ("min", E.Binary(A.Minus, UA, E.Lit(7))), ("sum", E.Unary(A.Negate, UB))]:
        qs.append(AggQuery([], [ROWNO], Measure(kind, e)))
    return qs


def filter_queries():
    """(query, hoisted): Float32 `column CMP literal` with float and int literals, uint32 against int32 literals, and
    the chains as non-hoisted filter roots."""
    out = []
    for f in [E.lt(FA, E.Lit(0.1)), E.ge(FA, E.Lit(16777217.0)), E.eq(FA, E.Lit(-0.0)), E.gt(FA, E.Lit(-1)),
              E.lt(UA, E.Lit(-1)), E.ge(UA, E.Lit(2 ** 31)), E.lt(UB, E.Lit(0.5)), E.ne(FA, E.Lit(2 ** 31))]:
        out.append((AggQuery([f], [ROWNO], Measure("count")), True))
    mul = E.mul(FA, FB)
    for f in [E.lt(E.Binary(A.Minus, E.mul(FA, E.Lit(3.0)), E.Lit(0.3)), E.Lit(0.0)), E.lt(E.add(mul, FC), FD),
              E.ge(E.Binary(A.Minus, FC, mul), E.Lit(0.0)), E.and_(E.lt(FA, FB), E.ne(FC, FD)),
              E.or_(E.gt(FA, E.Lit(1.0)), E.lt(FB, E.Lit(0.0))), E.Unary(A.Not, E.eq(FA, FB))]:
        out.append((AggQuery([f], [ROWNO], Measure("count")), False))
    return out


def member_filter_groups():
    """Four queries with different filters over the same dimension: one kernel, each filter a member filter."""
    fs = [E.lt(E.add(E.mul(FA, FB), FC), E.Lit(0.0)), E.and_(E.gt(FA, FB), E.Unary(A.IsNull, FC)),
          E.or_(E.lt(UA, E.Lit(-1)), E.eq(FD, E.Lit(0.1))), E.Unary(A.Not, E.ge(E.Binary(A.Minus, UA, UB), E.Lit(0))),
          E.lt(UA, UB), E.ne(E.div(FA, FB), FC), E.gt(E.Binary(A.Minus, FC, E.mul(FA, FB)), E.Lit(-0.0)), E.eq(FA, FA)]
    return [[AggQuery([f], [ROWNO], Measure("count")) for f in c] for c in chunks(fs, 4)]


def _sass_ffma(dump):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    out = {}
    for cubin in sorted(Path(dump).glob("*.cubin")):
        sass = subprocess.run([cuobjdump, "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout
        out[cubin.name] = (len(re.findall(r"\bFFMA\b", sass)), len(re.findall(r"\bFMUL\b", sass)))
    return out


def sass_guard_queries():
    """The Float32 chains without a division (the IEEE division routine contracts its own Newton steps into FFMAs): as
    dimensions, measures and filter roots."""
    mul = E.mul(FA, FB)
    dims = [E.add(mul, FC), E.Binary(A.Minus, mul, FC), E.Binary(A.Minus, FC, mul), E.add(mul, E.mul(FC, FD)),
            E.Binary(A.Minus, E.mul(FA, E.Lit(3.0)), E.Lit(0.3))]
    return [AggQuery([], [ROWNO] + dims, Measure("count"))] + chain_queries()[3:7] + [q for q, _ in filter_queries()[8:11]]


def test_float_chains_are_rounded_per_functor(monkeypatch):
    """The kernels of the Float32 chains over mode-1 and mode-0 columns (no null bitmap between the multiply and the
    add) contain FMULs and no FFMA: each functor's result is rounded once."""
    dump = tempfile.mkdtemp(prefix="aresjit_functor_")
    try:
        monkeypatch.setenv("ARESDB_B200_JIT_DUMP_DIR", dump)
        monkeypatch.delenv("ARESDB_B200_JIT_GENERATE_ONLY", raising=False)
        for modes in (CHAIN_MODES[0], CHAIN_MODES[2]):
            for q in sass_guard_queries():
                dry(q, CHAIN_DTS, modes)
        counts = _sass_ffma(dump)
        assert len(counts) == 2 * len(sass_guard_queries()) and sum(m for _, m in counts.values()) > 0, counts
        assert all(f == 0 for f, _ in counts.values()), counts
    finally:
        shutil.rmtree(dump, ignore_errors=True)


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("da,db", PAIRINGS, ids=[f"{NAMES[a]}-{NAMES[b]}" for a, b in PAIRINGS])
def test_binary_functors_as_dimensions_on_gpu(da, db):
    eng = H.get_backend("b200")
    table = pair_table(da, db)
    rows = spread([(r[0], r[2]) for r in table])
    vflags = spread([(r[1], r[3]) for r in table])
    dts, modes = [A.Uint32, da, db], [1, 2, 2]
    vf = lambda r, i: vflags[r][i - 1]
    batch = upload(eng, dts, rows, vf, modes, start_bits={1: 5, 2: 3})
    view = row_view(rows, vf, modes, None, dts)
    for q in binary_dim_queries(da, db):
        check_dims(eng, q, batch, view, dts, (NAMES[da], NAMES[db]))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", P.COLUMN_TYPES, ids=[NAMES[d] for d in P.COLUMN_TYPES])
def test_unary_functors_as_dimensions_on_gpu(dt):
    """Every unary functor (but the calendar and HLL ones) on modes 0 (valid and invalid default), 1 and 2."""
    eng = H.get_backend("b200")
    ev = edges(dt)
    rows = spread([(v,) for v in ev] * 2)
    flags = spread([True] * len(ev) + [False] * len(ev))
    dts = [A.Uint32, dt]
    for modes, defaults in ([1, 2], None), ([1, 1], None), ([1, 0], {1: (ev[-1], True)}), ([1, 0], {1: (ev[-1], False)}):
        if modes[1] == 0 and dt == A.Float32:
            defaults = {1: (float(R.bits_f32(ev[3])), defaults[1][1])}
        vf = lambda r, i: flags[r]
        batch = upload(eng, dts, rows, vf, modes, defaults, start_bits={1: 6})
        view = row_view(rows, vf, modes, defaults, dts)
        for q in unary_dim_queries(dt):
            check_dims(eng, q, batch, view, dts, (NAMES[dt], modes, defaults))


def _chain_batch(eng, modes, zone_map=None):
    """The chain table over columns of `modes`; `zone_map`: the (min, max) announced for the row number (direct-indexed
    forms; rows above a narrow maximum take the cold path)."""
    table, valid = chain_rows()
    rows = spread(table, copies=31)          # more than one full tile: the zone-map batch runs direct-indexed
    vmat = np.asarray(spread([tuple(v) for v in valid], copies=31))
    defaults = {3: (0.3, True), 4: (0.0, False)}
    vf = lambda r, i: bool(vmat[r][i - 1])
    batch = upload(eng, CHAIN_DTS, rows, vf, modes, defaults)
    assert len(rows) == CHAIN_BATCH_ROWS
    if zone_map:
        batch.ranges = {0: zone_map if zone_map != "exact" else (0, len(rows) - 1)}
    return batch, row_view(rows, vf, modes, defaults, CHAIN_DTS)


def _measure_expected(q, view):
    """{row number: measure bits} of a query grouped by the row number alone (a NULL measure is the identity)."""
    oc = R.sink_class(q.measure_data_type, False)
    ident = {A.AGGR_MIN_FLOAT: R.f32_bits(3.402823466e38), A.AGGR_MAX_FLOAT: R.f32_bits(1.175494351e-38),
             A.AGGR_MIN_SIGNED: 2 ** 31 - 1, A.AGGR_MAX_SIGNED: 2 ** 31, A.AGGR_MIN_UNSIGNED: M32}.get(q.agg_func, 0)
    out = {}
    for r, row in enumerate(view):
        c, cls = eval_expr(q.measure, row, CHAIN_DTS)
        out[r] = R.cvt(c[0], cls, oc) if c[1] else ident      # (None: an undefined conversion)
    return out


def _measure_got(res):
    w = res.query.measure_bytes
    raw = res.measures.view(np.uint8).reshape(res.groups, w)
    return {int.from_bytes(res.dim_values[0][g].tobytes(), "little"): int.from_bytes(raw[g].tobytes(), "little")
            for g in range(res.groups)}


def _nan_equal(a, b, w):
    """Same bits; an expectation of None (an undefined conversion) takes any bits; two Float64 NaNs are equal (the F32
    -> F64 conversion of a NaN keeps no pattern the reference states)."""
    if a == b or b is None:
        return True
    return w == 8 and a is not None and np.isnan(R.bits_f64(a)) and np.isnan(R.bits_f64(b))


@pytest.mark.gpu
@pytest.mark.parametrize("modes", CHAIN_MODES, ids=["mode1", "mode2", "mode0"])
def test_chains_on_gpu(modes):
    """a*b + c, a*b - c, c - a*b, a*b + c*d, a/b + c, unsigned Minus, Negate of INT_MIN as dimensions (hash form) and as
    measures: hash table (no zone map), global slots (the row number's exact range), CTA slots with the rows above a
    narrow range on the cold path.  MIN / MAX of a NaN row is NaN."""
    eng = H.get_backend("b200")
    batch, view = _chain_batch(eng, modes)
    zoned = {zm: _chain_batch(eng, modes, zone_map=zm)[0] for zm in ("exact", NARROW)}
    for q in chain_queries():
        if q.measure_kind == "count":
            for b in [batch] + list(zoned.values()):
                before = J.T.dense_launches(eng)
                check_dims(eng, q, b, view, CHAIN_DTS, (modes, b.ranges))
                assert J.T.dense_launches(eng) - before == (b.ranges is not None and measure_form(q, b.ranges[0]) != 0)
            continue
        exp, w = _measure_expected(q, view), q.measure_bytes
        for b in [batch] + list(zoned.values()):
            before = J.T.dense_launches(eng)
            got = _measure_got(run(eng, q, b))
            bad = [(r, hex(got.get(r, -1)), hex(exp[r])) for r in exp if not _nan_equal(got.get(r, -1), exp[r], w)]
            assert not bad and len(got) == len(exp), (q.measure_kind, q.measure, b.ranges, bad[:6])
            assert J.T.dense_launches(eng) - before == (b.ranges is not None and measure_form(q, b.ranges[0]) != 0)
        per_node = _measure_got(run(eng, q, batch, fused=False))
        assert len(per_node) == len(got) and all(_nan_equal(per_node[r], got[r], w) for r in got), (q.measure, "per-node")


@pytest.mark.gpu
@pytest.mark.parametrize("modes", CHAIN_MODES, ids=["mode1", "mode2", "mode0"])
def test_filters_on_gpu(modes):
    """Filter roots (hoisted `column CMP literal` and chains), and member filters of a shared scan: the rows kept."""
    eng = H.get_backend("b200")
    batch, view = _chain_batch(eng, modes)
    dense, _ = _chain_batch(eng, modes, zone_map="exact")
    before = J.T.dense_launches(eng)
    for q, _ in filter_queries():
        want = [r for r, row in enumerate(view) if R.keep(*eval_expr(q.filters[0], row, CHAIN_DTS))]
        for b in (batch, dense):
            got = rows_kept(run(eng, q, b))
            assert got == want, (q.filters, b.ranges, sorted(set(got) ^ set(want))[:8])
        assert rows_kept(run(eng, q, batch, fused=False)) == want, (q.filters, "per-node")
    assert J.T.dense_launches(eng) - before == len(filter_queries())       # one direct-indexed launch per zone-map run
    for qs in member_filter_groups():
        batch = dense
        ex = FusedRequestExecutor(eng.lib, eng.space, qs)
        ex.process_batch(batch)
        for q, res in zip(qs, ex.results()):
            want = [r for r, row in enumerate(view) if R.keep(*eval_expr(q.filters[0], row, CHAIN_DTS))]
            assert rows_kept(res) == want, (q.filters, sorted(set(rows_kept(res)) ^ set(want))[:8])
            assert rows_kept(run(eng, q, batch, fused=False)) == want, (q.filters, "per-node")
        ex.close()
