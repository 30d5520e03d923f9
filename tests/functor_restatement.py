"""Plain-Python restatement of the AQL functor set over 32-bit `<value, valid>` cells, written from the reference's own
definitions (not from csrc/cell.cuh):

  functors         query/functor.hpp:30-78 (And / Or / Not: NULL AND x is NULL, TRUE OR NULL is TRUE), :83-198
                   (comparisons: NULL operand -> (false, false)), :205-352 (arithmetic, Negate, bitwise, Floor = a - a % b),
                   :356-380 (IsNull / IsNotNull always valid, Noop passes value and validity through)
  dispatch         query/functor.hpp:663-698 (UnaryFunctor: an unknown functor returns its argument), :924-970
                   (BinaryFunctor<O, T, T>: `default: return t1`), :746-770 and :1037-1076 (the float specialisations:
                   only Not / IsNull / IsNotNull / Negate / Noop and And / Or / comparisons / + - * / exist; every other
                   functor on a float operand returns its first argument)
  operand classes  query/binder.hpp:209-264: a column yields bool, int32_t (Int8 / Int16 / Int32, sign-extended),
                   uint32_t (Uint8 / Uint16 / Uint32) or float; a ConstInt literal is int32_t, a ConstFloat float
  common class     query/utils.hpp:83-94: float if either operand is float, else int64 if either is, else int32 if either
                   is signed, else uint32 (bool counts as unsigned)
  conversions      the C++ implicit conversions of thrust::tuple<T, bool> between the operand, common, result and sink
                   types; a bool is the byte it is stored in (`v & 0xff` of a wider cell is its value)

Values are Python ints holding the cell's raw bits (the low 32 bits for the 32-bit classes, 64 for I64 / F64).  Float32
arithmetic is one numpy float32 operation per functor: each result is rounded once, as the reference's per-node calls
round it when they write their float scratch vector.

Two things the C++ leaves to the machine, where the engine's DEVICE build and an x86 HOST build legitimately differ:

  * NaN bit patterns of arithmetic results (`device=True` gives the CUDA build's, `device=False` x86's).  PTX produces
    the canonical NaN 0x7FFFFFFF for every NaN result of add / sub / mul / div and of negation (nvcc emits `neg.f32`, which sm_90 runs as FADD -x, -0); x86 SSE returns the
    default NaN 0xFFC00000 for an invalid operation, the first NaN operand made quiet otherwise, and negates by flipping
    the sign bit.  Moving bits (Noop, a Float32 dimension of a column) keeps a NaN's pattern on both.
  * Float -> integer conversions of NaN, of +-inf or of a value whose truncation is outside the destination (int32 for
    the 1- and 2-byte sinks), which C++ leaves undefined.  The engine converts through double with nvcc's
    F2I.{S32,U32,S64}.F64.TRUNC; x86 uses cvttss2si / cvttsd2si ("integer indefinite" 0x80000000).  The tests do not model
    these bytes: `cvt` returns None for them, and a test pins only such a result's validity and that the fused and the
    per-node paths of the engine agree on its bytes.
"""
from __future__ import annotations

import math
import struct

import numpy as np

from aresdb_b200 import cabi as A

M32, M64 = 0xFFFFFFFF, 0xFFFFFFFFFFFFFFFF
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
CANONICAL_NAN = 0x7FFFFFFF

# value classes: what an operand, a result and a sink can be
BOOL, I32, U32, F32, I64, F64, I8, U8, I16, U16 = "bool", "i32", "u32", "f32", "i64", "f64", "i8", "u8", "i16", "u16"


def operand_class(dt: int) -> str:
    """What a column of data type `dt` yields (binder.hpp:209-264)."""
    return {A.Bool: BOOL, A.Int8: I32, A.Int16: I32, A.Int32: I32, A.Uint8: U32, A.Uint16: U32, A.Uint32: U32,
            A.Float32: F32, A.Int64: I64}[dt]


def sink_class(dt: int, dim: bool) -> str:
    """The class a result is converted to when it is written to a vector of type `dt` (dimension, scratch or measure)."""
    if dim:
        return {A.Bool: BOOL, A.Int8: I8, A.Uint8: U8, A.Int16: I16, A.Uint16: U16, A.Int32: I32, A.Uint32: U32,
                A.Float32: F32, A.Int64: I64}[dt]
    return {A.Int32: I32, A.Uint32: U32, A.Float32: F32, A.Int64: I64, A.Float64: F64}[dt]


def f32_bits(x) -> int:
    return struct.unpack("<I", struct.pack("<f", np.float32(x)))[0]


def bits_f32(b: int) -> np.float32:
    return np.frombuffer(struct.pack("<I", b & M32), np.float32)[0]


def f64_bits(x) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b & M64))[0]


def load(dt: int, stored) -> int:
    """Cell bits of a stored column value of type `dt`: Int8 / Int16 sign-extend to int32, Float32 keeps its bits."""
    if dt == A.Float32:
        return f32_bits(stored) if not isinstance(stored, int) else stored & M32
    if dt == A.Bool:
        return 1 if stored else 0
    return int(stored) & M32


def i32(x: int) -> int:
    x &= M32
    return x - 2 ** 32 if x >= 2 ** 31 else x


def i64(x: int) -> int:
    x &= M64
    return x - 2 ** 64 if x >= 2 ** 63 else x


# ---- conversions -------------------------------------------------------------------------------------------------
def value_of(bits: int, cls: str):
    """The C++ value of a cell: an int for the integer classes (bool: its byte, 0 or 1), a float for F32 / F64."""
    if cls == BOOL:
        return 1 if bits & 0xFF else 0
    if cls == I32:
        return i32(bits)
    if cls == U32:
        return bits & M32
    if cls == F32:
        return float(bits_f32(bits))
    if cls == I64:
        return i64(bits)
    if cls == F64:
        return bits_f64(bits)
    if cls == I8:
        return ((bits & 0xFF) ^ 0x80) - 0x80
    if cls == U8:
        return bits & 0xFF
    if cls == I16:
        return ((bits & 0xFFFF) ^ 0x8000) - 0x8000
    return bits & 0xFFFF


def _f2i(x: float, lo: int, hi: int):
    """Truncating float -> integer conversion into [lo, hi]; None where C++ leaves it undefined."""
    if math.isnan(x) or math.isinf(x) or not lo <= math.trunc(x) <= hi:
        return None
    return math.trunc(x)


def cvt(bits: int, frm: str, to: str):
    """`static_cast<To>(From value)` on cell bits; None for a float -> integer conversion C++ leaves undefined."""
    if frm == to:
        return bits
    x = value_of(bits, frm)
    isf = frm in (F32, F64)
    if to == BOOL:
        return 1 if x != 0 else 0                        # NaN != 0: true
    if to == F32:
        return f32_bits(np.float32(x))                   # (an int rounds to nearest even: 16777217 -> 16777216)
    if to == F64:
        if frm == F32:
            return f64_bits(float(bits_f32(bits)))
        return f64_bits(float(x))
    lo, hi = {I64: (-2 ** 63, 2 ** 63 - 1), U32: (0, M32)}.get(to, (INT_MIN, INT_MAX))
    v = _f2i(x, lo, hi) if isf else x
    if v is None:
        return None
    if to == I64:
        return v & M64
    if to in (I32, U32):
        return v & M32
    return v & (0xFF if to in (I8, U8) else 0xFFFF)      # 1- and 2-byte sinks: a float goes through int32 first


def host_defined(bits: int, frm: str, to: str) -> bool:
    """Is `cvt` defined by C++ (so that every build agrees on it)?"""
    return cvt(bits, frm, to) is not None


def common_class(a: str, b: str) -> str:
    """common_type of two operand classes (utils.hpp:83-94)."""
    if F32 in (a, b):
        return F32
    if I64 in (a, b):
        return I64
    if I32 in (a, b):
        return I32
    return U32


# ---- functors ----------------------------------------------------------------------------------------------------
NULL = (0, False)


def _truth(bits: int, cls: str) -> bool:
    return value_of(bits, cls) != 0                      # (NaN != 0: true)


def _f32_result(z: np.float32, device: bool) -> int:
    return CANONICAL_NAN if device and np.isnan(z) else f32_bits(z)


def _f32_arith(fn: int, x: np.float32, y: np.float32) -> np.float32:
    with np.errstate(all="ignore"):
        if fn == A.Plus:
            return np.float32(x + y)
        if fn == A.Minus:
            return np.float32(x - y)
        if fn == A.Multiply:
            return np.float32(x * y)
        return np.float32(x / y)


def eval_unary(fn: int, a: tuple, ic: str, device: bool = True):
    """(result cell, result class) of unary functor `fn` on cell `a` of class `ic` (calendar and HLL functors are
    restated by their own tests)."""
    v, ok = a
    if fn == A.Not:
        return (NULL if not ok else (0 if _truth(v, ic) else 1, True)), BOOL
    if fn == A.IsNull:
        return (0 if ok else 1, True), BOOL
    if fn == A.IsNotNull:
        return (1 if ok else 0, True), BOOL
    if fn == A.Negate:
        if not ok:
            return NULL, ic
        if ic == F32:
            x = bits_f32(v)
            return (CANONICAL_NAN if device and np.isnan(x) else v ^ 0x80000000, True), ic
        if ic == BOOL:
            return (1 if v & 0xFF else 0, True), ic        # -(true) = -1: true
        return ((-v) & M32, True), ic
    if fn == A.BitwiseNot and ic != F32:
        if not ok:
            return NULL, ic
        if ic == BOOL:
            return (1, True), ic                            # ~0 = -1 and ~1 = -2: both true
        return ((~v) & M32, True), ic
    # Noop, BitwiseNot of a float and any functor the class does not implement: the argument itself
    return a, ic


def _int_arith(fn: int, x: int, y: int, signed: bool) -> int:
    """Integer arithmetic in the common class; divisors 0 and -1 give the engine's stated results (C leaves
    x / 0, x % 0 and INT_MIN / -1 undefined)."""
    if fn == A.Plus:
        return (x + y) & M32
    if fn == A.Minus:
        return (x - y) & M32
    if fn == A.Multiply:
        return (x * y) & M32
    if fn == A.BitwiseAnd:
        return (x & y) & M32
    if fn == A.BitwiseOr:
        return (x | y) & M32
    if fn == A.BitwiseXor:
        return (x ^ y) & M32

    def cdiv(p, q):
        r = abs(p) // abs(q)
        return -r if (p < 0) != (q < 0) else r

    if signed:
        if fn == A.Divide:
            return M32 if y == 0 else (-x) & M32 if y == -1 else cdiv(x, y) & M32
        if fn == A.Mod:
            return x & M32 if y == 0 else 0 if y == -1 else (x - y * cdiv(x, y)) & M32
        return 0 if y == 0 else x & M32 if y == -1 else (y * cdiv(x, y)) & M32                 # Floor: x - x % y
    if fn == A.Divide:
        return M32 if y == 0 else x // y
    if fn == A.Mod:
        return x if y == 0 else x % y
    return 0 if y == 0 else x - x % y                                                          # Floor


CMP = {A.Equal: lambda x, y: x == y, A.NotEqual: lambda x, y: x != y, A.LessThan: lambda x, y: x < y,
       A.LessThanOrEqual: lambda x, y: x <= y, A.GreaterThan: lambda x, y: x > y,
       A.GreaterThanOrEqual: lambda x, y: x >= y}
ARITH = (A.Plus, A.Minus, A.Multiply, A.Divide)
INT_ONLY = (A.Mod, A.BitwiseAnd, A.BitwiseOr, A.BitwiseXor, A.Floor)


def eval_binary(fn: int, a: tuple, b: tuple, tc: str, device: bool = True):
    """(result cell, result class) of binary functor `fn` on cells already converted to the common class `tc`
    (I32, U32 or F32)."""
    (x, xo), (y, yo) = a, b
    if fn == A.And:
        return (NULL if not (xo and yo) else (int(_truth(x, tc) and _truth(y, tc)), True)), BOOL
    if fn == A.Or:
        if (_truth(x, tc) and xo) or (_truth(y, tc) and yo):
            return (1, True), BOOL
        return (NULL if not (xo and yo) else (0, True)), BOOL
    if fn in CMP:
        if not (xo and yo):
            return NULL, BOOL
        return (int(bool(CMP[fn](value_of(x, tc), value_of(y, tc)))), True), BOOL
    if fn in ARITH or (fn in INT_ONLY and tc != F32):
        if not (xo and yo):
            return NULL, tc
        if tc == F32:
            return (_f32_result(_f32_arith(fn, bits_f32(x), bits_f32(y)), device), True), tc
        return (_int_arith(fn, value_of(x, tc), value_of(y, tc), tc == I32), True), tc
    return a, tc                                           # "return t1"


def binary(fn: int, a: tuple, ac: str, b: tuple, bc: str, device: bool = True):
    """Operands of classes ac, bc: converted to their common class, then the functor."""
    tc = common_class(ac, bc)
    ca = (cvt(a[0], ac, tc), a[1])
    cb = (cvt(b[0], bc, tc), b[1])
    return eval_binary(fn, ca, cb, tc, device)


def keep(cell: tuple, rc: str) -> bool:
    """A filter keeps a row when the result's value converts to true; its validity is not consulted (comparisons
    already give false on NULL; Noop and "return t1" pass the stored value)."""
    return _truth(cell[0], rc)
