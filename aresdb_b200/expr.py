"""A small typed expression AST — the subset of the reference's query/expr package that the hot
path consumes, with the bottom-up type resolution of QueryContextHelper.Rewrite
(reference query/context/query_context_helper.go:132-330): Boolean < Unsigned < Signed < Float,
comparison operands are cast to the higher type, FLOOR / bitwise / CONVERT_TZ are unsigned,
DIV is float, SUB is at least signed, calendar functors and GET_HLL_VALUE are unsigned.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from enum import IntEnum

from . import cabi as A


class Type(IntEnum):
    Unknown = 0
    Boolean = 1
    Unsigned = 2
    Signed = 3
    Float = 4
    UUID = 7


DATA_TYPE_TO_EXPR_TYPE = {A.Bool: Type.Boolean, A.Int8: Type.Signed, A.Int16: Type.Signed, A.Int32: Type.Signed,
                          A.Int64: Type.Signed, A.Uint8: Type.Unsigned, A.Uint16: Type.Unsigned,
                          A.Uint32: Type.Unsigned, A.Float32: Type.Float, A.UUID: Type.UUID}


class Expr:
    type: Type = Type.Unknown


@dataclass
class Col(Expr):
    """VarRef of main-table column `index` (position in the batch's column list)."""
    index: int
    data_type: int
    name: str = ""

    @property
    def type(self):
        return DATA_TYPE_TO_EXPR_TYPE[self.data_type]


@dataclass
class ForeignCol(Expr):
    """VarRef of column `index` of joined dimension table `table` (0-based position in AggQuery.joins; the reference's
    VarRef.TableID - 1): read at the RecordID the join found for the row (ForeignColumnInput)."""
    table: int
    index: int
    data_type: int
    name: str = ""
    timezone: bool = False   # enum column mapped through the query's timezone-offset table (makeForeignColumnInput)

    @property
    def type(self):
        return DATA_TYPE_TO_EXPR_TYPE[self.data_type]


@dataclass
class Lit(Expr):
    """NumberLiteral; `type` Float makes it a ConstFloat, anything else a ConstInt
    (makeConstantInput, reference query/time_series_aggregate.go:239-270)."""
    value: float
    type: Type = Type.Unknown

    def __post_init__(self):
        if self.type == Type.Unknown:
            self.type = Type.Float if isinstance(self.value, float) else (Type.Signed if self.value < 0 else Type.Unsigned)


@dataclass
class Unary(Expr):
    op: int  # cabi UnaryFunctorType
    expr: Expr
    type: Type = Type.Unknown


@dataclass
class Binary(Expr):
    op: int  # cabi BinaryFunctorType
    lhs: Expr
    rhs: Expr
    type: Type = Type.Unknown


@dataclass
class Bucket(Expr):
    """A numeric bucketizer over `expr` (PLAN_FN_NUMERIC_BUCKET, a dimension root): the dimension holds the bucket ordinal.
    `spec` is the bucketizer's identity: ("width", w), ("log", b, log_min, number of bounds) or ("partitions", p0, ...).
    `bounds` is the log table / the partitions as doubles, `bounds_ptr` their copy in the executor's memory space (what
    BatchPlan.Bucketizers points at); neither is part of the expression's identity beyond `spec`."""
    expr: Expr
    spec: tuple
    bounds: tuple = field(default=(), repr=False, compare=False)
    bounds_ptr: int = field(default=0, repr=False, compare=False)
    keep: object = field(default=None, repr=False, compare=False)   # the device copy of the bounds

    @property
    def kind(self) -> str:
        return self.spec[0]

    @property
    def type(self):
        return Type.Signed if self.kind == "width" else Type.Unsigned

    @property
    def data_type(self) -> int:
        """Type of the ordinal: Int32 (width), Uint16 (log base), Uint8 (manual partitions)."""
        return {"width": A.Int32, "log": A.Uint16, "partitions": A.Uint8}[self.kind]


def _cast(e: Expr, t: Type) -> Expr:
    """expr.Cast: literals change type in place; other nodes keep theirs (the functor promotes)."""
    if isinstance(e, Lit) and t in (Type.Float, Type.Signed, Type.Unsigned) and e.type != t:
        if t == Type.Float:
            return Lit(float(e.value), Type.Float)
        if e.type == Type.Float:
            return Lit(int(e.value), t)
        return Lit(e.value, t)
    return e


def resolve(e: Expr) -> Expr:
    """Bottom-up type resolution (returns a new tree)."""
    if isinstance(e, (Col, Lit, ForeignCol)):
        return e
    if isinstance(e, Bucket):
        return Bucket(resolve(e.expr), e.spec, e.bounds, e.bounds_ptr, e.keep)
    if isinstance(e, Unary):
        c = resolve(e.expr)
        t = c.type
        if e.op == A.Not:
            t = Type.Boolean
        elif e.op == A.Negate:
            t = max(t, Type.Signed)
        elif e.op in (A.IsNull, A.IsNotNull):
            t = Type.Boolean
        elif e.op == A.BitwiseNot or A.GetWeekStart <= e.op <= A.GetHLLValue:
            t = Type.Unsigned
            c = _cast(c, Type.Unsigned)
        return Unary(e.op, c, t)
    if isinstance(e, Binary):
        l, r = resolve(e.lhs), resolve(e.rhs)
        hi = max(l.type, r.type)
        op = e.op
        if op in (A.Plus, A.Minus):
            t = hi
            if hi == Type.Float:
                l, r = _cast(l, Type.Float), _cast(r, Type.Float)
            elif op == A.Minus:
                t = Type.Signed
        elif op in (A.Multiply, A.Mod):
            t = hi
            l, r = _cast(l, hi), _cast(r, hi)
        elif op == A.Divide:
            t = Type.Float
            l, r = _cast(l, Type.Float), _cast(r, Type.Float)
        elif op in (A.BitwiseAnd, A.BitwiseOr, A.BitwiseXor, A.Floor):
            t = Type.Unsigned
            l, r = _cast(l, Type.Unsigned), _cast(r, Type.Unsigned)
        elif op in (A.And, A.Or):
            t = Type.Boolean
        elif A.Equal <= op <= A.GreaterThanOrEqual:
            t = Type.Boolean
            l, r = _cast(l, hi), _cast(r, hi)
        else:
            raise ValueError(f"unsupported binary operator {op}")
        return Binary(op, l, r, t)
    raise TypeError(e)


def scratch_data_type(t: Type) -> int:
    """getOutputDataType(exprType, 4) — reference query/time_series_aggregate.go:337-363."""
    return A.Float32 if t == Type.Float else (A.Uint32 if t == Type.Unsigned else A.Int32)


def dimension_data_type(e: Expr) -> int:
    """GetDimensionDataType — reference query/common/dim_util.go:9-40."""
    if isinstance(e, (Col, ForeignCol, Bucket)):
        return e.data_type
    return {Type.Boolean: A.Bool, Type.Unsigned: A.Uint32, Type.Signed: A.Int32, Type.Float: A.Float32,
            Type.UUID: A.UUID}.get(e.type, A.Uint32)


# ---- conveniences --------------------------------------------------------------------------------
def eq(l, r): return Binary(A.Equal, l, r)
def ne(l, r): return Binary(A.NotEqual, l, r)
def lt(l, r): return Binary(A.LessThan, l, r)
def le(l, r): return Binary(A.LessThanOrEqual, l, r)
def gt(l, r): return Binary(A.GreaterThan, l, r)
def ge(l, r): return Binary(A.GreaterThanOrEqual, l, r)
def and_(l, r): return Binary(A.And, l, r)
def or_(l, r): return Binary(A.Or, l, r)
def floor(l, r): return Binary(A.Floor, l, r)
def add(l, r): return Binary(A.Plus, l, r)
def mul(l, r): return Binary(A.Multiply, l, r)
def mod(l, r): return Binary(A.Mod, l, r)
def div(l, r): return Binary(A.Divide, l, r)


def uses_foreign(e: Expr) -> bool:
    """Does the expression read a joined table's column?"""
    if isinstance(e, ForeignCol):
        return True
    if isinstance(e, (Unary, Bucket)):
        return uses_foreign(e.expr)
    if isinstance(e, Binary):
        return uses_foreign(e.lhs) or uses_foreign(e.rhs)
    return False


def uses_bucket(e: Expr) -> bool:
    """Is the expression a numeric bucketizer (or does it contain one)?"""
    if isinstance(e, Bucket):
        return True
    if isinstance(e, Unary):
        return uses_bucket(e.expr)
    if isinstance(e, Binary):
        return uses_bucket(e.lhs) or uses_bucket(e.rhs)
    return False
