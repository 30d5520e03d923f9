"""AQL front-end subset: a JSON AQL query (the form of the reference's examples/1k_trips/queries/*.aql)
-> `AggQuery`, i.e. the part of the reference's query compiler that produces what the hot path consumes
(SURVEY.md §8 f1).  Mirrors, for a single fact table and a time zone whose offset does not change inside the
query's time range (UTC, numeric offsets like "-8" / "05:30", or an IANA name without a daylight-saving switch in range):

* time filters            query/common/time_filter.go:100-420 (calendar-aligned relative / absolute
                          expressions -> `col >= from AND col < to`)
* time bucketizers        query/time_bucketizer.go:36-299, query/common/time_bucketizer.go:60-140
                          (regular -> FLOOR, recurring -> FLOOR(MOD) [/ unit], irregular -> calendar functors)
* numeric bucketizers     query/common/aql.go:24-45 (bucketWidth / logBase / manualPartitions -> E.Bucket, a plan-only
                          functor of the fused path; the dimension is the bucket ordinal, formatted as its lower bound)
* measures                query/aql_compiler.go:1139-1250 (count -> sum(1), sum widening, hll) and
                          query/context/query_context_helper.go:540-575 (countdistincthll)
* row / common filters    SQL-ish boolean expressions over columns and literals with the reference parser's operator
                          precedence (query/expr/token.go:302-331): comparisons, AND / OR / NOT, + - * / %, & | ^ ~,
                          IN / NOT IN lists (expanded into OR chains, query_context_helper.go:93-130), IS [NOT] NULL; enum
                          literals translated through the column's dictionary (query/aql_compiler.go:540-600)

* time zones              query/common/time_filter.go:69-85 (ParseTimezone), query/time_bucketizer.go:72-146 (the time
                          column is shifted with CONVERT_TZ = Plus before it is bucketized), utils/time.go:110-116

* joins                   query/aql_compiler.go:168-282 (processJoinConditions / matchEqualJoin): up to 8 dimension tables,
                          each joined directly to the main table by ONE equality between a main-table column and the
                          table's single primary-key column; `alias.column` references become foreign-column operands
                          (VarRef.TableID = position in `joins` + 1); filters that read a joined table run after the join

* time-zone columns       query/aql_compiler.go:439-465 (processTimezone), query/aql_processor.go:459-508
                          (prepareTimezoneTable), query/time_bucketizer.go:78-92: `"timezone": "tzcolumn(join_key)"` joins the
                          configured timezone table on `join_key = alias.id` (alias `__timezone_lookup` unless the query joins
                          that table itself), maps the enum column `tzcolumn` — its dictionary holds IANA names — to the
                          zones' offsets at `now` (an int16 table on the device), and shifts the time column by the joined
                          row's offset before bucketizing

Not covered (they raise): geo joins, MORE than one daylight-saving switch inside the range of a named zone (one switch
is handled as the reference does, query/time_bucketizer.go:94-133), array functions, non-aggregate queries.
"""
from __future__ import annotations

import calendar
import datetime as _dt
import math
import re
from dataclasses import dataclass, field

from . import cabi as A
from . import expr as E
from .query import AggQuery, Join, Measure

SECONDS = {"m": 60, "h": 3600, "d": 86400}
SECONDS_PER_WEEK = 7 * 86400
SECONDS_PER_4_DAYS = 4 * 86400

_TIME_UNIT = {"year": "y", "quarter": "q", "month": "M", "week": "w", "day": "d", "hour": "h", "quarter-hour": "15m",
              "minute": "m", "second": "s"}
_REGULAR_UNIT = {"minutes": "m", "minute": "m", "day": "d", "hours": "h", "hour": "h"}
_RECURRING = {"time of day": (1, 86400), "hour of day": (3600, 86400), "hour of week": (3600, SECONDS_PER_WEEK),
              "day of week": (86400, SECONDS_PER_WEEK)}
_IRREGULAR = {"month": A.GetMonthStart, "quarter": A.GetQuarterStart, "year": A.GetYearStart, "week": A.GetWeekStart}
_IRREGULAR_RECURRING = {"day of month": A.GetDayOfMonth, "day of year": A.GetDayOfYear,
                        "month of year": A.GetMonthOfYear, "quarter of year": A.GetQuarterOfYear}


class AQLError(ValueError):
    pass


@dataclass
class Column:
    name: str
    data_type: int                       # cabi data type of the stored values (SmallEnum -> Uint8, BigEnum -> Uint16)
    enum: dict | None = None             # enum columns: literal -> dictionary id
    hll: bool = False                    # Uint32 column that already holds rho << 16 | reg values


@dataclass
class Table:
    name: str
    columns: list = field(default_factory=list)
    primary_key: list = field(default_factory=list)   # column names (dimension tables: the join key)
    is_fact_table: bool = True

    def index_of(self, name: str) -> int:
        for i, c in enumerate(self.columns):
            if c.name == name:
                return i
        raise AQLError(f"unknown column {name}")

    def ref(self, name: str) -> E.Col:
        i = self.index_of(name)
        return E.Col(i, self.columns[i].data_type, name)


@dataclass
class JoinedTable:
    """A dimension table a query may join: its schema and the resident table the executors read (joins.DimensionTable)."""
    schema: Table
    resident: object = None


# ---- time filter -----------------------------------------------------------------------------------
def parse_timezone(text: str | None) -> _dt.tzinfo:
    """ParseTimezone (query/common/time_filter.go:69-85): "hours[:minutes]" is a fixed zone, anything else an IANA name."""
    if not text or text == "UTC":
        return _dt.timezone.utc
    seg = text.split(":")
    try:
        hours = int(seg[0])
        minutes = int(seg[1]) if len(seg) > 1 else 0
        if hours < 0 or seg[0].startswith("-"):
            minutes = -minutes
        return _dt.timezone(_dt.timedelta(seconds=hours * 3600 + minutes * 60))
    except ValueError:
        pass
    try:
        import zoneinfo
        return zoneinfo.ZoneInfo(text)
    except Exception as e:  # unknown name / no tz database
        raise AQLError(f"timezone Failed to parse: {text}") from e


def _add_months(t: _dt.datetime, months: int) -> _dt.datetime:
    m = t.month - 1 + months
    return t.replace(year=t.year + m // 12, month=m % 12 + 1)


def _apply_offset(base: _dt.datetime, amount: int, unit: str):
    """start / end of the calendar unit `amount` units away from the one containing `base` (in base's time zone)."""
    def _utc(*a):   # wall-clock constructor of the query's zone (UTC unless the query names another one)
        return _dt.datetime(*a, tzinfo=base.tzinfo)
    day = _utc(base.year, base.month, base.day)
    month = _utc(base.year, base.month, 1)
    if unit == "y":
        return _utc(base.year + amount, 1, 1), _utc(base.year + 1 + amount, 1, 1)
    if unit == "q":
        start = _add_months(month, -((base.month - 1) % 3) + 3 * amount)
        return start, _add_months(start, 3)
    if unit == "M":
        start = _add_months(month, amount)
        return start, _add_months(start, 1)
    if unit == "w":  # weeks start on Monday
        start = day - _dt.timedelta(days=base.weekday()) + _dt.timedelta(days=7 * amount)
        return start, start + _dt.timedelta(days=7)
    if unit == "d":
        start = day + _dt.timedelta(days=amount)
        return start, start + _dt.timedelta(days=1)
    if unit == "h":
        start = _utc(base.year, base.month, base.day, base.hour) + _dt.timedelta(hours=amount)
        return start, start + _dt.timedelta(hours=1)
    if unit == "15m":
        start = _utc(base.year, base.month, base.day, base.hour, base.minute - base.minute % 15) + _dt.timedelta(minutes=15 * amount)
        return start, start + _dt.timedelta(minutes=15)
    if unit == "m":
        start = _utc(base.year, base.month, base.day, base.hour, base.minute) + _dt.timedelta(minutes=amount)
        return start, start + _dt.timedelta(minutes=1)
    raise AQLError(f"Unknown time filter unit: {unit}")


def _absolute(date_expr: str, time_expr: str, tz: _dt.tzinfo = _dt.timezone.utc):
    seg = date_expr.split("-")
    if len(seg) > 3:
        raise AQLError(f"Unknown time expression: {date_expr} {time_expr}")
    year, month, day, hour, minute, unit = int(seg[0]), 1, 1, 0, 0, "y"
    if len(seg) >= 2:
        if seg[1].startswith("Q"):
            if len(seg) == 3:
                raise AQLError(f"Unknown time expression: {date_expr} {time_expr}")
            month, unit = 1 + (int(seg[1][1:]) - 1) * 3, "q"
        else:
            month, unit = int(seg[1]), "M"
    if len(seg) == 3:
        day, unit = int(seg[2]), "d"
    elif time_expr:
        raise AQLError(f"Unknown time expression: {date_expr} {time_expr}")
    if time_expr:
        ts = time_expr.split(":")
        if len(ts) > 2:
            raise AQLError(f"Unknown time expression: {date_expr} {time_expr}")
        hour, unit = int(ts[0]), "h"
        if len(ts) == 2:
            minute = int(ts[1])
            unit = "15m" if minute % 15 == 0 else "m"
    start, end = _apply_offset(_dt.datetime(year, month, day, hour, minute, tzinfo=tz), 0, unit)
    return start, end, unit


def _time_expression(expression: str, now: _dt.datetime):
    """(start, end, unit) of the calendar unit an expression names."""
    if expression == "now":
        return now, now, "s"
    expression = {"today": "this day", "yesterday": "last day"}.get(expression, expression)
    seg = expression.split(" ")
    if seg[0] in ("this", "last"):
        if len(seg) != 2 or seg[1] not in _TIME_UNIT:
            raise AQLError(f"Unknown time filter expression: {expression}")
        unit = _TIME_UNIT[seg[1]]
        return (*_apply_offset(now, 0 if seg[0] == "this" else -1, unit), unit)
    if seg[-1] == "ago":
        if len(seg) != 3 or seg[1][:-1] not in _TIME_UNIT:
            raise AQLError(f"Unknown time filter expression: {expression}")
        unit = _TIME_UNIT[seg[1][:-1]]
        return (*_apply_offset(now, -int(seg[0]), unit), unit)
    if len(seg) == 1:
        m = re.fullmatch(r"(-?\d+)([yqMwdhm])", expression)
        if m:
            return (*_apply_offset(now, int(m.group(1)), m.group(2)), m.group(2))
        if re.fullmatch(r"\d+", expression):
            seconds = int(expression)
            if seconds > 99999999999:      # milliseconds
                seconds //= 1000
            if seconds > 9999999:
                t = _dt.datetime.fromtimestamp(seconds, now.tzinfo)
                return t, t, "m" if seconds % 60 == 0 else "s"
    if len(seg) > 2:
        raise AQLError(f"Unknown time filter expression: {expression}")
    return _absolute(seg[0], seg[1] if len(seg) == 2 else "", now.tzinfo)


def parse_time_filter(time_filter: dict, now: int, tz: _dt.tzinfo = _dt.timezone.utc):
    """-> (from_ts | None, to_ts | None) in epoch seconds; `to` defaults to now when only `from` is given.  Calendar
    units are those of `tz` (ParseTimeFilter's location argument)."""
    now_t = _dt.datetime.fromtimestamp(int(now), tz)
    frm = to = None
    if time_filter.get("from"):
        frm = int(_time_expression(time_filter["from"], now_t)[0].timestamp())
    if time_filter.get("to"):
        to = int(_time_expression(time_filter["to"], now_t)[1].timestamp())
    elif frm is not None:
        to = int(now)
    return frm, to


# ---- time bucketizer -------------------------------------------------------------------------------
def _bucket_size(text: str, unit: str) -> int:
    if unit in ("m", "h") and text.isdigit():
        n = int(text)
        if 0 < n < 60 and ((unit == "m" and 60 % n == 0) or (unit == "h" and 24 % n == 0)):
            return n
    raise AQLError(f"failed to parse time bucketizer: {text}: invalid bucket size for {unit}")


def _regular_bucket_seconds(s: str) -> int:
    """"3m", "4 hours", "hour", "day", "quarter-hour" ... -> seconds (ParseRegularTimeBucketizer)."""
    s = "15m" if s == "quarter-hour" else s.lower()
    seg = s.split(" ", 1)
    if len(seg) == 2:
        if seg[1] not in _REGULAR_UNIT:
            raise AQLError(f"failed to parse time bucketizer: {s}")
        unit = _REGULAR_UNIT[seg[1]]
        return _bucket_size(seg[0], unit) * SECONDS[unit]
    s = _REGULAR_UNIT.get(s, s)
    unit = s[-1:]
    if unit not in SECONDS:
        raise AQLError(f"failed to parse time bucketizer: {s}")
    return (_bucket_size(s[:-1], unit) if len(s) > 1 else 1) * SECONDS[unit]


def time_dimension_expr(bucketizer: str, time_col: E.Expr) -> E.Expr:
    """The expression a time dimension with `timeBucketizer` evaluates (UTC)."""
    unsigned = E.Type.Unsigned
    rec = None
    if bucketizer.endswith("minutes of day"):
        comps = bucketizer.split()
        if len(comps) < 4 or not comps[0].isdigit():
            raise AQLError(f"Must put number before minutes of day: got {bucketizer}")
        n = int(comps[0])
        if n < 2 or n > 30 or 30 % n:
            raise AQLError(f"Only {{2,3,4,5,6,10,15,20,30}} minutes of day are allowed: got {bucketizer}")
        rec = (60 * n, 86400)
    elif bucketizer in _RECURRING:
        rec = _RECURRING[bucketizer]
    if rec:
        base_unit, bucket = rec
        if base_unit > 1:
            t = time_col
            if bucket == SECONDS_PER_WEEK:   # 1970-01-01 is a Thursday: shift to Monday-based weeks
                t = E.Binary(A.Minus, t, E.Lit(SECONDS_PER_4_DAYS, unsigned))
            e = E.Binary(A.Floor, E.Binary(A.Mod, t, E.Lit(bucket, unsigned)), E.Lit(base_unit, unsigned))
        else:
            e = E.Binary(A.Mod, time_col, E.Lit(bucket, unsigned))
        if base_unit >= 86400:
            e = E.Binary(A.Divide, e, E.Lit(float(base_unit), E.Type.Float))
        return e
    if bucketizer in _IRREGULAR_RECURRING:
        return E.Unary(_IRREGULAR_RECURRING[bucketizer], time_col)
    if bucketizer in _IRREGULAR:
        return E.Unary(_IRREGULAR[bucketizer], time_col)
    return E.Binary(A.Floor, time_col, E.Lit(_regular_bucket_seconds(bucketizer), unsigned))


# ---- SQL-ish expressions ---------------------------------------------------------------------------
_TOKEN = re.compile(r"\s*(?:(\d+\.\d*|\.\d+|\d+)|'((?:[^']|'')*)'|([A-Za-z_][A-Za-z_0-9.]*)|(<>|!=|<=|>=|[-+*/%()=<>,&|^~]))")
# operator precedence of the reference's expression parser (query/expr/token.go:302-331), bitwise XOR above * / % included
_BINARY = {"or": (1, A.Or), "and": (2, A.And), "=": (4, A.Equal), "!=": (4, A.NotEqual), "<>": (4, A.NotEqual),
           "<": (4, A.LessThan), "<=": (4, A.LessThanOrEqual), ">": (4, A.GreaterThan), ">=": (4, A.GreaterThanOrEqual),
           "in": (4, "in"), "is": (4, "is"),
           "|": (5, A.BitwiseOr), "&": (6, A.BitwiseAnd),
           "+": (8, A.Plus), "-": (8, A.Minus), "*": (9, A.Multiply), "/": (9, A.Divide), "%": (9, A.Mod), "^": (10, A.BitwiseXor)}
AGGREGATES = ("count", "sum", "min", "max", "avg", "hll", "countdistincthll")


@dataclass
class _Call:
    name: str
    args: list


@dataclass
class _Str:
    value: str


class _Parser:
    def __init__(self, text: str, table: Table, foreign=()):
        # foreign: (alias, Table schema) per joined table, in `joins` order
        self.table, self.foreign, self.toks, pos = table, list(foreign), [], 0
        while pos < len(text):
            if text[pos:].strip() == "":
                break
            m = _TOKEN.match(text, pos)
            if not m:
                raise AQLError(f"cannot parse expression near: {text[pos:]}")
            num, s, ident, op = m.groups()
            if num is not None:
                self.toks.append(("num", num))
            elif s is not None:
                self.toks.append(("str", s.replace("''", "'")))
            elif ident is not None:
                self.toks.append(("id", ident))
            else:
                self.toks.append(("op", op))
            pos = m.end()
        self.i = 0

    def peek(self):
        return self.toks[self.i] if self.i < len(self.toks) else (None, None)

    def take(self):
        t = self.peek()
        self.i += 1
        return t

    def expect(self, op):
        if self.take() != ("op", op):
            raise AQLError(f"expected {op}")

    def parse(self):
        e = self.expression(0)
        if self.i != len(self.toks):
            raise AQLError(f"unexpected token {self.peek()[1]}")
        return e

    def expression(self, min_prec: int):
        lhs = self.unary()
        while True:
            kind, v = self.peek()
            key = v.lower() if kind == "id" else v
            negated = False
            if kind == "id" and key == "not":       # only as NOT IN here (query/expr/parser.go:319-329)
                nxt = self.toks[self.i + 1] if self.i + 1 < len(self.toks) else (None, None)
                if nxt[0] != "id" or nxt[1].lower() != "in":
                    raise AQLError("expected IN after NOT")
                negated, key = True, "in"
            if kind not in ("op", "id") or key not in _BINARY or _BINARY[key][0] < min_prec:
                return lhs
            prec, op = _BINARY[key]
            self.take()
            if negated:
                self.take()
            if op == "in":
                lhs = self.inclusion(lhs, negated)
            elif op == "is":
                lhs = self.is_test(lhs)
            else:
                rhs = self.expression(prec + 1)
                lhs = self.binary(op, lhs, rhs)

    def inclusion(self, lhs, negated: bool):
        """`column IN (a, b, ...)` -> ((column = a) OR (column = b)) OR ...; NOT IN -> NOT of that (expandINop,
        query/context/query_context_helper.go:93-130, 335-341).  An empty list is the literal false."""
        if not isinstance(lhs, (E.Col, E.ForeignCol)):
            raise AQLError("lhs of IN or NOT_IN must be a valid column")
        self.expect("(")
        values = []
        if self.peek() != ("op", ")"):
            values.append(self.expression(0))
            while self.peek() == ("op", ","):
                self.take()
                values.append(self.expression(0))
        self.expect(")")
        e = E.Lit(0, E.Type.Boolean)
        for i, v in enumerate(values):
            eq = self.binary(A.Equal, lhs, v)
            e = eq if i == 0 else E.Binary(A.Or, e, eq)
        return E.Unary(A.Not, e) if negated else e

    def is_test(self, lhs):
        """`x IS [NOT] NULL` (rewriteIsOp, query/expr/parser.go:240-270)."""
        kind, v = self.take()
        affirmative = True
        if kind == "id" and v.lower() == "not":
            affirmative = False
            kind, v = self.take()
        if kind == "id" and v.lower() in ("null", "unknown"):
            return E.Unary(A.IsNull if affirmative else A.IsNotNull, lhs)
        raise AQLError(f"bad literal {v} following IS" + ("" if affirmative else " NOT"))

    def binary(self, op, lhs, rhs):
        # enum literal against an enum column -> its dictionary id (unknown literal: matches nothing, id -1)
        for a, b in ((lhs, rhs), (rhs, lhs)):
            if isinstance(b, _Str):
                column = (self.table.columns[a.index] if isinstance(a, E.Col)
                          else self.foreign[a.table][1].columns[a.index] if isinstance(a, E.ForeignCol) else None)
                if column is None or column.enum is None:
                    raise AQLError("string literals are only comparable with enum columns")
                lit = E.Lit(column.enum.get(b.value, -1))
                lhs, rhs = (a, lit) if b is rhs else (lit, a)
        return E.Binary(op, lhs, rhs)

    def column(self, v: str):
        """`column`, `main_table.column` or `alias.column` of a joined table."""
        if "." in v:
            prefix, name = v.split(".", 1)
            for t, (alias, schema) in enumerate(self.foreign):
                if prefix == alias:
                    i = schema.index_of(name)
                    return E.ForeignCol(t, i, schema.columns[i].data_type, name)
            if prefix != self.table.name:
                raise AQLError(f"unknown table {prefix}")
            v = name
        return self.table.ref(v)

    def unary(self):
        kind, v = self.take()
        if kind == "num":
            return E.Lit(float(v)) if "." in v else E.Lit(int(v))
        if kind == "str":
            return _Str(v)
        if kind == "op" and v == "(":
            e = self.expression(0)
            self.expect(")")
            return e
        if kind == "op" and v == "-":
            e = self.unary()
            return E.Lit(-e.value) if isinstance(e, E.Lit) else E.Unary(A.Negate, e)
        if kind == "op" and v == "~":
            return E.Unary(A.BitwiseNot, self.unary())
        if kind == "id" and v.lower() == "not":
            return E.Unary(A.Not, self.expression(3))
        if kind == "id":
            if self.peek() == ("op", "("):
                self.take()
                args = []
                if self.peek() == ("op", "*"):
                    self.take()
                    args.append("*")
                elif self.peek() != ("op", ")"):
                    args.append(self.expression(0))
                    while self.peek() == ("op", ","):
                        self.take()
                        args.append(self.expression(0))
                self.expect(")")
                return self.call(v.lower(), args)
            if v.lower() in ("true", "false"):
                return E.Lit(1 if v.lower() == "true" else 0, E.Type.Boolean)
            return self.column(v)
        raise AQLError(f"unexpected token {v}")

    def call(self, name, args):
        if name in AGGREGATES:
            return _Call(name, args)
        if name == "floor" and len(args) == 2:
            return E.Binary(A.Floor, args[0], args[1])
        raise AQLError(f"unsupported function {name}")


def parse_expression(text: str, table: Table, foreign=()):
    return _Parser(text, table, foreign).parse()


MAX_FOREIGN_TABLES = 8


def process_joins(query: dict, table: Table, dimension_tables: dict | None):
    """The query's `joins` clause -> ([Join], [(alias, schema)]).  Same acceptance rules as the reference
    (query/aql_compiler.go:168-282): at most 8 tables; one condition per join, an equality of two columns, one of the main
    table and one of THIS joined table (either order); the joined table is a dimension table with a single-column primary
    key, and the joined column is that key (many-to-one)."""
    specs = query.get("joins") or []
    if len(specs) > MAX_FOREIGN_TABLES:
        raise AQLError(f"At most {MAX_FOREIGN_TABLES} foreign tables allowed, got: {len(specs)}")
    foreign, residents = [], []
    for spec in specs:
        known = (dimension_tables or {}).get(spec.get("table"))
        if known is None:
            raise AQLError(f"unknown table {spec.get('table')}")
        foreign.append((spec.get("alias") or spec["table"], known.schema))
        residents.append(known.resident)
    joins = []
    for t, spec in enumerate(specs):
        schema = foreign[t][1]
        conditions = spec.get("conditions") or []
        if any("geography_intersects" in c.lower() for c in conditions):
            raise AQLError("geo joins are outside this engine")
        if len(conditions) != 1:
            raise AQLError(f"1 join conditions expected, got {len(conditions)}")
        if schema.is_fact_table:
            raise AQLError(f"join table {schema.name} is fact table, only dimension table supported")
        if len(schema.primary_key) > 1:
            raise AQLError("composite key not supported")
        e = parse_expression(conditions[0], table, foreign)
        if not isinstance(e, E.Binary):
            raise AQLError("binary expression expected in join condition")
        if e.op != A.Equal:
            raise AQLError("equal join expected")
        left, right = e.lhs, e.rhs
        for side in (left, right):
            if not isinstance(side, (E.Col, E.ForeignCol)):
                raise AQLError("column in join condition expected")
        if isinstance(left, E.ForeignCol):     # main table at left, foreign table at right
            left, right = right, left
        if not isinstance(left, E.Col) or not isinstance(right, E.ForeignCol) or right.table != t:
            raise AQLError(f"foreign table must be joined directly to the main table, join condition: {conditions[0]}")
        if not schema.primary_key or schema.primary_key[0] != right.name:
            raise AQLError("join column is not primary key of foreign table")
        joins.append(Join(residents[t], left))
    return joins, foreign


# ---- query -----------------------------------------------------------------------------------------
DEFAULT_TIMEZONE_ALIAS = "__timezone_lookup"


def parse_timezone_column(text) -> tuple | None:
    """`column(join_key)` -> (column of the timezone table, join key of the main table); anything else: None
    (parseTimezoneColumnString, query/aql_compiler.go:1395-1406)."""
    m = re.fullmatch(r"\s*([A-Za-z_][A-Za-z_0-9]*)\s*\(\s*([A-Za-z_][A-Za-z_0-9.]*)\s*\)\s*", str(text or ""))
    return (m.group(1), m.group(2)) if m else None


def compile_query(query: dict, table: Table, now: int, reduce_mode: int = A.ARES_REDUCE_SORT,
                  dimension_tables: dict | None = None, timezone_table: str | None = None, upload=None) -> AggQuery:
    """One element of the AQL `queries` array -> AggQuery.  `now` (epoch seconds) anchors relative time filters;
    `dimension_tables` {name: JoinedTable} are the tables the `joins` clause may name; `timezone_table` is the configured
    timezone table (utils config Query.TimezoneTable.TableName) and `upload(int16 array) -> buffer with .ptr` places the
    offset table of a time-zone column in the executor's memory space."""
    if query.get("table") != table.name:
        raise AQLError(f"unknown table {query.get('table')}")
    tz_column = parse_timezone_column(query.get("timezone"))
    tz_alias = None
    if tz_column is not None:       # processTimezone: the timezone table joins the query (once)
        if not timezone_table:
            raise AQLError("a time-zone column needs the configured timezone table")
        specs = list(query.get("joins") or [])
        tz_alias = next((j.get("alias") or j["table"] for j in specs if j.get("table") == timezone_table), None)
        if tz_alias is None:
            tz_alias = DEFAULT_TIMEZONE_ALIAS
            specs.append({"table": timezone_table, "alias": tz_alias, "conditions": [f"{tz_column[1]}={tz_alias}.id"]})
        query = dict(query, joins=specs)
    joins, foreign = process_joins(query, table, dimension_tables)
    tz = _dt.timezone.utc if tz_column is not None else parse_timezone(query.get("timezone"))
    tz_operand = None
    if tz_column is not None:       # prepareTimezoneTable: dictionary id -> the zone's offset at `now`
        t = next(i for i, (alias, _) in enumerate(foreign) if alias == tz_alias)
        schema = foreign[t][1]
        try:
            ci = schema.index_of(tz_column[0])
        except AQLError:
            raise AQLError(f"unknown timezone column {tz_column[0]}") from None
        names = schema.columns[ci].enum
        if names is None:
            raise AQLError(f"unknown timezone column {tz_column[0]}")
        import numpy as np
        seconds = np.zeros(max(names.values(), default=-1) + 1, np.int64)
        for zone, i in names.items():
            try:
                import zoneinfo
                seconds[i] = int(_dt.datetime.fromtimestamp(int(now), zoneinfo.ZoneInfo(zone)).utcoffset().total_seconds())
            except Exception as e:
                raise AQLError(f"error parsing timezone {zone}") from e
        # the table is int16, filled with Go's int16(offset): offsets from +9:06:08 on (Sydney, Auckland ...) WRAP, there
        # as here (aql_processor.go:488-492)
        lookup = seconds.astype(np.int16)
        if upload is None:
            raise AQLError("a time-zone column needs `upload` (the offset table lives in the executor's memory space)")
        buf = upload(lookup)
        joins[t].timezone_ptr, joins[t].timezone_size, joins[t].timezone_keep = buf.ptr, len(lookup), buf
        tz_operand = E.ForeignCol(t, ci, schema.columns[ci].data_type, tz_column[0], timezone=True)
    measures = query.get("measures") or []
    if len(measures) != 1:
        raise AQLError("expect one measure per query")   # aql_compiler.go:1140-1146
    m = measures[0]
    agg = parse_expression(m.get("sqlExpression") or m.get("expr"), table, foreign)
    if not isinstance(agg, _Call):
        raise AQLError("expect aggregate function")
    if agg.name == "count":
        measure = Measure("count")
    elif len(agg.args) != 1 or agg.args[0] == "*":
        raise AQLError(f"expect one parameter for {agg.name}")
    else:
        arg = agg.args[0]
        if agg.name == "countdistincthll" and isinstance(arg, E.Col) and table.columns[arg.index].hll:
            measure = Measure("hll", arg)      # noop when the column itself is an hll column
        else:
            measure = Measure(agg.name, arg)

    filters = [parse_expression(f, table, foreign) for f in (m.get("rowFilters") or []) + (query.get("rowFilters") or [])]
    tf = query.get("timeFilter") or {}
    time_col = None
    time_filters = []        # kept apart from the common filters (OOPK.TimeFilters): archive batches inside the range skip them
    if tf.get("column"):
        time_col = table.ref(tf["column"])
        frm, to = parse_time_filter(tf, now, tz)
        if frm is not None:
            time_filters.append(E.Binary(A.GreaterThanOrEqual, time_col, E.Lit(frm, E.Type.Unsigned)))
        if to is not None:
            time_filters.append(E.Binary(A.LessThan, time_col, E.Lit(to, E.Type.Unsigned)))

    # fixed offset of the query's zone over [from, to): buildTimeDimensionExpr (query/time_bucketizer.go:72-146) shifts
    # the time column by it (CONVERT_TZ is Plus, query/time_series_aggregate.go:87) before bucketizing
    tz_offset, tz_to_offset, dst_switch = 0, 0, 0
    if tz is not _dt.timezone.utc:
        ends = [t for t in ((frm, to) if tf.get("column") else ()) if t is not None]
        offset_at = lambda t: int(_dt.datetime.fromtimestamp(int(t), tz).utcoffset().total_seconds())
        if isinstance(tz, _dt.timezone):                     # numeric offset: constant by definition
            tz_offset = tz_to_offset = offset_at((ends or [now])[0])
        else:
            if len(ends) < 2:
                raise AQLError("a named time zone needs a time filter with both ends (its offset is taken at the ends of the range)")
            lo, hi = int(ends[0]), int(ends[1])
            tz_offset, tz_to_offset = offset_at(lo), offset_at(hi)
            # every offset change inside [from, to) matters — a range can cross TWO switches and end at the offset it started
            # with (January to January; the reference compares the two ends only and would then shift the whole range by one
            # offset): walk the range in steps no transition pair can hide in (7 days is far below the shortest gap
            # between two switches) and count the changes
            probe = list(range(lo, max(hi, lo + 1), 7 * 86400)) + [max(hi - 1, lo), hi]
            seen = [offset_at(t) for t in probe]
            changes = sum(1 for a, b in zip(seen, seen[1:]) if a != b)
            if changes > 1 or (changes == 1 and tz_offset == tz_to_offset):
                raise AQLError("more than one daylight-saving switch inside the time range is outside this front-end")
            if tz_offset != tz_to_offset:
                # ONE switch: utils.CalculateDSTSwitchTs (utils/time.go:93-107) — bisect down to an hour, round down
                f, t = lo, hi
                while t - f > 3600:
                    mid = f + (t - f) // 2
                    if offset_at(f) != offset_at(mid):
                        t = mid
                    else:
                        f = mid
                dst_switch = t - t % 3600
    dims = []
    for d in query.get("dimensions") or []:
        e = parse_expression(d.get("sqlExpression") or d.get("expr"), table, foreign)
        if d.get("numericBucketizer"):
            if d.get("timeBucketizer"):
                raise AQLError("a dimension has a timeBucketizer or a numericBucketizer, not both")
            e = numeric_bucket_expr(d["numericBucketizer"], e, table, upload)
        if d.get("timeBucketizer"):
            if tz_operand is not None:      # (timeColumn CONVERT_TZ timezoneColumn): the joined row's offset
                e = E.Binary(A.Plus, e, tz_operand)
            if dst_switch:
                # buildTimeDimensionExpr's "simulated IF" (query/time_bucketizer.go:96-133, its test
                # time_bucketizer_test.go:256-330), verbatim: timeCol + (fromOffset + (fromOffset - toOffset) * (timeCol >= switchTs))
                shift = E.Binary(A.Plus, E.Lit(tz_offset, E.Type.Signed),
                                 E.Binary(A.Multiply, E.Lit(tz_offset - tz_to_offset, E.Type.Signed),
                                          E.Binary(A.GreaterThanOrEqual, e, E.Lit(dst_switch))))
                e = E.Binary(A.Plus, e, shift)
            elif tz_offset:
                e = E.Binary(A.Plus, e, E.Lit(tz_offset, E.Type.Signed if tz_offset < 0 else E.Type.Unsigned))
            e = time_dimension_expr(d["timeBucketizer"], e)
        dims.append(e)
    q = AggQuery(filters, dims, measure, reduce_mode, joins=joins, time_filters=time_filters)
    q.time_range = (frm, to) if tf.get("column") else (None, None)
    # result formatting: DimensionMeta.from_offset / to_offset / dst_switch (utils.AdjustOffset, utils/time.go:110-116)
    q.tz_offset, q.tz_to_offset, q.dst_switch = tz_offset, tz_to_offset, dst_switch
    return q


def time_bucket_start(ts: int, bucketizer: str) -> int:
    """Host-side statement of the irregular bucket starts (tests / result formatting)."""
    t = _dt.datetime.fromtimestamp(ts, _dt.timezone.utc)
    if bucketizer == "month":
        return calendar.timegm((t.year, t.month, 1, 0, 0, 0))
    if bucketizer == "year":
        return calendar.timegm((t.year, 1, 1, 0, 0, 0))
    if bucketizer == "quarter":
        return calendar.timegm((t.year, 1 + (t.month - 1) // 3 * 3, 1, 0, 0, 0))
    if bucketizer == "week":   # Monday 00:00 (reference query/functor.cu:207-212)
        return ts - (ts - SECONDS_PER_4_DAYS) % SECONDS_PER_WEEK
    return ts - ts % _regular_bucket_seconds(bucketizer)


# ---- numeric bucketizer ------------------------------------------------------------------------------
FLT_MAX = 3.4028234663852886e38
MAX_LOG_BOUNDS = 65536        # a log table's ordinals are Uint16
MAX_PARTITIONS = 255          # manual partitions' ordinals are Uint8


def _number(v, what: str) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise AQLError(f"numericBucketizer: {what} must be a number")
    return float(v)


def _pow(b: float, k: int) -> float:
    try:
        return b ** k
    except OverflowError:
        return math.inf


def log_table(b: float, is_float: bool) -> tuple:
    """(exponent of t[0], t): the bounds t[j] = b ** (kmin + j) of a log-base bucketizer, strictly increasing, covering the
    positive values of the operand's class: from t[0] <= 2^-149 to t[-1] > FLT_MAX for Float32 values, from t[0] <= 1 to
    t[-1] > 2^32 for integers."""
    lo, hi = (2.0 ** -149, FLT_MAX) if is_float else (1.0, 2.0 ** 32)
    k = math.floor(math.log(lo) / math.log(b))
    while _pow(b, k) > lo:
        k -= 1
    while _pow(b, k + 1) <= lo:
        k += 1
    t = [_pow(b, k)]
    while t[-1] <= hi:
        if len(t) >= MAX_LOG_BOUNDS:
            raise AQLError(f"numericBucketizer: logBase {b!r} needs more than {MAX_LOG_BOUNDS} buckets")
        t.append(_pow(b, k + len(t)))
    if any(x >= y for x, y in zip(t, t[1:])):
        raise AQLError(f"numericBucketizer: the bounds of logBase {b!r} are not strictly increasing")
    return k, tuple(t)


def numeric_bucket_expr(defn, e: E.Expr, table: Table, upload=None) -> E.Expr:
    """numericBucketizer (NumericBucketizerDef, query/common/aql.go:24-45) of dimension expression `e` -> E.Bucket.  As in
    the Go struct, a zero field is an unset field, and nothing set ({}) leaves the dimension as it is.  The bounds of the
    log-base and manual-partition forms go to the executor's memory space through `upload(float64 array) -> buffer with
    .ptr`."""
    if not isinstance(defn, dict):
        raise AQLError("numericBucketizer must be an object")
    unknown = set(defn) - {"bucketWidth", "logBase", "manualPartitions"}
    if unknown:
        raise AQLError(f"numericBucketizer: unknown field {sorted(unknown)[0]}")
    width, base, parts = defn.get("bucketWidth") or 0, defn.get("logBase") or 0, defn.get("manualPartitions") or []
    given = [name for name, v in (("bucketWidth", width), ("logBase", base), ("manualPartitions", parts)) if v]
    if not given:
        return e
    if len(given) > 1:
        raise AQLError("numericBucketizer: set one of bucketWidth, logBase and manualPartitions")
    r = E.resolve(e)
    if E.uses_foreign(r):
        raise AQLError("numericBucketizer: a joined table's column cannot be bucketized")
    if isinstance(r, E.Col) and (table.columns[r.index].enum is not None or table.columns[r.index].hll):
        raise AQLError(f"numericBucketizer: {table.columns[r.index].name} is an enum or hll column")
    if r.type not in (E.Type.Boolean, E.Type.Unsigned, E.Type.Signed, E.Type.Float) or E.dimension_data_type(r) in (A.Int64, A.UUID):
        raise AQLError("numericBucketizer: the dimension must be a Bool, 1-, 2-, 4-byte integer or Float32 value")
    if width:
        w = _number(width, "bucketWidth")
        if not (0 < w < math.inf):
            raise AQLError("numericBucketizer: bucketWidth must be finite and > 0")
        return E.Bucket(e, ("width", w))
    if base:
        b = _number(base, "logBase")
        if not (1 < b < math.inf):
            raise AQLError("numericBucketizer: logBase must be finite and > 1")
        kmin, bounds = log_table(b, r.type == E.Type.Float)
        spec = ("log", b, kmin, len(bounds))
    else:
        if not isinstance(parts, list) or not 1 <= len(parts) <= MAX_PARTITIONS:
            raise AQLError(f"numericBucketizer: manualPartitions must be a list of 1 to {MAX_PARTITIONS} numbers")
        bounds = tuple(_number(p, "a manual partition") for p in parts)
        if not all(-math.inf < p < math.inf for p in bounds) or any(x >= y for x, y in zip(bounds, bounds[1:])):
            raise AQLError("numericBucketizer: manualPartitions must be finite and strictly increasing")
        spec = ("partitions",) + bounds
    if upload is None:
        raise AQLError("numericBucketizer: the bounds need `upload` (they live in the executor's memory space)")
    import numpy as np
    buf = upload(np.array(bounds, np.float64))
    return E.Bucket(e, spec, bounds, buf.ptr, buf)


def bucket_lower_bound(spec: tuple, ordinal: int) -> float:
    """The lower bound of bucket `ordinal` of a numeric bucketizer (E.Bucket.spec): fl(k * w), t[j], or -inf / p[i - 1]."""
    if spec[0] == "width":
        return float(ordinal) * spec[1]
    if spec[0] == "log":
        return _pow(spec[1], spec[2] + ordinal)
    return -math.inf if ordinal == 0 else spec[ordinal]


def compile_request(request, table: Table, now: int, **kwargs) -> list:
    """A whole AQL request — the JSON text (or parsed object) of a `.aql` file: {"queries": [...]} — -> one AggQuery per
    element, in order (the handler runs them one after the other, api/query_handler.go)."""
    import json
    if isinstance(request, (str, bytes)):
        request = json.loads(request)
    queries = request.get("queries") if isinstance(request, dict) else None
    if not isinstance(queries, list):
        raise AQLError("expect {\"queries\": [...]}")
    return [compile_query(q, table, now, **kwargs) for q in queries]
