"""Result post-processing (SURVEY.md §8 f2): the binary dimension / measure vectors of an aggregate
query -> the nested `{dim0: {dim1: value}}` result the reference returns as JSON
(query/aql_postprocessor.go:34-170 flushResultBuffer + readMeasure :232-264, query/common/dimval.go:36-212
ReadDimension / formatTimeDimension, query/common/aql_query_result.go:45-68 Set), and the HyperLogLog
estimate of an hll query's register sets (query/common/hll.go:735-775 Compute).  UTC only.
"""
from __future__ import annotations

import datetime as _dt
import math
from dataclasses import dataclass

import numpy as np

from . import cabi as A
from . import expr as E
from .aql import _regular_bucket_seconds, AQLError, SECONDS_PER_4_DAYS, bucket_lower_bound
from .query import HLL_REGISTERS, HLLResult, QueryResult

NULL_STRING = "NULL"


@dataclass
class DimensionMeta:
    """What the reference keeps per query dimension: enum reverse dictionary and time formatting."""
    enum_names: list | None = None
    time_bucketizer: str | None = None     # set for time dimensions
    time_unit: str = ""                    # "", "second", "minute", "hour", "day", "millisecond"
    from_offset: int = 0                   # seconds the query's time zone is ahead of UTC (AggQuery.tz_offset)
    to_offset: int = 0                     # ... at the end of the range, and the switch instant when they differ
    dst_switch: int = 0                    # (AggQuery.tz_to_offset / dst_switch)
    numeric_bucketizer: tuple | None = None  # E.Bucket.spec of a numeric bucketizer: the value is the bucket ordinal


def format_float64(x) -> str:
    """strconv.FormatFloat(v, 'g', -1, 64): the 64-bit sibling of format_float32 (shortest digits that round-trip a
    double; exponent form when the decimal exponent is < -4 or >= 6)."""
    f = float(x)
    if math.isnan(f):
        return "NaN"
    if math.isinf(f):
        return "+Inf" if f > 0 else "-Inf"
    if f == 0:
        return "-0" if math.copysign(1.0, f) < 0 else "0"
    mant, exp = np.format_float_scientific(np.float64(f), unique=True, trim="-", exp_digits=2).split("e")
    e = int(exp)
    if e < -4 or e >= 6:
        return f"{mant}e{'+' if e >= 0 else '-'}{abs(e):02d}"
    return np.format_float_positional(np.float64(f), unique=True, trim="-")


def format_float32(x) -> str:
    """strconv.FormatFloat(float64(float32), 'g', -1, 32): shortest digits that round-trip a float32;
    exponent form when the decimal exponent is < -4 or >= 6 (strconv's rule for the shortest precision)."""
    f = np.float32(x)
    if np.isnan(f):
        return "NaN"
    if np.isinf(f):
        return "+Inf" if f > 0 else "-Inf"
    if f == 0:
        return "-0" if np.signbit(f) else "0"
    sci = np.format_float_scientific(f, unique=True, trim="-", exp_digits=2)   # d.ddde+XX
    mant, exp = sci.split("e")
    e = int(exp)
    if e < -4 or e >= 6:
        return f"{mant}e{'+' if e >= 0 else '-'}{abs(e):02d}"
    return np.format_float_positional(f, unique=True, trim="-")


def _utc(ts: int) -> _dt.datetime:
    return _dt.datetime.fromtimestamp(ts, _dt.timezone.utc)


def format_time_dimension(val: int, meta: DimensionMeta) -> str:
    if meta.time_unit:
        # numeric output is an instant again (utils.AdjustOffset, utils/time.go:110-116)
        offset = meta.from_offset
        if meta.dst_switch > 0 and val >= meta.dst_switch + meta.to_offset:
            offset = meta.to_offset
        val -= offset
        div = {"day": 86400, "hour": 3600, "minute": 60}.get(meta.time_unit)
        if div:
            val = int(val / div) if val < 0 else val // div   # Go integer division truncates
        elif meta.time_unit == "millisecond":
            val *= 1000
        return str(val)
    b = meta.time_bucketizer
    if b == "time of day":
        return _utc(val).strftime("%H:%M")
    if b == "hour of day":
        return _utc(val - val % 3600).strftime("%H:%M")
    if b == "hour of week":
        return _utc(val + SECONDS_PER_4_DAYS).strftime("%A %H:%M")
    if b == "day of week":     # 1970-01-01 was a Thursday
        return _utc(((val + 4) % 7) * 86400).strftime("%A")
    try:
        seconds = _regular_bucket_seconds(b)
    except (AQLError, TypeError, AttributeError):
        return str(val)
    if seconds % 86400 == 0:
        return _utc(val - val % 86400).strftime("%Y-%m-%d")
    if seconds % 3600 == 0:
        return _utc(val - val % 3600).strftime("%Y-%m-%d %H:00")
    return _utc(val).strftime("%Y-%m-%d %H:%M")


def read_dimension(raw, valid, data_type: int, meta: DimensionMeta | None) -> str | None:
    """One dimension value of one result row -> its string form (None for NULL)."""
    if not valid:
        return None
    if meta is not None and meta.numeric_bucketizer is not None:
        return format_float64(bucket_lower_bound(meta.numeric_bucketizer, int(raw)))
    is_time = meta is not None and meta.time_bucketizer is not None
    if data_type == A.Float32:
        if not is_time:
            return format_float32(raw)
        val = int(raw)                       # a time dimension that went through a float division
    elif data_type in (A.Int64, A.Int32, A.Int16, A.Int8, A.Bool):
        return str(int(raw))
    elif data_type in (A.Uint32, A.Uint16, A.Uint8):
        val = int(raw)
    elif data_type == A.UUID:
        h = bytes(raw).hex()
        return f"{h[0:8]}-{h[8:12]}-{h[12:16]}-{h[16:20]}-{h[20:32]}"
    else:
        return None
    names = meta.enum_names if meta else None
    if names is not None and 0 <= val < len(names):
        return names[val]
    if is_time:
        return format_time_dimension(val, meta)
    return str(val)


def default_metas(q) -> list:
    """The formatting a query's dimensions carry by themselves: the lower bounds of numeric bucketizers."""
    return [DimensionMeta(numeric_bucketizer=d.spec) if isinstance(d, E.Bucket) else None for d in q.dimensions]


def nested_result(result: QueryResult, metas: list | None = None) -> dict:
    """QueryResult -> nested dict keyed by the formatted dimension values, leaves = float measures."""
    q = result.query
    metas = metas or default_metas(q)
    cols = result.decoded_dims()
    out: dict = {}
    for g in range(result.groups):
        cur = out
        for d in range(len(q.dimensions)):
            v = cols[d][g]
            key = read_dimension(v, v is not None, q.dim_types[d], metas[d])
            key = NULL_STRING if key is None else key
            if d == len(q.dimensions) - 1:
                cur[key] = float(result.measures[g])
            else:
                cur = cur.setdefault(key, {})
    return out


# ---- HyperLogLog estimate ----------------------------------------------------------------------------
HLL_THRESHOLD = 15500.0
HLL_DENSE_THRESHOLD = HLL_REGISTERS // 4   # query/common/hll.go DenseThreshold


def hll_estimate_bias(estimate: float) -> float:
    """getEstimateBias (reference query/common/hll.go:639-667): mean bias of the k = 6 raw estimates nearest to
    `estimate` among the (up to 2k + 1) table entries around its insertion point; ties keep table order, as Go's
    sort.Sort does on an already ordered window of distinct distances."""
    import bisect
    from .hll_bias_p14 import BIASES, RAW_ESTIMATES
    i = bisect.bisect_right(RAW_ESTIMATES, estimate)        # first index with estimate < RAW_ESTIMATES[i]
    k = 6
    lo, hi = max(i - 1 - k, 0), min(i + k, len(RAW_ESTIMATES))
    window = sorted(((RAW_ESTIMATES[j] - estimate) ** 2, j) for j in range(lo, hi))
    return sum(BIASES[j] for _, j in window[:k]) / float(k)


def hll_estimate(dense: np.ndarray) -> float:
    """HLL.Compute on one register set (uint8[16384] of rho+1, 0 = empty) — reference query/common/hll.go:735-775:
    raw estimate alpha m^2 / sum 2^-rho, empirical bias correction up to 5m, linear counting below the threshold,
    truncation to an integer."""
    m = float(HLL_REGISTERS)
    nonzero = float(np.count_nonzero(dense))
    # float64 accumulation in the order of the Go loops (the sum is order-sensitive in its last bits and the result is
    # truncated): a sparse register set (fewer than DenseThreshold = 4096 registers, readHLL :547-581) adds its registers
    # in vector order (ascending register id) and then m - nonzero; a dense one walks all 16384 bytes (an empty
    # register's byte 0 contributes 1 / 2^0)
    s = 0.0
    regs = dense.tolist()
    if nonzero < HLL_DENSE_THRESHOLD:
        for r in regs:
            if r:
                s += 1.0 / float(1 << r)
        s += m - nonzero
    else:
        for r in regs:
            s += 1.0 / float(1 << r)
    estimate = 0.7213 / (1 + 1.079 / m) * m * m / s
    if estimate <= 5.0 * m:
        estimate -= hll_estimate_bias(estimate)
    estimate_h = estimate
    if nonzero < m:
        estimate_h = m * math.log(m / (m - nonzero))
    if estimate_h <= HLL_THRESHOLD:
        estimate = estimate_h
    return float(int(estimate))


def hll_nested_result(result: HLLResult, metas: list | None = None) -> dict:
    q = result.query
    metas = metas or default_metas(q)
    cols = result.dims.decoded_dims()
    dense = result.dense_registers()
    out: dict = {}
    for g in range(result.groups):
        cur = out
        for d in range(len(q.dimensions)):
            v = cols[d][g]
            key = read_dimension(v, v is not None, q.dim_types[d], metas[d])
            key = NULL_STRING if key is None else key
            if d == len(q.dimensions) - 1:
                cur[key] = hll_estimate(dense[result.dims.rows[g]])
            else:
                cur = cur.setdefault(key, {})
    return out


# ---- merging the nested results of several nodes -------------------------------------------------------------------
class MergeError(ValueError):
    pass


def merge_nested_results(lhs: dict, rhs: dict, agg: str) -> dict:
    """The merge a broker applies to its nodes' nested results, in place into `lhs` (reference broker/result_merge.go:44-140;
    the device-side counterpart of this engine is AggStateMerge / the exchange step).  `agg`: "count" / "sum" add, "max" /
    "min" keep the extreme, "hll" merges register sets (hll_data.HLL.merge), "avg" divides lhs (the sum query's result) by rhs
    (the count query's) and needs every key on both sides.  A key on one side only is taken as it is."""
    if agg not in ("count", "sum", "max", "min", "avg", "hll"):
        raise MergeError(f"unknown aggregation {agg}")

    def leaf(l, r, path):
        if hasattr(l, "merge") and hasattr(l, "non_zero_registers"):      # an HLL register set
            if agg != "hll":
                raise MergeError("error merging: HLL value found for non Hll aggregation")
            l.merge(r)
            return l
        if agg in ("count", "sum"):
            return l + r
        if agg == "max":
            return r if r > l else l
        if agg == "min":
            return r if r < l else l
        if agg == "avg":
            return l / r
        raise MergeError(f"error merging: number found for {agg} aggregation, path: {path}")

    def walk(l: dict, r: dict, path: list):
        for k in list(l):
            if k not in r or r[k] is None:
                if agg == "avg":
                    raise MergeError(f"error calculating avg: some dimension has only sum. path: {path + [k]}")
                continue
            if l[k] is None:
                l[k] = r[k]
            elif type(l[k]) is not type(r[k]) and not (isinstance(l[k], (int, float)) and isinstance(r[k], (int, float))):
                raise MergeError(f"error merging: different type lhs: {type(l[k]).__name__} vs. rhs: {type(r[k]).__name__}")
            elif isinstance(l[k], dict):
                walk(l[k], r[k], path + [k])
            else:
                l[k] = leaf(l[k], r[k], path + [k])
        for k in r:
            if k not in l:
                if agg == "avg":
                    raise MergeError(f"error calculating avg: some dimension has only count. path: {path + [k]}")
                l[k] = r[k]

    walk(lhs, rhs, [])
    return lhs
