"""Time bucketing on the fused kernel at calendar and time-zone edges, against a restatement built on numpy's
proleptic-Gregorian datetime64 (itself pinned to Python's `datetime` on the edge table).

Every time dimension `aql.time_dimension_expr` accepts, shifted by every kind of zone `aql.compile_query` compiles, over
an edge table of instants where calendars and 32-bit arithmetic go wrong.  The restatement follows the calendar except
where the reference departs from it, and then follows the reference:

  * day of month, day of year, month of year and quarter of year count from 0 (resolveTimeBucketizer);
  * week start is 0 for every instant before 1970-01-05, the first Monday;
  * every integer literal is a ConstInt (an int32 cell), and common_type(uint32, int32) is int32: the zone shift
    `t + offset`, MINUS, MOD and FLOOR all run in the int32 class.  An instant at or above 2^31 is negative there, so
    its FLOOR rounds toward zero (2106-02-07 ends at -25,200 s, already a multiple of 3,600) and its MOD is negative;
    the calendar functors read the shifted bits as uint32, so an instant within a negative offset of 0 wraps to the top
    of the uint32 range;
  * hour of week and day of week subtract four days first: every instant before 1970-01-05 has a negative remainder,
    which the next FLOOR (C truncation) keeps negative;
  * "day of week" is a Float32 dimension (the unsigned FLOOR converted to float, divided by 86400.0);
  * the one-switch daylight-saving expression is the reference's, verbatim:
    `t + (fromOffset + (fromOffset - toOffset) * (t >= switch))`, the comparison in the int32 class too;
  * a Float32 time column is not a timestamp: the calendar functors pass it through (Noop), MOD and FLOOR of a float
    return their left operand, and a Uint32 dimension sink truncates (bucket_of_float);
  * the time filter compares the Uint32 column with ConstInt literals in the int32 class, after a literal at or above
    2^32 kept its low 32 bits (makeConstantInput): a `to` at or above 2^31 lets no instant pass (time_filter_keep).

Edge table (`edge_instants`): midnight and the second before it of 1970-01-01 .. 05, the month ends of 2023, 1972-02-29,
2000-02-29, 2100-02-28, 2100-03-01, 31 December 2000 / 2004 / 2096; 2038-01-19 03:14:07 and :08, 2106-02-07 06:28:15;
the first and last 14 hours of the uint32 range every 30 minutes; a dense stretch of hourly rows over six weeks around the
2024 daylight-saving switch of Los Angeles.  Blocks of all edge instants open each batch at offsets 0..3 (every quad
position, one block each) and sit at the end of the last full tile and in the tail.

Matrix (bucketizer x zone x form); every cell names its test, or why it is left out:

  bucketizer                          UTC    05:30  -8     14     -12    LA (one switch)
  regular: minute 3m quarter-hour     G      G      G      G      G      G
           4 hours 12h hour day
  recurring: time of day hour of day  G      G      G      G      G      G
           hour of week day of week
           10 minutes of day
  irregular: week month quarter year  G      G      G      G      G      G
  irregular recurring: day of month   G      G      G      G      G      G
           day of year month of year
           quarter of year

  G  test_bucketizer_on_gpu: every zone, both reduce modes, exact / narrow / stale / absent zone maps of the time
     column, bypass (ExpectedGroups 100,000) and the one-CTA tail (batches without a full tile), sum(v) against the
     restatement.  LA cases run on the rows of the time filter around the 2024 switch (the edge instants fall outside
     it, by definition of a one-switch range).
  Forms (test_form_of_every_case, asserted on the dry run and, on the GPU, by the direct-indexed launch count): the edge
  rows reach 2^32 - 1, so no zone map of these batches bounds a dimension below 2^31.  The four recurring calendar
  functors, whose ranges need no zone map, are direct-indexed value dimensions in every zone and with every zone map;
  hour of day and 10 minutes of day (UTC) index by quotient under a too-narrow zone map; everything else takes the hash
  table: week, month, quarter and year start (no direct-indexed form, out of scope), day of week (a Float32 dimension),
  and every zone-shifted chain (a shifted range can start below 0).  test_quotient_forms_on_gpu covers the quotient
  forms on batches whose zone map stays below 2^31 (count(*): the global slot array needs a neutral-safe aggregate):
  span division for hour over one day and for hour of day (a FLOOR of a MOD result), the plain quotient for day over
  1970 .. 1990 (span * 86400 > 2^32), the global slot array for minute over two weeks (20,160 slots).
  Time-column types (test_time_column_types_on_gpu): Int32 holding negative values, Uint16, Float32, NULL rows with
  garbage underneath, a mode-0 default, and an RLE archive batch sorted by time (Uint32 is every other test).  Not run
  for the LA zone: its time filter is defined on the Uint32 time column only (the reference refuses any other type).
  Float32 runs in UTC only, without hour of week and day of week: a shifted or week-aligned float goes negative, and a
  negative float converted to uint32 is undefined.
  test_dashboard_request_on_gpu: one compiled request of four panels on FusedRequestExecutor (member dimensions).
  test_time_filter_at_the_int32_boundary_on_gpu: `from` / `to` at and above 2^31, and a `to` beyond 2^32.

The CPU tests pin the restatement to Python's `datetime`, to the oracle's per-node UnaryTransform and its legacy call
sequence of every compiled query, and to the reference's HOST build (stored digests).

Engine mutations and what catches them (each run on an H100; reverting it restores the pass):
  * the calendar functors' direct-indexed ranges from 1 instead of 0 (jitAnalyzeDense): no result test fails, since a
    row outside the range takes the hash table and the result is the same; tools/time_bucket_bench.py times it;
  * the sign-aware quad path of fast division never taken: test_bucketizer_on_gpu[hour of week] and [day of week]
    (the negative remainders of instants before 1970-01-05 take the unsigned quotient);
  * daysBeforeMonth ignoring `leap`: test_bucketizer_on_gpu[month].
"""
from __future__ import annotations

import calendar
import ctypes as C
import datetime as dt
import functools
import gc
import json
import re

import numpy as np
import pytest

import harness as H
import parity_cases as P
import test_aggregate_forms as AF
import test_member_dimensions as MD
import test_pipeline_parity as T
import test_shared_scan as S
from aresdb_b200 import aql, cabi as A
from aresdb_b200 import columns
from aresdb_b200.executor import Batch, FusedBatchExecutor, LegacyBatchExecutor

DAY, WEEK, U32 = 86400, 7 * 86400, 1 << 32
DENSE_LO = calendar.timegm((2024, 10, 6, 0, 0, 0))        # six weeks of hourly rows around the LA switch of 2024-11-03
DENSE_HOURS = 6 * 7 * 24
LA_FILTER = {"from": "2024-10-27", "to": "2024-11-10"}      # one switch inside, in the zone's calendar


# ---- the edge table ------------------------------------------------------------------------------------------------
def _midnights():
    days = [(1970, 1, d) for d in range(1, 6)]
    days += [(2023, m, calendar.monthrange(2023, m)[1]) for m in range(1, 13)]
    days += [(2023, m, 1) for m in range(1, 13)] + [(2024, 1, 1)]
    days += [(1972, 2, 29), (2000, 2, 29), (2100, 2, 28), (2100, 3, 1), (2000, 12, 31), (2004, 12, 31), (2096, 12, 31)]
    out = []
    for y, m, d in days:
        t = calendar.timegm((y, m, d, 0, 0, 0))
        out += [t, t - 1] if t > 0 else [t]
        nxt = t + DAY                                          # the day's last second and the next midnight
        out += [nxt - 1, nxt]
    return out


@functools.lru_cache(maxsize=None)
def edge_instants():
    """uint32 instants where the calendar or the 32-bit arithmetic turns."""
    e = _midnights()
    e += [2 ** 31 - 1, 2 ** 31, U32 - 1]                        # 2038-01-19 03:14:07 / :08, 2106-02-07 06:28:15
    e += list(range(0, 14 * 3600 + 1, 1800)) + [1, 59, 3599, 4 * DAY - 1, 4 * DAY]
    e += [U32 - 1 - s for s in range(0, 14 * 3600 + 1, 1800)] + [U32 - 60, U32 - 3600]
    return np.unique(np.asarray([x for x in e if 0 <= x < U32], np.int64)).astype(np.uint32)


def _quad_blocks(rows):
    """Start rows of the edge blocks: the batch's opening rows at every quad position, the end of the last full tile and
    the tail of every tile size the engine picks."""
    n = len(edge_instants())
    stride = (n + 3) // 4 * 4 + 4
    starts = {k * stride + k for k in range(4)} | {rows - n}
    for tr in (3968, 1920, 896):
        tail = max(rows - 128, 0) // tr * tr
        starts |= {tail - n, tail, tail + 1}
    return sorted(s for s in starts if 0 <= s <= rows - n)


def time_batch(seed, rows, edges=True):
    """uint32 instants of one batch: hourly rows of the dense stretch (some seconds past the hour), edge blocks."""
    rng = np.random.default_rng(seed)
    ts = (DENSE_LO + rng.integers(0, DENSE_HOURS, rows) * 3600 + rng.integers(0, 4, rows) * 900).astype(np.uint32)
    if edges:
        e = edge_instants()
        for s in _quad_blocks(rows):
            ts[s:s + len(e)] = e
    v = rng.integers(0, 1000, rows).astype(np.uint16)
    return {"ts": ts, "v": v, "rows": rows}


@functools.lru_cache(maxsize=None)
def batches(kind="gpu"):
    if kind == "tail":
        return [time_batch(31, 3001), time_batch(32, 1999)]
    if kind == "cpu":
        return [time_batch(41, 20011), time_batch(42, 9001)]
    return [time_batch(11, 200_003), time_batch(12, 120_001)]


# ---- the restatement -----------------------------------------------------------------------------------------------
def i32(x):
    x = np.asarray(x, np.int64) & 0xFFFFFFFF
    return np.where(x >= 2 ** 31, x - U32, x)


def c_mod(a, b):
    """C remainder of int64 arrays: the dividend's sign."""
    return np.sign(a) * (np.abs(a) % b)


def calendar_of(u, fn):
    """The calendar functors on uint32 instants `u` (int64 array), from numpy's datetime64."""
    u = np.asarray(u, np.int64)
    d = u.astype("datetime64[s]")
    day, month, year = d.astype("datetime64[D]"), d.astype("datetime64[M]"), d.astype("datetime64[Y]")
    moy = (month - year).astype(np.int64)
    if fn == A.GetWeekStart:
        return np.where(u < 4 * DAY, 0, u - (u - 4 * DAY) % WEEK)
    if fn == A.GetMonthStart:
        return month.astype("datetime64[s]").astype(np.int64)
    if fn == A.GetQuarterStart:
        return (year + (moy // 3 * 3).astype("timedelta64[M]")).astype("datetime64[s]").astype(np.int64)
    if fn == A.GetYearStart:
        return year.astype("datetime64[s]").astype(np.int64)
    if fn == A.GetDayOfMonth:
        return (day - month.astype("datetime64[D]")).astype(np.int64)
    if fn == A.GetDayOfYear:
        return (day - year.astype("datetime64[D]")).astype(np.int64)
    if fn == A.GetMonthOfYear:
        return moy
    return moy // 3


def calendar_by_datetime(t, fn):
    """One instant through Python's datetime (the pin of calendar_of)."""
    c = dt.datetime.fromtimestamp(int(t), dt.timezone.utc)
    utc = lambda *a: calendar.timegm((*a, 0, 0, 0))
    if fn == A.GetWeekStart:
        return 0 if t < 4 * DAY else utc(c.year, c.month, c.day) - c.weekday() * DAY
    return {A.GetMonthStart: lambda: utc(c.year, c.month, 1), A.GetYearStart: lambda: utc(c.year, 1, 1),
            A.GetQuarterStart: lambda: utc(c.year, (c.month - 1) // 3 * 3 + 1, 1),
            A.GetDayOfMonth: lambda: c.day - 1, A.GetDayOfYear: lambda: c.timetuple().tm_yday - 1,
            A.GetMonthOfYear: lambda: c.month - 1, A.GetQuarterOfYear: lambda: (c.month - 1) // 3}[fn]()


CALENDAR_FNS = [A.GetWeekStart, A.GetMonthStart, A.GetQuarterStart, A.GetYearStart, A.GetDayOfMonth, A.GetDayOfYear,
                A.GetMonthOfYear, A.GetQuarterOfYear]
REGULAR = ["minute", "3m", "quarter-hour", "4 hours", "12h", "hour", "day"]
RECURRING = ["time of day", "hour of day", "hour of week", "day of week", "10 minutes of day"]
IRREGULAR = ["week", "month", "quarter", "year"]
IRREGULAR_RECURRING = ["day of month", "day of year", "month of year", "quarter of year"]
BUCKETIZERS = REGULAR + RECURRING + IRREGULAR + IRREGULAR_RECURRING
ZONES = ["UTC", "05:30", "-8", "14", "-12", "America/Los_Angeles"]


@functools.lru_cache(maxsize=None)
def la_zone():
    """(from offset, to offset, switch) of the LA time filter, or None without a tz database."""
    try:
        q = compile_query("hour", "America/Los_Angeles")
    except aql.AQLError:
        return None
    return q.tz_offset, q.tz_to_offset, q.dst_switch


def shifted(t, zone):
    """The time dimension's operand: `t` (int64 values of the time column) shifted as compile_query shifts it, with
    32-bit wraparound (the bits are what the next operator reads)."""
    if zone == "UTC":
        return t
    if zone == "America/Los_Angeles":
        frm, to, sw = la_zone()
        return t + frm + (frm - to) * (i32(t) >= sw)
    return t + int(aql.parse_timezone(zone).utcoffset(None).total_seconds())


def bucket(name, x):
    """Dimension cells (uint32 bits) of bucketizer `name` on operand bits x.  Every integer literal is a ConstInt, so
    every MOD / FLOOR / MINUS with one runs in the int32 class (C remainder, dividend's sign); the calendar functors
    read the bits as uint32; day of week converts the FLOOR's uint32 scratch value to float."""
    s = i32(x)
    if name in aql._IRREGULAR or name in aql._IRREGULAR_RECURRING:
        fn = {**aql._IRREGULAR, **aql._IRREGULAR_RECURRING}[name]
        return calendar_of(s & 0xFFFFFFFF, fn) & 0xFFFFFFFF
    rec = None
    if name.endswith("minutes of day"):
        rec = (60 * int(name.split()[0]), DAY)
    elif name in aql._RECURRING:
        rec = aql._RECURRING[name]
    if rec is None:
        sec = aql._regular_bucket_seconds(name)
        return (s - c_mod(s, sec)) & 0xFFFFFFFF
    base, size = rec
    if size == WEEK:
        s = i32(s - 4 * DAY)
    m = c_mod(s, size)
    if base == 1:
        return m & 0xFFFFFFFF
    f = (m - c_mod(m, base)) & 0xFFFFFFFF
    if base >= DAY:
        q = (f.astype(np.float32) / np.float32(base)).astype(np.float32)
        return q.view(np.uint32).astype(np.int64)
    return f


def bucket_of_float(name, f):
    """A Float32 time column: MOD and FLOOR of a float return their left operand, the calendar functors pass it
    through, and a Uint32 dimension sink truncates (time of day, a MOD, is a Float32 dimension); DIV and MINUS are
    float arithmetic."""
    f = np.asarray(f, np.float32)
    rec = aql._RECURRING.get(name)
    assert rec is None or rec[1] != WEEK, "f - 4 days goes negative, and a negative float to uint32 is undefined"
    if rec is not None and rec[0] == 1:             # MOD alone: a Float32 dimension
        return f.view(np.uint32).astype(np.int64)
    return f.astype(np.int64) & 0xFFFFFFFF


def column_values(hb, col_type):
    """(stored values of the time column, their int64 reading) for each time-column type."""
    ts = hb["ts"].astype(np.int64)
    if col_type == A.Int32:             # negative instants: a mirror of the table before 1970
        raw = np.where(np.arange(len(ts)) % 3 == 0, -(ts % (2 ** 31)), ts % (2 ** 31)).astype(np.int32)
        return raw, raw.astype(np.int64)
    if col_type == A.Uint16:
        raw = (ts & 0xFFFF).astype(np.uint16)
        return raw, raw.astype(np.int64)
    if col_type == A.Float32:           # values exact in float32
        raw = (ts % (1 << 24)).astype(np.float32)
        return raw, raw.astype(np.int64)
    return hb["ts"], ts


def expected_dims(hb, name, zone, col_type=A.Uint32, valid=None):
    """(cells, row validity) of the time dimension over a batch."""
    raw, t = column_values(hb, col_type)
    assert col_type != A.Float32 or zone == "UTC"
    cells = bucket_of_float(name, raw) if col_type == A.Float32 else bucket(name, shifted(t, zone))
    ok = np.ones(len(t), bool) if valid is None else valid
    return np.where(ok, cells, 0), ok


def time_filter_mask(hb, zone):
    if zone != "America/Los_Angeles":
        return np.ones(hb["rows"], bool)
    frm, to = aql.parse_time_filter(LA_FILTER, 0, aql.parse_timezone(zone))
    return (hb["ts"] >= frm) & (hb["ts"] < to)


def restate(hbs, name, zone, mode=A.ARES_REDUCE_SORT, kind="sum", col_type=A.Uint32, keep=None, valids=None, mults=None):
    """AF.Expected of sum(v) (or count) grouped by the time dimension."""
    rows, vals, mult = [], [], []
    for i, hb in enumerate(hbs):
        cells, ok = expected_dims(hb, name, zone, col_type, None if valids is None else valids[i])
        alive = time_filter_mask(hb, zone) if keep is None else keep[i]
        packed = np.hstack([cells.astype("<u4").view(np.uint8).reshape(-1, 4), ok.astype(np.uint8).reshape(-1, 1)])
        rows.append(packed[alive])
        vals.append(hb["v"][alive].astype(np.int64))
        mult.append((np.ones(hb["rows"], np.int64) if mults is None else mults[i])[alive])
    rows, v, m = np.vstack(rows), np.concatenate(vals), np.concatenate(mult)
    if mode == A.ARES_REDUCE_SORT:
        key = np.zeros(len(rows), np.uint64)
        for b in range(rows.shape[1]):
            key |= rows[:, b].astype(np.uint64) << np.uint64(8 * b)
    else:
        key = AF.hashes.murmur3_32(rows)
    uniq, first, inv = np.unique(key, return_index=True, return_inverse=True)
    meas = np.zeros(len(uniq), np.int64)
    np.add.at(meas, inv, m if kind == "count" else v * m)
    meas = (meas & 0xFFFFFFFF).astype(np.uint32) if kind == "count" else meas.view(np.uint64)
    if mode == A.ARES_REDUCE_SORT:
        grows = rows[first]
        order = np.argsort(AF.hashes.murmur3_128_lo(grows), kind="stable")
        return AF.Expected([r.tobytes() for r in grows[order]], meas[order])
    return AF.Expected(uniq.tolist(), meas)


# ---- compiled queries ----------------------------------------------------------------------------------------------
def table(col_type=A.Uint32):
    return aql.Table("trips", [aql.Column("request_at", col_type), aql.Column("v", A.Uint16)])


def aql_query(name, zone, measure="sum(v)", time_filter=None):
    q = {"table": "trips", "measures": [{"sqlExpression": measure}],
         "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": name}]}
    if zone != "UTC":
        q["timezone"] = zone
    if zone == "America/Los_Angeles":
        q["timeFilter"] = {"column": "request_at", **LA_FILTER}
    if time_filter:
        q["timeFilter"] = {"column": "request_at", **time_filter}
    return q


NOW = calendar.timegm((2024, 11, 20, 0, 0, 0))


def compile_query(name, zone, col_type=A.Uint32, mode=A.ARES_REDUCE_SORT, measure="sum(v)", time_filter=None):
    return aql.compile_query(aql_query(name, zone, measure, time_filter), table(col_type), NOW, reduce_mode=mode)


def zones():
    return [z for z in ZONES if z != "America/Los_Angeles" or la_zone() is not None]


def upload(be, hb, col_type=A.Uint32, ranges=None, valid=None, default=None):
    raw, _ = column_values(hb, col_type)
    keep, cols = [], []
    if default is not None:
        cols.append(columns.constant_column(col_type, *default))
    else:
        buf, vp = columns.make_column(be.space, col_type, raw, valid=valid)
        keep.append(buf)
        cols.append(vp)
    buf, vp = columns.make_column(be.space, A.Uint16, hb["v"])
    keep.append(buf)
    cols.append(vp)
    return Batch(cols, hb["rows"], keep=keep, ranges=ranges)


def zone_map(hb, how):
    lo, hi = int(hb["ts"].min()), int(hb["ts"].max())
    if how is None:
        return None
    if how == "exact":
        return {0: (lo, hi)}
    if how == "narrow":
        return {0: (lo, lo + (hi - lo) // 2)}
    return {0: (lo + 90 * DAY, hi + 90 * DAY)}                 # stale: another batch's


# ---- CPU: the restatement ------------------------------------------------------------------------------------------
def test_calendar_restatement_matches_datetime():
    """calendar_of (numpy datetime64) against Python's datetime on every edge instant and a stretch of 2024."""
    e = np.concatenate([edge_instants().astype(np.int64), np.arange(DENSE_LO, DENSE_LO + 400 * DAY, 86399)])
    for fn in CALENDAR_FNS:
        got = calendar_of(e, fn)
        want = [calendar_by_datetime(t, fn) for t in e.tolist()]
        assert got.tolist() == want, fn


def test_edge_table_has_the_edges():
    e = set(edge_instants().tolist())
    for t in (calendar.timegm((2000, 2, 29, 0, 0, 0)), calendar.timegm((2100, 3, 1, 0, 0, 0)) - 1, 2 ** 31 - 1, 2 ** 31,
              U32 - 1, 0, 4 * DAY - 1, calendar.timegm((2096, 12, 31, 0, 0, 0))):
        assert t in e, t
    hb = batches("gpu")[0]
    ts = hb["ts"]
    stride = (len(e) + 3) // 4 * 4 + 4
    for k in range(4):                                      # every quad position
        s = k * stride + k
        assert s % 4 == k and ts[s:s + len(e)].tolist() == sorted(e)
    quirks = {name: bucket(name, np.asarray([0, 3 * DAY, U32 - 25200], np.int64)).tolist()
              for name in ("hour of week", "week", "hour")}
    assert quirks["week"][:2] == [0, 0]                      # week start clamps to 0 before the first Monday
    assert quirks["hour of week"][:2] == [(-4 * DAY) & 0xFFFFFFFF, (-DAY) & 0xFFFFFFFF]   # negative remainders
    assert quirks["hour"][2] == U32 - 25200                  # FLOOR in the int32 class: -25200 is a multiple of 3600


@pytest.mark.parametrize("col_type", [A.Uint32, A.Int32, A.Uint16, A.Float32], ids=["u32", "i32", "u16", "f32"])
def test_calendar_functors_per_node(col_type):
    """UnaryTransform of every calendar functor over the edge table (NULLs with garbage under them) into a Uint32
    dimension: the restatement, the oracle and the reference's HOST build (stored digest)."""
    orc = H.get_backend("oracle")
    hb = {"ts": np.concatenate([edge_instants(), batches("cpu")[0]["ts"][:500]]), "rows": 0}
    hb["rows"] = len(hb["ts"])
    raw, t = column_values(hb, col_type)
    valid = np.arange(hb["rows"]) % 7 != 3
    spec = P.InputSpec("column", col_type, raw, valid, mode=2)
    results = []
    for fn in CALENDAR_FNS:
        got = P.run_transform(orc, [spec], fn, ("dim", A.Uint32), hb["rows"])
        vals = got["values"].view(np.uint32).astype(np.int64)
        want = (t & 0xFFFFFFFF) if col_type == A.Float32 else calendar_of(t & 0xFFFFFFFF, fn)
        assert got["valid"].tolist() == valid.astype(np.uint8).tolist()
        assert vals[valid].tolist() == want[valid].tolist(), fn
        results.append(got)
    H.assert_matches_reference(f"time_bucketing/per_node/{col_type}", H.digest(results),
                               lambda: H.digest([P.run_transform(H.get_backend("ref"), [spec], fn, ("dim", A.Uint32),
                                                                 hb["rows"]) for fn in CALENDAR_FNS]))


def _legacy(be, q, hbs, col_type=A.Uint32):
    ex = LegacyBatchExecutor(be.lib, be.space, q)
    for hb in hbs:
        ex.process_batch(upload(be, hb, col_type))
    return ex.result()


@pytest.mark.parametrize("zone", ZONES)
def test_compiled_queries_on_the_checkers(zone):
    """Every bucketizer in this zone, compiled by aql.compile_query, through the reference call sequence on the oracle
    (against the restatement) and the reference's HOST build (stored digest)."""
    if zone == "America/Los_Angeles" and la_zone() is None:
        pytest.skip("no tz database on this box")
    orc = H.get_backend("oracle")
    hbs = batches("cpu")
    results = []
    for name in BUCKETIZERS:
        q = compile_query(name, zone)
        got = _legacy(orc, q, hbs)
        AF.assert_matches(got, restate(hbs, name, zone), "sum", A.Uint16, ctx=f"oracle {name} {zone}")
        results.append(got)
    H.assert_matches_reference(f"time_bucketing/aql/{zone}", H.digest(results),
                               lambda: H.digest([_legacy(H.get_backend("ref"), compile_query(n, zone), hbs)
                                                 for n in BUCKETIZERS]))


def test_compiled_query_structure():
    """The chains the fused kernel specialises: MINUS (signed), MOD, FLOOR for the weekly recurring bucketizers; a zone
    shift below the bucketizer; day of week divides in float."""
    E = aql.E
    d = compile_query("hour of week", "-8").dimensions[0]
    assert d.op == A.Floor and d.lhs.op == A.Mod and d.lhs.lhs.op == A.Minus and d.lhs.lhs.lhs.op == A.Plus
    assert d.lhs.lhs.lhs.rhs.type == E.Type.Signed and int(d.lhs.lhs.lhs.rhs.value) == -28800
    d = compile_query("day of week", "14").dimensions[0]
    assert d.op == A.Divide and d.rhs.type == E.Type.Float and d.lhs.op == A.Floor
    assert d.lhs.lhs.lhs.lhs.rhs.type == E.Type.Unsigned
    q = compile_query("day of week", "UTC")
    assert q.dim_types == [A.Float32]
    for name in IRREGULAR + IRREGULAR_RECURRING:
        assert compile_query(name, "05:30").dimensions[0].op == {**aql._IRREGULAR, **aql._IRREGULAR_RECURRING}[name]
    if la_zone() is not None:
        frm, to, sw = la_zone()
        assert (frm, to) == (-25200, -28800) and calendar.timegm((2024, 11, 3, 9, 0, 0)) == sw


# ---- CPU: the form every GPU case reaches --------------------------------------------------------------------------
def _plan(q, rows, ranges=None, col_type=A.Uint32, queries=None):
    p = A.BatchPlan()
    insts = q.plan_instructions(measures=queries) if queries else q.plan_instructions()
    p.NumInsts = len(insts)
    for i, pi in enumerate(insts):
        p.Insts[i] = pi
    p.NumColumns = 2
    for i, t in enumerate((col_type, A.Uint16)):
        p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), t, rows, 0, 64 * 200 * 4, 2, 0)
    p.NumRows = rows
    for col, (lo, hi) in (ranges or {}).items():
        p.Ranges[col].Known, p.Ranges[col].Min, p.Ranges[col].Max = 1, lo, hi
    return p


def dry_run(q, rows, ranges=None, expected_groups=0, col_type=A.Uint32):
    fn = A.load_engine().alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    p = _plan(q, rows, ranges, col_type)
    src = C.c_char_p()
    h = fn(q.agg_spec(expected_groups), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return (src.value or b"").decode()


def expected_form(name, zone, how):
    """'dense' or 'hash' for a batch of batches('gpu'): its edge rows reach 2^32 - 1, so no zone map of the time column
    bounds a dimension below 2^31 (jitAnalyzeDense), and only the recurring calendar functors, whose ranges need no
    zone map, index directly."""
    if name in IRREGULAR_RECURRING:
        return "dense"
    # a too-narrow zone map ends below 2^31: the FLOOR of a UTC MOD result indexes by quotient (rows outside it take the
    # hash table); under a zone shift the sum's range starts below 0 and is not tracked
    return "dense" if how == "narrow" and zone == "UTC" and name in ("hour of day", "10 minutes of day") else "hash"


def form_of(src):
    return {0: "hash", 1: "dense", 2: "global"}[AF._macro(src, "JIT_DENSE")]


def test_form_of_every_case(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    hb = batches("gpu")[0]
    for name in BUCKETIZERS:
        for zone in zones():
            q = compile_query(name, zone)
            texts = set()
            for how in ("exact", "narrow", "stale", None):
                src = dry_run(q, hb["rows"], zone_map(hb, how))
                assert form_of(src) == expected_form(name, zone, how), (name, zone, how)
                texts.add(src)
            if name in IRREGULAR_RECURRING:             # one kernel whatever the zone map: the ranges are parameters
                assert len(texts) == 1, (name, zone)
            tail = batches("tail")[0]
            assert form_of(dry_run(q, tail["rows"], zone_map(tail, "exact"))) == "hash", (name, zone)
            assert AF._macro(dry_run(q, hb["rows"], None, 100_000), "JIT_BYPASS") == 1, (name, zone)
    # the quotient forms (count(*): the global slot array needs a neutral-safe aggregate)
    for name, ranges, form, span in QUOTIENT_CASES:
        src = dry_run(compile_query(name, "UTC", measure="count(*)"), 200_000, ranges)
        assert form_of(src) == form and ("P.dBase[0]" in src) == span, name
    # the recurring chains on the stack: the sign-aware quad path for the signed MOD of hour of week
    src = dry_run(compile_query("hour of week", "UTC"), 200_000, {0: (0, U32 - 1)})
    assert "(int32_t)(x[0] | x[1] | x[2] | x[3]) < 0" in src
    # the ranges of the calendar functors are parameters: the kernel text does not depend on them
    for name in IRREGULAR_RECURRING:
        assert "JIT_DENSE 1" in dry_run(compile_query(name, "UTC"), 200_000)


Y1990 = calendar.timegm((1990, 1, 1, 0, 0, 0))
# (bucketizer, zone map, form, span division): hour over one day (span division), day over 1970 .. 1990 (plain quotient:
# span * 86400 > 2^32), minute over two weeks (20,160 slots: the global slot array), hour of day over two weeks (the
# FLOOR of a MOD result: span division)
QUOTIENT_CASES = [("hour", {0: (DENSE_LO, DENSE_LO + DAY - 1)}, "dense", True),
                  ("day", {0: (0, Y1990 - 1)}, "dense", False),
                  ("minute", {0: (DENSE_LO, DENSE_LO + 14 * DAY - 1)}, "global", True),
                  ("hour of day", {0: (DENSE_LO, DENSE_LO + 14 * DAY - 1)}, "dense", True)]


def _uniform_batch(seed, rows, lo, span):
    rng = np.random.default_rng(seed)
    ts = (lo + rng.integers(0, span, rows)).astype(np.uint32)
    ts[:4] = [lo, lo + span - 1, lo, lo + span - 1]
    return {"ts": ts, "v": rng.integers(0, 1000, rows).astype(np.uint16), "rows": rows}


# ---- GPU -----------------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    gc.collect()
    try:
        import torch
        if torch.cuda.is_available() and torch.cuda.is_initialized():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    except ImportError:
        pass


def _run(eng, q, bs, expected_groups=0):
    ex = FusedBatchExecutor(eng.lib, eng.space, q, expected_groups)
    for b in bs:
        ex.process_batch(b)
    r = ex.result()
    ex.close()
    return r


MODES = [(A.ARES_REDUCE_SORT, "sort"), (A.ARES_REDUCE_HASH, "hash")]


@pytest.mark.gpu
@pytest.mark.parametrize("name", BUCKETIZERS)
def test_bucketizer_on_gpu(name):
    eng = H.get_backend("b200")
    for zone in zones():
        for mode, mname in MODES:
            q = compile_query(name, zone, mode=mode)
            exp = restate(batches("gpu"), name, zone, mode)
            for how in ("exact", "narrow", "stale", None):
                d0 = T.dense_launches(eng)
                got = _run(eng, q, [upload(eng, hb, ranges=zone_map(hb, how)) for hb in batches("gpu")])
                AF.assert_matches(got, exp, "sum", A.Uint16, mode, ctx=f"{name}/{zone}/{mname}/{how}")
                want = len(batches("gpu")) if expected_form(name, zone, how) != "hash" else 0
                assert T.dense_launches(eng) - d0 == want, f"{name}/{zone}/{mname}/{how}: direct-indexed launches"
            # bypass, and the one-CTA tail
            got = _run(eng, q, [upload(eng, hb) for hb in batches("gpu")], 100_000)
            AF.assert_matches(got, exp, "sum", A.Uint16, mode, ctx=f"{name}/{zone}/{mname}/bypass")
            tails = batches("tail")
            got = _run(eng, q, [upload(eng, hb, ranges=zone_map(hb, "exact")) for hb in tails])
            AF.assert_matches(got, restate(tails, name, zone, mode), "sum", A.Uint16, mode, ctx=f"{name}/{zone}/{mname}/tail")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [m for m, _ in MODES], ids=[n for _, n in MODES])
def test_quotient_forms_on_gpu(mode):
    """The quotient forms of QUOTIENT_CASES with exact, too narrow and stale zone maps; count(*) by the bucket."""
    eng = H.get_backend("b200")
    for name, ranges, form, _ in QUOTIENT_CASES:
        lo, hi = ranges[0]
        hbs = [_uniform_batch(21 + i, rows, lo, hi - lo + 1) for i, rows in enumerate((150_001, 90_001))]
        q = compile_query(name, "UTC", mode=mode, measure="count(*)")
        exp = restate(hbs, name, "UTC", mode, kind="count")
        for how in ("exact", "narrow", "stale"):
            zm = {"exact": (lo, hi), "narrow": (lo, lo + (hi - lo) // 2), "stale": (lo + (hi - lo) // 3, hi + (hi - lo) // 3)}[how]
            d0 = T.dense_launches(eng)
            got = _run(eng, q, [upload(eng, hb, ranges={0: zm}) for hb in hbs])
            AF.assert_matches(got, exp, "count", None, mode, ctx=f"{name}/{how}")
            assert T.dense_launches(eng) - d0 == len(hbs), f"{name}/{how}"


TYPE_CASES = {"i32": A.Int32, "u16": A.Uint16, "f32": A.Float32}


@pytest.mark.gpu
@pytest.mark.parametrize("type_name", ["i32", "u16", "f32", "nulls", "default", "rle"])
def test_time_column_types_on_gpu(type_name):
    """Every bucketizer in every fixed zone over one kind of time column, against the restatement and the oracle's
    reference call sequence."""
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    hbs = batches("gpu")
    col_type = TYPE_CASES.get(type_name, A.Uint32)
    for name in BUCKETIZERS:
        if col_type == A.Float32 and name in ("hour of week", "day of week"):
            continue    # bucket_of_float: a negative float converted to uint32 is undefined
        for zone in ["UTC"] if col_type == A.Float32 else [z for z in ZONES if z != "America/Los_Angeles"]:
            q = compile_query(name, zone, col_type)
            if type_name == "nulls":
                valids = [np.random.default_rng(7 + i).random(hb["rows"]) >= 0.2 for i, hb in enumerate(hbs)]
                bs = [upload(eng, hb, ranges=zone_map(hb, "exact"), valid=ok) for hb, ok in zip(hbs, valids)]
                exp = restate(hbs, name, zone, valids=valids)
            elif type_name == "default":
                t0 = calendar.timegm((2024, 2, 29, 23, 59, 59))
                const = [{"ts": np.full(hb["rows"], t0, np.uint32), "v": hb["v"], "rows": hb["rows"]} for hb in hbs]
                bs = [upload(eng, hb, default=(t0, True)) for hb in const]
                exp = restate(const, name, zone)
            elif type_name == "rle":
                bs, views = zip(*[_rle_batch(eng, hb, 60 + i) for i, hb in enumerate(hbs)])
                exp = restate(views, name, zone, mults=[v["mult"] for v in views])
            else:
                bs = [upload(eng, hb, col_type) for hb in hbs]
                exp = restate(hbs, name, zone, col_type=col_type)
            got = _run(eng, q, bs)
            AF.assert_matches(got, exp, "sum", A.Uint16, ctx=f"{type_name}/{name}/{zone}")
            if type_name in TYPE_CASES:
                T.assert_same_result(got, _legacy(orc, q, hbs, col_type), ctx=f"{type_name}/{name}/{zone} vs oracle")


def _rle_batch(eng, hb, seed):
    """An archive batch: sorted by time, the time column run-length encoded (its counts are the batch's base counts, one
    index position per run)."""
    rng = np.random.default_rng(seed)
    ts = np.sort(hb["ts"])
    runs = np.unique(ts)
    lens = rng.integers(1, 6, len(runs))
    base = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    v = rng.integers(0, 1000, len(runs)).astype(np.uint16)
    tbuf, tvp = columns.make_column(eng.space, A.Uint32, runs, counts=base)
    vbuf, vvp = columns.make_column(eng.space, A.Uint16, v)
    bc = eng.put(base)
    view = {"ts": runs, "v": v, "rows": len(runs), "mult": lens.astype(np.int64)}
    return Batch([tvp, vvp], len(runs), base_counts=bc, start_count=0, keep=[tbuf, vbuf, bc]), view


DASHBOARD = {"queries": [
    {"table": "trips", "timezone": "-8", "measures": [{"sqlExpression": "count(*)"}],
     "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "hour of day"}]},
    {"table": "trips", "timezone": "-8", "measures": [{"sqlExpression": "sum(v)"}],
     "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "day of week"}]},
    {"table": "trips", "timezone": "-8", "measures": [{"sqlExpression": "count(*)"}],
     "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "month of year"}]},
    {"table": "trips", "timezone": "-8", "measures": [{"sqlExpression": "sum(v)"}],
     "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "day of month"}]}]}


def dashboard():
    qs = aql.compile_request(json.dumps(DASHBOARD), table(), NOW)
    kinds = [q["measures"][0]["sqlExpression"].split("(")[0] for q in DASHBOARD["queries"]]
    names = [q["dimensions"][0]["timeBucketizer"] for q in DASHBOARD["queries"]]
    return qs, kinds, names


def test_dashboard_request_forms_one_pass(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    qs, _, _ = dashboard()
    from aresdb_b200.executor import shared_scan_groups, shared_scan_passes
    assert shared_scan_passes(qs, shared_scan_groups(qs, member_filters=True)) == [[0, 1, 2, 3]]
    hb = batches("gpu")[0]
    try:
        _, src = S.dry_run_multi(A.load_engine(), qs, _plan(qs[0], hb["rows"], zone_map(hb, "exact"), queries=qs))
        kernels = 1
        assert "#define JIT_MDIMS 1" in src
    except A.AresError as e:
        kernels = int(re.search(r"run (\d+) kernels", str(e)).group(1))
    assert kernels == dashboard_kernels()


def dashboard_kernels():
    """Kernels per batch of the dashboard over batches('gpu'): hour of day and day of week cannot index directly (the
    zone map reaches 2^32 - 1; day of week is a Float32 dimension), so each query runs its own kernel."""
    return 4


@pytest.mark.gpu
def test_dashboard_request_on_gpu():
    eng = H.get_backend("b200")
    qs, kinds, names = dashboard()
    bs = [upload(eng, hb, ranges=zone_map(hb, "exact")) for hb in batches("gpu")]
    per_batch, got = MD._run(eng, qs, bs)
    assert [k for k, _ in per_batch] == [dashboard_kernels()] * len(bs), per_batch
    for r, q, kind, name in zip(got, qs, kinds, names):
        AF.assert_matches(r, restate(batches("gpu"), name, "-8", kind=kind), kind, A.Uint16, ctx=f"dashboard {name}")


TIME_FILTERS = {
    # `to` at or above 2^31 is negative in the int32 class: no instant passes
    "to_above_2^31": {"from": "2037-12-31", "to": "2038-01-20"},
    # `to` beyond 2^32 keeps its low 32 bits (1970-01-02 17:31:44), `from` is negative: the first 41 hours of 1970 and
    # every instant from `from` on pass
    "to_beyond_2^32": {"from": "2038-01-20", "to": "2106-02-08"},
    # `from` at or above 2^31 alone (`to` is now): every instant before now, and those from `from` to 2^32 - 1
    "from_above_2^31": {"from": "2038-01-20"},
    # both ends below 2^31: the calendar's answer
    "below_2^31": {"from": "2024-10-20", "to": "2024-11-01"},
}


def time_filter_keep(tf, hb):
    """The reference's time filter: a Uint32 column against a ConstInt literal compares in the common class, int32
    (query/utils.hpp common_type), after the literal kept its low 32 bits: an instant at or above 2^31 is negative."""
    frm, to = aql.parse_time_filter(tf, NOW)
    t = i32(hb["ts"])
    return (t >= i32(frm)) & (t < i32(to))


def test_time_filter_literals_at_the_int32_boundary():
    """What the checkers do with the compiled filters at the int32 boundary (time_filter_keep)."""
    orc = H.get_backend("oracle")
    hbs = batches("cpu")
    counts = {}
    for key, tf in TIME_FILTERS.items():
        q = compile_query("day", "UTC", time_filter=tf)
        keep = [time_filter_keep(tf, hb) for hb in hbs]
        AF.assert_matches(_legacy(orc, q, hbs), restate(hbs, "day", "UTC", keep=keep), "sum", A.Uint16, ctx=key)
        counts[key] = sum(int(k.sum()) for k in keep)
    assert counts["to_above_2^31"] == 0
    frm, to = aql.parse_time_filter(TIME_FILTERS["to_beyond_2^32"], NOW)
    assert counts["to_beyond_2^32"] == sum(int(((hb["ts"] < to - U32) | (hb["ts"] >= frm)).sum()) for hb in hbs) > 0
    frm = aql.parse_time_filter(TIME_FILTERS["from_above_2^31"], NOW)[0]
    assert counts["from_above_2^31"] == sum(int(((hb["ts"] < NOW) | (hb["ts"] >= frm)).sum()) for hb in hbs)
    assert 0 < counts["below_2^31"] < sum(hb["rows"] for hb in hbs)


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(TIME_FILTERS))
def test_time_filter_at_the_int32_boundary_on_gpu(key):
    eng = H.get_backend("b200")
    hbs = batches("gpu")
    keep = [time_filter_keep(TIME_FILTERS[key], hb) for hb in hbs]
    for name in ("day", "month of year", "hour of day"):
        q = compile_query(name, "UTC", time_filter=TIME_FILTERS[key])
        exp = restate(hbs, name, "UTC", keep=keep)
        for how in ("exact", None):
            got = _run(eng, q, [upload(eng, hb, ranges=zone_map(hb, how)) for hb in hbs])
            AF.assert_matches(got, exp, "sum", A.Uint16, ctx=f"{key}/{name}/{how}")
