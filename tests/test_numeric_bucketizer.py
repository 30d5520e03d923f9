"""Numeric bucketizer dimensions (AQL `numericBucketizer`): bucket width, log base and manual partitions on the fused kernel.

The restatement below is built on numpy, `fractions` and torch.bucketize and shares no code with aresdb_b200/aql.py: the
width ordinal is the k with fl(k * w) <= x < fl((k + 1) * w) (fl: one double multiply), found from the exact quotient;
the log ordinal indexes a table [b ** k ...] built here; the partition ordinal is torch.bucketize(x, p, right=True).

CPU: the restatement at its pinned edges, the AQL front-end (compiles, errors, `{}` is a plain dimension), the lower-bound
formatting, and dry runs (AresJitDryRun) that check which form every case reaches, with the digests of the new kernel
texts in tests/golden/numeric_bucket_kernel_sha256.json.  GPU: an edge table of every form on every column type against
the restatement; a four-query request (one pass, and a simulated two-rank exchange); a 2 x 1.25e8-row fare histogram.
"""
from __future__ import annotations

import bisect
import ctypes as C
import gc
import hashlib
import json
import math
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

from aresdb_b200 import aql, cabi as A, columns, expr as E, synth
from aresdb_b200.executor import Batch, FusedBatchExecutor, LegacyBatchExecutor, _BatchPlans
from aresdb_b200.postprocess import DimensionMeta, format_float64, nested_result, read_dimension
from aresdb_b200.query import AggQuery, Measure

GOLDEN = Path(__file__).resolve().parent / "golden" / "numeric_bucket_kernel_sha256.json"
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
F32_MAX = float(np.finfo(np.float32).max)
F32_TINY = float(np.float32(1.4e-45))   # 2^-149


# ---- the restatement ---------------------------------------------------------------------------------------------------
def r_width(x: float, w: float):
    """Int32 k with fl(k * w) <= x < fl((k + 1) * w), or None."""
    if math.isnan(x) or math.isinf(x):
        return None
    k0 = math.floor(Fraction(x) / Fraction(w))
    if not I32_MIN - 2 <= k0 <= I32_MAX + 2:   # (k is k0 or k0 + 1: far outside Int32)
        return None
    for k in (k0 - 1, k0, k0 + 1):
        if float(k) * w <= x < float(k + 1) * w:
            return k if I32_MIN <= k <= I32_MAX else None
    raise AssertionError((x, w))


def r_log_table(b: float, is_float: bool):
    """(kmin, [b ** k for k = kmin ...]) from at most 2^-149 (Float32) or 1 (integers) to beyond FLT_MAX / 2^32."""
    lo, hi = (2.0 ** -149, F32_MAX) if is_float else (1.0, 2.0 ** 32)
    k = 0
    while b ** k > lo:
        k -= 1
    while b ** (k + 1) <= lo:
        k += 1
    t = []
    j = k
    while True:
        try:
            v = b ** j
        except OverflowError:
            v = math.inf
        t.append(v)
        if v > hi:
            return k, t
        j += 1


def r_log(x: float, table):
    if math.isnan(x) or not 0 < x < math.inf:
        return None
    j = bisect.bisect_right(table, x) - 1
    return j if 0 <= j < len(table) - 1 else None


def r_partitions(xs, p):
    import torch
    xs = np.asarray(xs, np.float64)
    out = torch.bucketize(torch.from_numpy(xs), torch.tensor(p, dtype=torch.float64), right=True).numpy()
    return [None if math.isnan(x) else int(o) for x, o in zip(xs, out)]


def restate(spec, xs, is_float):
    """Ordinals (None = NULL) of the doubles xs under an E.Bucket spec."""
    if spec[0] == "width":
        return [r_width(float(x), spec[1]) for x in xs]
    if spec[0] == "log":
        _, t = r_log_table(spec[1], is_float)
        return [r_log(float(x), t) for x in xs]
    return r_partitions(xs, list(spec[1:]))


def r_lower_bound(spec, k, is_float):
    if spec[0] == "width":
        return float(k) * spec[1]
    if spec[0] == "log":
        return r_log_table(spec[1], is_float)[1][k]
    return -math.inf if k == 0 else spec[k]


# ---- CPU: the restatement ----------------------------------------------------------------------------------------------
def test_width_restatement_at_its_edges():
    # floor(x / w) alone is off by one in each direction against the bound definition
    assert math.floor(16.5 / 1.1) == 14 and r_width(16.5, 1.1) == 15
    assert math.floor(93.5 / 1.1) == 85 and r_width(93.5, 1.1) == 84
    # integers: floor division toward -inf, not truncation
    for x, w in ((-7, 2), (-1, 5), (-10, 5), (7, 2), (-2 ** 31, 3), (2 ** 31 - 1, 7)):
        assert r_width(float(x), float(w)) == x // w
    assert r_width(-0.0, 1.0) == 0 and r_width(0.0, 1.0) == 0
    assert r_width(math.inf, 1.0) is None and r_width(math.nan, 1.0) is None
    assert r_width(2.0 ** 40, 1.0) is None and r_width(-(2.0 ** 31), 1.0) == I32_MIN
    # a value exactly on a bound, and its float32 neighbours
    for w in (0.1, 2.5, 1.1):
        for k in (3, 17, -4):
            b = float(k) * w
            f = np.float32(b)
            for x in (f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))):
                x = float(x)
                got = r_width(x, w)
                assert float(got) * w <= x < float(got + 1) * w
            assert r_width(b, w) == k


def test_log_and_partition_restatements():
    k, t = r_log_table(2.0, False)
    assert k == 0 and t[:3] == [1.0, 2.0, 4.0] and t[-1] == 2.0 ** 33 and len(t) == 34
    k, t = r_log_table(10.0, True)
    assert t == [10.0 ** j for j in range(k, k + len(t))] and t[0] <= 2.0 ** -149 < t[1] and t[-2] <= F32_MAX < t[-1]
    assert r_log(1.0, r_log_table(2.0, False)[1]) == 0 and r_log(3.0, r_log_table(2.0, False)[1]) == 1
    assert r_log(0.0, t) is None and r_log(-1.0, t) is None and r_log(math.inf, t) is None
    assert r_log(F32_TINY, t) == 0 and r_log(F32_MAX, t) == len(t) - 2
    p = [-1.0, 0.0, 2.5, 10.0]
    assert r_partitions([-math.inf, -1.0, -0.5, 0.0, -0.0, 2.5, 9.99, 10.0, math.inf, math.nan], p) == \
        [0, 1, 1, 2, 2, 3, 3, 4, 4, None]


def test_log_table_of_the_front_end_equals_the_restatement():
    for b in (2.0, 10.0, 1.5, 1.01, 1e300):
        for is_float in (False, True):
            k, t = aql.log_table(b, is_float)
            assert (k, list(t)) == r_log_table(b, is_float), (b, is_float)
    with pytest.raises(aql.AQLError):
        aql.log_table(1.002, True)


# ---- CPU: AQL ----------------------------------------------------------------------------------------------------------
class FakeBuf:
    def __init__(self, a):
        self.a, self.ptr = a, 0x7D0000000000


TABLE = aql.Table("trips", [aql.Column(n, t) for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)] +
                  [aql.Column("status_name", A.Uint8, enum={"a": 0}), aql.Column("hll", A.Uint32, hll=True),
                   aql.Column("big", A.Int64), aql.Column("id", A.UUID), aql.Column("i32", A.Int32)])


def aql_query(dims, measure="count(*)"):
    return {"table": "trips", "measures": [{"sqlExpression": measure}], "dimensions": dims}


def compile_q(dims, measure="count(*)", mode=A.ARES_REDUCE_SORT, upload=FakeBuf):
    return aql.compile_query(aql_query(dims, measure), TABLE, synth.BASE_TS, mode, upload=upload)


def plan_bytes(q):
    return [bytes(pi) for pi in q.plan_instructions()]


def test_aql_compiles_the_three_forms():
    q = compile_q([{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 5}}])
    d = q.dimensions[0]
    assert isinstance(d, E.Bucket) and d.spec == ("width", 5.0) and q.dim_types == [A.Int32]
    insts = q.plan_instructions()
    assert insts[0].Functor == A.PLAN_FN_NUMERIC_BUCKET and insts[0].Bucket == 0 and insts[0].SinkDataType == A.Int32
    q = compile_q([{"sqlExpression": "city_id", "numericBucketizer": {"logBase": 2}},
                   {"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": [1, 2.5, 10]}}])
    assert q.dim_types == [A.Uint16, A.Uint8]
    assert q.dimensions[0].spec == ("log", 2.0, 0, 34) and q.dimensions[1].spec == ("partitions", 1.0, 2.5, 10.0)
    insts = q.plan_instructions()
    assert [i.Bucket for i in insts if i.Functor == A.PLAN_FN_NUMERIC_BUCKET] == [0, 1] and len(q.bucketizers) == 2
    uploads = []
    q = compile_q([{"sqlExpression": "fare", "numericBucketizer": {"logBase": 10}}], upload=lambda a: uploads.append(a) or FakeBuf(a))
    assert uploads[0].dtype == np.float64 and uploads[0].tolist() == r_log_table(10.0, True)[1]


def test_empty_bucketizer_is_a_plain_dimension():
    plain = compile_q([{"sqlExpression": "fare"}, {"sqlExpression": "city_id"}])
    zero = compile_q([{"sqlExpression": "fare", "numericBucketizer": {}}, {"sqlExpression": "city_id", "numericBucketizer": {}}])
    assert plan_bytes(plain) == plan_bytes(zero) and zero.dim_types == plain.dim_types


@pytest.mark.parametrize("dim", [
    {"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 5, "logBase": 2}},
    {"sqlExpression": "fare", "numericBucketizer": {"logBase": 2, "manualPartitions": [1]}},
    {"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": -1}},
    {"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": "5"}},
    {"sqlExpression": "fare", "numericBucketizer": {"logBase": 0.5}},
    {"sqlExpression": "fare", "numericBucketizer": {"logBase": 1.001}},
    {"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": [2, 1]}},
    {"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": [1, 1]}},
    {"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": list(range(256))}},
    {"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 1, "unknown": 1}},
    {"sqlExpression": "request_at", "timeBucketizer": "hour", "numericBucketizer": {"bucketWidth": 5}},
    {"sqlExpression": "status_name", "numericBucketizer": {"bucketWidth": 5}},
    {"sqlExpression": "hll", "numericBucketizer": {"bucketWidth": 5}},
    {"sqlExpression": "big", "numericBucketizer": {"bucketWidth": 5}},
    {"sqlExpression": "id", "numericBucketizer": {"bucketWidth": 5}},
], ids=lambda d: json.dumps(d["numericBucketizer"])[:40] + d["sqlExpression"])
def test_aql_errors(dim):
    with pytest.raises(aql.AQLError):
        compile_q([dim])


def test_aql_needs_upload_for_bounds_and_legacy_refuses():
    with pytest.raises(aql.AQLError):
        compile_q([{"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": [1]}}], upload=None)
    q = compile_q([{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 5}}], upload=None)
    with pytest.raises(ValueError, match="fused path"):
        LegacyBatchExecutor(None, None, q)


def test_two_widths_never_share_a_dimension():
    a = compile_q([{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 5}}])
    b = compile_q([{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 2}}])
    c = compile_q([{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 5}}], "sum(fare)")
    assert plan_bytes(a) == plan_bytes(b)   # (the instruction names its bucketizer by index)
    assert a.shared_scan_key() != b.shared_scan_key() and a.shared_scan_key() == c.shared_scan_key()
    assert a.shared_scan_key(member_filters=True) != b.shared_scan_key(member_filters=True)
    from aresdb_b200.query import member_dimensions
    union = member_dimensions([a, b])
    assert [d.spec for d, _, _ in union] == [("width", 5.0), ("width", 2.0)]


# ---- CPU: formatting ---------------------------------------------------------------------------------------------------
def test_formatting():
    for v, s in ((-math.inf, "-Inf"), (2.5, "2.5"), (1e6, "1e+06"), (0.1 + 0.2, "0.30000000000000004"), (-3.0, "-3"),
                 (123456.0, "123456"), (1e-5, "1e-05"), (0.0, "0"), (1.5e300, "1.5e+300"), (16.5, "16.5")):
        assert format_float64(v) == s
    meta = lambda spec: DimensionMeta(numeric_bucketizer=spec)
    assert read_dimension(15, True, A.Int32, meta(("width", 1.1))) == "16.5"
    assert read_dimension(-2, True, A.Int32, meta(("width", 0.1))) == "-0.2"
    assert read_dimension(3, True, A.Uint16, meta(("log", 10.0, -45, 85))) == "1e-42"
    assert read_dimension(0, True, A.Uint8, meta(("partitions", 1.0, 2.5))) == "-Inf"
    assert read_dimension(2, True, A.Uint8, meta(("partitions", 1.0, 2.5))) == "2.5"
    assert read_dimension(2, False, A.Uint8, meta(("partitions", 1.0, 2.5))) is None
    for spec, k, f in ((("width", 1.1), 15, False), (("log", 10.0, -45, 85), 3, True), (("partitions", 1.0, 2.5), 1, False)):
        assert aql.bucket_lower_bound(spec, k) == r_lower_bound(spec, k, f)


# ---- CPU: the form every case reaches ----------------------------------------------------------------------------------
FAKE = 0x7F0000000000


def fake_batch(types, rows, ranges=None):
    cols = [columns.slice_of(FAKE + i * (1 << 32), t, rows, 0, 64 * 200 * 4, 2, 0) for i, t in enumerate(types)]
    return Batch(cols, rows, ranges=ranges)


def dry_run(q, batch, expected_groups=0):
    fn = A.load_engine().alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    p = _BatchPlans(q, lambda tf, co: q.plan_instructions(time_filters=tf, cutoff=co)).plan_for(batch, True, 0)
    src = C.c_char_p()
    h = fn(q.agg_spec(expected_groups), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return (src.value or b"").decode()


def form_of(src):
    for line in src.splitlines():
        if line.startswith("#define JIT_DENSE "):
            return {0: "hash", 1: "cta", 2: "global"}[int(line.split()[2])]
    raise AssertionError("no JIT_DENSE")


F100 = int(np.float32(100.0).view(np.uint32))
TYPES5 = [A.Uint32, A.Uint16, A.Int32, A.Float32, A.Uint32]   # request_at, city, i32, fare, v
HOUR = E.floor(E.Col(0, A.Uint32, "request_at"), E.Lit(3600))
DAY0 = synth.BASE_TS


def bucket(col, spec, is_float=False):
    bounds = ()
    if spec[0] == "log":
        bounds = tuple(r_log_table(spec[1], is_float)[1])
        spec = ("log", spec[1], r_log_table(spec[1], is_float)[0], len(bounds))
    elif spec[0] == "partitions":
        bounds = tuple(spec[1:])
    return E.Bucket(col, spec, bounds, 0x7D0000000000 if bounds else 0)


FARE = E.Col(3, A.Float32, "fare")
U32 = E.Col(4, A.Uint32, "v")
I32 = E.Col(2, A.Int32, "i32")
P16 = ("partitions",) + tuple(float(x) for x in range(0, 96, 6))
SHAPES = {
    # name: (dimensions, measure, zone map, rows, expected groups, form)
    "partitions16/fare/zone": ([bucket(FARE, P16, True)], Measure("count"), {3: (0, F100)}, 1_000_000, 0, "cta"),
    "partitions16/fare/none": ([bucket(FARE, P16, True)], Measure("count"), None, 1_000_000, 0, "cta"),
    "partitions16_x_hour/zone": ([HOUR, bucket(FARE, P16, True)], Measure("count"), {0: (DAY0, DAY0 + 86399), 3: (0, F100)},
                                 1_000_000, 0, "cta"),
    "partitions255/sum": ([bucket(FARE, ("partitions",) + tuple(float(x) for x in range(255)), True)], Measure("sum", FARE),
                          None, 1_000_000, 0, "cta"),
    "width/fare/zone": ([bucket(FARE, ("width", 2.5), True)], Measure("sum", FARE), {3: (0, F100)}, 1_000_000, 0, "cta"),
    "width/u32/zone": ([bucket(U32, ("width", 5.0))], Measure("max", U32), {4: (0, 1000)}, 1_000_000, 0, "cta"),
    "width_x_hour/u32": ([HOUR, bucket(U32, ("width", 10.0))], Measure("count"), {0: (DAY0, DAY0 + 86399), 4: (0, 999)},
                         1_000_000, 0, "cta"),
    "width/u32/many": ([bucket(U32, ("width", 1.0))], Measure("count"), {4: (0, 1_000_000)}, 1_000_000, 0, "global"),
    "width/u32/none": ([bucket(U32, ("width", 5.0))], Measure("count"), None, 1_000_000, 0, "hash"),
    "width/i32/negative": ([bucket(I32, ("width", 5.0))], Measure("count"), None, 1_000_000, 0, "hash"),
    "width/u32/bypass": ([bucket(U32, ("width", 5.0))], Measure("count"), None, 1_000_000, 100_000, "hash"),
    "width/u32/tail": ([bucket(U32, ("width", 5.0))], Measure("count"), {4: (0, 1000)}, 900, 0, "hash"),
    "log/u32/zone": ([bucket(U32, ("log", 2.0))], Measure("avg", FARE), {4: (0, 1_000_000)}, 1_000_000, 0, "cta"),
    "log/fare/zone": ([bucket(FARE, ("log", 1.5), True)], Measure("min", FARE), {3: (0, F100)}, 1_000_000, 0, "cta"),
    "log/fare/none": ([bucket(FARE, ("log", 1.5), True)], Measure("count"), None, 1_000_000, 0, "hash"),
}


def shape_sources():
    out = {}
    for name, (dims, m, ranges, rows, eg, _) in SHAPES.items():
        q = AggQuery([], dims, m)
        out[name] = dry_run(q, fake_batch(TYPES5, rows, ranges), eg)
    return out


def test_forms_and_kernel_texts(monkeypatch):
    """Every shape reaches its form; the texts are those recorded (the bucketizers' numbers are not in them)."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    srcs = shape_sources()
    for name, src in srcs.items():
        assert form_of(src) == SHAPES[name][5], name
        assert "numericBucket<" in src, name
    assert "JIT_BYPASS 1" in srcs["width/u32/bypass"]
    assert "jitStageBuckets" in srcs["partitions16/fare/zone"] and "jitStageBuckets" not in srcs["width/u32/zone"]
    # another width / table is the same kernel
    q = AggQuery([], [bucket(U32, ("width", 7.25))], Measure("max", U32))
    assert dry_run(q, fake_batch(TYPES5, 1_000_000, {4: (0, 1000)})) == srcs["width/u32/zone"]
    got = {n: hashlib.sha256(s.encode()).hexdigest() for n, s in srcs.items()}
    assert got == json.loads(GOLDEN.read_text())


def test_new_shapes_compile_for_sm_90a():
    """NVRTC compiles the new shapes (the partition table in shared memory, the log table through L1)."""
    for name in ("partitions16_x_hour/zone", "log/u32/zone", "width/fare/zone", "width/u32/none"):
        dims, m, ranges, rows, eg, _ = SHAPES[name]
        dry_run(AggQuery([], dims, m), fake_batch(TYPES5, rows, ranges), eg)


def test_plan_validation():
    q = AggQuery([], [bucket(U32, ("width", 5.0))], Measure("count"))
    b = fake_batch(TYPES5, 1000)
    fn = A.load_engine().alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle

    def run(mutate):
        p = _BatchPlans(q, lambda tf, co: q.plan_instructions(time_filters=tf, cutoff=co)).plan_for(b, True, 0)
        mutate(p)
        os.environ["ARESDB_B200_JIT_GENERATE_ONLY"] = "1"
        try:
            h = fn(q.agg_spec(), C.byref(p), C.byref(C.c_char_p()))
        finally:
            del os.environ["ARESDB_B200_JIT_GENERATE_ONLY"]
        return C.string_at(h.pStrErr).decode() if h.pStrErr else None

    import os
    assert run(lambda p: None) is None
    assert "outside BatchPlan.Bucketizers" in run(lambda p: setattr(p.Insts[0], "Bucket", 1))
    assert "width" in run(lambda p: setattr(p.Bucketizers[0], "Param", -1.0))
    assert "unknown kind" in run(lambda p: setattr(p.Bucketizers[0], "Kind", 9))
    assert "Int32 (width)" in run(lambda p: setattr(p.Insts[0], "SinkDataType", A.Uint16))
    assert "number of numeric bucketizers" in run(lambda p: setattr(p, "NumBucketizers", 5))

    def log_bad(p):
        p.Bucketizers[0].Kind, p.Bucketizers[0].Param, p.Bucketizers[0].NumBounds = A.PLAN_BUCKET_LOG, 2.0, 70000
        p.Bucketizers[0].Bounds = FAKE
    assert "log table" in run(log_bad)

    def part_bad(p):
        p.Bucketizers[0].Kind, p.Bucketizers[0].NumBounds, p.Bucketizers[0].Bounds = A.PLAN_BUCKET_PARTITIONS, 0, FAKE
    assert "manual partitions" in run(part_bad)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
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


NP = {A.Int8: np.int8, A.Int16: np.int16, A.Int32: np.int32, A.Uint8: np.uint8, A.Uint16: np.uint16, A.Uint32: np.uint32,
      A.Float32: np.float32}
COL_TYPES = list(NP)


def edge_values(dt, nonneg):
    """Bounds and their neighbours, zeros, negatives, denormals, extremes, infinities and NaN that the type holds."""
    base = [0.0, -0.0, 1.0, 2.0, 2.5, 3.0, 4.0, 5.0, 6.0, 9.99, 10.0, 15.0, 16.5, 93.5, 100.0, 127.0, 255.0, 1000.0, 65535.0,
            2.0 ** 31 - 1, 2.0 ** 32 - 1, -1.0, -2.5, -5.0, -6.0, -128.0, -(2.0 ** 31), 1e-45, 1.2e-38, F32_MAX, -F32_MAX,
            math.inf, -math.inf, math.nan, 0.1, 0.7, 1.1]
    for b in (1.0, 2.5, 6.0, 10.0, 1.5 ** 5, 16.5):
        f = np.float32(b)
        base += [float(np.nextafter(f, np.float32(np.inf))), float(np.nextafter(f, np.float32(-np.inf)))]
    out = []
    for v in base:
        if nonneg and not (v >= 0 and v < math.inf) or (nonneg and math.copysign(1, v) < 0):
            continue
        if dt == A.Float32:
            out.append(np.float32(v))
        elif math.isfinite(v) and v == math.floor(v) and np.iinfo(NP[dt]).min <= v <= np.iinfo(NP[dt]).max:
            out.append(NP[dt](v))
    return np.unique(np.array(out, NP[dt]))


def edge_batch(dt, nonneg, rows, seed):
    """Values drawn from the edge list (every quad position sees every value), the whole list at the start, around the
    first tile boundaries, at the end (the tail); ~3 % NULL rows that hold an edge value underneath."""
    rng = np.random.default_rng(seed)
    ev = edge_values(dt, nonneg)
    x = ev[rng.integers(0, len(ev), rows)]
    for at in (0, 896 - 3, 1920 - 5, 3968 - 7, 2 * 3968 - 2, rows - len(ev)):
        if 0 <= at and at + len(ev) <= rows:
            x[at:at + len(ev)] = ev
    valid = rng.random(rows) > 0.03
    valid[:len(ev)] = True
    v = rng.integers(0, 1000, rows).astype(np.uint32)
    return {"x": x, "valid": valid, "v": v, "rows": rows}


def expected_groups(spec, hbs, dt, kind):
    is_float = dt == A.Float32
    acc = {}
    for hb in hbs:
        xs = hb["x"].astype(np.float64)
        ords = restate(spec, xs, is_float)
        for o, ok, v in zip(ords, hb["valid"], hb["v"].tolist()):
            key = o if ok else None
            a = acc.setdefault(key, [0, 0, None, None])
            a[0] += 1
            a[1] += v
            a[2] = v if a[2] is None else min(a[2], v)
            a[3] = v if a[3] is None else max(a[3], v)
    idx = {"count": 0, "sum": 1, "min": 2, "max": 3}
    if kind == "avg":
        return {k: a[1] / a[0] for k, a in acc.items()}
    return {k: a[idx[kind]] for k, a in acc.items()}


def got_groups(r, kind):
    dims = r.decoded_dims()[0]
    out = {d: float(m) if kind == "avg" else int(m) for d, m in zip(dims, r.measures.tolist())}
    assert len(out) == r.groups
    return out


def _upload(eng, hb, dt, ranges):
    xb, xvp = columns.make_column(eng.space, dt, hb["x"], valid=hb["valid"])
    vb, vvp = columns.make_column(eng.space, A.Uint32, hb["v"])
    return Batch([xvp, vvp], hb["rows"], keep=[xb, vb], ranges=ranges)


def zone_map(eng, b, how):
    from aresdb_b200.executor import compute_zone_map
    zm = compute_zone_map(eng.lib, eng.space, b.columns[:1])
    if how is None or 0 not in zm:
        return None
    lo, hi = zm[0]
    return {"exact": {0: (lo, hi)}, "narrow": {0: (lo, lo + (hi - lo) // 2)}, "stale": {0: (lo + (hi - lo) // 3 + 1, hi + (hi - lo))}}[how]


SPECS = {"width": [("width", 2.5), ("width", 1.1), ("width", 3.0)], "log": [("log", 2.0), ("log", 10.0)],
         "partitions": [("partitions", -5.0, -1.0, 0.0, 1.0, 2.5, 6.0, 10.0, 16.5, 100.0, 2.0 ** 31 - 1)]}
KINDS = ["count", "sum", "min", "max", "avg"]


def _run(eng, q, bs, eg=0):
    ex = FusedBatchExecutor(eng.lib, eng.space, q, eg)
    for b in bs:
        ex.process_batch(b)
    r = ex.result()
    ex.close()
    return r


def _compare(got, exp, kind, ctx):
    assert set(got) == set(exp), f"{ctx}: groups {sorted(got, key=repr)[:8]} vs {sorted(exp, key=repr)[:8]}"
    for k in exp:
        if kind == "avg":
            assert abs(got[k] - exp[k]) <= 1e-4 * max(1.0, abs(exp[k])), f"{ctx}: {k}: {got[k]} vs {exp[k]}"
        else:
            assert got[k] == exp[k], f"{ctx}: {k}: {got[k]} vs {exp[k]}"


@pytest.mark.gpu
@pytest.mark.parametrize("dt", COL_TYPES, ids=lambda d: {v: k for k, v in vars(A).items() if k in
                                                         ("Int8", "Int16", "Int32", "Uint8", "Uint16", "Uint32", "Float32")}[d])
def test_edge_table_on_gpu(dt):
    """Every form of every kind on one column type: edge values at every quad position, first full tiles and the tail,
    NULL rows with values underneath; exact / narrow / stale / absent zone maps; both reduce modes; count, sum, min, max,
    avg by the bucket."""
    import harness as H
    import test_pipeline_parity as T
    eng = H.get_backend("b200")
    n = 0
    for nonneg in (False, True):
        hbs = [edge_batch(dt, nonneg, rows, 11 + i + 7 * nonneg) for i, rows in enumerate((60_013, 20_001))]
        plain = [_upload(eng, hb, dt, None) for hb in hbs]
        for form, specs in SPECS.items():
            for spec in specs:
                b = bucket(E.Col(0, dt, "x"), spec, dt == A.Float32)
                keep = [eng.space.put(np.array(b.bounds, np.float64))] if b.bounds else []
                if keep:
                    b = E.Bucket(b.expr, b.spec, b.bounds, keep[0].ptr, keep[0])
                for how in ("exact", "narrow", "stale", None):
                    kind = KINDS[n % len(KINDS)]
                    mode = (A.ARES_REDUCE_SORT, A.ARES_REDUCE_HASH)[n % 2]
                    n += 1
                    m = Measure("count") if kind == "count" else Measure(kind, E.Col(1, A.Uint32, "v"))
                    q = AggQuery([], [b], m, reduce_mode=mode)
                    bs = [Batch(p.columns, p.num_rows, keep=p.keep, ranges=zone_map(eng, p, how)) for p in plain]
                    ctx = f"{dt}/{spec[:2]}/nonneg={nonneg}/{how}/{kind}/mode{mode}"
                    d0 = T.dense_launches(eng)
                    got = got_groups(_run(eng, q, bs), kind)
                    _compare(got, expected_groups(spec, hbs, dt, kind), kind, ctx)
                    if form == "partitions":
                        assert T.dense_launches(eng) - d0 == len(bs), f"{ctx}: direct-indexed launches"
                # bypass, and a mode-0 (constant) column
                q = AggQuery([], [b], Measure("count"))
                _compare(got_groups(_run(eng, q, plain, 100_000), "count"), expected_groups(spec, hbs, dt, "count"), "count",
                         f"{dt}/{spec[:2]}/bypass")
                c = hbs[0]["x"][5]
                const = Batch([columns.constant_column(dt, c.item()), plain[0].columns[1]], hbs[0]["rows"], keep=plain[0].keep)
                got = got_groups(_run(eng, q, [const]), "count")
                o = restate(spec, [float(c)], dt == A.Float32)[0]
                assert got == {o: hbs[0]["rows"]}, f"{dt}/{spec[:2]}/mode-0 {c}"


@pytest.mark.gpu
def test_rle_column_on_gpu():
    """A run-length encoded (archive) column under each form."""
    import harness as H
    eng = H.get_backend("b200")
    rng = np.random.default_rng(5)
    runs = 3000
    vals = rng.integers(0, 200, runs).astype(np.uint32)
    lens = rng.integers(1, 40, runs)
    counts = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    rows = int(counts[-1])
    xb, xvp = columns.make_column(eng.space, A.Uint32, vals, valid=np.ones(runs, bool), counts=counts)
    full = np.repeat(vals, lens)
    v = rng.integers(0, 1000, rows).astype(np.uint32)
    vb, vvp = columns.make_column(eng.space, A.Uint32, v)
    batch = Batch([xvp, vvp], rows, keep=[xb, vb], ranges={0: (0, 199)})
    hb = {"x": full, "valid": np.ones(rows, bool), "v": v, "rows": rows}
    for spec in (("width", 7.0), ("log", 2.0), ("partitions", 3.0, 50.0, 150.0)):
        b = bucket(E.Col(0, A.Uint32, "x"), spec)
        keep = [eng.space.put(np.array(b.bounds, np.float64))] if b.bounds else []
        if keep:
            b = E.Bucket(b.expr, b.spec, b.bounds, keep[0].ptr, keep[0])
        for kind in ("count", "sum"):
            m = Measure("count") if kind == "count" else Measure("sum", E.Col(1, A.Uint32, "v"))
            got = got_groups(_run(eng, AggQuery([], [b], m), [batch]), kind)
            _compare(got, expected_groups(spec, [hb], A.Uint32, kind), kind, f"rle/{spec[:2]}/{kind}")


REQUEST = {"queries": [
    {"table": "trips", "measures": [{"sqlExpression": "count(*)"}],
     "dimensions": [{"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": [5, 10, 20, 40, 80]}}]},
    {"table": "trips", "measures": [{"sqlExpression": "sum(fare)"}],
     "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "hour"},
                    {"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": [5, 10, 20, 40, 80]}}]},
    {"table": "trips", "measures": [{"sqlExpression": "max(fare)"}], "dimensions": [{"sqlExpression": "city_id"}]},
    {"table": "trips", "measures": [{"sqlExpression": "count(*)"}],
     "dimensions": [{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 12.5}}]},
]}


@pytest.mark.gpu
def test_request_in_one_pass_and_exchange_on_gpu():
    """Four queries grouping by a bucket, by hour x bucket, by city and by a width bucket: one pass of
    FusedRequestExecutor and the simulated two-rank exchange give each query its own FusedBatchExecutor result."""
    import harness as H
    import test_pipeline_parity as T
    import test_shared_scan as S
    import test_sharded_request as SR
    from aresdb_b200.executor import FusedRequestExecutor
    eng = H.get_backend("b200")
    qs = aql.compile_request(REQUEST, TABLE, synth.BASE_TS, upload=eng.space.put)
    hbs = [synth.generate_batch(d, 30000, num_cities=30) for d in range(4)]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs]
    full = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert len(full.passes) == 1, full.passes
    d0 = T.dense_launches(eng)
    for b in batches:
        full.process_batch(b)
    assert full.calls == len(batches) and T.dense_launches(eng) - d0 == len(batches)
    got = full.results()
    for q, g in zip(qs, got):
        S._same(g, _run(eng, q, batches), q, "request")
    # the histogram itself against the restatement
    fare = np.concatenate([hb.values[synth.COL_FARE] for hb in hbs]).astype(np.float64)
    valid = np.concatenate([hb.valid[synth.COL_FARE] for hb in hbs]).astype(bool)
    ords = np.array(r_partitions(fare, [5, 10, 20, 40, 80]))
    exp = {int(k): int(c) for k, c in zip(*np.unique(ords[valid], return_counts=True))}
    if (~valid).any():
        exp[None] = int((~valid).sum())
    assert got_groups(got[0], "count") == exp
    nested = nested_result(got[0])
    assert set(nested) == {"-Inf", "5", "10", "20", "40", "80"} | ({"NULL"} if (~valid).any() else set())
    locals_ = [FusedRequestExecutor(eng.lib, eng.space, qs) for _ in range(2)]
    for i, b in enumerate(batches):
        locals_[i % 2].process_batch(b)
    xqs, out = SR._exchange_on_one_device(eng, locals_, 32768, (1,))
    SR._check_exchange(xqs, out, got, 32768, "numeric bucket request")


@pytest.mark.gpu
def test_fare_histograms_at_scale():
    """2 x 1.25e8 rows: count(*) by 16 fare partitions x hour, and by a fare width, against a torch restatement."""
    import torch
    import harness as H
    eng = H.get_backend("b200")
    dev = eng.space.dev
    rows = 125_000_000
    parts = [float(x) for x in range(0, 96, 6)]
    hp = torch.tensor(parts, dtype=torch.float64, device=dev)
    q1 = aql.compile_query({"table": "trips", "measures": [{"sqlExpression": "count(*)"}],
                            "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "hour"},
                                           {"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": parts}}]},
                           TABLE, synth.BASE_TS, upload=eng.space.put)
    q2 = aql.compile_query({"table": "trips", "measures": [{"sqlExpression": "count(*)"}],
                            "dimensions": [{"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 0.7}}]},
                           TABLE, synth.BASE_TS, upload=eng.space.put)
    ex1, ex2 = FusedBatchExecutor(eng.lib, eng.space, q1), FusedBatchExecutor(eng.lib, eng.space, q2)
    from aresdb_b200.executor import compute_zone_map
    exp1, exp2, keep = {}, {}, []
    bits = torch.arange(8, device=dev, dtype=torch.uint8)

    def column(bufs, off, c, dtype):
        valid = ((bufs[c][:(rows + 7) // 8].unsqueeze(1) >> bits) & 1).reshape(-1)[:rows].bool()
        return bufs[c][off:off + rows * dtype.itemsize].view(dtype), valid

    for d in range(2):
        bufs, off = synth.generate_batch_cuda(d, rows, dev, exact_fares=False)
        cols = [columns.slice_of(t.data_ptr(), dt, rows, 0, off, 2) for t, dt in zip(bufs, synth.COLUMN_TYPES)]
        b = Batch(cols, rows, keep=bufs, ranges=compute_zone_map(eng.lib, eng.space, cols))
        keep.append(b)
        ex1.process_batch(b)
        ex2.process_batch(b)
        ts, ok_ts = column(bufs, off, synth.COL_REQUEST_AT, torch.int32)
        fare, ok = column(bufs, off, synth.COL_FARE, torch.float32)
        f64 = fare.to(torch.float64)
        key = (ts.to(torch.int64) // 3600) * 64 + torch.bucketize(f64, hp, right=True)
        for kk, c in zip(*[t.tolist() for t in torch.unique(key[ok & ok_ts], return_counts=True)]):
            exp1[(kk // 64 * 3600, kk % 64)] = exp1.get((kk // 64 * 3600, kk % 64), 0) + c
        k = torch.floor(f64 / 0.7)
        k = torch.where(k * 0.7 > f64, k - 1, torch.where((k + 1) * 0.7 <= f64, k + 1, k)).to(torch.int64)
        for kk, c in zip(*[t.tolist() for t in torch.unique(k[ok], return_counts=True)]):
            exp2[kk] = exp2.get(kk, 0) + c
        del ts, fare, f64, key, k
    r1, r2 = ex1.result(), ex2.result()
    d1 = r1.decoded_dims()
    got1 = {(h, p): int(m) for h, p, m in zip(d1[0], d1[1], r1.measures.tolist()) if h is not None and p is not None}
    assert got1 == exp1
    assert {k: v for k, v in got_groups(r2, "count").items() if k is not None} == exp2
