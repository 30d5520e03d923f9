"""Queries of one AQL request that share filters and dimensions, run in one pass over the batches.

CPU: the generated text of every single-measure plan shape is unchanged (SHA-256 recorded before the multi-measure
form existed), multi-measure plans of the cfg3 shape compile for sm_90a, and FusedRequestExecutor groups exactly the
compatible queries.  GPU: every query of a request equals the same query run alone on FusedBatchExecutor."""
import ctypes as C
import hashlib
import json
from pathlib import Path

import numpy as np
import pytest

from aresdb_b200 import cabi as A
from aresdb_b200 import columns, synth
from aresdb_b200 import expr as E
from aresdb_b200.query import AggQuery, Measure
import test_jit_codegen as J
import test_pipeline_parity as T

GOLDEN = Path(__file__).resolve().parent / "golden" / "single_measure_kernel_sha256.json"
ALIGNED_BC = 0x7E0000000000


def single_measure_shapes():
    """name -> (query, dry-run keyword arguments): every plan shape the codegen and parity suites build."""
    import harness as H
    import test_hll_pipeline as HP
    import test_joins as TJ
    wide = dict(J.DAY_RANGES)
    wide[synth.COL_CITY_ID] = (0, 65535)
    range_sets = {"none": None, "day": J.DAY_RANGES, "day_fare": {**J.DAY_RANGES, **J.FARE_RANGE}, "wide": wide}
    shapes = {}
    suites = {**T.queries(), **T.avg_queries()}
    q = T.queries()["cfg3_sum"]
    suites["doubled_fare"] = AggQuery(q.filters, [E.floor(T.TS, E.Lit(3600)), T.CITY], Measure("sum", E.mul(T.FARE, E.Lit(2.0))))
    suites["wide_int"] = AggQuery(q.filters, [E.floor(T.TS, E.Lit(3600)), T.CITY], Measure("sum", T.CITY))
    suites["wide_count"] = AggQuery(q.filters, [E.floor(T.TS, E.Lit(3600)), T.CITY], Measure("count"))
    suites["ts_city_count"] = AggQuery([], [T.TS, T.CITY], Measure("count"))
    for name, qq in suites.items():
        for rname, r in range_sets.items():
            shapes[f"{name}/{rname}"] = (qq, {"ranges": r})
        shapes[f"{name}/rle"] = (qq, {"base_counts": ALIGNED_BC})
        shapes[f"{name}/rle_day"] = (qq, {"base_counts": ALIGNED_BC, "ranges": J.DAY_RANGES})
        shapes[f"{name}/bypass"] = (qq, {"expected_groups": 100000})
    for name, qq in HP.hll_queries().items():
        shapes[f"hll_{name}/entry"] = (qq, {"expected_groups": 100000})
        shapes[f"hll_{name}/dense"] = (qq, {})
        shapes[f"hll_{name}/day"] = (qq, {"ranges": J.DAY_RANGES})
    orc = H.get_backend("oracle")
    table, _ = TJ._dimension_table(orc)
    for name, qq in TJ.join_queries(table, 0x7E0000000000, 12).items():
        shapes[f"join_{name}/none"] = (qq, {})
        shapes[f"join_{name}/day"] = (qq, {"ranges": J.DAY_RANGES})
    shapes["_keep"] = (table, {})
    return shapes


def shape_digests(lib):
    out = {}
    for name, (q, kw) in single_measure_shapes().items():
        if name == "_keep":
            continue
        _, src = J._dry_run(lib, q, **kw)
        out[name] = hashlib.sha256(src.encode()).hexdigest()
    return out


def test_single_measure_kernel_text_is_unchanged(monkeypatch):
    """The generated text of every single-measure shape is byte-identical to what it was before plans could carry
    several measures: the kernels bench.py and the rest of the suite run are the same kernels."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    got = shape_digests(A.load_engine())
    want = json.loads(GOLDEN.read_text())
    assert sorted(got) == sorted(want)
    changed = [n for n in want if got[n] != want[n]]
    assert not changed, f"generated text changed for {changed}"


def cfg3_request(k):
    """k queries of one dashboard panel over the cfg3 slice: the first k of sum(fare) (exact-integer form), count(*),
    avg(fare), max(city_id)."""
    q = T.queries()["cfg3_sum"]
    dims = [E.floor(T.TS, E.Lit(3600)), T.CITY]
    measures = [Measure("sum", T.FARE), Measure("count"), Measure("avg", T.FARE), Measure("max", T.CITY)]
    return [AggQuery(q.filters, dims, m) for m in measures[:k]]


def shared_plan(queries, rows=100000, ranges=None, base_counts=None):
    """The BatchPlan of a group over fake, aligned device addresses (nothing is dereferenced)."""
    p = A.BatchPlan()
    insts = queries[0].plan_instructions(measures=queries)
    p.NumInsts = len(insts)
    for i, pi in enumerate(insts):
        p.Insts[i] = pi
    p.NumColumns = len(synth.COLUMN_TYPES)
    for i, dt in enumerate(synth.COLUMN_TYPES):
        p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, rows, 0, 64 * 200, 2, 0)
    p.NumRows = rows
    if base_counts is not None:
        p.BaseCounts = base_counts
    for col, (lo, hi) in (ranges or {}).items():
        p.Ranges[col].Known, p.Ranges[col].Min, p.Ranges[col].Max = 1, lo, hi
    return p


def dry_run_multi(lib, queries, plan, specs=None):
    fn = lib.alg.AresJitDryRunMulti
    fn.argtypes = [C.POINTER(A.AggSpec), C.c_int, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    specs = specs or [q.agg_spec() for q in queries]
    arr = (A.AggSpec * len(specs))(*specs)
    src = C.c_char_p()
    h = fn(arr, len(specs), C.byref(plan), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return int(h.res or 0), (src.value or b"").decode()


CFG3_RANGES = synth.zone_map_of_day(0)


@pytest.mark.parametrize("k", [2, 3, 4])
def test_cfg3_requests_compile_in_the_shared_form(k):
    """K measures of the cfg3 shape: one kernel; each measure keeps the form it takes alone (sum(fare): exact integers,
    count(*): flag-less 32-bit adds, avg: split CAS / RED, max of an integer column: flagged 32-bit atomics)."""
    lib = A.load_engine()
    qs = cfg3_request(k)
    size, src = dry_run_multi(lib, qs, shared_plan(qs, rows=125_000_000, ranges=CFG3_RANGES))
    assert size > 0 and f"#define JIT_NMEAS {k}" in src and "#define JIT_DENSE 1" in src
    acc = {2: "{4, 1}", 3: "{4, 1, 2}", 4: "{4, 1, 2, 1}"}[k]
    assert f"kMeasAcc[JIT_NMEAS] = {acc};" in src
    # rows are evaluated once: the filters appear once, every measure has its own root
    assert src.count("if (!__any_sync(__activemask(), al[0]") == 2          # rowEval and rowEvalGeneric
    for m in range(1, k):
        assert f"meas{m}[r]" in src


def test_one_state_is_the_single_measure_kernel(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    q = T.queries()["cfg3_sum"]
    plan = shared_plan([q], ranges=CFG3_RANGES)
    assert dry_run_multi(lib, [q], plan)[1] == J._dry_run(lib, q, ranges=CFG3_RANGES)[1]


def test_shared_form_needs_every_measure_direct_indexed(monkeypatch):
    """No zone map, too many slots for K measures, or a batch that is all tail: each state runs its own kernel."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    qs = cfg3_request(2)
    for plan in (shared_plan(qs), shared_plan(qs, rows=3000, ranges=CFG3_RANGES)):
        with pytest.raises(A.AresError, match="one kernel per state"):
            dry_run_multi(lib, qs, plan)
    # 25 hour buckets x 300 cities (7,826 slots with the NULL ones) fit a CTA for each measure alone and for two, not for four
    wide = dict(CFG3_RANGES)
    wide[synth.COL_CITY_ID] = (1, 300)
    q4 = cfg3_request(4)
    for q in q4:
        assert "#define JIT_DENSE 1" in J._dry_run(lib, q, ranges=wide)[1]
    assert "#define JIT_NMEAS 2" in dry_run_multi(lib, qs, shared_plan(qs, ranges=wide))[1]
    with pytest.raises(A.AresError, match="one kernel per state"):
        dry_run_multi(lib, q4, shared_plan(q4, ranges=wide))


def test_plan_errors_are_reported(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    qs = cfg3_request(2)
    plan = shared_plan(qs, ranges=CFG3_RANGES)
    specs = [q.agg_spec() for q in qs]
    with pytest.raises(A.AresError, match="numSpecs must be 1..4"):
        dry_run_multi(lib, qs * 3, shared_plan(qs * 3, ranges=CFG3_RANGES))
    last = plan.NumInsts - 1
    plan.Insts[last].SinkArg = 0
    with pytest.raises(A.AresError, match="duplicate SinkArg"):
        dry_run_multi(lib, qs, plan)
    plan.Insts[last].SinkArg = 2
    with pytest.raises(A.AresError, match="SinkArg 2"):
        dry_run_multi(lib, qs, plan)
    plan.NumInsts = last
    with pytest.raises(A.AresError, match="missing SinkArg"):
        dry_run_multi(lib, qs, plan)
    plan = shared_plan(qs, ranges=CFG3_RANGES)
    with pytest.raises(A.AresError, match="MeasureDataType"):
        dry_run_multi(lib, qs, plan, specs=specs[::-1])


def test_grouping_of_a_request():
    """The reference's example pair (total_fare.aql / total_trips.aql: same table, filter, time filter and hour
    bucketizer) groups; a different filter literal, time range, dimension, join, reduce mode or an HLL measure does not."""
    from aresdb_b200.executor import shared_scan_groups
    from aresdb_b200.query import Join
    t0 = synth.BASE_TS
    dims = [E.floor(T.TS, E.Lit(3600)), T.CITY]
    base = [E.eq(T.STATUS, E.Lit(1))]
    tf = [E.ge(T.TS, E.Lit(t0)), E.lt(T.TS, E.Lit(t0 + 86400))]
    def q(m, filters=base, d=dims, time=tf, **kw):
        return AggQuery(filters, d, m, time_filters=time, **kw)
    fare, trips = q(Measure("sum", T.FARE)), q(Measure("count"))
    assert shared_scan_groups([fare, trips]) == [[0, 1]]
    others = [q(Measure("count"), filters=[E.eq(T.STATUS, E.Lit(2))]),
              q(Measure("count"), time=[E.ge(T.TS, E.Lit(t0)), E.lt(T.TS, E.Lit(t0 + 7200))]),
              q(Measure("count"), d=[E.floor(T.TS, E.Lit(60)), T.CITY]),
              q(Measure("count"), reduce_mode=A.ARES_REDUCE_HASH),
              q(Measure("countdistincthll", T.CITY)),
              q(Measure("countdistincthll", T.CITY)),
              q(Measure("count"), joins=[Join(object(), T.CITY)])]
    groups = shared_scan_groups([fare] + others + [trips])
    assert groups == [[0, len(others) + 1]] + [[i] for i in range(1, len(others) + 1)]
    # at most four per group, in request order
    many = [q(Measure(k, T.FARE)) for k in ("sum", "min", "max", "avg", "sum", "min")]
    assert shared_scan_groups(many) == [[0, 1, 2, 3], [4, 5]]
    # one query's plan is what it was; a group's plan ends with one measure root per query, SinkArg = its ordinal
    assert [bytes(i) for i in fare.plan_instructions(measures=[fare])] == [bytes(i) for i in fare.plan_instructions()]
    roots = [i for i in fare.plan_instructions(measures=[fare, trips]) if i.Sink == A.PLAN_SINK_MEASURE]
    assert [r.SinkArg for r in roots] == [0, 1]


# ---- on the GPU: every query of a request equals the same query run alone --------------------------------------------
def _same(got, exp, q, ctx):
    """Bit-identical (counts, integer sums, min / max, float sums on the 1/64 grid of the synthetic fares); AVG: counts
    exact, averages to the tolerance of tests/test_pipeline_parity.py (the rolling float average depends on row order)."""
    if q.agg_func == A.AGGR_AVG_FLOAT:
        g = {r: (c, m) for r, c, m in zip(got.rows, got.counts.tolist(), got.measures.tolist())}
        e = {r: (c, m) for r, c, m in zip(exp.rows, exp.counts.tolist(), exp.measures.tolist())}
        assert g.keys() == e.keys(), f"{ctx}: groups differ"
        assert [g[r][0] for r in e] == [e[r][0] for r in e], f"{ctx}: counts differ"
        np.testing.assert_allclose([g[r][1] for r in e], [e[r][1] for r in e], rtol=2e-5, atol=1e-6, err_msg=ctx)
    elif q.agg_func in (A.AGGR_MIN_FLOAT, A.AGGR_MAX_FLOAT):
        # the minimum of +0.0 and -0.0 is whichever an atomic meets first, in a solo run as much as in a shared one
        assert got.rows == exp.rows if q.reduce_mode == A.ARES_REDUCE_SORT else sorted(got.rows) == sorted(exp.rows), ctx
        g, e = got.as_dict(), exp.as_dict()
        assert all(g[r] == e[r] for r in e), f"{ctx}: measures differ"
    else:
        T.assert_same_result(got, exp, ordered=q.reduce_mode == A.ARES_REDUCE_SORT, ctx=ctx)


def _launches(eng):
    return eng.lib.kernel_launch_count(), T.dense_launches(eng)


def _request_vs_solo(eng, qs, batches, expected_groups=0):
    """batches: executor.Batch objects.  Runs the request on FusedRequestExecutor and every query alone; returns the
    (kernel launches, direct-indexed launches) of the request per batch."""
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    req = FusedRequestExecutor(eng.lib, eng.space, qs, expected_groups)
    solos = [FusedBatchExecutor(eng.lib, eng.space, q, expected_groups) for q in qs]
    per_batch = []
    for b in batches:
        k0, d0 = _launches(eng)
        req.process_batch(b)
        k1, d1 = _launches(eng)
        per_batch.append((k1 - k0, d1 - d0))
        for ex in solos:
            ex.process_batch(b)
    got = req.results()
    for i, (q, ex) in enumerate(zip(qs, solos)):
        _same(got[i], ex.result(), q, f"query {i} ({q.measure_kind})")
    req.close()
    for ex in solos:
        ex.close()
    return per_batch, got


def _cfg3_queries(reduce_mode, days=2):
    import test_at_size as AS
    q = AS._queries(days)["cfg3"]
    dims = [E.floor(T.TS, E.Lit(3600)), T.CITY]
    ms = [Measure("sum", T.FARE), Measure("count"), Measure("avg", T.FARE), Measure("max", T.CITY)]
    return [AggQuery(q.filters, dims, m, reduce_mode=reduce_mode) for m in ms]


@pytest.mark.gpu
@pytest.mark.parametrize("reduce_mode", [A.ARES_REDUCE_SORT, A.ARES_REDUCE_HASH], ids=["sort", "hash"])
@pytest.mark.parametrize("city_dist", ["uniform", "zipf"])
def test_cfg3_request_at_scale_equals_solo_runs(city_dist, reduce_mode):
    """2 x 1.25e8 rows with zone maps: one fused launch per batch feeds the four states, and each query equals its solo
    run; sum(fare) also equals tests/independent.py."""
    import torch
    import harness as H
    import independent as I
    import test_at_size as AS
    from aresdb_b200.executor import Batch
    eng, dev, rows = H.get_backend("b200"), torch.device("cuda:0"), AS.BATCH_ROWS
    t0 = synth.BASE_TS
    exp = I.Expected("cfg3", 2, dev, t0, t0 + 1800, t0 + 2 * 86400 - 1800)
    qs = _cfg3_queries(reduce_mode)

    def batches():
        for d in range(2):
            bufs, voff, cols = AS._batch(d, rows, dev, city_dist=city_dist)
            exp.add_batch(bufs, voff, rows)
            yield Batch(cols, rows, ranges=synth.zone_map_of_day(d), keep=[bufs])

    per_batch, got = _request_vs_solo(eng, qs, batches())
    assert per_batch == [(1, 1), (1, 1)], per_batch
    if reduce_mode == A.ARES_REDUCE_SORT:
        assert exp.check(got[0])["groups"] == 2 * 24 * 100


def _edge_batches(eng, n=200_000, days=2, zone_maps="exact"):
    """NULL fares and cities, -0.0 and +0.0 fares, one city whose fares are all zero (its sums are 0)."""
    out = []
    for d in range(days):
        hb = synth.generate_batch(d, n, num_cities=100, null_rate=0.05)
        fare, city = hb.values[3], hb.values[1]
        fare[::97] = -0.0
        fare[5::89] = 0.0
        fare[city == 7] = 0.0
        zm = {"exact": synth.zone_map(hb), "stale": synth.zone_map_of_day(days - 1 - d), "narrow": {**synth.zone_map(hb), 1: (1, 10)},
              "none": None}[zone_maps]
        out.append(T.upload(eng, hb, 0, zm))
    return out


def _status_queries(reduce_mode=A.ARES_REDUCE_SORT):
    """No filter on fare: NULL / zero / -0.0 fares reach the measures (split CAS / RED float sum, flagged integer sum)."""
    dims = [E.floor(T.TS, E.Lit(3600)), T.CITY]
    f = [E.eq(T.STATUS, E.Lit(1))]
    return [AggQuery(f, dims, m, reduce_mode=reduce_mode)
            for m in (Measure("sum", T.FARE), Measure("count"), Measure("sum", T.CITY), Measure("min", T.FARE))]


@pytest.mark.gpu
@pytest.mark.parametrize("zone_maps", ["exact", "stale", "narrow"])
@pytest.mark.parametrize("request_of", ["cfg3", "status"])
def test_edge_inputs_equal_solo_runs(request_of, zone_maps):
    """Rows outside a too-narrow or stale zone map take every state's cold path; NULL and -0.0 measures and groups whose
    sum is 0 keep the flag / neutral-value rules of each measure."""
    import harness as H
    eng = H.get_backend("b200")
    qs = _cfg3_queries(A.ARES_REDUCE_SORT, days=2) if request_of == "cfg3" else _status_queries()
    per_batch, got = _request_vs_solo(eng, qs, _edge_batches(eng, zone_maps=zone_maps))
    assert all(p == (1, 1) for p in per_batch), per_batch
    if request_of == "status":
        zero = [v for v, c in zip(got[0].measures.tolist(), got[0].decoded_dims()[1]) if c == 7]
        assert zero and all(v == 0.0 for v in zero)


@pytest.mark.gpu
def test_out_of_range_rows_claiming_many_groups_spill_per_state():
    """A zone map that claims 16 seconds of a batch whose rows span a day, grouped by the raw time: more than 2^20 new
    groups arrive through the cold path of every state (parked while each table is at its growth threshold)."""
    import harness as H
    eng = H.get_backend("b200")
    qs = [AggQuery([], [T.TS, T.CITY], m) for m in (Measure("sum", T.FARE), Measure("count"), Measure("max", T.CITY))]
    hb = synth.generate_batch(0, 1_500_000, num_cities=100, null_rate=0.0)
    zm = {**synth.zone_map(hb), 0: (synth.BASE_TS, synth.BASE_TS + 15)}
    per_batch, got = _request_vs_solo(eng, qs, [T.upload(eng, hb, 0, zm)])
    assert per_batch == [(1, 1)] and got[0].groups > (1 << 20)


@pytest.mark.gpu
def test_fallback_runs_each_state_and_gives_the_same_results():
    """No zone map (hash-table form), and 25 x 300 city slots that one measure fits in a CTA but four do not: one kernel
    per state and batch."""
    import harness as H
    eng = H.get_backend("b200")
    qs = _cfg3_queries(A.ARES_REDUCE_SORT)
    per_batch, _ = _request_vs_solo(eng, qs, _edge_batches(eng, zone_maps="none"))
    assert per_batch == [(4, 0), (4, 0)], per_batch
    batches = []
    for d in range(2):
        hb = synth.generate_batch(d, 200_000, num_cities=300, null_rate=0.01)
        batches.append(T.upload(eng, hb, 0, synth.zone_map_of_day(d, 300)))
    per_batch, _ = _request_vs_solo(eng, qs, batches)
    assert per_batch == [(4, 4), (4, 4)], per_batch
    # two of them do fit: one kernel
    per_batch, _ = _request_vs_solo(eng, qs[:2], batches)
    assert per_batch == [(1, 1), (1, 1)], per_batch


@pytest.mark.gpu
def test_archive_shard_scan_and_join_requests():
    """An RLE archive scan through archive.scan_shard (live batches with the cutoff filter, archive days with and without
    the time filter) and a request of join queries give what the queries give alone."""
    import harness as H
    import test_joins as TJ
    from aresdb_b200 import aql, archive
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    eng = H.get_backend("b200")
    table = aql.Table("trips", [aql.Column(n, t) for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)])
    day0 = synth.BASE_TS // 86400
    cutoff = synth.BASE_TS + 3 * 86400
    arch = {day0 + d: synth.generate_batch(d, 20000, num_cities=12, null_rate=0.0) for d in range(3)}
    live = [synth.generate_batch(3 + i, 25000, num_cities=12, null_rate=0.0) for i in range(2)]
    frm, to = synth.BASE_TS + 86400 + 1800, synth.BASE_TS + 5 * 86400 - 1800
    text = {"table": "trips", "measures": [{"sqlExpression": m, "rowFilters": ["status = 1"]} for m in ("sum(fare)", "count(*)")],
            "timeFilter": {"column": "request_at", "from": str(frm), "to": str(to)},
            "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "hour"}, {"sqlExpression": "city_id"}]}
    qs = [aql.compile_query({**text, "measures": [m]}, table, synth.BASE_TS + 30 * 86400) for m in text["measures"]]
    keep_live = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in live]
    keep_arch = {d: T.upload(eng, hb, 0, synth.zone_map(hb)) for d, hb in arch.items()}
    req = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert req.groups == [[0, 1]]
    k0, d0 = _launches(eng)
    archive.scan_shard(req, keep_live, keep_arch, cutoff, qs[0].time_range, 0)
    k1, d1 = _launches(eng)
    for q, got in zip(qs, req.results()):
        ex = FusedBatchExecutor(eng.lib, eng.space, q)
        archive.scan_shard(ex, keep_live, keep_arch, cutoff, q.time_range, 0)
        _same(got, ex.result(), q, f"archive scan {q.measure_kind}")
    assert d1 - d0 >= 1
    # RLE archive batches: SUM / COUNT count run lengths, MIN does not, in one kernel
    rle = []
    for seed in (1, 2):
        b = T._archive_batch(eng, seed, 150000)
        b.ranges = {0: (synth.BASE_TS, synth.BASE_TS + 3 * 86400), 1: (1, 40), 2: (0, 3)}
        rle.append(b)
    per_batch, _ = _request_vs_solo(eng, _status_queries(), rle)
    assert [p[1] for p in per_batch] == [1, 1], per_batch
    # join: the lookup is shared; the dimension-table dimension has no zone map, so each state runs its own kernel
    etable, _ = TJ._dimension_table(eng)
    etz, tzn = TJ._tz_table(eng)
    by_region = TJ.join_queries(etable, etz.ptr, tzn)["by_region"]
    jq = [by_region, AggQuery([E.eq(T.STATUS, E.Lit(1)), E.gt(E.ForeignCol(0, 3, A.Float32, "surge"), E.Lit(1.0))],
                              [E.ForeignCol(0, 1, A.Uint8, "region"), E.floor(T.TS, E.Lit(3600))], Measure("count"),
                              joins=by_region.joins)]
    from aresdb_b200.executor import shared_scan_groups
    assert shared_scan_groups(jq) == [[0, 1]]
    hbs = [synth.generate_batch(d, 30000, num_cities=80, null_rate=0.03) for d in range(2)]
    _request_vs_solo(eng, jq, [T.upload(eng, hb) for hb in hbs])


@pytest.mark.gpu
def test_abi_rejections():
    import harness as H
    from aresdb_b200.executor import FusedBatchExecutor
    eng = H.get_backend("b200")
    qs = _cfg3_queries(A.ARES_REDUCE_SORT)[:2]
    hb = synth.generate_batch(0, 20000, num_cities=20)
    b = T.upload(eng, hb, 0, synth.zone_map(hb))
    solo = FusedBatchExecutor(eng.lib, eng.space, qs[0])
    plan = solo.plans.plan_for(b, True, 0)
    base = qs[0].plan_instructions(measures=qs)

    def run(queries, insts=base, n=None):
        exs = [FusedBatchExecutor(eng.lib, eng.space, q) for q in queries]
        plan.NumInsts = len(insts)
        for i, pi in enumerate(insts):
            plan.Insts[i] = pi
        states = (C.c_void_p * max(len(exs), 1))(*[e.state.value for e in exs])
        eng.lib.ExecuteBatchPlanMulti(states, len(exs) if n is None else n, C.byref(plan), eng.space.stream, eng.space.device)

    run(qs)
    for n in (0, 5):
        with pytest.raises(A.AresError, match="numStates must be 1..4"):
            run(qs, n=n)
    other_dims = AggQuery(qs[1].filters, [E.floor(T.TS, E.Lit(3600))], Measure("count"))
    with pytest.raises(A.AresError, match="NumDimsPerDimWidth"):
        run([qs[0], other_dims])
    with pytest.raises(A.AresError, match="ReduceMode"):
        run([qs[0], AggQuery(qs[1].filters, qs[1].dimensions, Measure("count"), reduce_mode=A.ARES_REDUCE_HASH)])
    with pytest.raises(A.AresError, match="AGGR_HLL"):
        run([qs[0], AggQuery(qs[1].filters, qs[1].dimensions, Measure("countdistincthll", T.CITY))])
    with pytest.raises(A.AresError, match="MeasureDataType"):
        run(qs[::-1])
    dup = list(base)
    dup[-1] = A.PlanInst.from_buffer_copy(bytes(base[-1]))
    dup[-1].SinkArg = 0
    with pytest.raises(A.AresError, match="duplicate SinkArg"):
        run(qs, dup)
    with pytest.raises(A.AresError, match="missing SinkArg"):
        run(qs, base[:-1])
    dup[-1].SinkArg = 3
    with pytest.raises(A.AresError, match="SinkArg 3"):
        run(qs, dup)
    solo.close()


if __name__ == "__main__":   # records the digests (run once, at the commit before the multi-measure form)
    import os
    os.environ["ARESDB_B200_JIT_GENERATE_ONLY"] = "1"
    GOLDEN.write_text(json.dumps(shape_digests(A.load_engine()), indent=1, sort_keys=True) + "\n")
