"""Queries of one AQL request that differ in their row filters, run in one pass over the batches.

A group's plan carries the filters every member has (PLAN_SINK_FILTER), then each member's own filters as member filter
roots (PLAN_SINK_MEASURE_FILTER, SinkArg = the member), then the dimensions and one measure root per member.

CPU: the generated text of every multi-measure plan without member filters is unchanged (SHA-256 recorded before member
filters existed), differing-filter requests compile in the shared form with per-member masks, the ABI rejects malformed
member filters, and FusedRequestExecutor groups queries by dimensions, time filter, joins and reduce mode.  GPU: every
member's result equals the same query run alone on FusedBatchExecutor."""
import ctypes as C
import hashlib
import json
import re
from pathlib import Path

import numpy as np
import pytest

from aresdb_b200 import cabi as A
from aresdb_b200 import columns, synth
from aresdb_b200 import expr as E
from aresdb_b200.query import AggQuery, Join, Measure
import test_jit_codegen as J
import test_pipeline_parity as T
import test_shared_scan as S

GOLDEN = Path(__file__).resolve().parent / "golden" / "multi_measure_kernel_sha256.json"
TS, CITY, STATUS, FARE = T.TS, T.CITY, T.STATUS, T.FARE
HOUR_CITY = [E.floor(TS, E.Lit(3600)), CITY]
T0 = synth.BASE_TS
TIME = [E.ge(TS, E.Lit(T0 + 1800)), E.lt(TS, E.Lit(T0 + 3 * 86400 - 1800))]


def plan_of(queries, rows=100000, ranges=None, base_counts=None):
    """The BatchPlan of a group over fake, aligned device addresses (nothing is dereferenced); joined tables as
    test_jit_codegen._dry_run sets them up.  Returns (plan, arrays the plan points into)."""
    p = S.shared_plan(queries, rows=rows, ranges=ranges, base_counts=base_counts)
    lead, keep = queries[0], []
    if lead.joins:
        p.NumForeignTables = len(lead.joins)
        for t, j in enumerate(lead.joins):
            p.ForeignTables[t].JoinColumn = j.on.index
            p.ForeignTables[t].Index = j.table.hash_index()
        p.NumForeignColumns = len(lead.foreign_columns)
        for k, (t, col, tz) in enumerate(lead.foreign_columns):
            f, arr = lead.joins[t].table.foreign_column(col, None, 0x7E0000000000 if tz else None, 12 if tz else 0)
            keep.append(arr)
            p.ForeignColumns[k].Table, p.ForeignColumns[k].Column = t, f
    return p, keep


def _dimension_table():
    import harness as H
    import test_joins as TJ
    return TJ._dimension_table(H.get_backend("oracle"))[0]


SURGE = E.ForeignCol(0, 3, A.Float32, "surge")


def multi_measure_shapes():
    """name -> (queries, plan keyword arguments): multi-measure requests whose members share every filter."""
    wide = dict(S.CFG3_RANGES)
    wide[synth.COL_CITY_ID] = (1, 300)
    rle_ranges = {0: (T0, T0 + 3 * 86400), 1: (1, 40), 2: (0, 3)}
    table = _dimension_table()
    joined = [AggQuery([E.eq(STATUS, E.Lit(1)), E.gt(SURGE, E.Lit(1.0))], HOUR_CITY, m, joins=[Join(table, CITY)])
              for m in (Measure("sum", FARE), Measure("count"))]
    shapes = {f"cfg3_k{k}": (S.cfg3_request(k), {"rows": 125_000_000, "ranges": S.CFG3_RANGES}) for k in (2, 3, 4)}
    shapes["wide_city_k2"] = (S.cfg3_request(2), {"ranges": wide})
    shapes["rle_status_k4"] = (S._status_queries(), {"base_counts": S.ALIGNED_BC, "ranges": rle_ranges})
    shapes["rle_cfg3_k4"] = (S.cfg3_request(4), {"base_counts": S.ALIGNED_BC, "ranges": S.CFG3_RANGES})
    shapes["join_k2"] = (joined, {"ranges": J.DAY_RANGES})
    return shapes, table


def shape_digests(lib):
    shapes, _keep = multi_measure_shapes()
    out = {}
    for name, (qs, kw) in shapes.items():
        plan, _arrays = plan_of(qs, **kw)
        _, src = S.dry_run_multi(lib, qs, plan)
        out[name] = hashlib.sha256(src.encode()).hexdigest()
    return out


def test_multi_measure_kernel_text_is_unchanged(monkeypatch):
    """Plans without member filters generate the text they generated before member filters existed."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    got = shape_digests(A.load_engine())
    want = json.loads(GOLDEN.read_text())
    assert sorted(got) == sorted(want)
    changed = [n for n in want if got[n] != want[n]]
    assert not changed, f"generated text changed for {changed}"


def diff_request(k=4, base=None, reduce_mode=A.ARES_REDUCE_SORT):
    """The first k members of a panel whose queries differ in their filters.  `base`: the cfg3 filters (status = 1,
    fare > 5, city_id != 0, then the time range); the common part is city_id != 0 and the time range.  Members:
    sum(fare) where status = 1 and fare > 5 (the cfg3 query), count(*) where status = 1, count(*) where status = 2,
    count(*)."""
    base = base or T.queries()["cfg3_sum"].filters
    status1, fare5, rest = base[0], base[1], base[2:]
    status2 = E.eq(STATUS, E.Lit(2))
    members = [(base, Measure("sum", FARE)), ([status1] + rest, Measure("count")), ([status2] + rest, Measure("count")),
               (rest, Measure("count"))]
    return [AggQuery(f, HOUR_CITY, m, reduce_mode=reduce_mode) for f, m in members[:k]]


def _sinks(insts):
    return [(pi.Sink, pi.SinkArg) for pi in insts if pi.Sink != A.PLAN_SINK_STACK]


def test_plan_carries_common_then_member_filters():
    """Common filters once, in the lead's order; each member's own filters as member filter roots; a group whose filters
    are identical keeps today's plan."""
    qs = diff_request()
    insts = qs[0].plan_instructions(measures=qs)
    F, MF, D, M = A.PLAN_SINK_FILTER, A.PLAN_SINK_MEASURE_FILTER, A.PLAN_SINK_DIMENSION, A.PLAN_SINK_MEASURE
    assert _sinks(insts) == [(F, 0)] * 3 + [(MF, 0), (MF, 0), (MF, 1), (MF, 2)] + [(D, 0), (D, 1)] + [(M, k) for k in range(4)]
    # the cutoff filter and the time filters stay in the common section
    assert _sinks(qs[0].plan_instructions(cutoff=5, measures=qs))[:4] == [(F, 0)] * 4
    assert _sinks(qs[0].plan_instructions(time_filters=False, measures=qs))[:1] == [(F, 0)]
    same = S.cfg3_request(4)
    ref = [bytes(i) for i in same[0].plan_instructions()]
    got = [bytes(i) for i in same[0].plan_instructions(measures=same)]
    assert got[:len(ref) - 1] == ref[:-1] and not any(i.Sink == MF for i in same[0].plan_instructions(measures=same))


@pytest.mark.parametrize("k", [2, 3, 4])
def test_differing_filter_requests_compile_in_the_shared_form(k):
    """One kernel; one warp skip per evaluator, taken only when no row is alive for any member; sum(fare) under its
    member filter fare > 5 keeps the exact-integer form it takes alone."""
    lib = A.load_engine()
    qs = diff_request(k)
    plan, _ = plan_of(qs, rows=125_000_000, ranges=S.CFG3_RANGES)
    size, src = S.dry_run_multi(lib, qs, plan)
    assert size > 0 and f"#define JIT_NMEAS {k}" in src and "#define JIT_LIVE_ARG(x) , x" in src
    assert "#define JIT_DENSE 1" in src
    assert re.search(r"kMeasAcc\[JIT_NMEAS\] = \{4[,}]", src)
    assert src.count("__any_sync(") == 2                                 # rowEval and rowEvalGeneric
    for m in range(k):
        assert src.count(f"live[{m}] = ") == 2


def test_member_filter_does_not_prove_shared_columns_valid(monkeypatch):
    """city_id > 3 as a member filter proves city_id non-NULL for its member only: the city dimension keeps its validity
    test (it is constant true when the filter is common), while the member's own measure sum(city_id) may count it."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    gt3 = E.gt(CITY, E.Lit(3))

    def city_dim_valid(qs):
        insts = qs[0].plan_instructions(measures=qs)
        i = [n for n, pi in enumerate(insts) if pi.Sink == A.PLAN_SINK_DIMENSION and pi.SinkArg == 1][0]
        j = [n for n, pi in enumerate(insts) if pi.Sink == A.PLAN_SINK_MEASURE and pi.SinkArg == 0][0]
        src = S.dry_run_multi(lib, qs, plan_of(qs, ranges=J.DAY_RANGES)[0])[1]
        return f"v{i}[r] = (uint32_t)x.v; m{i}[r] = true;" in src, f"v{j}[r] = (uint32_t)x.v; m{j}[r] = true;" in src
    common = [AggQuery([gt3], HOUR_CITY, Measure("sum", CITY)), AggQuery([gt3], HOUR_CITY, Measure("count"))]
    member = [AggQuery([gt3], HOUR_CITY, Measure("sum", CITY)), AggQuery([], HOUR_CITY, Measure("count"))]
    assert city_dim_valid(common) == (True, True)
    assert city_dim_valid(member) == (False, True)


def test_one_state_with_member_filters_is_the_plan_with_filters(monkeypatch):
    """numStates == 1: the member filters of the only state are ordinary filters (the single-measure kernel)."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    f = T.queries()["cfg3_sum"].filters
    q = AggQuery(f[2:] + f[:2], HOUR_CITY, Measure("sum", FARE))   # status = 1 and fare > 5 last
    plan, _ = plan_of([q], ranges=S.CFG3_RANGES)
    roots = [i for i in range(plan.NumInsts) if plan.Insts[i].Sink == A.PLAN_SINK_FILTER]
    for i in roots[3:]:
        plan.Insts[i].Sink = A.PLAN_SINK_MEASURE_FILTER
    assert S.dry_run_multi(lib, [q], plan)[1] == J._dry_run(lib, q, ranges=S.CFG3_RANGES)[1]


def test_member_filter_errors_are_reported(monkeypatch):
    """Member filters in a plan for ExecuteBatchPlan, a SinkArg outside the states, and member filter roots after a
    dimension root or before a filter root."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    qs = diff_request(3)
    plan, _ = plan_of(qs, ranges=S.CFG3_RANGES)
    mf = [i for i in range(plan.NumInsts) if plan.Insts[i].Sink == A.PLAN_SINK_MEASURE_FILTER]
    assert mf == [3, 4, 5, 6]
    with pytest.raises(A.AresError, match="need ExecuteBatchPlanMulti"):
        fn = lib.alg.AresJitDryRun
        fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
        fn.restype = A.CGoCallResHandle
        h = fn(qs[0].agg_spec(), C.byref(plan), None)
        if h.pStrErr:
            raise A.AresError(C.string_at(h.pStrErr).decode())
    bad = A.BatchPlan.from_buffer_copy(bytes(plan))
    bad.Insts[6].SinkArg = 3
    with pytest.raises(A.AresError, match="member filter root with SinkArg 3"):
        S.dry_run_multi(lib, qs, bad)
    bad = A.BatchPlan.from_buffer_copy(bytes(plan))   # city_id != 0 (a filter root) after the member filters
    bad.Insts[0], bad.Insts[3] = plan.Insts[3], plan.Insts[0]
    with pytest.raises(A.AresError, match="follow the last PLAN_SINK_FILTER"):
        S.dry_run_multi(lib, qs, bad)
    bad = A.BatchPlan.from_buffer_copy(bytes(plan))   # a member filter after the first dimension root
    dim = [i for i in range(plan.NumInsts) if plan.Insts[i].Sink == A.PLAN_SINK_DIMENSION][0]
    assert plan.Insts[dim].NumOperands == 2 and plan.Insts[dim - 1].Sink == A.PLAN_SINK_MEASURE_FILTER
    moved = [plan.Insts[i] for i in range(plan.NumInsts) if i != 6]
    moved.insert(dim, plan.Insts[6])
    for i, pi in enumerate(moved):
        bad.Insts[i] = pi
    with pytest.raises(A.AresError, match="precede the first dimension root"):
        S.dry_run_multi(lib, qs, bad)
    with pytest.raises(A.AresError, match="member filter root with SinkArg 1"):   # numStates == 1
        S.dry_run_multi(lib, qs[:1], plan)


def _trips_table():
    from aresdb_b200 import aql
    return aql.Table("trips", [aql.Column("request_at", A.Uint32), aql.Column("city_id", A.Uint16),
                               aql.Column("status", A.Uint8, enum={"completed": 0, "cancelled": 1, "other": 2}),
                               aql.Column("fare", A.Float32)])


def test_grouping_by_dimensions_time_filter_joins_and_reduce_mode():
    """Queries that differ only in their filters share a pass; different dimensions, time range, join, reduce mode or an
    HLL measure do not; the instruction limit splits a group."""
    from aresdb_b200.executor import shared_scan_groups
    tf = [E.ge(TS, E.Lit(T0)), E.lt(TS, E.Lit(T0 + 86400))]

    def q(m, filters=(E.eq(STATUS, E.Lit(1)),), d=HOUR_CITY, time=tf, **kw):
        return AggQuery(list(filters), d, m, time_filters=time, **kw)
    fare, trips = q(Measure("sum", FARE)), q(Measure("count"))
    cancelled, everything = q(Measure("count"), filters=[E.eq(STATUS, E.Lit(2))]), q(Measure("count"), filters=[])
    assert shared_scan_groups([fare, cancelled, trips, everything], member_filters=True) == [[0, 1, 2, 3]]
    assert shared_scan_groups([fare, cancelled, trips, everything]) == [[0, 2], [1], [3]]
    others = [q(Measure("count"), time=[E.ge(TS, E.Lit(T0)), E.lt(TS, E.Lit(T0 + 7200))]),
              q(Measure("count"), d=[E.floor(TS, E.Lit(60)), CITY]),
              q(Measure("count"), reduce_mode=A.ARES_REDUCE_HASH),
              q(Measure("countdistincthll", CITY)),
              q(Measure("countdistincthll", CITY)),
              q(Measure("count"), joins=[Join(object(), CITY)])]
    groups = shared_scan_groups([fare] + others + [cancelled], member_filters=True)
    assert groups == [[0, len(others) + 1]] + [[i] for i in range(1, len(others) + 1)]
    # long member filters: a query that would take the plan past ARES_MAX_PLAN_INSTS opens a new group
    chain = E.Lit(1)
    for _ in range(23):
        chain = E.add(chain, CITY)
    long_ = [q(Measure("count"), filters=[E.gt(chain, E.Lit(n))]) for n in range(4)]
    assert len(long_[0].plan_instructions(measures=long_[:2])) <= A.ARES_MAX_PLAN_INSTS - 1   # (room for the cutoff filter)
    with pytest.raises(ValueError, match="plan too long"):
        long_[0].plan_instructions(measures=long_[:3])
    assert shared_scan_groups(long_, member_filters=True) == [[0, 1], [2, 3]]


def test_compiled_request_with_a_cancelled_trips_panel_is_one_group():
    """The reference's total_trips.aql next to the same query for cancelled trips: one pass, the status filters as member
    filters."""
    from aresdb_b200 import aql
    from aresdb_b200.executor import shared_scan_groups
    import test_aql_frontend as F
    trips = F._queries()["total_trips"]
    cancelled = json.loads(json.dumps(trips))
    cancelled["measures"][0]["rowFilters"] = ["status='cancelled'"]
    qs = aql.compile_request({"queries": [trips, cancelled]}, _trips_table(), T0 + 86400)
    assert shared_scan_groups(qs, member_filters=True) == [[0, 1]]
    sinks = _sinks(qs[0].plan_instructions(measures=qs))
    assert (A.PLAN_SINK_MEASURE_FILTER, 0) in sinks and (A.PLAN_SINK_MEASURE_FILTER, 1) in sinks


# ---- on the GPU: every member equals the same query run alone ------------------------------------------------------
def _run(eng, qs, batches, expected_groups=0):
    """S._request_vs_solo, and every query's skipped batches equal to its solo run's.  Returns (launches per batch,
    results)."""
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    req = FusedRequestExecutor(eng.lib, eng.space, qs, expected_groups)
    solos = [FusedBatchExecutor(eng.lib, eng.space, q, expected_groups) for q in qs]
    per_batch = []
    for b in batches:
        k0, d0 = S._launches(eng)
        req.process_batch(b)
        k1, d1 = S._launches(eng)
        per_batch.append((k1 - k0, d1 - d0))
        for ex in solos:
            ex.process_batch(b)
    got = req.results()
    for i, (q, ex) in enumerate(zip(qs, solos)):
        S._same(got[i], ex.result(), q, f"query {i} ({q.measure_kind})")
        assert req.executors[i].skipped == ex.skipped, f"query {i}: skipped batches differ"
    req.close()
    for ex in solos:
        ex.close()
    return per_batch, got


@pytest.mark.gpu
@pytest.mark.parametrize("reduce_mode", [A.ARES_REDUCE_SORT, A.ARES_REDUCE_HASH], ids=["sort", "hash"])
@pytest.mark.parametrize("city_dist", ["uniform", "zipf"])
def test_differing_filter_request_at_scale_equals_solo_runs(city_dist, reduce_mode):
    """2 x 1.25e8 rows with zone maps: one fused launch per batch feeds the four members; sum(fare) (the cfg3 query) also
    equals tests/independent.py."""
    import torch
    import harness as H
    import independent as I
    import test_at_size as AS
    from aresdb_b200.executor import Batch
    eng, dev, rows = H.get_backend("b200"), torch.device("cuda:0"), AS.BATCH_ROWS
    exp = I.Expected("cfg3", 2, dev, T0, T0 + 1800, T0 + 2 * 86400 - 1800)
    qs = diff_request(4, AS._queries(2)["cfg3"].filters, reduce_mode)

    def batches():
        for d in range(2):
            bufs, voff, cols = AS._batch(d, rows, dev, city_dist=city_dist)
            exp.add_batch(bufs, voff, rows)
            yield Batch(cols, rows, ranges=synth.zone_map_of_day(d), keep=[bufs])

    per_batch, got = _run(eng, qs, batches())
    assert per_batch == [(1, 1), (1, 1)], per_batch
    if reduce_mode == A.ARES_REDUCE_SORT:
        assert exp.check(got[0])["groups"] == 2 * 24 * 100
    assert all(r.groups > 0 for r in got)


def _nullable_request():
    """Member filters on NULL-able columns: fare > 5 (exact-integer sum), city_id > 50 (a dimension: its rows are never
    NULL for that member, for the others they may be), status = 2 (flagged min), none (sum(city_id))."""
    return [AggQuery([E.gt(FARE, E.Lit(5.0))], HOUR_CITY, Measure("sum", FARE)),
            AggQuery([E.gt(CITY, E.Lit(50))], HOUR_CITY, Measure("count")),
            AggQuery([E.eq(STATUS, E.Lit(2))], HOUR_CITY, Measure("min", FARE)),
            AggQuery([], HOUR_CITY, Measure("sum", CITY))]


@pytest.mark.gpu
@pytest.mark.parametrize("zone_maps", ["exact", "stale", "narrow"])
@pytest.mark.parametrize("request_of", ["cfg3", "nullable"])
def test_edge_inputs_equal_solo_runs(request_of, zone_maps):
    """NULL fares and cities, -0.0 / +0.0 fares and NULL-able filtered columns; rows outside a too-narrow or stale zone map
    take the cold path of the members they are alive for.  The narrow zone map (cities 1..10) contradicts city_id > 50:
    that member skips the batches, as it does alone."""
    import harness as H
    eng = H.get_backend("b200")
    qs = diff_request(4) if request_of == "cfg3" else _nullable_request()
    per_batch, got = _run(eng, qs, S._edge_batches(eng, zone_maps=zone_maps))
    assert all(p == (1, 1) for p in per_batch), per_batch
    if request_of == "nullable":
        null_city = [c is None for c in got[3].decoded_dims()[1]]
        assert any(null_city) and not any(c is None for c in got[1].decoded_dims()[1])


@pytest.mark.gpu
def test_empty_member_and_groups_of_one_member():
    """A member whose filter matches no row has an empty result; groups that only one member's rows reach (city 7) are
    absent from the others, whatever their form: flag-less count, exact-integer sum, flagged max."""
    import harness as H
    eng = H.get_backend("b200")
    not7, is7 = E.ne(CITY, E.Lit(7)), E.eq(CITY, E.Lit(7))
    qs = [AggQuery([not7, E.eq(STATUS, E.Lit(2))], HOUR_CITY, Measure("count")),
          AggQuery([not7, E.gt(FARE, E.Lit(5.0))], HOUR_CITY, Measure("sum", FARE)),
          AggQuery([not7], HOUR_CITY, Measure("max", CITY)),
          AggQuery([is7], HOUR_CITY, Measure("count"))]
    hbs = [synth.generate_batch(d, 200_000, num_cities=20, null_rate=0.02) for d in range(2)]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs]
    per_batch, got = _run(eng, qs, batches)
    assert per_batch == [(1, 1), (1, 1)], per_batch
    cities = [set(r.decoded_dims()[1]) for r in got]
    assert cities[3] == {7} and all(7 not in c and c for c in cities[:3])
    none = qs[:1] + [AggQuery([E.lt(FARE, E.Lit(-1.0))], HOUR_CITY, Measure("sum", FARE))]
    per_batch, got = _run(eng, none, batches)
    assert per_batch == [(1, 1), (1, 1)] and got[1].groups == 0 and got[0].groups > 0


@pytest.mark.gpu
def test_member_contradicted_by_the_zone_map_is_left_out():
    """city_id > 1000 cannot hold on these batches: that member skips them (its skipped count is its solo run's), the
    others run together; when one member is left it runs its own plan; when all are contradicted nothing is launched."""
    import harness as H
    eng = H.get_backend("b200")
    hbs = [synth.generate_batch(d, 100_000, num_cities=50, null_rate=0.02) for d in range(2)]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs]
    big = E.gt(CITY, E.Lit(1000))
    qs = diff_request(2) + [AggQuery(T.queries()["cfg3_sum"].filters[2:] + [big], HOUR_CITY, Measure("count"))]
    per_batch, got = _run(eng, qs, batches)
    assert per_batch == [(1, 1), (1, 1)] and got[2].groups == 0
    per_batch, _ = _run(eng, [qs[0], qs[2]], batches)
    assert per_batch == [(1, 1), (1, 1)], per_batch
    per_batch, _ = _run(eng, [qs[2], AggQuery([big, E.eq(STATUS, E.Lit(1))], HOUR_CITY, Measure("sum", FARE))], batches)
    assert per_batch == [(0, 0), (0, 0)], per_batch


@pytest.mark.gpu
def test_member_filter_on_a_joined_table_column():
    """surge > 1.0 (a dimension-table column; unmatched rows read NULL) filters one member; the lookup serves both."""
    import harness as H
    import test_joins as TJ
    eng = H.get_backend("b200")
    table, _ = TJ._dimension_table(eng)
    j = [Join(table, CITY)]
    qs = [AggQuery([E.eq(STATUS, E.Lit(1)), E.gt(SURGE, E.Lit(1.0))], HOUR_CITY, Measure("sum", FARE), joins=j),
          AggQuery([E.eq(STATUS, E.Lit(1))], HOUR_CITY, Measure("count"), joins=j),
          AggQuery([E.Unary(A.IsNull, E.ForeignCol(0, 1, A.Uint8, "region"))], HOUR_CITY, Measure("max", CITY), joins=j)]
    hbs = [synth.generate_batch(d, 30000, num_cities=80, null_rate=0.03) for d in range(2)]
    per_batch, got = _run(eng, qs, [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs])
    assert per_batch == [(1, 1), (1, 1)], per_batch
    assert all(r.groups > 0 for r in got)


def _aql_request(rows_filters):
    from aresdb_b200 import aql
    table = aql.Table("trips", [aql.Column(n, t) for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)])
    frm, to = T0 + 86400 + 1800, T0 + 5 * 86400 - 1800
    text = {"table": "trips", "timeFilter": {"column": "request_at", "from": str(frm), "to": str(to)},
            "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "hour"}, {"sqlExpression": "city_id"}]}
    return [aql.compile_query({**text, "measures": [{"sqlExpression": m, "rowFilters": f}]}, table, T0 + 30 * 86400)
            for m, f in rows_filters]


AQL_MEMBERS = [("sum(fare)", ["status = 1", "fare > 5"]), ("count(*)", ["status = 1"]), ("count(*)", ["status = 2"]),
               ("max(city_id)", [])]


@pytest.mark.gpu
def test_archive_shard_scan_and_rle_batches():
    """archive.scan_shard (live batches with the cutoff filter, archive days with and without the time filter) and RLE
    archive batches (SUM / COUNT count run lengths, MAX does not) give what the members give alone."""
    import harness as H
    from aresdb_b200 import archive
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    eng = H.get_backend("b200")
    day0, cutoff = T0 // 86400, T0 + 3 * 86400
    arch = {day0 + d: synth.generate_batch(d, 20000, num_cities=12, null_rate=0.02) for d in range(3)}
    live = [synth.generate_batch(3 + i, 25000, num_cities=12, null_rate=0.02) for i in range(2)]
    qs = _aql_request(AQL_MEMBERS)
    keep_live = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in live]
    keep_arch = {d: T.upload(eng, hb, 0, synth.zone_map(hb)) for d, hb in arch.items()}
    req = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert req.groups == [[0, 1, 2, 3]]
    k0, d0 = S._launches(eng)
    archive.scan_shard(req, keep_live, keep_arch, cutoff, qs[0].time_range, 0)
    k1, d1 = S._launches(eng)
    for q, got in zip(qs, req.results()):
        ex = FusedBatchExecutor(eng.lib, eng.space, q)
        archive.scan_shard(ex, keep_live, keep_arch, cutoff, q.time_range, 0)
        S._same(got, ex.result(), q, f"archive scan {q.measure_kind}")
        assert got.groups > 0
    assert d1 - d0 >= 1
    rle = []
    for seed in (1, 2):
        b = T._archive_batch(eng, seed, 150000)
        b.ranges = {0: (T0, T0 + 3 * 86400), 1: (1, 40), 2: (0, 3)}
        rle.append(b)
    qs = [AggQuery([E.eq(STATUS, E.Lit(1))], HOUR_CITY, Measure("sum", FARE)),
          AggQuery([E.eq(STATUS, E.Lit(2)), E.gt(FARE, E.Lit(20.0))], HOUR_CITY, Measure("count")),
          AggQuery([], HOUR_CITY, Measure("max", FARE)),
          AggQuery([E.ne(STATUS, E.Lit(1))], HOUR_CITY, Measure("sum", CITY))]
    per_batch, _ = _run(eng, qs, rle)
    assert [p[1] for p in per_batch] == [1, 1], per_batch


@pytest.mark.gpu
def test_out_of_range_rows_claiming_many_groups_spill_per_state():
    """A zone map that claims 16 seconds of a day of rows, grouped by the raw time: more than 2^20 new groups arrive
    through the cold path of every member, each claiming only the groups of its own rows."""
    import harness as H
    eng = H.get_backend("b200")
    dims = [TS, CITY]
    qs = [AggQuery([E.gt(FARE, E.Lit(5.0))], dims, Measure("sum", FARE)), AggQuery([], dims, Measure("count")),
          AggQuery([E.eq(STATUS, E.Lit(1))], dims, Measure("max", CITY))]
    hb = synth.generate_batch(0, 1_500_000, num_cities=100, null_rate=0.0)
    zm = {**synth.zone_map(hb), 0: (T0, T0 + 15)}
    per_batch, got = _run(eng, qs, [T.upload(eng, hb, 0, zm)])
    assert per_batch == [(1, 1)] and got[1].groups > (1 << 20) and got[2].groups < got[1].groups


@pytest.mark.gpu
def test_fallback_without_a_zone_map():
    """No zone map: each member runs its own single-measure plan (its member filters as filters), one kernel per member."""
    import harness as H
    eng = H.get_backend("b200")
    per_batch, _ = _run(eng, diff_request(4), S._edge_batches(eng, zone_maps="none"))
    assert per_batch == [(4, 0), (4, 0)], per_batch


@pytest.mark.gpu
def test_sharded_request_on_simulated_ranks():
    """Batches dealt to two simulated ranks (a FusedRequestExecutor each, as ShardedFusedRequest runs them), exchanged
    with one export, merge and finalize: every rank has the request's results; ShardedFusedRequest without a process
    group equals FusedRequestExecutor through scan_shard."""
    import harness as H
    import test_sharded_request as SR
    from aresdb_b200 import archive
    from aresdb_b200.executor import FusedRequestExecutor
    from aresdb_b200.sharding import ShardedFusedRequest
    eng = H.get_backend("b200")
    qs = diff_request(4)
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in (synth.generate_batch(d, 20000, num_cities=30) for d in range(4))]
    full = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert full.groups == [[0, 1, 2, 3]]
    locals_ = [FusedRequestExecutor(eng.lib, eng.space, qs) for _ in range(2)]
    for i, b in enumerate(batches):
        full.process_batch(b)
        locals_[i % 2].process_batch(b)
    expected = full.results()
    xqs, out = SR._exchange_on_one_device(eng, locals_, 32768, (1,))
    SR._check_exchange(xqs, out, expected, 32768, "W2")
    for ex in locals_ + [full]:
        ex.close()
    day0, cutoff = T0 // 86400, T0 + 3 * 86400
    arch = {day0 + d: T.upload(eng, synth.generate_batch(d, 20000, num_cities=12), 0) for d in range(3)}
    live = [T.upload(eng, synth.generate_batch(3 + i, 25000, num_cities=12), 0) for i in range(2)]
    qs = _aql_request(AQL_MEMBERS)
    req, ref = ShardedFusedRequest(eng.lib, eng.space, qs), FusedRequestExecutor(eng.lib, eng.space, qs)
    archive.scan_shard(req, live, arch, cutoff, qs[0].time_range, 0)
    archive.scan_shard(ref, live, arch, cutoff, qs[0].time_range, 0)
    SR._same_results(qs, req.finalize(), ref.results(), "scan_shard")
    req.close()
    ref.close()


@pytest.mark.gpu
def test_abi_rejections():
    import harness as H
    from aresdb_b200.executor import FusedBatchExecutor
    eng = H.get_backend("b200")
    qs = diff_request(3)
    hb = synth.generate_batch(0, 20000, num_cities=20)
    b = T.upload(eng, hb, 0, synth.zone_map(hb))
    exs = [FusedBatchExecutor(eng.lib, eng.space, q) for q in qs]
    plan = exs[0].plans.plan_for(b, True, 0)
    insts = qs[0].plan_instructions(measures=qs)

    def run(ins, n=3):
        plan.NumInsts = len(ins)
        for i, pi in enumerate(ins):
            plan.Insts[i] = pi
        states = (C.c_void_p * 3)(*[e.state.value for e in exs])
        eng.lib.ExecuteBatchPlanMulti(states, n, C.byref(plan), eng.space.stream, eng.space.device)

    run(insts)
    with pytest.raises(A.AresError, match="need ExecuteBatchPlanMulti"):
        eng.lib.ExecuteBatchPlan(exs[0].state, C.byref(plan), eng.space.stream, eng.space.device)
    bad = [A.PlanInst.from_buffer_copy(bytes(i)) for i in insts]
    bad[6].SinkArg = 3
    with pytest.raises(A.AresError, match="member filter root with SinkArg 3"):
        run(bad)
    with pytest.raises(A.AresError, match="member filter root with SinkArg 1"):
        run(insts[:], n=1)
    with pytest.raises(A.AresError, match="follow the last PLAN_SINK_FILTER"):
        run([insts[3], insts[1], insts[2], insts[0]] + insts[4:])
    dim = [i for i, pi in enumerate(insts) if pi.Sink == A.PLAN_SINK_DIMENSION][0]
    with pytest.raises(A.AresError, match="precede the first dimension root"):
        run(insts[:6] + insts[7:dim + 1] + [insts[6]] + insts[dim + 1:])
    for e in exs:
        e.close()


if __name__ == "__main__":   # records the digests (run once, at the commit before member filters)
    import os
    os.environ["ARESDB_B200_JIT_GENERATE_ONLY"] = "1"
    GOLDEN.write_text(json.dumps(shape_digests(A.load_engine()), indent=1, sort_keys=True) + "\n")
