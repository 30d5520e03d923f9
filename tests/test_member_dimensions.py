"""Queries of one AQL request that differ in their dimensions, run in one pass over the batches.

A pass's plan carries the union of its members' dimensions as member dimension roots (PLAN_SINK_MEMBER_DIMENSION,
SinkArg = the mask of the members that group by the dimension), after the member filters and before the measure roots.
Per batch the engine runs one kernel for every member, one kernel per set of members with the same dimensions, or one
kernel per member.

CPU: plan emission, packing of groups into passes, the form each dry run takes, the ABI rejections and the generated
text of the new shapes (SHA-256 in tests/golden/member_dimension_kernel_sha256.json).  GPU: every member's result
equals the same query run alone on FusedBatchExecutor, and the launches per batch are those of the chosen form."""
import ctypes as C
import hashlib
import json
import re
from pathlib import Path

import pytest

from aresdb_b200 import cabi as A
from aresdb_b200 import synth
from aresdb_b200 import expr as E
from aresdb_b200.query import AggQuery, Join, Measure
import test_member_filters as MF
import test_pipeline_parity as T
import test_shared_scan as S

GOLDEN = Path(__file__).resolve().parent / "golden" / "member_dimension_kernel_sha256.json"
TS, CITY, STATUS, FARE = T.TS, T.CITY, T.STATUS, T.FARE
HOUR = E.floor(TS, E.Lit(3600))
T0 = synth.BASE_TS
F, MFL, D, MD, M = (A.PLAN_SINK_FILTER, A.PLAN_SINK_MEASURE_FILTER, A.PLAN_SINK_DIMENSION, A.PLAN_SINK_MEMBER_DIMENSION,
                    A.PLAN_SINK_MEASURE)


def panel(k=4, filters=None, reduce_mode=A.ARES_REDUCE_SORT):
    """The first k panels of a dashboard over the cfg3 slice, all with the cfg3 filters: sum(fare) by hour x city (the
    cfg3 query), count(*) by hour, count(*) by city, count(*) by status."""
    f = T.queries()["cfg3_sum"].filters if filters is None else filters
    members = [([HOUR, CITY], Measure("sum", FARE)), ([HOUR], Measure("count")), ([CITY], Measure("count")),
               ([STATUS], Measure("count"))]
    return [AggQuery(f, d, m, reduce_mode=reduce_mode) for d, m in members[:k]]


def forms_panel(filters=None, reduce_mode=A.ARES_REDUCE_SORT):
    """Each accumulation form with a dimension set of its own: exact-integer sum(fare) by hour x city, flag-less count by
    hour, split CAS / RED avg(fare) by city, flagged 32-bit max(city_id) by status."""
    f = T.queries()["cfg3_sum"].filters if filters is None else filters
    ms = [([HOUR, CITY], Measure("sum", FARE)), ([HOUR], Measure("count")), ([CITY], Measure("avg", FARE)),
          ([STATUS], Measure("max", CITY))]
    return [AggQuery(f, d, m, reduce_mode=reduce_mode) for d, m in ms]


def sets_panel():
    """Two members by hour x city and two by two-hour buckets x city: with 300 cities each set fits a CTA, both do not."""
    f = T.queries()["cfg3_sum"].filters
    h2 = [E.floor(TS, E.Lit(7200)), CITY]
    return [AggQuery(f, [HOUR, CITY], Measure("sum", FARE)), AggQuery(f, [HOUR, CITY], Measure("count")),
            AggQuery(f, h2, Measure("count")), AggQuery(f, h2, Measure("max", CITY))]


def mixed_panel():
    """Two members by hour x city and two by status: without a zone-map range for status only the first set takes a
    direct-indexed kernel, and the members by status run their own kernels."""
    f = T.queries()["cfg3_sum"].filters
    return [AggQuery(f, [HOUR, CITY], Measure("sum", FARE)), AggQuery(f, [HOUR, CITY], Measure("count")),
            AggQuery(f, [STATUS], Measure("count")), AggQuery(f, [STATUS], Measure("max", CITY))]


def without_status(ranges):
    return {c: r for c, r in ranges.items() if c != synth.COL_STATUS}


def filtered_panel(reduce_mode=A.ARES_REDUCE_SORT):
    """Member filters with member dimensions: the common part is city_id != 0 and the time range."""
    base = T.queries()["cfg3_sum"].filters
    rest = base[2:]
    ms = [(base, [HOUR, CITY], Measure("sum", FARE)), ([base[0]] + rest, [HOUR], Measure("count")),
          ([E.eq(STATUS, E.Lit(2))] + rest, [CITY], Measure("count")), (rest, [STATUS], Measure("count"))]
    return [AggQuery(f, d, m, reduce_mode=reduce_mode) for f, d, m in ms]


WIDE = {**S.CFG3_RANGES, synth.COL_CITY_ID: (1, 300)}


def _sinks(insts):
    return [(pi.Sink, pi.SinkArg) for pi in insts if pi.Sink != A.PLAN_SINK_STACK]


def member_dimension_shapes():
    """name -> (queries, plan keyword arguments): requests whose members differ in their dimensions."""
    table = MF._dimension_table()
    region = E.ForeignCol(0, 1, A.Uint8, "region")
    j = [Join(table, CITY)]
    f = [E.eq(STATUS, E.Lit(1))]
    joined = [AggQuery(f, [HOUR, CITY], Measure("sum", FARE), joins=j), AggQuery(f, [region], Measure("count"), joins=j)]
    shapes = {f"cfg3_k{k}": (panel(k), {"rows": 125_000_000, "ranges": S.CFG3_RANGES}) for k in (2, 3, 4)}
    shapes["forms_k4"] = (forms_panel(), {"rows": 125_000_000, "ranges": S.CFG3_RANGES})
    shapes["member_filters_k4"] = (filtered_panel(), {"rows": 125_000_000, "ranges": S.CFG3_RANGES})
    shapes["rle_k4"] = (forms_panel(), {"base_counts": S.ALIGNED_BC, "ranges": S.CFG3_RANGES})
    # the joined column has no zone map: its member runs its own kernel, the digest is of the other member's set
    shapes["join_k2"] = (joined, {"ranges": {**S.CFG3_RANGES}})
    return shapes, table


def _digest_source(lib, qs, kw):
    """The kernel text of the pass's plan in the shared form, or, when that form is not taken, the texts of its
    members' own plans."""
    try:
        return S.dry_run_multi(lib, qs, MF.plan_of(qs, **kw)[0])[1]
    except A.AresError as e:
        assert "one kernel per" in str(e), e
    return "".join(S.dry_run_multi(lib, [q], MF.plan_of([q], **kw)[0])[1] for q in qs)


def shape_digests(lib):
    shapes, _keep = member_dimension_shapes()
    return {name: hashlib.sha256(_digest_source(lib, qs, kw).encode()).hexdigest() for name, (qs, kw) in shapes.items()}


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_plan_carries_the_union_of_the_dimensions():
    """Common filters, then member filters, then the union of the dimensions as member dimension roots with the masks of
    their members, then the measure roots; a pass whose members share their dimensions keeps today's bytes."""
    qs = panel()
    assert _sinks(qs[0].plan_instructions(measures=qs)) == [(F, 0)] * 5 + [(MD, 0b0011), (MD, 0b0101), (MD, 0b1000)] + \
        [(M, k) for k in range(4)]
    fq = filtered_panel()
    sinks = _sinks(fq[0].plan_instructions(measures=fq))
    assert sinks[3:7] == [(MFL, 0), (MFL, 0), (MFL, 1), (MFL, 2)]
    assert sinks[7:10] == [(MD, 0b0011), (MD, 0b0101), (MD, 0b1000)]
    same = S.cfg3_request(4)
    ref = [bytes(i) for i in same[0].plan_instructions()]
    got = [bytes(i) for i in same[0].plan_instructions(measures=same)]
    assert got[:len(ref) - 1] == ref[:-1] and not any(i.Sink == MD for i in same[0].plan_instructions(measures=same))
    # the union keeps each member's layout order (city, status and hour, status): city, hour, status
    from aresdb_b200.query import member_dimensions
    u = member_dimensions([AggQuery([], [STATUS, CITY], Measure("count")), AggQuery([], [HOUR, STATUS], Measure("count"))])
    assert [(e.name if isinstance(e, E.Col) else "hour", mask) for e, _, mask in u] == [("city_id", 0b01), ("hour", 0b10),
                                                                                          ("status", 0b11)]


def test_packing_of_groups_into_passes():
    from aresdb_b200.executor import shared_scan_groups, shared_scan_passes
    import test_sharded_request as SR

    def passes(qs):
        return shared_scan_passes(qs, shared_scan_groups(qs, member_filters=True))
    assert passes(panel()) == [[0, 1, 2, 3]]
    req = [q for q in SR._request() if not q.is_hll and q.reduce_mode == A.ARES_REDUCE_SORT]
    assert len(req) == 4 and len(shared_scan_groups(req, member_filters=True)) == 2 and passes(req) == [[0, 1, 2, 3]]
    tf = [E.ge(TS, E.Lit(T0)), E.lt(TS, E.Lit(T0 + 86400))]

    def q(m, d, time=tf, **kw):
        return AggQuery([E.eq(STATUS, E.Lit(1))], d, m, time_filters=time, **kw)
    by_hour = q(Measure("count"), [HOUR])
    outsiders = {
        "time filter": q(Measure("count"), [CITY], time=[E.ge(TS, E.Lit(T0)), E.lt(TS, E.Lit(T0 + 7200))]),
        "join": q(Measure("count"), [CITY], joins=[Join(object(), CITY)]),
        "reduce mode": q(Measure("count"), [CITY], reduce_mode=A.ARES_REDUCE_HASH),
        "hll": q(Measure("countdistincthll", CITY), [CITY]),
        "no dimensions": q(Measure("count"), []),
    }
    for why, other in outsiders.items():
        assert passes([by_hour, other]) == [[0], [1]], why
    # two members order two 4-byte dimensions (hour, minute) differently
    minute = E.floor(TS, E.Lit(60))
    a, b = q(Measure("count"), [HOUR, minute]), q(Measure("sum", FARE), [minute, HOUR])
    assert passes([a, b]) == [[0], [1]]
    # a fifth state opens a new pass
    five = panel() + [q(Measure("max", CITY), [TS])]
    assert passes(five) == [[0, 1, 2, 3], [4]]
    # more than 8 union dimensions
    nine = [q(Measure("count"), [E.floor(TS, E.Lit(60 * (n + 1))) for n in range(5)]),
            q(Measure("count"), [E.floor(TS, E.Lit(7 * (n + 1))) for n in range(4)])]
    assert passes(nine) == [[0], [1]]
    # a plan past ARES_MAX_PLAN_INSTS
    chain = E.Lit(1)
    for _ in range(30):
        chain = E.add(chain, CITY)
    long_ = [q(Measure("count"), [chain]), q(Measure("count"), [E.add(chain, E.Lit(1))]), q(Measure("count"), [HOUR])]
    with pytest.raises(ValueError, match="plan too long"):
        long_[0].plan_instructions(cutoff=1, measures=long_[:2])
    assert passes(long_) == [[0], [1, 2]]


def test_dry_runs_choose_the_form():
    """The cfg3 panel: one kernel with the day's zone map (each member keeps the form it takes alone); two hour x city
    members and two two-hour x city members over 300 cities: one kernel per dimension set; no zone map: one kernel per
    state; a set that fits next to a set without a zone map: the set's kernel and one kernel per other member.  With 300
    cities the cfg3 panel itself still fits one kernel: only one member groups by hour x city."""
    lib = A.load_engine()
    qs = panel()
    size, src = S.dry_run_multi(lib, qs, MF.plan_of(qs, rows=125_000_000, ranges=S.CFG3_RANGES)[0])
    assert size > 0 and "#define JIT_NMEAS 4" in src and "#define JIT_MDIMS 1" in src and "#define JIT_DENSE 1" in src
    assert "kMeasAcc[JIT_NMEAS] = {4, 1, 1, 1};" in src and "kMeasDims[JIT_NMEAS] = {3, 1, 2, 4};" in src
    assert src.count("if (!__any_sync(__activemask(), al[0]") == 2
    fq = forms_panel()
    src = S.dry_run_multi(lib, fq, MF.plan_of(fq, rows=125_000_000, ranges=S.CFG3_RANGES)[0])[1]
    assert "kMeasAcc[JIT_NMEAS] = {4, 1, 2, 1};" in src
    assert "#define JIT_NMEAS 4" in S.dry_run_multi(lib, qs, MF.plan_of(qs, ranges=WIDE)[0])[1]
    sq = sets_panel()
    with pytest.raises(A.AresError, match="one kernel per dimension set"):
        S.dry_run_multi(lib, sq, MF.plan_of(sq, rows=125_000_000, ranges=WIDE)[0])
    for plan_qs in (sq[:2], sq[2:]):
        assert "#define JIT_NMEAS 2" in S.dry_run_multi(lib, plan_qs, MF.plan_of(plan_qs, rows=125_000_000, ranges=WIDE)[0])[1]
    with pytest.raises(A.AresError, match="one kernel per state"):
        S.dry_run_multi(lib, qs, MF.plan_of(qs, rows=125_000_000)[0])
    mq = mixed_panel()
    with pytest.raises(A.AresError, match=r"run 3 kernels, one kernel per group of states: \{0, 1\} direct-indexed, \{2\}, \{3\}$"):
        S.dry_run_multi(lib, mq, MF.plan_of(mq, rows=125_000_000, ranges=without_status(S.CFG3_RANGES))[0])


def test_one_state_with_member_dimensions_is_its_own_plan(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    import test_jit_codegen as J
    q = panel(1)[0]
    plan, _ = MF.plan_of([q], ranges=S.CFG3_RANGES)
    for i in range(plan.NumInsts):
        if plan.Insts[i].Sink == D:
            plan.Insts[i].Sink, plan.Insts[i].SinkArg = MD, 1
    assert S.dry_run_multi(lib, [q], plan)[1] == J._dry_run(lib, q, ranges=S.CFG3_RANGES)[1]


def test_member_dimension_errors_are_reported(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    qs = panel(3)
    plan, _ = MF.plan_of(qs, ranges=S.CFG3_RANGES)
    md = [i for i in range(plan.NumInsts) if plan.Insts[i].Sink == MD]
    assert [plan.Insts[i].SinkArg for i in md] == [0b011, 0b101]
    fn = lib.alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    h = fn(qs[0].agg_spec(), C.byref(plan), None)
    assert h.pStrErr and b"need ExecuteBatchPlanMulti" in C.string_at(h.pStrErr)

    def bad(edit, match):
        p = A.BatchPlan.from_buffer_copy(bytes(plan))
        edit(p)
        with pytest.raises(A.AresError, match=match):
            S.dry_run_multi(lib, qs, p)

    def zero(p): p.Insts[md[0]].SinkArg = 0
    def high(p): p.Insts[md[1]].SinkArg = 0b1001
    def mixed(p): p.Insts[md[1]].Sink, p.Insts[md[1]].SinkArg = D, 0
    def widths(p): p.Insts[md[1]].SinkArg = 0b111    # state 1 (count by hour) would get a 2-byte dimension as its second
    def after_measure(p):
        moved = [p.Insts[i] for i in range(plan.NumInsts) if i != md[1]]
        moved.append(A.PlanInst.from_buffer_copy(bytes(plan.Insts[md[1]])))
        for i, pi in enumerate(moved):
            p.Insts[i] = pi
    bad(zero, "empty state mask")
    bad(high, "state mask 9: there are 3 states")
    bad(mixed, "not both")
    bad(widths, "member dimension roots of state 1 do not match its NumDimsPerDimWidth")
    bad(after_measure, "precede the measure roots")
    # states that differ in their layout stay refused without member dimensions
    same = A.BatchPlan.from_buffer_copy(bytes(MF.plan_of(S.cfg3_request(2), ranges=S.CFG3_RANGES)[0]))
    with pytest.raises(A.AresError, match="states differ in NumDimsPerDimWidth"):
        S.dry_run_multi(lib, qs[:2], same)


def test_member_dimension_kernel_text_is_unchanged(monkeypatch):
    """The kernel text of the member dimension shapes is the one recorded when they were added."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    got = shape_digests(A.load_engine())
    want = json.loads(GOLDEN.read_text())
    assert sorted(got) == sorted(want)
    changed = [n for n in want if got[n] != want[n]]
    assert not changed, f"generated text changed for {changed}"


# ---- on the GPU: every member equals the same query run alone ------------------------------------------------------
def _run(eng, qs, batches, expected_groups=0):
    """MF._run on a request; also checks that the request forms one pass."""
    from aresdb_b200.executor import FusedRequestExecutor
    probe = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert probe.passes == [list(range(len(qs)))], probe.passes
    probe.close()
    return MF._run(eng, qs, batches, expected_groups)


@pytest.mark.gpu
@pytest.mark.parametrize("zone_maps", ["exact", "stale", "narrow", "none"])
def test_panel_on_edge_batches_equals_solo_runs(zone_maps):
    """NULL fares and cities (garbage under NULL), -0.0 / +0.0 fares; rows outside a too-narrow or stale zone map take the
    cold path of every member; without a zone map each member runs its own kernel."""
    import harness as H
    eng = H.get_backend("b200")
    per_batch, got = _run(eng, panel(), S._edge_batches(eng, zone_maps=zone_maps))
    assert per_batch == [(4, 0)] * 2 if zone_maps == "none" else all(p == (1, 1) for p in per_batch), per_batch
    assert all(r.groups > 0 for r in got)


@pytest.mark.gpu
@pytest.mark.parametrize("reduce_mode", [A.ARES_REDUCE_SORT, A.ARES_REDUCE_HASH], ids=["sort", "hash"])
@pytest.mark.parametrize("request_of", ["forms", "member_filters"])
def test_forms_and_member_filters_equal_solo_runs(request_of, reduce_mode):
    """Every accumulation form as a member with its own dimension set, and member filters with member dimensions, in
    both reduce modes, on day batches with NULLs."""
    import harness as H
    eng = H.get_backend("b200")
    qs = forms_panel(reduce_mode=reduce_mode) if request_of == "forms" else filtered_panel(reduce_mode)
    per_batch, _ = _run(eng, qs, S._edge_batches(eng, zone_maps="exact"))
    assert per_batch == [(1, 1), (1, 1)], per_batch


@pytest.mark.gpu
def test_launches_follow_the_form():
    """(1, 1) when the pass fits a CTA; one launch per dimension set when only the sets fit (300 cities); nothing when
    the zone map contradicts every member; a direct-indexed set next to members without a zone map: the kernels the dry
    run reports for each batch's plan."""
    import harness as H
    eng = H.get_backend("b200")
    batches = []
    for d in range(2):
        hb = synth.generate_batch(d, 200_000, num_cities=300, null_rate=0.01)
        batches.append(T.upload(eng, hb, 0, synth.zone_map_of_day(d, 300)))
    per_batch, _ = _run(eng, sets_panel(), batches)
    assert per_batch == [(2, 2), (2, 2)], per_batch
    big = E.gt(CITY, E.Lit(1000))
    gone = [AggQuery([big], [HOUR], Measure("count")), AggQuery([big, E.eq(STATUS, E.Lit(1))], [CITY], Measure("sum", FARE))]
    per_batch, got = _run(eng, gone, batches)
    assert per_batch == [(0, 0), (0, 0)] and all(r.groups == 0 for r in got), per_batch
    mixed, reported = mixed_panel(), []
    for b in batches:
        b.ranges = without_status(b.ranges)
        with pytest.raises(A.AresError) as e:
            S.dry_run_multi(eng.lib, mixed, MF.plan_of(mixed, rows=b.num_rows, ranges=b.ranges)[0])
        reported.append(int(re.search(r"run (\d+) kernels", str(e.value)).group(1)))
    per_batch, _ = _run(eng, mixed, batches)
    assert reported == [3, 3] and per_batch == [(k, 1) for k in reported], (reported, per_batch)


@pytest.mark.gpu
def test_rle_batches_and_an_all_tail_batch():
    """RLE archive batches (SUM / COUNT count run lengths, MAX does not) and a batch too small for a full tile."""
    import harness as H
    eng = H.get_backend("b200")
    rle = []
    for seed in (1, 2):
        b = T._archive_batch(eng, seed, 150000)
        b.ranges = {0: (T0, T0 + 3 * 86400), 1: (1, 40), 2: (0, 3)}
        rle.append(b)
    qs = [AggQuery([E.eq(STATUS, E.Lit(1))], [HOUR, CITY], Measure("sum", FARE)), AggQuery([], [HOUR], Measure("count")),
          AggQuery([], [CITY], Measure("max", FARE)), AggQuery([E.ne(STATUS, E.Lit(1))], [STATUS], Measure("sum", CITY))]
    per_batch, _ = _run(eng, qs, rle)
    assert [p[1] for p in per_batch] == [1, 1], per_batch
    hb = synth.generate_batch(0, 3000, num_cities=20, null_rate=0.05)
    _run(eng, panel(), [T.upload(eng, hb, 0, synth.zone_map(hb))])


@pytest.mark.gpu
def test_member_grouped_by_a_joined_column():
    """count(*) by a dimension-table column (no zone map) next to members by hour x city and by hour: the joined member
    runs its own kernel, the others share theirs."""
    import harness as H
    import test_joins as TJ
    eng = H.get_backend("b200")
    table, _ = TJ._dimension_table(eng)
    j = [Join(table, CITY)]
    f = [E.eq(STATUS, E.Lit(1))]
    qs = [AggQuery(f, [HOUR, CITY], Measure("sum", FARE), joins=j), AggQuery(f, [HOUR], Measure("count"), joins=j),
          AggQuery(f, [E.ForeignCol(0, 1, A.Uint8, "region")], Measure("count"), joins=j)]
    hbs = [synth.generate_batch(d, 30000, num_cities=80, null_rate=0.03) for d in range(2)]
    per_batch, got = _run(eng, qs, [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs])
    assert all(r.groups > 0 for r in got)
    assert all(k == 3 for k, _ in per_batch), per_batch


@pytest.mark.gpu
def test_one_member_outgrows_its_table():
    """A member grouped by the raw time under a zone map that claims 16 seconds: more than 2^20 groups arrive through its
    cold path (parked and grown per state) while the members by hour and by city stay small."""
    import harness as H
    eng = H.get_backend("b200")
    qs = [AggQuery([], [TS, CITY], Measure("count")), AggQuery([], [HOUR], Measure("sum", FARE)),
          AggQuery([E.eq(STATUS, E.Lit(1))], [CITY], Measure("max", CITY))]
    hb = synth.generate_batch(0, 1_500_000, num_cities=100, null_rate=0.0)
    zm = {**synth.zone_map(hb), 0: (T0, T0 + 15)}
    per_batch, got = _run(eng, qs, [T.upload(eng, hb, 0, zm)])
    assert per_batch == [(1, 1)] and got[0].groups > (1 << 20) and got[1].groups <= 25 and got[2].groups <= 101


def _aql_panels():
    from aresdb_b200 import aql
    table = aql.Table("trips", [aql.Column(n, t) for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)])
    frm, to = T0 + 86400 + 1800, T0 + 5 * 86400 - 1800
    hour = {"sqlExpression": "request_at", "timeBucketizer": "hour"}
    city = {"sqlExpression": "city_id"}

    def panel_(m, dims):
        return {"table": "trips", "measures": [{"sqlExpression": m, "rowFilters": ["status = 1"]}], "dimensions": dims,
                "timeFilter": {"column": "request_at", "from": str(frm), "to": str(to)}}
    request = {"queries": [panel_("count(*)", [hour]), panel_("sum(fare)", [city]), panel_("count(*)", [hour, city])]}
    return aql.compile_request(json.dumps(request), table, T0 + 30 * 86400)


@pytest.mark.gpu
def test_compiled_request_and_exchange():
    """A request compiled from JSON panels by hour, by city and by hour x city is one pass (archive.scan_shard); a pass
    dealt to two simulated ranks and exchanged equals the single-GPU result, and so does a 2-rank ShardedFusedRequest
    when two GPUs are present (ShardedFusedRequest without a process group otherwise)."""
    import harness as H
    import test_sharded_request as SR
    from aresdb_b200 import archive
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    from aresdb_b200.sharding import ShardedFusedRequest
    eng = H.get_backend("b200")
    qs = _aql_panels()
    day0, cutoff = T0 // 86400, T0 + 3 * 86400
    arch = {day0 + d: T.upload(eng, hb, 0, synth.zone_map(hb))
            for d, hb in enumerate(synth.generate_batch(d, 20000, num_cities=12, null_rate=0.02) for d in range(3))}
    live = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in (synth.generate_batch(3 + i, 25000, num_cities=12) for i in range(2))]
    req = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert len(req.groups) == 3 and req.passes == [[0, 1, 2]]
    k0, d0 = S._launches(eng)
    archive.scan_shard(req, live, arch, cutoff, qs[0].time_range, 0)
    k1, d1 = S._launches(eng)
    results = req.results()
    for q, got in zip(qs, results):
        ex = FusedBatchExecutor(eng.lib, eng.space, q)
        archive.scan_shard(ex, live, arch, cutoff, q.time_range, 0)
        S._same(got, ex.result(), q, f"archive scan {q.measure_kind}")
        assert got.groups > 0
        ex.close()
    assert d1 - d0 >= 1
    sharded = ShardedFusedRequest(eng.lib, eng.space, qs)
    archive.scan_shard(sharded, live, arch, cutoff, qs[0].time_range, 0)
    SR._same_results(qs, sharded.finalize(), results, "scan_shard")
    sharded.close()
    req.close()
    qs = panel()
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in (synth.generate_batch(d, 20000, num_cities=30) for d in range(4))]
    full = FusedRequestExecutor(eng.lib, eng.space, qs)
    locals_ = [FusedRequestExecutor(eng.lib, eng.space, qs) for _ in range(2)]
    for i, b in enumerate(batches):
        full.process_batch(b)
        locals_[i % 2].process_batch(b)
    expected = full.results()
    xqs, out = SR._exchange_on_one_device(eng, locals_, 32768, (1,))
    SR._check_exchange(xqs, out, expected, 32768, "W2")
    for ex in locals_ + [full]:
        ex.close()


if __name__ == "__main__":   # records the digests (run once, when the member dimension shapes were added)
    import os
    os.environ["ARESDB_B200_JIT_GENERATE_ONLY"] = "1"
    GOLDEN.write_text(json.dumps(shape_digests(A.load_engine()), indent=1, sort_keys=True) + "\n")
