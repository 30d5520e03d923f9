"""Distinct-count estimates on the device: AggStateFinalizeHLLEstimate / FusedBatchExecutor.hll_estimates give, for every
group of an hll query, the float64 that postprocess.hll_estimate (the reference's HLL.Compute, query/common/hll.go:735-775)
computes from that group's register vector, bit for bit.

CPU: the claim the kernel rests on (when every v = rho+1 of a group is <= 39, the float64 sum of 2^-v in the reference's
order is the exact sum), the fixture that shows why groups with a larger v take the ordered walk, the tie in the bias
window that decides which bias is subtracted, and the library's copy of the bias tables.
GPU: the estimates of real queries (both state forms, zone maps, RLE batches, no groups), of register sets injected
through AggStateMerge at every edge of HLL.Compute, nested AQL results, the two-rank exchange, reuse after a reset, the
error strings, and two queries at size."""
import ctypes as C
import re
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

from aresdb_b200 import cabi as A
from aresdb_b200 import expr as E
from aresdb_b200 import synth
from aresdb_b200.hll_bias_p14 import BIASES, RAW_ESTIMATES
from aresdb_b200.postprocess import HLL_THRESHOLD, hll_estimate, hll_estimate_bias, hll_nested_result, nested_result
from aresdb_b200.query import AggQuery, Measure

ROOT = Path(__file__).resolve().parent.parent
M = 16384
M_F = float(M)
ALPHA_MM = 0.7213 / (1 + 1.079 / M_F) * M_F * M_F    # HLL.Compute's numerator, in its order
UNIT = 2.0 ** -39                                   # the integer sum counts units of 2^-39


# ---- the host-side facts -------------------------------------------------------------------------------------------
def go_order_sum(dense: np.ndarray) -> float:
    """The float64 sum of hll_estimate: sparse (< 4096 hit registers) in register order then m - nonzero; dense over all
    16384 registers in order."""
    nonzero = int(np.count_nonzero(dense))
    s = 0.0
    if nonzero < M // 4:
        for r in dense.tolist():
            if r:
                s += 1.0 / float(1 << r)
        return s + (M_F - nonzero)
    for r in dense.tolist():
        s += 1.0 / float(1 << r)
    return s


def exact_sum(dense: np.ndarray) -> Fraction:
    n = np.bincount(dense, minlength=256)
    return sum(Fraction(int(c), 1 << v) for v, c in enumerate(n) if c)


def registers_for_units(units: int, rng, n: int = M) -> np.ndarray:
    """n registers, all hit (v in 1..39), whose sum of 2^-v is units * 2^-39: the binary digits of the sum, then the
    largest terms split in two until there are n of them.  Shuffled (the order of a sum of such terms does not matter)."""
    counts, rem = [0] * 40, units
    counts[1], rem = rem // (1 << 38), rem % (1 << 38)
    for v in range(2, 40):
        if rem >= 1 << (39 - v):
            counts[v], rem = 1, rem - (1 << (39 - v))
    assert rem == 0 and sum(counts) <= n, "no such register set"
    total = sum(counts)
    while total < n:
        v = next(v for v in range(1, 39) if counts[v])
        k = min(counts[v], n - total)
        counts[v] -= k
        counts[v + 1] += 2 * k
        total += k
    out = np.concatenate([np.full(c, v, np.uint8) for v, c in enumerate(counts) if c])
    rng.shuffle(out)
    return out


def hits(n: int, rng, vmax: int = 20) -> np.ndarray:
    """n hit registers at random places, v from a geometric law (what hashing gives) capped at vmax."""
    dense = np.zeros(M, np.uint8)
    regs = rng.choice(M, n, replace=False)
    dense[regs] = np.minimum(rng.geometric(0.5, n), vmax).astype(np.uint8)
    return dense


def estimate_of_sum(s: float, nonzero: int) -> float:
    """hll_estimate's steps after the sum."""
    import math
    e = ALPHA_MM / s
    if e <= 5.0 * M_F:
        e -= hll_estimate_bias(e)
    h = M_F * math.log(M_F / (M_F - nonzero)) if nonzero < M else e
    return float(int(h if h <= HLL_THRESHOLD else e))


FALLBACK = ROOT / "tests" / "golden" / "hll_fallback_registers.npy"
# A sum of 2^-39 units whose raw estimate lies equally far (after rounding the squares) from RAW_ESTIMATES[60] and [66],
# the 6th and 7th nearest entries: the tie order decides which bias is subtracted.
TIE_UNITS, TIE_LOW = 3707410371442175, 60


def test_go_order_sum_is_the_exact_sum_up_to_v39():
    """Every partial sum is a multiple of 2^-39 no larger than 2^14: 53 bits, so each addition is exact."""
    rng = np.random.default_rng(7)
    sets = [hits(n, rng, vmax) for n in (1, 17, 4095, 4096, 9000, 16384) for vmax in (20, 39)]
    sets += [np.full(M, 39, np.uint8), np.where(np.arange(M) % 2 == 0, 0, 39).astype(np.uint8),
             np.where(np.arange(M) % 2 == 0, 1, 39).astype(np.uint8), np.concatenate([np.full(4095, 39, np.uint8), np.zeros(M - 4095, np.uint8)]),
             np.concatenate([np.zeros(M - 4096, np.uint8), np.full(4096, 39, np.uint8)]),
             np.concatenate([np.full(M // 2, 1, np.uint8), np.full(M // 2, 39, np.uint8)])]
    sets += [registers_for_units(int(u), rng) for u in rng.integers(M, 8192 * 2 ** 39, 4)]
    for dense in sets:
        assert int(dense.max()) <= 39
        assert Fraction(go_order_sum(dense)) == exact_sum(dense)
        assert exact_sum(dense) == Fraction(int(exact_sum(dense) / Fraction(UNIT)), 1) * Fraction(UNIT)


def test_fallback_fixture_needs_the_reference_order():
    """The fixture: 8192 registers of v = 1, a few tuning registers, then 7800 of v = 42, each a quarter of an ulp of the
    running sum in the reference's order and so lost.  Its ordered sum is not the correctly rounded exact sum, and the
    estimates of the two differ (46000 vs 45999)."""
    dense = np.load(FALLBACK)
    assert dense.dtype == np.uint8 and dense.size == M and int(dense.max()) >= 40
    go, exact = go_order_sum(dense), exact_sum(dense)
    assert go != float(exact)
    assert hll_estimate(dense) == estimate_of_sum(go, M) == 46000.0
    assert estimate_of_sum(float(exact), M) == 45999.0


def test_tie_in_the_bias_window_decides_the_estimate():
    import bisect
    s = TIE_UNITS * UNIT
    e = ALPHA_MM / s
    lo, hi = RAW_ESTIMATES[TIE_LOW], RAW_ESTIMATES[TIE_LOW + 6]
    assert (lo - e) ** 2 == (hi - e) ** 2 and (lo - e) * (lo - e) == (hi - e) * (hi - e)
    i = bisect.bisect_right(RAW_ESTIMATES, e)
    assert max(i - 7, 0) <= TIE_LOW and TIE_LOW + 6 < min(i + 6, len(RAW_ESTIMATES))
    # the smaller index wins: the other order subtracts another bias and truncates to another count
    later = sorted(((RAW_ESTIMATES[j] - e) ** 2, -j) for j in range(max(i - 7, 0), min(i + 6, len(RAW_ESTIMATES))))
    other = sum(BIASES[-j] for _, j in later[:6]) / 6.0
    assert float(int(e - other)) != float(int(e - hll_estimate_bias(e)))
    dense = registers_for_units(TIE_UNITS, np.random.default_rng(3))
    assert hll_estimate(dense) == float(int(e - hll_estimate_bias(e)))


def test_library_bias_tables_are_the_published_data():
    src = (ROOT / "aresdb_b200" / "csrc" / "hll_estimate.cu").read_text()

    def table(name):
        body = re.search(name + r"\[kBiasEntries\] = \{(.*?)\};", src, re.S).group(1)
        return tuple(float(x) for x in body.replace("\n", " ").split(",") if x.strip())
    assert table("cRawEstimates") == tuple(RAW_ESTIMATES)
    assert table("cBiases") == tuple(BIASES)


# ---- GPU -----------------------------------------------------------------------------------------------------------
ENTRY_MODE, DENSE_MODE = 100000, 0   # AggSpec.ExpectedGroups: (group, register) entries / dense register arrays


def _check(est, res, ctx, sample=None):
    """HLLEstimates vs the HLLResult of the same state: same groups and dimension rows in the same order, and every
    estimate (or those of `sample`) equal to hll_estimate of its registers."""
    assert est.groups == res.groups, ctx
    assert est.rows == res.dims.rows, f"{ctx}: groups differ"
    assert est.measures.dtype == np.float64
    dense = res.dense_registers()
    for g in (range(res.groups) if sample is None else sample):
        want = hll_estimate(dense[res.dims.rows[g]])
        assert est.measures[g] == want, f"{ctx}: group {g}: {est.measures[g]!r} != {want!r}"


def _fused(eng, q, batches, mode):
    from aresdb_b200.executor import FusedBatchExecutor
    ex = FusedBatchExecutor(eng.lib, eng.space, q, mode)
    for b in batches:
        ex.process_batch(b)
    return ex


@pytest.mark.gpu
@pytest.mark.parametrize("zone_maps", [False, True], ids=["plain", "zonemap"])
@pytest.mark.parametrize("mode", [ENTRY_MODE, DENSE_MODE], ids=["entries", "dense"])
def test_estimates_of_the_pipeline_queries(mode, zone_maps):
    import harness as H
    import test_hll_pipeline as HP
    import test_pipeline_parity as T
    eng = H.get_backend("b200")
    hbs = [synth.generate_batch(day, rows, num_cities=50, null_rate=0.02) for day, rows in HP.BATCHES]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb) if zone_maps else None) for hb in hbs]
    for name, q in HP.hll_queries().items():
        ex = _fused(eng, q, batches, mode)
        res = ex.hll_result()
        assert res.groups > 0
        if name == "dense_by_status":
            assert (res.counts >= 4096).any() and (res.counts < 4096).any()
        _check(ex.hll_estimates(), res, f"{name}/{mode}/{zone_maps}")
        ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [ENTRY_MODE, DENSE_MODE], ids=["entries", "dense"])
def test_estimates_on_rle_batches(mode):
    import harness as H
    import test_pipeline_parity as T
    eng = H.get_backend("b200")
    q = AggQuery([], [T.CITY], Measure("countdistincthll", T.TS))
    ex = _fused(eng, q, [T._archive_batch(eng, seed, 150000) for seed in (1, 2)], mode)
    res = ex.hll_result()
    assert res.groups > 0
    _check(ex.hll_estimates(), res, f"rle/{mode}")
    ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [ENTRY_MODE, DENSE_MODE], ids=["entries", "dense"])
def test_no_groups(mode):
    import harness as H
    import test_pipeline_parity as T
    eng = H.get_backend("b200")
    q = AggQuery([E.eq(T.STATUS, E.Lit(99))], [T.CITY], Measure("countdistincthll", T.TS))
    ex = _fused(eng, q, [T.upload(eng, synth.generate_batch(0, 5000))], mode)
    est = ex.hll_estimates()
    assert est.groups == 0 and est.measures.size == 0 and nested_result(est) == {}
    ex.close()


def _crafted_sets():
    """Register sets at the edges of HLL.Compute: the sparse / dense boundary, full saturation, a stride over the hit
    counts, v = 51, the fallback fixture, raw estimates either side of 5m, linear counting either side of 15500, bias
    windows clipped at both ends of the table, and the tie."""
    import math
    rng = np.random.default_rng(11)
    sets = [hits(n, rng) for n in (1, 4095, 4096, M)] + [hits(n, rng) for n in range(1, M, 397)]
    v51 = hits(5000, rng)
    v51[rng.choice(np.nonzero(v51)[0], 3, replace=False)] = 51
    sparse51 = hits(300, rng)
    sparse51[np.nonzero(sparse51)[0][0]] = 51
    sets += [v51, sparse51, np.load(FALLBACK)]
    five_m = int(ALPHA_MM / (5.0 * M_F) / UNIT)             # raw estimate 5m
    sets += [registers_for_units(five_m + d, rng) for d in (-4000, -1, 1, 4000)]
    n_lc = next(n for n in range(1, M) if M_F * math.log(M_F / (M_F - n)) > HLL_THRESHOLD)
    sets += [hits(n, rng) for n in (n_lc - 1, n_lc)]
    sets += [hits(200, rng, 3), hits(1000, rng, 2)]           # raw estimates below RAW_ESTIMATES[6]: window clipped low
    top = (RAW_ESTIMATES[-3] + RAW_ESTIMATES[-2]) / 2        # window clipped high
    sets += [registers_for_units(int(ALPHA_MM / top / UNIT), rng)]
    sets += [registers_for_units(TIE_UNITS, rng)]
    return sets


def _inject(eng, q, sets, mode):
    """One group per set (dimension value k + 1), its hit registers as carried (group, rho << 16 | reg) rows folded by
    AggStateMerge — the rows the exact-size exchange feeds an HLL state with."""
    from aresdb_b200.executor import FusedBatchExecutor, _ResultBuffers, dim_offsets
    groups, vals = [], []
    for k, dense in enumerate(sets):
        regs = np.nonzero(dense)[0].astype(np.uint32)
        groups.append(np.full(regs.size, k + 1, np.uint16))
        vals.append(((dense[regs].astype(np.uint32) - 1) << 16) | regs)
    g, v = np.concatenate(groups), np.concatenate(vals)
    n = g.size
    offs, nulls, _, total = dim_offsets(q.num_dims_per_width, n)
    block = np.zeros(total, np.uint8)
    block[offs[0]:offs[0] + 2 * n] = g.view(np.uint8)
    block[nulls[0]:nulls[0] + n] = 1
    buf = _ResultBuffers(eng.space, q, n)
    dims, meas = eng.put(block), eng.put(v)
    eng.lib.AsyncCopyDeviceToDevice(buf.dims.ptr, dims.ptr, total, eng.space.stream, 0)
    eng.lib.AsyncCopyDeviceToDevice(buf.measures.ptr, meas.ptr, 4 * n, eng.space.stream, 0)
    ex = FusedBatchExecutor(eng.lib, eng.space, q, mode)
    ex.merge(buf.dimension_vector(q), buf.measures.ptr, n)
    eng.lib.WaitForCudaStream(eng.space.stream, 0)
    return ex, (dims, meas, buf)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [ENTRY_MODE, DENSE_MODE], ids=["entries", "dense"])
def test_crafted_register_sets(mode):
    import harness as H
    import test_pipeline_parity as T
    eng = H.get_backend("b200")
    q = AggQuery([], [T.CITY], Measure("countdistincthll", T.TS))
    sets = _crafted_sets()
    ex, keep = _inject(eng, q, sets, mode)
    est, res = ex.hll_estimates(), ex.hll_result()
    assert est.groups == len(sets)
    dense = res.dense_registers()
    city = est.decoded_dims()[0]
    for g in range(est.groups):
        want = sets[city[g] - 1]
        assert np.array_equal(dense[res.dims.rows[g]], want), f"group {g}: registers were not injected as crafted"
        assert est.measures[g] == hll_estimate(want), f"set {city[g] - 1}: {est.measures[g]!r} != {hll_estimate(want)!r}"
    ex.close()


@pytest.mark.gpu
def test_nested_aql_result_with_time_enum_and_null_dimensions():
    import harness as H
    import test_pipeline_parity as T
    from aresdb_b200 import aql
    from aresdb_b200.executor import FusedRequestExecutor
    from aresdb_b200.postprocess import DimensionMeta
    eng = H.get_backend("b200")
    names = ["requested", "accepted", "completed", "cancelled"]
    cols = [aql.Column(n, t, enum={s: i for i, s in enumerate(names)} if n == "status" else None)
            for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)]
    table = aql.Table("trips", cols)
    text = {"table": "trips", "measures": [{"sqlExpression": "countdistincthll(request_at)"}],
            "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "day"}, {"sqlExpression": "status"},
                           {"sqlExpression": "city_id"}]}
    q = aql.compile_query(text, table, synth.BASE_TS + 30 * 86400)
    metas = [DimensionMeta(time_bucketizer="day"), DimensionMeta(enum_names=names), None]
    batches = [T.upload(eng, synth.generate_batch(d, 30000, num_cities=20, null_rate=0.05)) for d in range(2)]
    for mode in (ENTRY_MODE, DENSE_MODE):
        req = FusedRequestExecutor(eng.lib, eng.space, [q], mode)
        for b in batches:
            req.process_batch(b)
        got = nested_result(req.results(hll_estimates=True)[0], metas)
        want = hll_nested_result(req.executors[0].hll_result(), metas)
        assert got == want

        def keys(d, depth):
            return set(d) if depth == 0 else set().union(*(keys(v, depth - 1) for v in d.values()))
        assert "NULL" in keys(got, 0) | keys(got, 1) | keys(got, 2)
        assert keys(got, 1) - {"NULL"} <= set(names) and len(keys(got, 0)) >= 2
        req.close()


@pytest.mark.gpu
def test_exchange_between_simulated_ranks_and_sharded_results():
    """Two ranks' carried rows merged into one state (the exact-size exchange of an HLL query) estimate what the whole
    query run on one state estimates; ShardedFusedRequest / ShardedFusedQuery without a process group give the same."""
    import harness as H
    import test_hll_pipeline as HP
    import test_pipeline_parity as T
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    from aresdb_b200.sharding import ShardedFusedQuery, ShardedFusedRequest
    eng = H.get_backend("b200")
    q = HP.hll_queries()["two_dims"]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in (synth.generate_batch(d, 20000, num_cities=30) for d in range(4))]
    for mode in (ENTRY_MODE, DENSE_MODE):
        full = _fused(eng, q, batches, mode)
        ranks = [_fused(eng, q, batches[r::2], mode) for r in range(2)]
        merged = FusedBatchExecutor(eng.lib, eng.space, q, mode)
        for ex in ranks:
            g, o = ex.finalize_into()
            merged.merge(o.dimension_vector(q), o.measures.ptr, g)
        want, res = full.hll_estimates(), full.hll_result()
        _check(want, res, f"whole/{mode}")
        got = merged.hll_estimates()
        assert got.rows == want.rows and np.array_equal(got.measures, want.measures), mode
        for x in ranks + [merged, full]:
            x.close()
    qs = [T.queries()["cfg3_sum"], q]
    req, ref = ShardedFusedRequest(eng.lib, eng.space, qs), FusedRequestExecutor(eng.lib, eng.space, qs)
    one = ShardedFusedQuery(eng.lib, eng.space, q)
    for b in batches:
        req.process_batch(b)
        ref.process_batch(b)
        one.process_batch(b)
    want = ref.results(hll_estimates=True)[1]
    for got in (req.finalize(hll_estimates=True)[1], one.finalize_hll(hll_estimates=True)):
        assert got.rows == want.rows and np.array_equal(got.measures, want.measures)
    assert type(ref.results()[1]).__name__ == "QueryResult" and type(req.finalize()[1]).__name__ == "HLLResult"
    for x in (req, ref, one):
        x.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [ENTRY_MODE, DENSE_MODE], ids=["entries", "dense"])
def test_estimates_after_reset_and_another_batch(mode):
    import harness as H
    import test_hll_pipeline as HP
    import test_pipeline_parity as T
    eng = H.get_backend("b200")
    q = HP.hll_queries()["sparse_by_city"]
    b0, b1 = (T.upload(eng, synth.generate_batch(d, 40000, num_cities=40)) for d in (0, 1))
    ex = _fused(eng, q, [b0], mode)
    first = ex.hll_estimates()
    ex.reset()
    ex.process_batch(b1)
    est, res = ex.hll_estimates(), ex.hll_result()
    _check(est, res, f"reset/{mode}")
    fresh = _fused(eng, q, [b1], mode)
    again = fresh.hll_estimates()
    assert est.rows == again.rows and np.array_equal(est.measures, again.measures)
    assert first.rows != est.rows or not np.array_equal(first.measures, est.measures)
    ex.close()
    fresh.close()


@pytest.mark.gpu
def test_error_strings():
    import harness as H
    import test_hll_pipeline as HP
    import test_pipeline_parity as T
    from aresdb_b200.executor import FusedBatchExecutor
    eng = H.get_backend("b200")
    plain = FusedBatchExecutor(eng.lib, eng.space, T.queries()["cfg3_sum"])
    hll = FusedBatchExecutor(eng.lib, eng.space, HP.hll_queries()["two_dims"])
    d, e = C.c_void_p(), C.c_void_p()
    with pytest.raises(A.AresError, match="AggStateFinalizeHLLEstimate: .*needs a state created with AGGR_HLL"):
        eng.lib.AggStateFinalizeHLLEstimate(plain.state, C.byref(d), C.byref(e), eng.space.stream, 0)
    for args in ((None, C.byref(e)), (C.byref(d), None)):
        with pytest.raises(A.AresError, match="AggStateFinalizeHLLEstimate: null output pointer"):
            eng.lib.AggStateFinalizeHLLEstimate(hll.state, *args, eng.space.stream, 0)
    plain.close()
    hll.close()


@pytest.mark.gpu
def test_cfg4_hll_at_size():
    """cfg4 HLL (dense form) over 2 x 1.25e8 rows: every group."""
    import test_at_size as S
    ex, _, _ = S._run("cfg4_hll", S.BATCH_ROWS, 2, True)
    res = ex.hll_result()
    assert res.groups >= 200 and (res.counts >= 4096).any()
    _check(ex.hll_estimates(), res, "cfg4_hll")
    ex.close()


@pytest.mark.gpu
def test_hour_by_city_entries_form_at_size():
    """countdistincthll(request_at) by hour x city over 8 days (19,200 groups, entries form): 2,000 sampled groups and
    every group holding a register with v >= 40.  An hour holds at most 3,600 distinct request_at values, so every vector
    is sparse."""
    import torch
    import harness as H
    import test_at_size as S
    from aresdb_b200.executor import Batch
    eng = H.get_backend("b200")
    dev = torch.device("cuda:0")
    ts = E.Col(0, A.Uint32)
    q = AggQuery([], [E.floor(ts, E.Lit(3600)), E.Col(1, A.Uint16)], Measure("countdistincthll", ts))
    ex = _fused(eng, q, [], ENTRY_MODE)
    keep = []
    rows = 12_500_000
    for d in range(8):
        bufs, voff, cols = S._batch(d, rows, dev, null_rate=0.0)
        keep.append(bufs)
        ex.process_batch(Batch(cols, rows))
    res = ex.hll_result()
    assert res.groups == 8 * 24 * 100
    assert (res.counts > 1000).all() and (res.counts < 4096).all()
    dense = res.dense_registers()
    high = [g for g in range(res.groups) if int(dense[res.dims.rows[g]].max()) >= 40]
    sample = sorted(set(np.random.default_rng(5).choice(res.groups, 2000, replace=False).tolist()) | set(high))
    _check(ex.hll_estimates(), res, "hour x city", sample)
    ex.close()
