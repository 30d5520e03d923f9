"""One AQL request on several GPUs: AggStatesFinalize / AggStatesExportPartsToPeers / AggStatesMergeParts serve all of a
request's states with one launch each, and ShardedFusedRequest runs a rank's share of the request on them.

CPU: the slot layout of a request and the refusal of invalid requests before any device call.
GPU, one device: the K-state finalize equals per-state AggStateFinalize byte for byte; simulated ranks exchange through
receive buffers on one device (two epochs, truncated sub-parts, the all-gather form); ShardedFusedRequest without a
process group equals FusedRequestExecutor; every ABI rejection.  GPU, two devices: NCCL ranks over peer memory and over
the all-gather."""
import ctypes as C
import hashlib
import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from aresdb_b200 import cabi as A  # noqa: E402
from aresdb_b200 import expr as E  # noqa: E402
from aresdb_b200 import synth  # noqa: E402
from aresdb_b200.query import AggQuery, Measure  # noqa: E402
import test_pipeline_parity as T  # noqa: E402

FLAGS_PER_PARITY = 16 * 16 * 4


def _request():
    """Two shared-scan groups with different dimensions, one solo query (hash reduce) and one HLL query."""
    import test_hll_pipeline as HP
    q = T.queries()["cfg3_sum"]
    hour_city = [E.floor(T.TS, E.Lit(3600)), T.CITY]
    return [AggQuery(q.filters, hour_city, Measure("sum", T.FARE)), AggQuery(q.filters, hour_city, Measure("count")),
            AggQuery(q.filters, [T.CITY], Measure("max", T.CITY)), AggQuery(q.filters, [T.CITY], Measure("avg", T.FARE)),
            T.queries()["cfg4_hash"], HP.hll_queries()["two_dims"]]


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_slot_layout_is_aligned_and_sized_per_query():
    from aresdb_b200.executor import dim_offsets
    from aresdb_b200.sharding import request_slot_layout
    qs = [q for q in _request() if not q.is_hll] + [T.queries()["no_dims_wide"]]
    for cap in (64, 1000, 32768):
        parts, dims, values, slot = request_slot_layout(qs, cap)
        assert slot % 16 == 0
        end = 0
        for q, p, d, v in zip(qs, parts, dims, values):
            assert p % 16 == 0 and d % 16 == 0 and v % 16 == 0
            assert p >= end and d >= 16
            _, _, _, dim_bytes = dim_offsets(q.num_dims_per_width, cap)
            assert v >= d + dim_bytes and v - d - dim_bytes < 16
            end = p + v + q.measure_bytes * cap
        assert end <= slot


def test_invalid_requests_are_refused_before_any_device_call():
    from aresdb_b200.sharding import ShardedFusedRequest
    q = T.queries()["cfg3_sum"]
    # lib / space None: any device call would fail with an AttributeError instead
    with pytest.raises(ValueError, match="1..16 queries"):
        ShardedFusedRequest(None, None, [])
    with pytest.raises(ValueError, match="1..16 queries"):
        ShardedFusedRequest(None, None, [q] * 17)
    with pytest.raises(TypeError, match="AggQuery"):
        ShardedFusedRequest(None, None, [q, "sum(fare)"])
    for eg in (-1, [0], [0, -5], 1.5, True):
        with pytest.raises(ValueError, match="expected_groups"):
            ShardedFusedRequest(None, None, [q, q], eg)


# ---- GPU, one device ---------------------------------------------------------------------------------------------------
def _run(eng, q, batches, expected_groups=0):
    from aresdb_b200.executor import FusedBatchExecutor
    ex = FusedBatchExecutor(eng.lib, eng.space, q, expected_groups)
    for b in batches:
        ex.process_batch(b)
    return ex


def _states_finalize(eng, exs, caps):
    from aresdb_b200.executor import _ResultBuffers
    n = len(exs)
    bufs = [_ResultBuffers(eng.space, ex.q, c) for ex, c in zip(exs, caps)]
    groups = (C.c_int64 * n)()
    eng.lib.AggStatesFinalize((C.c_void_p * n)(*[ex.state.value for ex in exs]), n,
                              (A.DimensionVector * n)(*[b.dimension_vector(ex.q) for b, ex in zip(bufs, exs)]),
                              (C.c_void_p * n)(*[b.measures.ptr for b in bufs]), groups, eng.space.stream, 0)
    return list(groups), bufs


def _same_bytes(a, b, ctx):
    for f in ("dims", "hash", "measures"):
        assert np.array_equal(getattr(a, f).get(np.uint8), getattr(b, f).get(np.uint8)), f"{ctx}: {f} differ"


@pytest.mark.gpu
def test_states_finalize_equals_per_state_finalize():
    """cfg3 sum / count / avg / max, a hash-identity state, a state with 0 groups, one with more than 32768 groups (and one
    announcing more), and one with parked rows: AggStatesFinalize writes what AggStateFinalize writes, byte for byte."""
    import harness as H
    import test_shared_scan as S
    from aresdb_b200.executor import _ResultBuffers
    eng = H.get_backend("b200")
    hbs = [synth.generate_batch(d, 20000, num_cities=30) for d in range(3)]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs]
    big = T.upload(eng, synth.generate_batch(0, 200_000, num_cities=100, null_rate=0.0))
    hb = synth.generate_batch(0, 1_500_000, num_cities=100, null_rate=0.0)
    parked = T.upload(eng, hb, 0, {**synth.zone_map(hb), 0: (synth.BASE_TS, synth.BASE_TS + 15)})
    raw = AggQuery([], [T.TS, T.CITY], Measure("count"))
    exs = [_run(eng, q, batches) for q in S.cfg3_request(4)] + [_run(eng, T.queries()["cfg4_hash"], batches[:1]),
                                                              _run(eng, T.queries()["cfg3_count"], [])]
    small = len(exs)
    exs += [_run(eng, raw, [big]), _run(eng, raw, [big], 100000), _run(eng, AggQuery([], [T.TS, T.CITY], Measure("sum", T.FARE)), [parked])]
    caps = [32768] * small + [200_000, 200_000, 1_500_000]
    groups, bufs = _states_finalize(eng, exs, caps)
    assert groups[small - 1] == 0 and groups[small] > 32768 and groups[-1] > (1 << 20)
    for k, (ex, cap) in enumerate(zip(exs, caps)):
        ref = _ResultBuffers(eng.space, ex.q, cap)
        g = eng.lib.AggStateFinalize(ex.state, ref.dimension_vector(ex.q), ref.measures.ptr, eng.space.stream, 0)
        assert g == groups[k], k
        _same_bytes(bufs[k], ref, f"state {k}")
    # every state in the one-launch form: one kernel launch in all
    k0 = eng.lib.kernel_launch_count()
    groups2, _ = _states_finalize(eng, exs[:small], caps[:small])
    assert eng.lib.kernel_launch_count() - k0 == 1
    assert groups2 == groups[:small]
    for ex in exs:
        ex.close()


def _exchange_on_one_device(eng, locals_, cap, epochs, local_form=False):
    """Every simulated rank r exports its states (one AggStatesExportPartsToPeers) into every rank's receive buffer, then
    each rank folds its buffer (one AggStatesMergeParts) into fresh states and finalizes them (one AggStatesFinalize).
    Returns, per epoch and rank, the finalize outcome of every state and the part headers."""
    import torch
    from aresdb_b200.executor import FusedBatchExecutor, finalize_states
    from aresdb_b200.sharding import request_slot_layout
    W, dev, st = len(locals_), eng.space.dev, eng.space.stream
    exs = [[ex for ex in loc.executors if not ex.q.is_hll] for loc in locals_]
    qs, k = [ex.q for ex in exs[0]], len(exs[0])
    parts, dims, values, slot = request_slot_layout(qs, cap)
    po, do, vo = ((C.c_size_t * k)(*x) for x in (parts, dims, values))
    bufs = [torch.zeros(2 * FLAGS_PER_PARITY + 2 * W * slot, dtype=torch.uint8, device=dev) for _ in range(W)]
    out = []
    for epoch in epochs:
        par = epoch & 1
        base, fbase = 2 * FLAGS_PER_PARITY + par * W * slot, par * FLAGS_PER_PARITY
        for r in range(W):
            states = (C.c_void_p * k)(*[ex.state.value for ex in exs[r]])
            if local_form:   # the parts as an all-gather leaves them: rank r's slot at r * slot of one buffer
                mine = (C.c_void_p * 1)(bufs[0].data_ptr() + base + r * slot)
                eng.lib.AggStatesExportPartsToPeers(states, k, mine, None, 1, 0, slot, cap, po, do, vo, 0, st, 0)
            else:
                slots = (C.c_void_p * W)(*[bufs[p].data_ptr() + base + r * slot for p in range(W)])
                flags = (C.c_void_p * W)(*[bufs[p].data_ptr() + fbase + r * 4 for p in range(W)])
                eng.lib.AggStatesExportPartsToPeers(states, k, slots, flags, W, r, slot, cap, po, do, vo, epoch, st, 0)
        per_rank = []
        for r in range(1 if local_form else W):
            merged = [FusedBatchExecutor(eng.lib, eng.space, q) for q in qs]
            ms = (C.c_void_p * k)(*[m.state.value for m in merged])
            flags = None if local_form else bufs[r].data_ptr() + fbase
            eng.lib.AggStatesMergeParts(ms, k, bufs[r].data_ptr() + base, W, slot, cap, po, do, vo, flags, epoch, st, 0)
            res = finalize_states(merged)
            raw = bufs[r][base:base + W * slot].view(W, slot).cpu().numpy()
            claimed = [[int(raw[p, parts[j] + 8:parts[j] + 12].view(np.uint32)[0]) for p in range(W)] for j in range(k)]
            per_rank.append((merged, res, claimed))
        out.append(per_rank)
    return qs, out


def _check_exchange(qs, out, expected, cap, ctx):
    from aresdb_b200.executor import query_result
    import test_shared_scan as S
    for e, per_rank in enumerate(out):
        for r, (merged, res, claimed) in enumerate(per_rank):
            for j, q in enumerate(qs):
                c = f"{ctx}/epoch{e}/rank{r}/query{j}"
                if max(claimed[j]) > cap:
                    assert isinstance(res[j], A.AresError) and "exchange part truncated" in str(res[j]), c
                else:
                    assert not isinstance(res[j], Exception), f"{c}: {res[j]}"
                    S._same(query_result(q, *res[j]), expected[j], q, c)
            for m in merged:
                m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_exchange_of_a_request_between_simulated_ranks(world):
    """Batches dealt round-robin to `world` FusedRequestExecutors; one export, one merge and one finalize per rank give
    every rank the results of one FusedRequestExecutor over all batches, over two epochs on alternating buffers; with
    64-row sub-parts only the states with more groups report a truncated part; the all-gather form (no flags) agrees."""
    import harness as H
    from aresdb_b200.executor import FusedBatchExecutor, FusedRequestExecutor
    eng = H.get_backend("b200")
    qs = _request()
    hbs = [synth.generate_batch(d, 20000, num_cities=30) for d in range(5)]
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in hbs]
    full = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert len(full.groups) == 4   # {sum, count} by hour and city, {max, avg} by city, the hash query, the HLL query
    locals_ = [FusedRequestExecutor(eng.lib, eng.space, qs) for _ in range(world)]
    for i, b in enumerate(batches):
        full.process_batch(b)
        locals_[i % world].process_batch(b)
    expected = full.results()
    plain = [e for q, e in zip(qs, expected) if not q.is_hll]
    for cap in (32768, 64):
        xqs, out = _exchange_on_one_device(eng, locals_, cap, (1, 2))
        _check_exchange(xqs, out, plain, cap, f"W{world}/cap{cap}")
        if cap == 64:   # the small states fit, the hour x city ones do not
            claimed = out[0][0][2]
            assert any(max(c) > 64 for c in claimed) and any(max(c) <= 64 for c in claimed)
    xqs, out = _exchange_on_one_device(eng, locals_, 32768, (1,), local_form=True)
    _check_exchange(xqs, out, plain, 32768, f"W{world}/all-gather")
    # the HLL query keeps the exact protocol: carried rows of every rank merged into one state
    h = [i for i, q in enumerate(qs) if q.is_hll][0]
    merged = FusedBatchExecutor(eng.lib, eng.space, qs[h])
    for loc in locals_:
        g, o = loc.executors[h].finalize_into()
        merged.merge(o.dimension_vector(qs[h]), o.measures.ptr, g)
    got, exp = merged.hll_result().dense_registers(), full.executors[h].hll_result().dense_registers()
    assert got.keys() == exp.keys() and all(np.array_equal(got[k], exp[k]) for k in exp)
    merged.close()
    for ex in locals_ + [full]:
        ex.close()


def _same_results(qs, got, exp, ctx):
    import test_shared_scan as S
    for i, q in enumerate(qs):
        if q.is_hll:
            g, e = got[i].dense_registers(), exp[i].dense_registers()
            assert g.keys() == e.keys() and all(np.array_equal(g[k], e[k]) for k in e), f"{ctx}/query{i}"
        else:
            S._same(got[i], exp[i], q, f"{ctx}/query{i}")


@pytest.mark.gpu
def test_request_without_process_group_equals_request_executor():
    """world == 1: ShardedFusedRequest gives FusedRequestExecutor's results (HLLResults for HLL queries), for plain batches
    and for a shard scan (live batches behind the cutoff filter, then the archive days); so does a ShardedFusedQuery per
    query of the request."""
    import harness as H
    from aresdb_b200 import aql, archive
    from aresdb_b200.executor import FusedRequestExecutor, query_result
    from aresdb_b200.sharding import ShardedFusedQuery, ShardedFusedRequest
    eng = H.get_backend("b200")
    qs = _request()
    batches = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in (synth.generate_batch(d, 20000, num_cities=30) for d in range(3))]
    req, ref = ShardedFusedRequest(eng.lib, eng.space, qs), FusedRequestExecutor(eng.lib, eng.space, qs)
    for b in batches:
        req.process_batch(b)
        ref.process_batch(b)
    exp = [ex.hll_result() if q.is_hll else r for q, ex, r in zip(qs, ref.executors, ref.results())]
    _same_results(qs, req.finalize(), exp, "batches")
    # one ShardedFusedQuery per query (what bench.py runs): results left in device memory, HLLResults for HLL queries
    one = [ShardedFusedQuery(eng.lib, eng.space, q) for q in qs]
    for b in batches:
        for s in one:
            s.process_batch(b)
    got = [s.finalize_hll() if q.is_hll else query_result(q, *s.finalize()) for q, s in zip(qs, one)]
    _same_results(qs, got, exp, "one query")
    for x in one + [req, ref]:
        x.close()
    # archive.scan_shard
    table = aql.Table("trips", [aql.Column(n, t) for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)])
    day0, cutoff = synth.BASE_TS // 86400, synth.BASE_TS + 3 * 86400
    arch = {day0 + d: synth.generate_batch(d, 20000, num_cities=12, null_rate=0.0) for d in range(3)}
    live = [synth.generate_batch(3 + i, 25000, num_cities=12, null_rate=0.0) for i in range(2)]
    frm, to = synth.BASE_TS + 86400 + 1800, synth.BASE_TS + 5 * 86400 - 1800
    text = {"table": "trips", "rowFilters": ["status = 1"], "timeFilter": {"column": "request_at", "from": str(frm), "to": str(to)},
            "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": "hour"}, {"sqlExpression": "city_id"}]}
    qs = [aql.compile_query({**text, "measures": [{"sqlExpression": m}]}, table, synth.BASE_TS + 30 * 86400)
          for m in ("sum(fare)", "count(*)", "max(city_id)", "min(fare)")]
    keep_live = [T.upload(eng, hb, 0, synth.zone_map(hb)) for hb in live]
    keep_arch = {d: T.upload(eng, hb, 0, synth.zone_map(hb)) for d, hb in arch.items()}
    req, ref = ShardedFusedRequest(eng.lib, eng.space, qs), FusedRequestExecutor(eng.lib, eng.space, qs)
    archive.scan_shard(req, keep_live, keep_arch, cutoff, qs[0].time_range, 0)
    archive.scan_shard(ref, keep_live, keep_arch, cutoff, qs[0].time_range, 0)
    got, exp = req.finalize(), ref.results()
    assert sum(r.groups for r in exp) > 0
    _same_results(qs, got, exp, "scan_shard")
    req.close()
    ref.close()


@pytest.mark.gpu
def test_abi_rejections():
    import torch
    import harness as H
    import test_hll_pipeline as HP
    from aresdb_b200.executor import FusedBatchExecutor, _ResultBuffers
    from aresdb_b200.sharding import request_slot_layout
    eng = H.get_backend("b200")
    lib, st = eng.lib, eng.space.stream
    q = T.queries()["cfg3_sum"]
    ex = FusedBatchExecutor(lib, eng.space, q)
    hll = FusedBatchExecutor(lib, eng.space, HP.hll_queries()["two_dims"])
    other = FusedBatchExecutor(lib, eng.space, T.queries()["no_dims_wide"])
    twin = FusedBatchExecutor(lib, eng.space, q)
    cap = 64
    parts, dims, values, slot = request_slot_layout([q], cap)
    buf = torch.zeros(2 * FLAGS_PER_PARITY + 4 * slot, dtype=torch.uint8, device=eng.space.dev)
    b0 = buf.data_ptr() + 2 * FLAGS_PER_PARITY
    out = _ResultBuffers(eng.space, q, 64)

    def arr(t, xs):
        return (t * len(xs))(*xs)

    def states(*exs):
        return arr(C.c_void_p, [e.state.value for e in exs])

    def fin(sts, n, keys=None, vals=None, groups=None, o=out):
        keys = keys if keys is not None else arr(A.DimensionVector, [o.dimension_vector(q)] * max(n, 1))
        vals = vals if vals is not None else arr(C.c_void_p, [o.measures.ptr] * max(n, 1))
        groups = groups if groups is not None else (C.c_int64 * max(n, 1))()
        lib.AggStatesFinalize(sts, n, keys, vals, groups, st, 0)

    def exp_(sts, n, peers=1, rank=0, slot_bytes=slot, cap_rows=cap, po=parts, do=dims, vo=values, slots=None, flags=None):
        slots = slots if slots is not None else arr(C.c_void_p, [b0 + p * slot for p in range(max(peers, 1))])
        lib.AggStatesExportPartsToPeers(sts, n, slots, flags, peers, rank, slot_bytes, cap_rows,
                                        None if po is None else arr(C.c_size_t, po * max(n, 1)),
                                        None if do is None else arr(C.c_size_t, do * max(n, 1)),
                                        None if vo is None else arr(C.c_size_t, vo * max(n, 1)), 1, st, 0)

    def mrg(sts, n, parts_=2, stride=slot, cap_rows=cap, po=parts, do=dims, vo=values, slots=b0):
        lib.AggStatesMergeParts(sts, n, slots, parts_, stride, cap_rows,
                                None if po is None else arr(C.c_size_t, po * max(n, 1)),
                                None if do is None else arr(C.c_size_t, do * max(n, 1)),
                                None if vo is None else arr(C.c_size_t, vo * max(n, 1)), None, 0, st, 0)

    calls = {"AggStatesFinalize": fin, "AggStatesExportPartsToPeers": exp_, "AggStatesMergeParts": mrg}
    for name, call in calls.items():
        for n in (0, 17):
            with pytest.raises(A.AresError, match=f"{name}: numStates must be 1..16"):
                call(arr(C.c_void_p, [ex.state.value] * 17), n)
        with pytest.raises(A.AresError, match=f"{name}: states is null"):
            call(None, 1)
        with pytest.raises(A.AresError, match=f"{name}: state 1 is AGGR_HLL"):
            call(states(ex, hll), 2)
        with pytest.raises(A.AresError, match=f"{name}: state 1 appears twice"):
            call(states(ex, ex), 2)
    # null arrays
    with pytest.raises(A.AresError, match="AggStatesFinalize: outputKeys / outputValues / groups must not be null"):
        lib.AggStatesFinalize(states(ex), 1, None, arr(C.c_void_p, [out.measures.ptr]), (C.c_int64 * 1)(), st, 0)
    with pytest.raises(A.AresError, match="AggStatesExportPartsToPeers: peerSlots is null"):
        lib.AggStatesExportPartsToPeers(states(ex), 1, None, None, 1, 0, slot, cap, arr(C.c_size_t, parts), arr(C.c_size_t, dims),
                                        arr(C.c_size_t, values), 1, st, 0)
    with pytest.raises(A.AresError, match="AggStatesMergeParts: slots is null"):
        mrg(states(ex), 1, slots=None)
    for call in (exp_, mrg):
        with pytest.raises(A.AresError, match="must not be null"):
            call(states(ex), 1, po=None)
        with pytest.raises(A.AresError, match="must not be null"):
            call(states(ex), 1, vo=None)
    # capRows, alignment, fit
    for name, call in (("AggStatesExportPartsToPeers", exp_), ("AggStatesMergeParts", mrg)):
        for c in (0, 32769):
            with pytest.raises(A.AresError, match=f"{name}: capRows must be in \\[1, 32768\\]"):
                call(states(ex), 1, cap_rows=c)
        with pytest.raises(A.AresError, match=f"{name}: state 0: offsets must be multiples of 16"):
            call(states(ex), 1, po=[8])
        with pytest.raises(A.AresError, match=f"{name}: state 0: offsets must be multiples of 16"):
            call(states(ex), 1, vo=[values[0] + 4])
        with pytest.raises(A.AresError, match=f"{name}: state 0: the sub-part does not fit the slot"):
            call(states(ex), 1, po=[16])
        with pytest.raises(A.AresError, match=f"{name}: state 0: the header"):
            call(states(ex), 1, vo=[dims[0]])
        with pytest.raises(A.AresError, match=f"{name}: state 1: the sub-part overlaps that of state 0"):
            call(states(ex, twin), 2)
    with pytest.raises(A.AresError, match="AggStatesExportPartsToPeers: slotBytes must be a multiple of 16"):
        exp_(states(ex), 1, slot_bytes=slot + 8)
    with pytest.raises(A.AresError, match="AggStatesMergeParts: slotBytes must be a multiple of 16"):
        mrg(states(ex), 1, stride=slot + 8)
    # peers
    for peers, rank in ((0, 0), (17, 0), (2, 2), (2, -1)):
        with pytest.raises(A.AresError, match="AggStatesExportPartsToPeers: numPeers must be 1..16"):
            exp_(states(ex), 1, peers=peers, rank=rank)
    for n_parts in (0, 17):
        with pytest.raises(A.AresError, match="AggStatesMergeParts: numParts must be 1..16"):
            mrg(states(ex), 1, parts_=n_parts)
    # a DimensionVector whose layout differs from its state's AggSpec
    wrong = _ResultBuffers(eng.space, T.queries()["no_dims_wide"], 64)
    with pytest.raises(A.AresError, match="AggStatesFinalize: state 1: dimension layout differs from AggSpec"):
        fin(states(ex, other), 2, keys=arr(A.DimensionVector, [out.dimension_vector(q), wrong.dimension_vector(q)]))
    for e in (ex, hll, other, twin):
        e.close()


# ---- GPU, two devices --------------------------------------------------------------------------------------------------
def _rank_worker(rank, world, port, out_dir, exchange):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      ARESDB_B200_EXCHANGE=exchange)
    import torch
    import torch.distributed as dist
    import independent as I
    import test_at_size as AS
    import test_hll_pipeline as HP
    from aresdb_b200.executor import Batch, FusedRequestExecutor
    from aresdb_b200.memory import CudaSpace
    from aresdb_b200.sharding import ShardedFusedRequest
    torch.cuda.set_device(rank)
    dev = torch.device(f"cuda:{rank}")
    dist.init_process_group("nccl", device_id=dev)
    lib = A.load_engine()
    space = CudaSpace(rank, torch.cuda.current_stream().cuda_stream)
    days, rows, t0 = 4, 8_000_000, synth.BASE_TS
    base = AS._queries(days)["cfg3"]
    dims = [E.floor(T.TS, E.Lit(3600)), T.CITY]
    cfg3 = [AggQuery(base.filters, dims, m) for m in (Measure("sum", T.FARE), Measure("count"), Measure("avg", T.FARE), Measure("max", T.CITY))]
    qs = cfg3 + [HP.hll_queries()["two_dims"], AggQuery([], [T.TS, T.CITY], Measure("count"), reduce_mode=A.ARES_REDUCE_HASH)]
    eg = [0, 0, 0, 0, 0, 100000]
    exp = I.Expected("cfg3", days, dev, t0, t0 + 1800, t0 + days * 86400 - 1800)
    batches = []
    for d in range(days):
        bufs, voff, cols = AS._batch(d, rows, dev)
        exp.add_batch(bufs, voff, rows)
        batches.append(Batch(cols, rows, ranges=synth.zone_map_of_day(d), keep=[bufs]))
    report = []
    req = ShardedFusedRequest(lib, space, qs, eg)
    assert req.fixed == [0, 1, 2, 3]
    for d, b in enumerate(batches):
        if d % world == rank:
            req.process_batch(b)
    got = req.finalize()
    full = FusedRequestExecutor(lib, space, qs, eg)
    for b in batches:
        full.process_batch(b)
    want = [ex.hll_result() if q.is_hll else r for q, ex, r in zip(qs, full.executors, full.results())]
    _same_results(qs, got, want, f"rank{rank}/{exchange}")
    assert exp.check(got[0])["groups"] > 0
    # identical on every rank
    digest = hashlib.sha256()
    for q, r in zip(qs, got):
        if q.is_hll:
            for key, regs in sorted(r.dense_registers().items()):
                digest.update(repr(key).encode() + regs.tobytes())
        else:
            digest.update(repr(r.rows).encode() + r.measures.tobytes())
    every = [None] * world
    dist.all_gather_object(every, digest.hexdigest())
    assert all(e == every[0] for e in every)
    # the fixed exchange alone: 1 export + 1 merge + 1 finalize launch per rank
    small = ShardedFusedRequest(lib, space, cfg3)
    for d, b in enumerate(batches):
        if d % world == rank:
            small.process_batch(b)
    torch.cuda.synchronize()
    k0 = lib.kernel_launch_count()
    got4 = small.finalize()
    report.append(lib.kernel_launch_count() - k0)
    _same_results(cfg3, got4, want[:4], f"rank{rank}/{exchange}/fixed")
    for x in (req, full, small):
        x.close()
    (Path(out_dir) / f"rank{rank}.txt").write_text(f"ok {report[0]} {req._peer is not None}")
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("exchange", ["peer", "fixed"])
def test_two_ranks_with_nccl(tmp_path, exchange):
    """Two NCCL ranks run the cfg3 request plus an HLL query and a hash query announcing more than 32768 groups (both take
    the exact protocol): identical results on both ranks, equal to the single-GPU request, sum(fare) equal to
    tests/independent.py; the fixed exchange is one export, one merge and one finalize launch per rank."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs two GPUs, this machine has {torch.cuda.device_count()}")
    import torch.multiprocessing as mp
    port = 29700 + (os.getpid() % 2000) + (exchange == "fixed")
    mp.spawn(_rank_worker, args=(2, port, str(tmp_path), exchange), nprocs=2, join=True)
    for r in range(2):
        words = (tmp_path / f"rank{r}.txt").read_text().split()
        assert words[:2] == ["ok", "3"], words
        if exchange == "fixed":
            assert words[2] == "False"
