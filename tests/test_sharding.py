"""N > 1: batches are dealt round-robin to ranks, every rank aggregates its own, one exchange step
merges.  CPU: world_size-2 gloo processes run the reference call sequence on the C restatement (host
memory) and merge on the host; the result must equal the single-process run over all batches.
GPU: AggStateMerge (the device-side re-aggregation used after the NCCL all-gather) is checked by
folding two partial results into a fresh state."""
import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    import harness as H
    import test_pipeline_parity as T
    from aresdb_b200 import sharding, synth
    dist.init_process_group("gloo", rank=rank, world_size=world)
    orc = H.get_backend("oracle")
    hbs = [synth.generate_batch(d, 4000 + 137 * d, num_cities=20, null_rate=0.05) for d in range(5)]
    ok = True
    for name in ("cfg3_sum", "cfg3_count", "min_city", "nested"):
        q = T.queries()[name]
        mine = [hbs[i] for i in sharding.assign_batches(len(hbs), world, rank)]
        local = T.run_legacy(orc, q, mine)
        merged = sharding.merge_results_host(q, sharding.all_gather_results_host(dist, local))
        full = T.run_legacy(orc, q, hbs).as_dict()
        ok = ok and merged.keys() == full.keys() and all(np.array_equal(merged[k], full[k]) for k in full)
    # hll queries: per-register max of the ranks' register sets == the single-process run over all batches
    import test_hll_pipeline as HP
    for name, q in HP.hll_queries().items():
        mine = [hbs[i] for i in sharding.assign_batches(len(hbs), world, rank)]
        merged = sharding.merge_hll_results_host(sharding.all_gather_hll_host(dist, HP.run_hll_query(orc, q, mine)))
        full = HP.run_hll_query(orc, q, hbs).dense_registers()
        ok = ok and merged.keys() == full.keys() and all(np.array_equal(merged[k], full[k]) for k in full)
    (Path(out_dir) / f"rank{rank}.txt").write_text("ok" if ok else "mismatch")
    dist.destroy_process_group()


def test_two_rank_gloo_merge(tmp_path):
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "rank0.txt").read_text() == "ok"
    assert (tmp_path / "rank1.txt").read_text() == "ok"


def test_assign_batches_covers_everything():
    from aresdb_b200 import sharding
    for world in (1, 2, 4, 8):
        seen = sorted(b for r in range(world) for b in sharding.assign_batches(8, world, r))
        assert seen == list(range(8))


@pytest.mark.gpu
def test_agg_state_merge_on_device():
    import harness as H
    import test_pipeline_parity as T
    from aresdb_b200 import cabi as A
    from aresdb_b200 import synth
    from aresdb_b200.executor import FusedBatchExecutor
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    hbs = [synth.generate_batch(d, 20000, num_cities=30) for d in range(4)]
    for name in ("cfg3_sum", "cfg3_count", "cfg4_hash", "min_city", "no_dims_wide"):
        q = T.queries()[name]
        parts = []
        for half in (hbs[:2], hbs[2:]):
            ex = FusedBatchExecutor(eng.lib, eng.space, q)
            keep = []
            for hb in half:
                b = T.upload(eng, hb)
                keep.append(b)
                ex.process_batch(b)
            parts.append(ex.finalize_into())
            ex.close()
        merged = FusedBatchExecutor(eng.lib, eng.space, q)
        for g, out in parts:
            merged.merge(out.dimension_vector(q), out.measures.ptr, g)
        got = merged.result()
        merged.close()
        exp = T.run_legacy(orc, q, hbs)
        T.assert_same_result(got, exp, ordered=q.reduce_mode == A.ARES_REDUCE_SORT, ctx=name)


def _one_state_layout(q, cap):
    """The exchange layout of one query as a request of one state: [64-byte header | dimension block of `cap` rows |
    measures], 64-byte aligned.  Returns (part bytes, partOffset, dimOffset, valuesOffset) - the offsets as one-element
    arrays."""
    import ctypes as C
    from aresdb_b200.executor import dim_offsets
    _, _, _, dim_bytes = dim_offsets(q.num_dims_per_width, cap)
    dim_bytes = (dim_bytes + 15) // 16 * 16
    part = (64 + dim_bytes + q.measure_bytes * cap + 63) // 64 * 64
    return part, (C.c_size_t * 1)(0), (C.c_size_t * 1)(64), (C.c_size_t * 1)(64 + dim_bytes)


def _states(*exs):
    import ctypes as C
    return (C.c_void_p * len(exs))(*[ex.state.value for ex in exs])


@pytest.mark.gpu
def test_one_state_exchange_through_a_collective_on_device():
    """The device-only exchange of a sharded query through a collective (AggStatesExportPartsToPeers without flags ->
    [all-gather] -> AggStatesMergeParts without flags, one state each): two states' parts laid out as an all-gather leaves
    them are folded by one launch; counts never visit the host.  A part that cannot hold its sender's rows is reported by
    the receiver's finalize."""
    import ctypes as C
    import torch
    import harness as H
    import test_pipeline_parity as T
    from aresdb_b200 import cabi as A
    from aresdb_b200 import synth
    from aresdb_b200.executor import FusedBatchExecutor
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    hbs = [synth.generate_batch(d, 20000, num_cities=30) for d in range(4)]
    dev, st = eng.space.dev, eng.space.stream
    for name in ("cfg3_sum", "cfg3_count", "cfg4_hash", "min_city", "no_dims_wide"):
        q = T.queries()[name]
        exp = T.run_legacy(orc, q, hbs)
        for cap in (32768, 64):
            part, po, do, vo = _one_state_layout(q, cap)
            recv = torch.zeros(2 * part, dtype=torch.uint8, device=dev)
            keep = []
            for r, half in enumerate((hbs[:2], hbs[2:])):
                ex = FusedBatchExecutor(eng.lib, eng.space, q)
                for hb in half:
                    b = T.upload(eng, hb)
                    keep.append(b)
                    ex.process_batch(b)
                mine = (C.c_void_p * 1)(recv.data_ptr() + r * part)
                eng.lib.AggStatesExportPartsToPeers(_states(ex), 1, mine, None, 1, 0, part, cap, po, do, vo, 0, st, 0)
                keep.append(ex)
            merged = FusedBatchExecutor(eng.lib, eng.space, q)
            eng.lib.AggStatesMergeParts(_states(merged), 1, recv.data_ptr(), 2, part, cap, po, do, vo, None, 0, st, 0)
            hdr = recv.view(2, part)[:, :12].contiguous().view(torch.int32).cpu().numpy()
            if (hdr[:, 2] <= cap).all():
                assert (hdr[:, 1] == 0).all() and (hdr[:, 0] == hdr[:, 2]).all()
                got = merged.result()
                T.assert_same_result(got, exp, ordered=q.reduce_mode == A.ARES_REDUCE_SORT, ctx=f"{name}/cap{cap}")
            else:
                assert (hdr[:, 1] != 0).any()
                with pytest.raises(A.AresError, match="exchange part truncated"):
                    merged.result()
            merged.close()
            for k in keep:
                if isinstance(k, FusedBatchExecutor):
                    k.close()


@pytest.mark.gpu
def test_one_state_exchange_refuses_hll_states():
    """HLL states exchange through AggStateExport (carried rows): the fixed-size part entry points refuse them on the
    sending and on both receiving sides (with and without flags), in entry and in dense-register mode."""
    import ctypes as C
    import torch
    import harness as H
    import test_hll_pipeline as HP
    from aresdb_b200 import cabi as A
    from aresdb_b200.executor import FusedBatchExecutor
    eng = H.get_backend("b200")
    st = eng.space.stream
    q = HP.hll_queries()["two_dims"]
    cap = 64
    part, po, do, vo = _one_state_layout(q, cap)
    buf = torch.zeros(256 + 2 * part, dtype=torch.uint8, device=eng.space.dev)   # flags | two parts
    parts = buf.data_ptr() + 256
    refused = "state 0 is AGGR_HLL: HLL states exchange through AggStateExport"
    for mode in (HP.ENTRY_MODE, HP.DENSE_MODE):
        ex = FusedBatchExecutor(eng.lib, eng.space, q, mode)
        with pytest.raises(A.AresError, match=f"AggStatesExportPartsToPeers: {refused}"):
            eng.lib.AggStatesExportPartsToPeers(_states(ex), 1, (C.c_void_p * 1)(parts), None, 1, 0, part, cap, po, do, vo, 0, st, 0)
        with pytest.raises(A.AresError, match=f"AggStatesMergeParts: {refused}"):
            eng.lib.AggStatesMergeParts(_states(ex), 1, parts, 2, part, cap, po, do, vo, None, 0, st, 0)
        with pytest.raises(A.AresError, match=f"AggStatesMergeParts: {refused}"):
            eng.lib.AggStatesMergeParts(_states(ex), 1, parts, 2, part, cap, po, do, vo, buf.data_ptr(), 1, st, 0)
        ex.close()


@pytest.mark.gpu
def test_one_state_exchange_over_peer_memory_on_one_device():
    """AggStatesExportPartsToPeers / AggStatesMergeParts with flags, one state each, with both "ranks" on one GPU: two
    states export into each other's receive buffers (part in the sender's slot of BOTH buffers, flag raised to the epoch on
    both), each receive buffer is then folded by a merge kernel that waits for the two flags.  Same results as the
    collective form; two epochs on alternating buffers; a part that cannot hold its sender's rows, and a peer that never
    arrives (bounded wait), are reported by the receiver's finalize."""
    import ctypes as C
    import torch
    import harness as H
    import test_pipeline_parity as T
    from aresdb_b200 import cabi as A
    from aresdb_b200 import synth
    from aresdb_b200.executor import FusedBatchExecutor
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    hbs = [synth.generate_batch(d, 20000, num_cities=30) for d in range(4)]
    dev, st = eng.space.dev, eng.space.stream
    FLAGS = 256   # flags in front of the parts: state 0's uint32 flags[16 ranks] of parity p at p * 64
    for name in ("cfg3_sum", "cfg4_hash", "no_dims_wide"):
        q = T.queries()[name]
        exp = T.run_legacy(orc, q, hbs)
        for cap in (32768, 64):
            part, po, do, vo = _one_state_layout(q, cap)
            bufs = [torch.zeros(FLAGS + 2 * 2 * part, dtype=torch.uint8, device=dev) for _ in range(2)]   # flags | parity 0 | parity 1
            locals_, keep = [], []
            for half in (hbs[:2], hbs[2:]):
                ex = FusedBatchExecutor(eng.lib, eng.space, q)
                for hb in half:
                    b = T.upload(eng, hb)
                    keep.append(b)
                    ex.process_batch(b)
                locals_.append(ex)
            for epoch in (1, 2):
                par = epoch & 1
                base = FLAGS + par * 2 * part
                for r, ex in enumerate(locals_):
                    slots = (C.c_void_p * 2)(*[bufs[p].data_ptr() + base + r * part for p in range(2)])
                    flags = (C.c_void_p * 2)(*[bufs[p].data_ptr() + par * 64 + r * 4 for p in range(2)])
                    eng.lib.AggStatesExportPartsToPeers(_states(ex), 1, slots, flags, 2, r, part, cap, po, do, vo, epoch, st, 0)
                for r in range(2):
                    merged = FusedBatchExecutor(eng.lib, eng.space, q)
                    eng.lib.AggStatesMergeParts(_states(merged), 1, bufs[r].data_ptr() + base, 2, part, cap, po, do, vo,
                                                bufs[r].data_ptr() + par * 64, epoch, st, 0)
                    hdr = bufs[r][base:base + 2 * part].view(2, part)[:, :12].contiguous().view(torch.int32).cpu().numpy()
                    if (hdr[:, 2] <= cap).all():
                        got = merged.result()
                        T.assert_same_result(got, exp, ordered=q.reduce_mode == A.ARES_REDUCE_SORT, ctx=f"{name}/cap{cap}/epoch{epoch}/rank{r}")
                    else:
                        with pytest.raises(A.AresError, match="exchange part truncated"):
                            merged.result()
                    merged.close()
            for ex in locals_:
                ex.close()
    # a peer that never raises its flag: the merge kernel gives up after its bound and the finalize says so
    q = T.queries()["cfg3_count"]
    cap = 1024
    part, po, do, vo = _one_state_layout(q, cap)
    buf = torch.zeros(FLAGS + 2 * part, dtype=torch.uint8, device=dev)
    merged = FusedBatchExecutor(eng.lib, eng.space, q)
    eng.lib.AggStatesMergeParts(_states(merged), 1, buf.data_ptr() + FLAGS, 2, part, cap, po, do, vo, buf.data_ptr(), 7, st, 0)
    with pytest.raises(A.AresError, match="did not arrive"):
        merged.result()
    merged.close()
