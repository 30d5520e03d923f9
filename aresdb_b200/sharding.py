"""Multi-GPU execution of aggregate queries: table shards / archive batches are independent units (the reference
processes them one after the other and only couples them through the carried result vectors, SURVEY.md §8e), so batch i
goes to rank i mod N, every rank aggregates its batches into private group tables, and ONE exchange step merges the
per-rank results with each aggregate's combine rule — what the reference's broker does with JSON results
(broker/result_merge.go:80-105: sum/count add, min/max).  Results are identical on every rank.

ShardedFusedRequest runs a rank's share of an AQL request; ShardedFusedQuery is a request of one query.  The exchange
runs on the device: one export launch writes every query's rows as a fixed-capacity part and copies it into every peer's
receive buffer over peer memory (or, where the ranks cannot map each other's buffers, one NCCL all-gather moves the
parts), one merge launch folds the parts and one finalize launch completes every query.  Queries with more groups than a
part holds and HLL queries take the exact-size protocol (exchange_exact).  ARESDB_B200_EXCHANGE chooses the transport:
"peer" (the default), "fixed" (the all-gather) or "exact" (the exact-size protocol for every query).
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

from . import cabi as A
from .executor import MAX_LAUNCH_STATES, dim_offsets, finalize_states, query_result
from .query import AggQuery, QueryResult


EXCHANGE_ROWS = 32768   # rows of a fixed part (= what the engine's single-launch export handles)
_PART_HDR = 64          # a part's header (16 bytes used) in front of its dimension block


def assign_batches(num_batches: int, world: int, rank: int) -> list[int]:
    """Round-robin placement of batch ids."""
    return [b for b in range(num_batches) if b % world == rank]


def setup_peer_buffers(dist, space, world: int, nbytes: int):
    """Maps every rank's receive buffer of `nbytes` into every process (torch symmetric memory: CUDA IPC / fabric handles
    over NVLink) for the exchange over peer memory: dict(buf, hdl, ptrs, epoch=0), or None.  All ranks agree on the
    outcome; on failure (or with ARESDB_B200_EXCHANGE other than "peer") the NCCL all-gather stays."""
    import torch
    ok, peer = 0, None
    if os.environ.get("ARESDB_B200_EXCHANGE", "peer") == "peer" and world <= 16:
        try:
            import torch.distributed._symmetric_memory as symm
            buf = symm.empty(nbytes, dtype=torch.uint8, device=space.dev)
            buf.zero_()
            hdl = symm.rendezvous(buf, dist.group.WORLD)
            ptrs = [int(p) for p in hdl.buffer_ptrs]
            torch.cuda.synchronize()
            peer = dict(buf=buf, hdl=hdl, ptrs=ptrs, epoch=0)
            ok = 1
        except Exception as e:   # no peer access between these GPUs, or a torch without symmetric memory
            print(f"[aresdb_b200] exchange over peer memory unavailable ({type(e).__name__}: {e}); using the NCCL all-gather",
                  file=sys.stderr)
    agree = torch.tensor([ok], device=space.dev, dtype=torch.int32)
    dist.all_reduce(agree, op=dist.ReduceOp.MIN)   # (also: nobody writes before everybody has zeroed its flags)
    return peer if agree.item() else None


def exchange_exact(dist, world: int, rank: int, local, merged):
    """The exact-size exchange step of one query: every rank exports its table (AggStateExport: unordered rows, no sort),
    ONE all-gather moves [dim block | measure vector] of every rank, and every rank folds all of them into `merged` (a
    FusedBatchExecutor, reset first).  Returns (rows gathered — an upper bound of the merged group count —, the gathered
    tensor, which must stay alive until the merged state is finalized).  For hll queries the rows are the carried (group,
    register) entries."""
    import torch
    q, sp, lib = local.q, local.space, local.lib
    n = local.group_count()
    counts = torch.zeros(world, dtype=torch.int64, device=sp.dev)
    counts[rank] = n
    dist.all_reduce(counts)
    counts = counts.tolist()
    cap = max(max(counts), 1)
    _, _, _, dim_bytes = dim_offsets(q.num_dims_per_width, cap)
    dim_bytes = (dim_bytes + 15) // 16 * 16
    part = dim_bytes + q.measure_bytes * cap
    gathered = torch.empty(world * part, dtype=torch.uint8, device=sp.dev)
    mine = gathered[rank * part:(rank + 1) * part]
    if n:
        dv = A.make_dimension_vector(mine.data_ptr(), None, None, q.num_dims_per_width, cap)
        lib.AggStateExport(local.state, dv, mine.data_ptr() + dim_bytes, sp.stream, sp.device)
    dist.all_gather_into_tensor(gathered, mine.clone())
    merged.reset()
    base = gathered.data_ptr()
    for r in range(world):
        if counts[r]:
            dv = A.make_dimension_vector(base + r * part, None, None, q.num_dims_per_width, cap)
            merged.merge(dv, base + r * part + dim_bytes, counts[r])
    return int(sum(counts)), gathered


def request_slot_layout(queries: list, cap_rows: int = EXCHANGE_ROWS):
    """One rank's exchange slot of a request: per query a sub-part [header | dimension block of `cap_rows` rows |
    measures], each sized from the query's dimensions and measure width and 16-byte aligned.  Returns (part offsets,
    dimension-block offsets, measure offsets — the last two relative to their sub-part —, slot bytes)."""
    parts, dims, values, pos = [], [], [], 0
    for q in queries:
        _, _, _, dim_bytes = dim_offsets(q.num_dims_per_width, cap_rows)
        dim_bytes = (dim_bytes + 15) // 16 * 16
        parts.append(pos)
        dims.append(_PART_HDR)
        values.append(_PART_HDR + dim_bytes)
        pos += (_PART_HDR + dim_bytes + q.measure_bytes * cap_rows + 15) // 16 * 16
    return parts, dims, values, (pos + 63) // 64 * 64


class ShardedFusedRequest:
    """One rank's half of a sharded AQL request (torch.distributed / NCCL plumbing).  The rank's batches are scanned by a
    FusedRequestExecutor, so queries that share dimensions, time filter and joins share the scan on every rank.  finalize() exchanges
    every non-HLL query that announces at most EXCHANGE_ROWS groups in ONE export launch (the rank's slot holds one
    sub-part per query; over peer memory when every rank can map every other's receive buffer, else one NCCL all-gather
    — see ARESDB_B200_EXCHANGE in the module docstring), folds them with ONE merge launch and finalizes them with ONE
    AggStatesFinalize.  HLL queries, queries that announce more groups and queries whose sub-part was truncated take the
    exact-size protocol (exchange_exact)."""

    _FLAGS_PER_PARITY = MAX_LAUNCH_STATES * 16 * 4   # uint32 flags[state][16 ranks] of one epoch parity

    def __init__(self, lib, space, queries: list, expected_groups: int | list = 0):
        """`expected_groups`: one hint for every query, or a list with one per query."""
        from .executor import FusedBatchExecutor, FusedRequestExecutor
        queries = list(queries)
        if not queries or len(queries) > MAX_LAUNCH_STATES:
            raise ValueError(f"a sharded request holds 1..{MAX_LAUNCH_STATES} queries, not {len(queries)}")
        if not all(isinstance(q, AggQuery) for q in queries):
            raise TypeError("every query of a sharded request must be an AggQuery")
        eg = list(expected_groups) if isinstance(expected_groups, (list, tuple)) else [expected_groups] * len(queries)
        if len(eg) != len(queries) or not all(isinstance(g, int) and not isinstance(g, bool) and g >= 0 for g in eg):
            raise ValueError("expected_groups must be a non-negative int, or one per query")
        import torch.distributed as dist
        self.dist = dist
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.lib, self.space, self.queries = lib, space, queries
        self.local = FusedRequestExecutor(lib, space, queries, eg)
        self.merged = [FusedBatchExecutor(lib, space, q, g) for q, g in zip(queries, eg)] if self.world > 1 else None
        fixed_ok = self.world > 1 and os.environ.get("ARESDB_B200_EXCHANGE", "fixed") != "exact"
        self.fixed = [i for i, q in enumerate(queries) if fixed_ok and not q.is_hll and eg[i] <= EXCHANGE_ROWS]
        self._layout = request_slot_layout([queries[i] for i in self.fixed])
        self._send = self._recv = None
        self._peer, self._peer_ok = None, None   # exchange over peer memory: set up at the first exchange
        self._merged_dirty = False
        self._keep = []

    def process_batch(self, batch, stream=None, time_filters: bool = True, cutoff: int = 0):
        """Same meaning as FusedRequestExecutor.process_batch (archive.scan_shard drives a rank's share with it)."""
        self.local.process_batch(batch, stream, time_filters, cutoff)

    def reset(self):
        self.local.reset()

    def _exchange_fixed(self):
        """Export (one launch) -> peer copy or one all-gather -> merge (one launch) of the fixed-exchange queries."""
        import torch
        sp, lib, w, r = self.space, self.lib, self.world, self.rank
        parts, dims, values, slot = self._layout
        k = len(self.fixed)
        states = (C.c_void_p * k)(*[self.local.executors[i].state.value for i in self.fixed])
        merged = (C.c_void_p * k)(*[self.merged[i].state.value for i in self.fixed])
        po, do, vo = ((C.c_size_t * k)(*x) for x in (parts, dims, values))
        if self._peer is None and self._peer_ok is None:
            self._peer = setup_peer_buffers(self.dist, sp, w, 2 * self._FLAGS_PER_PARITY + 2 * w * slot)
            self._peer_ok = self._peer is not None
        if self._peer is not None:
            pe = self._peer
            pe["epoch"] += 1
            epoch, par = pe["epoch"], pe["epoch"] & 1   # receive buffers and flags alternate by parity
            base, fbase = 2 * self._FLAGS_PER_PARITY + par * w * slot, par * self._FLAGS_PER_PARITY
            slots = (C.c_void_p * w)(*[pe["ptrs"][p] + base + r * slot for p in range(w)])
            flags = (C.c_void_p * w)(*[pe["ptrs"][p] + fbase + r * 4 for p in range(w)])
            lib.AggStatesExportPartsToPeers(states, k, slots, flags, w, r, slot, EXCHANGE_ROWS, po, do, vo, epoch, sp.stream, sp.device)
            lib.AggStatesMergeParts(merged, k, pe["ptrs"][r] + base, w, slot, EXCHANGE_ROWS, po, do, vo, pe["ptrs"][r] + fbase, epoch,
                                    sp.stream, sp.device)
            return
        if self._send is None:
            self._send = torch.zeros(slot, dtype=torch.uint8, device=sp.dev)
            self._recv = torch.empty(w * slot, dtype=torch.uint8, device=sp.dev)
        mine = (C.c_void_p * 1)(self._send.data_ptr())
        lib.AggStatesExportPartsToPeers(states, k, mine, None, 1, 0, slot, EXCHANGE_ROWS, po, do, vo, 0, sp.stream, sp.device)
        self.dist.all_gather_into_tensor(self._recv, self._send)
        lib.AggStatesMergeParts(merged, k, self._recv.data_ptr(), w, slot, EXCHANGE_ROWS, po, do, vo, None, 0, sp.stream, sp.device)

    def finalize(self, hll_estimates: bool = False) -> list:
        """One result per query, in request order, identical on every rank: a QueryResult, or for HLL queries an HLLResult
        (`hll_estimates`: the HLLEstimates of the merged state, computed on the device)."""
        return [r if q.is_hll else query_result(q, *r) for q, r in zip(self.queries, self._finalize(hll_estimates))]

    def _finalize(self, hll_estimates: bool = False) -> list:
        """The exchange and finalize step: per query, in request order, (groups, _ResultBuffers) with the result left in
        device memory, or the HLLResult (HLLEstimates) of an HLL query."""
        if self.world == 1:
            return self._results(self.local.executors, {}, hll_estimates)
        if self._merged_dirty:
            for i in self.fixed:   # (exchange_exact resets the states it merges into)
                self.merged[i].reset()
        self._merged_dirty = True
        done, exact = {}, [i for i in range(len(self.queries)) if i not in self.fixed]
        if self.fixed:
            self._exchange_fixed()
            for i, res in zip(self.fixed, finalize_states([self.merged[i] for i in self.fixed])):
                if isinstance(res, A.AresError) and "exchange part truncated" in str(res):
                    exact.append(i)
                else:
                    done[i] = res
        self._keep = []
        for i in sorted(exact):
            rows, gathered = exchange_exact(self.dist, self.world, self.rank, self.local.executors[i], self.merged[i])
            self._keep.append(gathered)
            if not self.queries[i].is_hll:
                done[i] = self.merged[i].finalize_into(rows)
        return self._results(self.merged, done, hll_estimates)

    def _results(self, executors: list, done: dict, hll_estimates: bool) -> list:
        todo = [i for i, q in enumerate(self.queries) if not q.is_hll and i not in done]
        done.update(zip(todo, finalize_states([executors[i] for i in todo])))
        out = []
        for i, q in enumerate(self.queries):
            if q.is_hll:
                out.append(executors[i].hll_estimates() if hll_estimates else executors[i].hll_result())
            elif isinstance(done[i], Exception):
                raise done[i]
            else:
                out.append(done[i])
        return out

    def close(self):
        self.local.close()
        for m in self.merged or []:
            m.close()


class ShardedFusedQuery:
    """One rank's half of a sharded query: a ShardedFusedRequest of this one query, whose results stay in device memory."""

    def __init__(self, lib, space, q: AggQuery, expected_groups: int = 0):
        self.q = q
        self.request = ShardedFusedRequest(lib, space, [q], expected_groups)

    def process_batch(self, batch, stream=None):
        self.request.process_batch(batch, stream)

    def reset(self):
        self.request.reset()

    def finalize(self):
        """(groups, _ResultBuffers) of the WHOLE query, identical on every rank."""
        return self.request._finalize()[0]

    def finalize_hll(self, hll_estimates: bool = False):
        """HLL queries: the HLLResult of the WHOLE query (`hll_estimates`: its HLLEstimates), identical on every rank."""
        return self.request._finalize(hll_estimates)[0]

    def close(self):
        self.request.close()


# ---- host-side mirror (gloo / CPU): same protocol on QueryResults, used by the CPU test-suite ------
_COMBINE = {A.AGGR_SUM_UNSIGNED: np.add, A.AGGR_SUM_SIGNED: np.add, A.AGGR_SUM_FLOAT: np.add,
            A.AGGR_MIN_UNSIGNED: np.minimum, A.AGGR_MIN_SIGNED: np.minimum, A.AGGR_MIN_FLOAT: np.minimum,
            A.AGGR_MAX_UNSIGNED: np.maximum, A.AGGR_MAX_SIGNED: np.maximum, A.AGGR_MAX_FLOAT: np.maximum}


def merge_results_host(q: AggQuery, parts: list[dict]) -> dict:
    """Folds per-rank {packed dim row: measure} maps with the aggregate's combine rule."""
    op = _COMBINE[q.agg_func]
    out: dict = {}
    for part in parts:
        for k, v in part.items():
            out[k] = op(out[k], v) if k in out else v
    return out


def all_gather_results_host(dist, result: QueryResult) -> list[dict]:
    """all_gather_object of the compact result maps (gloo works on CPU tensors / objects)."""
    world = dist.get_world_size()
    gathered = [None] * world
    dist.all_gather_object(gathered, result.as_dict())
    return gathered


def merge_hll_results_host(parts: list[dict]) -> dict:
    """hll queries: per-rank {packed dim row: uint8[16384] registers} maps folded with the per-register
    maximum (broker/result_merge.go: HLL merge = Merge of the register sets)."""
    out: dict = {}
    for part in parts:
        for k, regs in part.items():
            out[k] = np.maximum(out[k], regs) if k in out else regs
    return out


def all_gather_hll_host(dist, result) -> list[dict]:
    """all_gather_object of the dense register maps of an HLLResult."""
    gathered = [None] * dist.get_world_size()
    dist.all_gather_object(gathered, result.dense_registers())
    return gathered
