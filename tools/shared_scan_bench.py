#!/usr/bin/env python
"""The cfg3 table (8 day-batches x 1.25e8 rows, zone maps) queried by one dashboard request: {sum(fare), count(*)},
a four-measure request {sum(fare), count(*), avg(fare), max(city_id)}, and a request whose queries differ in their filters
(common part: the time range and city_id != 0; members: sum(fare) where status = 1 and fare > 5, count(*) where
status = 1, count(*) where status = 2, count(*)), and a request whose queries differ in their dimensions (all with the cfg3
filters: sum(fare) by hour x city, count(*) by hour, count(*) by city, count(*) by status), each run in one pass
(FusedRequestExecutor) and as separate queries (one FusedBatchExecutor each), alternating in the same process; a request
of several groups of queries with the same dimensions is also run as it grouped before such groups shared a pass (one
FusedRequestExecutor per group).  Times are CUDA events around the batches of a step plus the finalize of every query; the results of both forms are compared before anything is timed.
Usage: python tools/shared_scan_bench.py [--steps N] [--batches B] [--rows R]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--rows", type=int, default=125_000_000)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from aresdb_b200 import cabi as A, columns, expr as E, synth
    from aresdb_b200.executor import Batch, FusedBatchExecutor, FusedRequestExecutor, shared_scan_groups
    from aresdb_b200.memory import CudaSpace
    from aresdb_b200.query import AggQuery, Measure

    lib = A.load_engine()
    dev = torch.device("cuda:0")
    space = CudaSpace(0)
    base = bench._q_cfg3()
    dims = base.dimensions
    ms = [Measure("sum", E.Col(3, A.Float32, "fare")), Measure("count"), Measure("avg", E.Col(3, A.Float32, "fare")),
          Measure("max", E.Col(1, A.Uint16, "city_id"))]
    status1, status2, rest = base.filters[0], E.eq(bench._columns()[2], E.Lit(2)), base.filters[2:]
    requests = {"sum_count": [AggQuery(base.filters, dims, m) for m in ms[:2]],
                "four_measures": [AggQuery(base.filters, dims, m) for m in ms],
                "differing_filters": [AggQuery(base.filters, dims, ms[0]), AggQuery([status1] + rest, dims, ms[1]),
                                      AggQuery([status2] + rest, dims, ms[1]), AggQuery(rest, dims, ms[1])],
                "differing_dimensions": [AggQuery(base.filters, d, m) for d, m in
                                         ((dims, ms[0]), (dims[:1], ms[1]), (dims[1:], ms[1]), ([bench._columns()[2]], ms[1]))]}
    keep, batches = [], []
    for d in range(args.batches):
        bufs, voff = synth.generate_batch_cuda(d, args.rows, dev)
        cols = [columns.slice_of(b.data_ptr(), dt, args.rows, 0, voff, 2) for b, dt in zip(bufs, synth.COLUMN_TYPES)]
        keep.append(bufs)
        batches.append(Batch(cols, args.rows, ranges=synth.zone_map_of_day(d)))
    torch.cuda.synchronize()

    def executors(kind, qs):
        """(executors, indexes of the queries each one runs): the whole request, one per group, or one per query."""
        if kind == "shared":
            return [FusedRequestExecutor(lib, space, qs)], [list(range(len(qs)))]
        if kind == "per_group":
            groups = shared_scan_groups(qs, member_filters=True)
            return [FusedRequestExecutor(lib, space, [qs[i] for i in g]) for g in groups], groups
        return [FusedBatchExecutor(lib, space, q) for q in qs], [[i] for i in range(len(qs))]

    def collect(run, idx):
        out = {}
        for ex, g in zip(run, idx):
            out.update(zip(g, ex.results() if isinstance(ex, FusedRequestExecutor) else [ex.result()]))
        return [out[i] for i in range(len(out))]

    def results(kind, qs):
        run, idx = executors(kind, qs)
        for b in batches:
            for ex in run:
                ex.process_batch(b)
        out = collect(run, idx)
        for ex in run:
            ex.close()
        return out

    def timed(kind, qs):
        run, idx = executors(kind, qs)
        times = []
        for step in range(args.steps + 1):   # step 0: warm-up (kernel compile, first launches)
            for e in run:
                e.reset()
            torch.cuda.synchronize()
            s, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for b in batches:
                for e in run:
                    e.process_batch(b)
            _ = collect(run, idx)
            e_.record()
            torch.cuda.synchronize()
            if step:
                times.append(s.elapsed_time(e_))
        for e in run:
            e.close()
        return times

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    report = {"gpu": smi, "rows": args.rows * args.batches, "batches": args.batches, "steps": args.steps, "requests": {}}
    for name, qs in requests.items():
        kinds = ["shared", "separate"] + (["per_group"] if len(shared_scan_groups(qs, member_filters=True)) > 1 else [])
        shared = results("shared", qs)
        for kind in kinds[1:]:
            for q, a, b in zip(qs, shared, results(kind, qs)):
                assert a.rows == b.rows and a.groups == b.groups, f"{name} ({kind}): groups differ"
                if q.agg_func == A.AGGR_AVG_FLOAT:
                    assert a.counts.tolist() == b.counts.tolist()
                    np.testing.assert_allclose(a.measures, b.measures, rtol=2e-5, atol=1e-6)
                else:
                    assert a.measures.tobytes() == b.measures.tobytes(), f"{name} ({kind}): {q.measure_kind} differs"
        t = {k: [] for k in kinds}
        for _ in range(2):   # alternate the forms
            for k in kinds:
                t[k] += timed(k, qs)
        med = {k: float(np.median(v)) for k, v in t.items()}
        entry = {"measures": len(qs), "groups": shared_scan_groups(qs, member_filters=True), "results_equal": True,
                 "speedup": med["separate"] / med["shared"]}
        for k in kinds:
            entry[f"{k}_ms"], entry[f"{k}_ms_all"] = med[k], t[k]
            entry[f"{k}_spread_ms"] = float(np.max(t[k]) - np.min(t[k]))
        report["requests"][name] = entry
        extra = f", per group {med['per_group']:.2f} ms" if "per_group" in med else ""
        print(f"{name}: one pass {med['shared']:.2f} ms, separate queries {med['separate']:.2f} ms "
              f"(x{med['separate'] / med['shared']:.2f}){extra}, {args.rows * args.batches:.3g} rows, {smi}", flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
