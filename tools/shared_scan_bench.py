#!/usr/bin/env python
"""The cfg3 table (8 day-batches x 1.25e8 rows, zone maps) queried by one dashboard request: {sum(fare), count(*)},
a four-measure request {sum(fare), count(*), avg(fare), max(city_id)}, and a request whose queries differ in their filters
(common part: the time range and city_id != 0; members: sum(fare) where status = 1 and fare > 5, count(*) where
status = 1, count(*) where status = 2, count(*)), each run in one pass (FusedRequestExecutor) and as separate queries (one
FusedBatchExecutor each), alternating in the same process.  Times are CUDA events around the batches of a step plus the finalize of every query; the results of both forms are compared before anything is timed.
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
                                      AggQuery([status2] + rest, dims, ms[1]), AggQuery(rest, dims, ms[1])]}
    keep, batches = [], []
    for d in range(args.batches):
        bufs, voff = synth.generate_batch_cuda(d, args.rows, dev)
        cols = [columns.slice_of(b.data_ptr(), dt, args.rows, 0, voff, 2) for b, dt in zip(bufs, synth.COLUMN_TYPES)]
        keep.append(bufs)
        batches.append(Batch(cols, args.rows, ranges=synth.zone_map_of_day(d)))
    torch.cuda.synchronize()

    def results(kind, qs):
        if kind == "shared":
            ex = FusedRequestExecutor(lib, space, qs)
            run = [ex]
        else:
            run = [FusedBatchExecutor(lib, space, q) for q in qs]
        for b in batches:
            for ex in run:
                ex.process_batch(b)
        out = ex.results() if kind == "shared" else [ex.result() for ex in run]
        for ex in run:
            ex.close()
        return out

    def timed(kind, qs):
        ex = FusedRequestExecutor(lib, space, qs) if kind == "shared" else None
        solos = None if ex else [FusedBatchExecutor(lib, space, q) for q in qs]
        times = []
        for step in range(args.steps + 1):   # step 0: warm-up (kernel compile, first launches)
            run = [ex] if ex else solos
            for e in run:
                e.reset()
            torch.cuda.synchronize()
            s, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for b in batches:
                for e in run:
                    e.process_batch(b)
            _ = ex.results() if ex else [x.result() for x in solos]
            e_.record()
            torch.cuda.synchronize()
            if step:
                times.append(s.elapsed_time(e_))
        for e in ([ex] if ex else solos):
            e.close()
        return times

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    report = {"gpu": smi, "rows": args.rows * args.batches, "batches": args.batches, "steps": args.steps, "requests": {}}
    for name, qs in requests.items():
        shared, separate = results("shared", qs), results("separate", qs)
        for q, a, b in zip(qs, shared, separate):
            assert a.rows == b.rows and a.groups == b.groups, f"{name}: groups differ"
            if q.agg_func == A.AGGR_AVG_FLOAT:
                assert a.counts.tolist() == b.counts.tolist()
                np.testing.assert_allclose(a.measures, b.measures, rtol=2e-5, atol=1e-6)
            else:
                assert a.measures.tobytes() == b.measures.tobytes(), f"{name}: {q.measure_kind} differs"
        t = {"shared": [], "separate": []}
        for _ in range(2):   # alternate the two forms
            t["shared"] += timed("shared", qs)
            t["separate"] += timed("separate", qs)
        med = {k: float(np.median(v)) for k, v in t.items()}
        report["requests"][name] = {"measures": len(qs), "groups": shared_scan_groups(qs, member_filters=True),
                                    "shared_ms": med["shared"], "separate_ms": med["separate"],
                                    "shared_ms_all": t["shared"], "separate_ms_all": t["separate"],
                                    "speedup": med["separate"] / med["shared"], "results_equal": True}
        print(f"{name}: one pass {med['shared']:.2f} ms, separate queries {med['separate']:.2f} ms "
              f"(x{med['separate'] / med['shared']:.2f}), {args.rows * args.batches:.3g} rows, {smi}", flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
