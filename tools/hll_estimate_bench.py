"""Times the distinct-count answer of countdistincthll queries: register vectors estimated on the host (today's path)
against estimates computed on the device (AggStateFinalizeHLLEstimate), over the cfg4-HLL table (bench.py's synthetic
trips: B batches of N rows).

  python tools/hll_estimate_bench.py [--rows N] [--batches B] [--reps R]

Queries: cfg4 HLL (status = 1, by day x city: 808 groups, dense register arrays) and countdistincthll(request_at) by
hour x city (19,200 groups over 8 days, (group, register) entries).  Per query, in alternating steps:
  (a) scan + hll_result() + postprocess.hll_nested_result (the register vectors read back, HLL.Compute in Python);
  (b) scan + hll_estimates() + postprocess.nested_result.
The nested results of (a) and (b) are compared first; then each step is timed with a host clock (each ends in a
synchronise), and the entry point alone with CUDA events over --reps calls.  Prints the card's name and power limit,
read in the same run.  Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=125_000_000)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=2, help="alternating (a) / (b) steps per query")
    args = ap.parse_args()
    import ctypes as C
    import torch
    from aresdb_b200 import cabi as A, columns, expr as E, synth
    from aresdb_b200.executor import Batch, FusedBatchExecutor, compute_zone_map
    from aresdb_b200.memory import CudaSpace
    from aresdb_b200.postprocess import hll_nested_result, nested_result
    from aresdb_b200.query import AggQuery, Measure
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("gpu:", smi.stdout.strip() or smi.stderr.strip(), flush=True)
    lib = A.load_engine()
    space = CudaSpace(0)
    dev = space.dev
    batches = []
    for d in range(args.batches):
        bufs, off = synth.generate_batch_cuda(d, args.rows, dev)
        cols = [columns.slice_of(b.data_ptr(), dt, args.rows, 0, off, 2) for b, dt in zip(bufs, synth.COLUMN_TYPES)]
        batches.append(Batch(cols, args.rows, keep=bufs, ranges=compute_zone_map(lib, space, cols)))
    TS, CITY, STATUS = (E.Col(i, t) for i, t in enumerate(synth.COLUMN_TYPES[:3]))
    qs = {
        "cfg4_hll_day_x_city": (AggQuery([E.eq(STATUS, E.Lit(1))], [E.floor(TS, E.Lit(86400)), CITY],
                                         Measure("countdistincthll", TS)), 0),
        "hll_hour_x_city": (AggQuery([], [E.floor(TS, E.Lit(3600)), CITY], Measure("countdistincthll", TS)), 24 * 100 * args.batches),
    }
    for name, (q, eg) in qs.items():
        ex = FusedBatchExecutor(lib, space, q, eg)

        def scan():
            ex.reset()
            for b in batches:
                ex.process_batch(b)

        def step_a():
            scan()
            return hll_nested_result(ex.hll_result())

        def step_b():
            scan()
            return nested_result(ex.hll_estimates())

        a, b = step_a(), step_b()   # (also the warm-up of both)
        assert a == b, f"{name}: the estimates differ from HLL.Compute on the host"
        groups = ex.hll_estimates().groups
        print(json.dumps({"query": name, "groups": groups, "checked": True}), flush=True)
        ta, tb = [], []
        for _ in range(args.steps):
            for fn, ts in ((step_a, ta), (step_b, tb)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                ts.append(1e3 * (time.perf_counter() - t0))
        # the entry point alone (the state holds the last scan): CUDA events around each call, outputs freed after it
        ev, dims, est = [], C.c_void_p(), C.c_void_p()
        for _ in range(args.reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            lib.AggStateFinalizeHLLEstimate(ex.state, C.byref(dims), C.byref(est), space.stream, space.device)
            e.record()
            torch.cuda.synchronize()
            ev.append(s.elapsed_time(e))
            for p in (dims, est):
                lib.DeviceFree(p, space.device)
        hv = []
        for _ in range(args.reps):   # the register-vector entry point, for scale
            t0 = time.perf_counter()
            ex.hll_result()
            hv.append(1e3 * (time.perf_counter() - t0))
        med = lambda xs: round(sorted(xs)[len(xs) // 2], 3)
        print(json.dumps({"query": name, "groups": groups, "rows": args.rows * args.batches,
                          "a_host_estimates_ms": [round(x, 1) for x in ta], "b_device_estimates_ms": [round(x, 1) for x in tb],
                          "AggStateFinalizeHLLEstimate_ms_median": med(ev), "min": round(min(ev), 3), "max": round(max(ev), 3),
                          "hll_result_ms_median": med(hv)}), flush=True)
        ex.close()


if __name__ == "__main__":
    main()
