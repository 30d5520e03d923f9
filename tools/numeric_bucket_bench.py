"""Times numeric-bucketizer histograms on the fused kernel over the cfg3 table (bench.py's synthetic trips: B batches of
N rows, zone maps from the engine), against count(*) by city_id x hour over the same batches.

  python tools/numeric_bucket_bench.py [--rows N] [--batches B] [--reps R]

Queries: count(*) by 16 and by 255 fare partitions, by a fare width x hour, by a log base of the fare, and the control.
Each result is first compared with a torch restatement (torch.bucketize / the width's floor) of the same rows; then the
queries are timed in alternating steps (one pass over all batches each, CUDA events) and the median per query printed
with the card's name and power limit, read in the same run.  Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

PARTS16 = [float(x) for x in range(0, 96, 6)]
PARTS255 = [100.0 * i / 255 for i in range(255)]


def queries():
    q = lambda dims: {"table": "trips", "measures": [{"sqlExpression": "count(*)"}], "dimensions": dims}
    hour = {"sqlExpression": "request_at", "timeBucketizer": "hour"}
    return {
        "partitions16": q([{"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": PARTS16}}]),
        "partitions255": q([{"sqlExpression": "fare", "numericBucketizer": {"manualPartitions": PARTS255}}]),
        "width2.5_x_hour": q([hour, {"sqlExpression": "fare", "numericBucketizer": {"bucketWidth": 2.5}}]),
        "log1.5": q([{"sqlExpression": "fare", "numericBucketizer": {"logBase": 1.5}}]),
        "city_x_hour": q([hour, {"sqlExpression": "city_id"}]),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=125_000_000)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    from aresdb_b200 import aql, cabi as A, columns, synth
    from aresdb_b200.executor import Batch, FusedBatchExecutor, compute_zone_map
    from aresdb_b200.memory import CudaSpace
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("gpu:", smi.stdout.strip() or smi.stderr.strip(), flush=True)
    lib = A.load_engine()
    space = CudaSpace(0)
    dev = space.dev
    table = aql.Table("trips", [aql.Column(n, t) for n, t in zip(synth.COLUMN_NAMES, synth.COLUMN_TYPES)])
    batches, keep = [], []
    bits = torch.arange(8, device=dev, dtype=torch.uint8)
    fares = []
    for d in range(args.batches):
        bufs, off = synth.generate_batch_cuda(d, args.rows, dev, exact_fares=False)
        cols = [columns.slice_of(b.data_ptr(), dt, args.rows, 0, off, 2) for b, dt in zip(bufs, synth.COLUMN_TYPES)]
        batches.append(Batch(cols, args.rows, keep=bufs, ranges=compute_zone_map(lib, space, cols)))
        f = bufs[synth.COL_FARE]
        ok = ((f[:(args.rows + 7) // 8].unsqueeze(1) >> bits) & 1).reshape(-1)[:args.rows].bool()
        fares.append((f[off:off + 4 * args.rows].view(torch.float32), ok))
    qs = {n: aql.compile_query(t, table, synth.BASE_TS, upload=space.put) for n, t in queries().items()}
    exs = {n: FusedBatchExecutor(lib, space, q) for n, q in qs.items()}
    # results first: every query once, each compared with its restatement (fare histograms) or its row count
    for n, ex in exs.items():
        for b in batches:
            ex.process_batch(b)
        r = ex.result()
        ex.reset()
        assert int(r.measures.sum()) == args.rows * args.batches, n
        if n.startswith("partitions"):
            p = torch.tensor(PARTS16 if n == "partitions16" else PARTS255, dtype=torch.float64, device=dev)
            exp = torch.zeros(len(p) + 1, dtype=torch.int64, device=dev)
            nulls = 0
            for f, ok in fares:
                exp += torch.bincount(torch.bucketize(f[ok].to(torch.float64), p, right=True), minlength=len(p) + 1)
                nulls += int((~ok).sum())
            got = {k: int(m) for k, m in zip(r.decoded_dims()[0], r.measures.tolist())}
            want = {k: int(c) for k, c in enumerate(exp.tolist()) if c}
            if nulls:
                want[None] = nulls
            assert got == want, f"{n}: histogram differs from torch.bucketize"
        print(json.dumps({"query": n, "groups": r.groups, "checked": True}), flush=True)
    # alternating steps: one pass of every query per step
    times = {n: [] for n in exs}
    for n, ex in exs.items():   # warm-up
        for b in batches:
            ex.process_batch(b)
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for n, ex in exs.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ex.reset()
            torch.cuda.synchronize()
            s.record()
            for b in batches:
                ex.process_batch(b)
            e.record()
            torch.cuda.synchronize()
            times[n].append(s.elapsed_time(e))
    for n, ts in times.items():
        ts.sort()
        print(json.dumps({"query": n, "ms_per_pass_median": round(ts[len(ts) // 2], 3), "min": round(ts[0], 3),
                          "max": round(ts[-1], 3), "rows": args.rows * args.batches}), flush=True)
    for ex in exs.values():
        ex.close()


if __name__ == "__main__":
    main()
