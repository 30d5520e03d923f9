"""Times a month-of-year and an hour-of-day count(*) over the same rows on the fused kernel, for one or two builds of
the engine, alternating them in one call.

Month of year is direct-indexed by the calendar functor's own range (jit.cu, jitAnalyzeDense); a range that does not
contain a row's value sends the row out of line to the global hash table.  Hour of day, indexed through the time
column's zone map, is the control.  Both queries read the same batches of a year of uniformly spread instants.

  python tools/time_bucket_bench.py [--lib DIR ...] [--rows N] [--batches B] [--reps R] [--rounds K]

Each `--lib` is a directory holding libalgorithm.so and libmem.so (default: the in-tree build).  Every (library, round)
runs in a process of its own; the line per run gives milliseconds per pass over all batches and a digest of each
result, which must agree between libraries.  Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import calendar
import hashlib
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def child(args):
    import numpy as np
    import torch
    from aresdb_b200 import aql, cabi as A, columns
    from aresdb_b200.executor import Batch, FusedBatchExecutor
    from aresdb_b200.memory import CudaSpace
    if args.lib:
        A.ENGINE_LIB_DIR = Path(args.lib)
    lib = A.load_engine()
    torch.zeros(1, device="cuda:0")
    space = CudaSpace(0)
    table = aql.Table("trips", [aql.Column("request_at", A.Uint32), aql.Column("v", A.Uint16)])
    lo = calendar.timegm((2024, 1, 1, 0, 0, 0))
    span = 366 * 86400
    rng = np.random.default_rng(1)
    batches = []
    for _ in range(args.batches):
        ts = (lo + rng.integers(0, span, args.rows)).astype(np.uint32)
        tb, tvp = columns.make_column(space, A.Uint32, ts)
        vb, vvp = columns.make_column(space, A.Uint16, np.ones(args.rows, np.uint16))
        batches.append(Batch([tvp, vvp], args.rows, keep=[tb, vb], ranges={0: (int(ts.min()), int(ts.max()))}))
    out = {"lib": args.lib or "in-tree", "gpu": torch.cuda.get_device_name(0)}
    for name in ("month of year", "hour of day"):
        q = aql.compile_query({"table": "trips", "measures": [{"sqlExpression": "count(*)"}],
                               "dimensions": [{"sqlExpression": "request_at", "timeBucketizer": name}]}, table, lo)
        ex = FusedBatchExecutor(lib, space, q)
        for _ in range(3):                          # warm-up: NVRTC compile, module load
            for b in batches:
                ex.process_batch(b)
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.reps):
            for b in batches:
                ex.process_batch(b)
        end.record()
        torch.cuda.synchronize()
        r = ex.result()
        ex.close()
        out[name] = {"ms_per_pass": start.elapsed_time(end) / args.reps, "groups": r.groups,
                     "digest": hashlib.sha256(r.packed_rows().tobytes() + r.measures.tobytes()).hexdigest()[:16]}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None)
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        args.lib = args.lib[0] if args.lib else None
        return child(args)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("gpu:", smi.stdout.strip() or smi.stderr.strip(), flush=True)
    libs = args.lib or [None]
    runs = []
    for _ in range(args.rounds):
        for lib in libs:
            cmd = [sys.executable, __file__, "--child", "--rows", str(args.rows), "--batches", str(args.batches),
                   "--reps", str(args.reps)] + (["--lib", lib] if lib else [])
            line = subprocess.run(cmd, check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1]
            print(line, flush=True)
            runs.append(json.loads(line))
    for name in ("month of year", "hour of day"):
        assert len({r[name]["digest"] for r in runs}) == 1, f"{name}: results differ between runs"
        for lib in libs:
            ms = sorted(r[name]["ms_per_pass"] for r in runs if r["lib"] == (lib or "in-tree"))
            print(f"{name:14s} {lib or 'in-tree':30s} median {ms[len(ms) // 2]:.3f} ms per pass "
                  f"({args.batches} x {args.rows:,} rows; min {ms[0]:.3f}, max {ms[-1]:.3f})")


if __name__ == "__main__":
    main()
