#!/usr/bin/env python
"""The 4-query cfg3 request {sum(fare), count(*), avg(fare), max(city_id)} over the cfg3 table (8 day-batches x 1.25e8
rows, zone maps), batch d on rank d mod N.

N > 1: ShardedFusedRequest (one shared scan, one export, one merge and one finalize launch for the request) against four
ShardedFusedQuery runs (a scan, an export, a merge and a finalize per query), alternating in one process per rank.
N = 1: FusedRequestExecutor.results() (one AggStatesFinalize) against four finalize_into calls on the same states.
Results of both forms are compared before anything is timed.  A step is the scan of the rank's batches plus the finalize
(host clock around work that ends in a synchronise, and the barrier of the exchange at N > 1); "finalize_ms" is the
finalize alone.  Reports the median of the steps, the engine's kernel launches per step (AresKernelLaunchCount), the card
and its power limit read in the same run, and N.
Usage: python tools/sharded_request_bench.py [--gpus N] [--steps K] [--batches B] [--rows R]"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _worker(rank, args, port, out):
    world = args.gpus
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import numpy as np
    import torch
    import torch.distributed as dist
    import bench
    from aresdb_b200 import cabi as A, columns, expr as E, synth
    from aresdb_b200.executor import Batch, FusedRequestExecutor, query_result
    from aresdb_b200.memory import CudaSpace
    from aresdb_b200.query import AggQuery, Measure
    from aresdb_b200.sharding import ShardedFusedQuery, ShardedFusedRequest

    torch.cuda.set_device(rank)
    dev = torch.device(f"cuda:{rank}")
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    lib = A.load_engine()
    space = CudaSpace(rank, torch.cuda.current_stream().cuda_stream)
    base = bench._q_cfg3()
    fare, city = E.Col(3, A.Float32, "fare"), E.Col(1, A.Uint16, "city_id")
    qs = [AggQuery(base.filters, base.dimensions, m) for m in (Measure("sum", fare), Measure("count"), Measure("avg", fare),
                                                                 Measure("max", city))]
    keep, batches = [], []
    for d in range(args.batches):
        if d % world != rank:
            continue
        bufs, voff = synth.generate_batch_cuda(d, args.rows, dev)
        keep.append(bufs)
        batches.append(Batch([columns.slice_of(b.data_ptr(), dt, args.rows, 0, voff, 2) for b, dt in zip(bufs, synth.COLUMN_TYPES)],
                             args.rows, ranges=synth.zone_map_of_day(d)))
    torch.cuda.synchronize()

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    # the two forms: (reset, scan, finalize), finalize returning QueryResults in request order
    if world > 1:
        one = ShardedFusedRequest(lib, space, qs)
        sep = [ShardedFusedQuery(lib, space, q) for q in qs]
        forms = {"request": (lambda: one.reset(), lambda b: one.process_batch(b), one.finalize),
                 "separate": (lambda: [s.reset() for s in sep], lambda b: [s.process_batch(b) for s in sep],
                              lambda: [query_result(s.q, *s.finalize()) for s in sep])}
    else:
        req = FusedRequestExecutor(lib, space, qs)
        forms = {"request": (req.reset, req.process_batch, req.results),
                 "separate": (req.reset, req.process_batch, lambda: [ex.result() for ex in req.executors])}

    def step(name):
        reset, scan, fin = forms[name]
        reset()
        sync()
        k0, t0 = lib.kernel_launch_count(), time.perf_counter()
        for b in batches:
            scan(b)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        res = fin()
        sync()
        t2 = time.perf_counter()
        return res, (t2 - t0) * 1e3, (t2 - t1) * 1e3, lib.kernel_launch_count() - k0

    got = {name: step(name)[0] for name in forms}   # results first
    for q, a, b in zip(qs, got["request"], got["separate"]):
        assert a.rows == b.rows and a.groups == b.groups, f"{q.measure_kind}: groups differ"
        if q.agg_func == A.AGGR_AVG_FLOAT:
            assert a.counts.tolist() == b.counts.tolist()
            np.testing.assert_allclose(a.measures, b.measures, rtol=2e-5, atol=1e-6)
        else:
            assert a.measures.tobytes() == b.measures.tobytes(), f"{q.measure_kind} differs"
    t = {n: {"step": [], "finalize": [], "launches": []} for n in forms}
    for _ in range(args.steps):   # alternate the two forms
        for name in forms:
            _, s, f, k = step(name)
            t[name]["step"].append(s)
            t[name]["finalize"].append(f)
            t[name]["launches"].append(k)
    if rank == 0:
        smi = subprocess.run(["nvidia-smi", f"--id={rank}", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        med = {n: {k: float(np.median(v)) for k, v in d.items()} for n, d in t.items()}
        report = {"gpu": smi, "gpus": world, "rows": args.rows * args.batches, "batches": args.batches, "steps": args.steps,
                  "queries": len(qs), "results_equal": True,
                  "request": {"step_ms": med["request"]["step"], "finalize_ms": med["request"]["finalize"],
                              "launches_per_step": med["request"]["launches"], "step_ms_all": t["request"]["step"]},
                  "separate": {"step_ms": med["separate"]["step"], "finalize_ms": med["separate"]["finalize"],
                               "launches_per_step": med["separate"]["launches"], "step_ms_all": t["separate"]["step"]}}
        Path(out).write_text(json.dumps(report))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--rows", type=int, default=125_000_000)
    args = ap.parse_args()
    import tempfile
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as tmp:
        out = str(Path(tmp) / "report.json")
        if args.gpus == 1:
            _worker(0, args, 0, out)
        else:
            mp.spawn(_worker, args=(args, 29600 + os.getpid() % 2000, out), nprocs=args.gpus, join=True)
        report = json.loads(Path(out).read_text())
    r, s = report["request"], report["separate"]
    print(f"N={report['gpus']} {report['gpu']}: request {r['step_ms']:.3f} ms/step (finalize {r['finalize_ms']:.3f} ms, "
          f"{r['launches_per_step']:.0f} launches) vs separate {s['step_ms']:.3f} ms/step (finalize {s['finalize_ms']:.3f} ms, "
          f"{s['launches_per_step']:.0f} launches), median of {report['steps']} steps", file=sys.stderr)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
