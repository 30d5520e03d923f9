"""The group table grows instead of failing (reference: a fresh map of 2 x rows per batch, query/hash_reduction.cu:211-292,
never runs out).  ARESDB_B200_TABLE_SLOTS starts the table small so that ordinary test sizes cross the threshold:
hash-table tile kernels stop at the threshold, the host doubles the table and resumes them; direct-indexed kernels (not
waited for) park new groups in the spill list, folded at the next synchronising call; merges get their room up front.
Results must equal the reference call sequence bit for bit."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

CHILD = r"""
import sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
import numpy as np
import harness as H, test_pipeline_parity as T
from aresdb_b200 import cabi as A, expr as E, synth
from aresdb_b200.query import AggQuery, Measure
eng, orc = H.get_backend("b200"), H.get_backend("oracle")
TS, CITY, STATUS, FARE = T.TS, T.CITY, T.STATUS, T.FARE
hbs = [synth.generate_batch(d, 60000, num_cities=50, null_rate=0.01) for d in range(3)]
for case in {cases!r}:
  if case == "hash":        # ~1.7e5 near-unique groups through the hash-table kernels: two doublings from 2^17 slots
      q = AggQuery([E.ne(CITY, E.Lit(0))], [TS, CITY], Measure("sum", FARE))
      exp = T.run_legacy(orc, q, hbs)
      got = T.run_fused(eng, q, hbs)
      assert exp.groups > 150000
      T.assert_same_result(got, exp, ctx=case)
  elif case == "hash_big":  # the DEFAULT table (2^21 slots) against 2 x 2.5e6 near-unique rows: every CTA folds several tiles,
      # the stop comes mid-batch, warps drain at different tiles and the resumed launch picks each of them up where it stopped
      big = [synth.generate_batch(d, 2500000, num_cities=200, null_rate=0.01) for d in range(2)]
      q = AggQuery([E.ne(CITY, E.Lit(0))], [TS, CITY], Measure("sum", FARE))
      exp = T.run_legacy(orc, q, big)
      got = T.run_fused(eng, q, big)
      assert exp.groups > 4000000
      assert (got.packed_rows() == exp.packed_rows()).all() and got.measures.tobytes() == exp.measures.tobytes()
  elif case == "hash32":    # hash-reduce mode with the bypass kernel
      q = AggQuery([], [CITY, E.floor(TS, E.Lit(2))], Measure("count"), reduce_mode=A.ARES_REDUCE_HASH)
      exp = T.run_legacy(orc, q, hbs)
      got = T.run_fused(eng, q, hbs, expected_groups=100000)
      assert exp.groups > 100000
      # group identity in this mode is the 32-bit hash: ~5 pairs of different rows collide at this size and merge; which
      # member names the merged group is unspecified on the reference's device path too (concurrent insert), so the
      # comparison is by hash, and every row named must be a row of the data
      import hashes as HS
      by_hash = lambda r: dict(zip(HS.murmur3_32(r.packed_rows()).tolist(), r.measures.tolist()))
      assert got.groups == exp.groups and by_hash(got) == by_hash(exp), "hash32: groups by hash differ"
      every = T.run_legacy(orc, AggQuery([], [CITY, E.floor(TS, E.Lit(2))], Measure("count")), hbs)
      assert every.groups > exp.groups and set(got.rows) <= set(every.rows)
  elif case == "spill":     # direct-indexed kernels with the zone map of ANOTHER batch: every row is out of range
      q = AggQuery([E.eq(STATUS, E.Lit(1))], [E.floor(TS, E.Lit(60)), CITY], Measure("sum", FARE))
      small = [synth.generate_batch(d, 30000, num_cities=50) for d in range(2)]
      exp = T.run_legacy(orc, q, small)
      zms = [synth.zone_map(hb) for hb in small][::-1]
      before = T.dense_launches(eng)
      got = T.run_fused(eng, q, small, zone_maps=zms)
      assert T.dense_launches(eng) - before == 2 and exp.groups > 4096
      T.assert_same_result(got, exp, ctx=case)
  elif case == "tail":      # batches without a full tile: one CTA folds them as its tail, its flush parks the groups the
      # table cannot take, the host grows the table and the resumed launch does not fold the tail again
      small = [synth.generate_batch(d, 4000, num_cities=50, null_rate=0.01) for d in range(3)]
      q = AggQuery([], [TS, CITY], Measure("sum", FARE))
      exp = T.run_legacy(orc, q, small)
      got = T.run_fused(eng, q, small)
      assert exp.groups > 4096
      T.assert_same_result(got, exp, ctx=case)
  elif case == "merge":     # AggStateMerge of more rows than the table holds
      from aresdb_b200.executor import FusedBatchExecutor
      q = AggQuery([], [TS, CITY], Measure("count"))
      parts = []
      for half in (hbs[:1], hbs[1:]):
          ex = FusedBatchExecutor(eng.lib, eng.space, q)
          keep = [T.upload(eng, hb) for hb in half]
          for b in keep:
              ex.process_batch(b)
          parts.append(ex.finalize_into())
          ex.close()
      merged = FusedBatchExecutor(eng.lib, eng.space, q)
      for g, out in parts:
          merged.merge(out.dimension_vector(q), out.measures.ptr, g)
      got = merged.result()
      merged.close()
      T.assert_same_result(got, T.run_legacy(orc, q, hbs), ctx=case)
print("ok")
"""


# one child process per table size, several cases in it: a child pays for the Python start-up, the library load and the
# NVRTC compiles once
GROUPS = [
    ("slots17-jit", ["hash", "hash32"], 1 << 17),
    ("default-jit", ["hash_big"], 0),
    ("slots12-jit", ["spill", "merge", "tail"], 1 << 12),
]


@pytest.mark.parametrize("name,cases,slots", GROUPS, ids=[g[0] for g in GROUPS])
def test_table_grows(name, cases, slots):
    code = CHILD.format(tests=str(ROOT / "tests"), root=str(ROOT), cases=cases)
    env = dict(os.environ)
    if slots:
        env["ARESDB_B200_TABLE_SLOTS"] = str(slots)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-1500:] + r.stderr[-4000:]
