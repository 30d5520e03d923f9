"""Group identity is the HASH of the packed dimension row, not the row (reference query/sort_reduce.cu:140-157,
query/hash_reduction.cu:216-243): rows whose hashes collide are ONE group.  Legacy Sort+Reduce and HashReduce keep
the dimension values of the first member in input order; the measures of all members are combined.

* 32-bit (HashReduce, the hash-reduce mode of the fused path): real murmur3-32 collisions are constructed by
  search (birthday bound: ~4e5 candidate rows give ~20 colliding pairs) — SURVEY.md 0.3 predicts ~116 such pairs at
  cfg4 scale.
* 64-bit (Sort+Reduce, the sort-reduce mode): collisions cannot be found by search; a test-only seam
  (ARESDB_B200_TEST_HASH64_MASK, same variable in the engine and the C restatement) masks the hash down to a
  few bits in a child process.
"""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import harness as H
import hashes
import parity_cases as P
from aresdb_b200 import cabi as A

ND = (0, 0, 1, 1, 0)   # one 4-byte + one 2-byte dimension: packed row = [u32][u16][valid][valid] = 8 bytes


def packed_rows(v4, v2):
    n = len(v4)
    rows = np.zeros((n, 8), np.uint8)
    rows[:, 0:4] = np.asarray(v4, "<u4").view(np.uint8).reshape(n, 4)
    rows[:, 4:6] = np.asarray(v2, "<u2").view(np.uint8).reshape(n, 2)
    rows[:, 6:8] = 1
    return rows


def find_collisions32(limit=8):
    """[(rowA, rowB)] of distinct (v4, v2) pairs with equal murmur3-32 of the packed row."""
    v4 = np.repeat(np.arange(4000, dtype=np.uint32) * 60 + 1_726_963_200, 100)
    v2 = np.tile(np.arange(1, 101, dtype=np.uint16), 4000)
    h = hashes.murmur3_32(packed_rows(v4, v2))
    order = np.argsort(h, kind="stable")
    hs = h[order]
    dup = np.nonzero(hs[1:] == hs[:-1])[0]
    out = [((int(v4[order[i]]), int(v2[order[i]])), (int(v4[order[i + 1]]), int(v2[order[i + 1]]))) for i in dup[:limit]]
    assert out, "no murmur3-32 collision among 4e5 rows"
    return out


def dim_block(v4, v2, capacity):
    offs, nulls, widths, total = H.dim_layout(ND, capacity)
    n = len(v4)
    block = np.zeros(total, np.uint8)
    block[offs[0]:offs[0] + 4 * n] = np.asarray(v4, "<u4").view(np.uint8)
    block[offs[1]:offs[1] + 2 * n] = np.asarray(v2, "<u2").view(np.uint8)
    block[nulls[0]:nulls[0] + n] = 1
    block[nulls[1]:nulls[1] + n] = 1
    return block


def test_numpy_hashes_match_the_oracle():
    orc = H.get_backend("oracle")
    dll = orc.lib.alg
    dll.oracle_murmur3_32.restype = C.c_uint32
    dll.oracle_murmur3_32.argtypes = [C.c_char_p, C.c_int, C.c_uint32]
    dll.oracle_murmur3_128.restype = None
    dll.oracle_murmur3_128.argtypes = [C.c_char_p, C.c_int, C.c_uint32, C.POINTER(C.c_uint64)]
    rng = np.random.default_rng(5)
    rows = rng.integers(0, 256, (200, 8), dtype=np.uint8)
    h32 = hashes.murmur3_32(rows)
    h64 = hashes.murmur3_128_lo(rows)
    for r, a, b in zip(rows, h32, h64):
        assert dll.oracle_murmur3_32(r.tobytes(), 8, 0) == int(a)
        out = (C.c_uint64 * 2)()
        dll.oracle_murmur3_128(r.tobytes(), 8, 0, out)
        assert out[0] == int(b)
    # known answers from the reference's own test (SortAndReduceTest.CheckHash, query/algorithm_unittest.cu:1160-1217)
    ka = {2: 0x60e187b4814392c4, 0: 0x7cb3f5c58dab264c, 3: 0xb73e42bb654cee53, 1: 0xca410abc0a9d4c6b}
    for v, want in ka.items():
        assert int(hashes.murmur3_128_lo(np.array([[v, 1]], np.uint8))[0]) == want


def test_numpy_murmur3_128_matches_the_oracle_up_to_32_bytes():
    """Every packed-row length the engine hashes (1..32 bytes: no body block, one and two 16-byte body blocks, each
    tail length), against the oracle's byte-wise x64_128."""
    dll = H.get_backend("oracle").lib.alg
    dll.oracle_murmur3_128.restype = None
    dll.oracle_murmur3_128.argtypes = [C.c_char_p, C.c_int, C.c_uint32, C.POINTER(C.c_uint64)]
    rng = np.random.default_rng(6)
    for ln in range(1, 33):
        rows = rng.integers(0, 256, (40, ln), dtype=np.uint8)
        rows[0] = 0
        rows[1] = 255
        got = hashes.murmur3_128_lo(rows)
        for r, h in zip(rows, got):
            out = (C.c_uint64 * 2)()
            dll.oracle_murmur3_128(r.tobytes(), ln, 0, out)
            assert out[0] == int(h), f"length {ln}"


def collision_case():
    """Input rows in which two colliding pairs interleave with ordinary rows; returns everything the checks need."""
    (a1, b1), (a2, b2) = find_collisions32(2)
    others = [(1_726_963_200 + 60 * k, 7 + k % 5) for k in range(40)]
    seq = [b1, others[0], a1, others[1], a1, b1, a2, others[2], b2, a2] + others + [b2, a1]
    rng = np.random.default_rng(11)
    meas = (rng.integers(1, 6400, len(seq)) / 64.0).astype(np.float64)
    return seq, meas, [(a1, b1), (a2, b2)]


def expected_hash_groups(seq, meas):
    """{hash32: (first row, sum)} — what HashReduce must produce (first member in input order names the group)."""
    rows = packed_rows([s[0] for s in seq], [s[1] for s in seq])
    h = hashes.murmur3_32(rows)
    out = {}
    for i, hv in enumerate(h.tolist()):
        if hv not in out:
            out[hv] = [rows[i].tobytes(), 0.0]
        out[hv][1] += float(meas[i])
    return {r: s for r, s in out.values()}


def run_hash_reduce(be, seq, meas):
    n = len(seq)
    block = dim_block([s[0] for s in seq], [s[1] for s in seq], n)
    r = P.run_hash_reduce(be, block, ND, n, n, meas, 8, A.AGGR_SUM_FLOAT)
    return {k: np.frombuffer(v, np.float64)[0] for k, v in r["groups"].items()}


@pytest.mark.parametrize("backend", ["ref", "oracle"])
def test_hash_reduce_merges_colliding_rows_cpu(backend):
    seq, meas, pairs = collision_case()
    got = run_hash_reduce(H.get_backend(backend), seq, meas)
    exp = expected_hash_groups(seq, meas)
    assert len(exp) == len(set(seq)) - len(pairs)        # each colliding pair is one group
    assert got == exp                                      # ... named by its first member, measures combined


@pytest.mark.gpu
def test_hash_reduce_merges_colliding_rows_b200():
    seq, meas, pairs = collision_case()
    assert run_hash_reduce(H.get_backend("b200"), seq, meas) == expected_hash_groups(seq, meas)


@pytest.mark.parametrize("backend", ["ref", "oracle"])
def test_sort_reduce_keeps_32bit_colliders_apart_cpu(backend):
    """The same rows through Sort + Reduce (64-bit identity): no merge."""
    seq, meas, _ = collision_case()
    n = len(seq)
    r = P.run_sort_reduce(H.get_backend(backend), dim_block([s[0] for s in seq], [s[1] for s in seq], n), ND, n, n, meas, 8,
                          A.AGGR_SUM_FLOAT)
    assert r["g"] == len(set(seq))


@pytest.mark.gpu
def test_fused_hash_mode_merges_colliding_rows_b200():
    """The fused path in hash-reduce mode: colliding rows are ONE group with the combined measure.  Which member
    names it is unspecified on the reference's DEVICE path as well (cudf's concurrent insert: the first thread to
    win the CAS, query/hash_reduction.cu:216-243), so any member is accepted."""
    import test_pipeline_parity as T
    from aresdb_b200 import expr as E, synth
    from aresdb_b200.query import AggQuery, Measure
    eng = H.get_backend("b200")
    (a1, b1), (a2, b2) = find_collisions32(2)
    members = {packed_rows([x[0]], [x[1]])[0].tobytes(): i for i, x in enumerate((a1, b1, a2, b2))}
    # a batch whose request_at / city_id make floor(ts, 60) x city hit the four colliding rows plus ordinary groups
    rows = 4000
    hb = synth.generate_batch(0, rows, num_cities=50, null_rate=0.0)
    for i, (t, c) in enumerate([a1, b1, a2, b2] * 25):
        hb.values[0][i * 7] = t + (i % 60)
        hb.values[1][i * 7] = c
    q = AggQuery([], [T.CITY, E.floor(T.TS, E.Lit(60))], Measure("sum", T.FARE), reduce_mode=A.ARES_REDUCE_HASH)
    for zm in (None, [synth.zone_map(hb)]):
        got = T.run_fused(eng, q, [hb], zone_maps=zm).as_dict()
        # expectation from first principles: group rows by murmur3-32 of their packed dimension row
        ts, city, fare = hb.values[0], hb.values[1], hb.values[3].astype(np.float64)
        prow = packed_rows(ts - ts % 60, city)
        h = hashes.murmur3_32(prow)
        classes = {}
        for i, hv in enumerate(h.tolist()):
            classes.setdefault(hv, [set(), 0.0])
            classes[hv][0].add(prow[i].tobytes())
            classes[hv][1] += fare[i]
        assert len(got) == len(classes)
        merged = 0
        for row, val in got.items():
            cls = classes[int(hashes.murmur3_32(np.frombuffer(row, np.uint8).reshape(1, 8))[0])]
            assert row in cls[0] and val == cls[1]
            merged += len(cls[0]) > 1
        assert merged == 2


# ---- 64-bit identity through the test-only seam (child process: the mask is read once per process) ------------
CHILD = r"""
import sys, numpy as np
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
import harness as H, hashes, parity_cases as P
from aresdb_b200 import cabi as A
import test_hash_collisions as T
mask = {mask}
rng = np.random.default_rng(3)
n = 600
v4 = rng.integers(0, 300, n).astype(np.uint32) + 1_726_963_200
v2 = rng.integers(1, 4, n).astype(np.uint16)
meas = (rng.integers(1, 6400, n) / 64.0).astype(np.float64)
rows = T.packed_rows(v4, v2)
h = hashes.murmur3_128_lo(rows) & np.uint64(mask)
exp = {{}}
for i, hv in enumerate(h.tolist()):          # first member in input order names the run; measures combine
    exp.setdefault(hv, [rows[i].tobytes(), 0.0])[1] += float(meas[i])
order = sorted(exp)                           # output order = ascending (masked) hash
want_rows = [exp[k][0] for k in order]
want_vals = [exp[k][1] for k in order]
assert len(order) < len(set(r.tobytes() for r in rows)), "the mask produced no collision"
for name in {backends!r}:
    be = H.get_backend(name)
    r = P.run_sort_reduce(be, T.dim_block(v4, v2, n), T.ND, n, n, meas, 8, A.AGGR_SUM_FLOAT)
    assert r["g"] == len(order), (name, r["g"], len(order))
    assert r["rows"] == want_rows, name
    assert np.frombuffer(r["measures"].tobytes(), np.float64).tolist() == want_vals, name
if {fused}:
    import test_pipeline_parity as TP
    from aresdb_b200 import expr as E, synth
    from aresdb_b200.query import AggQuery, Measure
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    hbs = [synth.generate_batch(d, 5000, num_cities=30) for d in range(2)]
    q = AggQuery([], [E.floor(TP.TS, E.Lit(3600)), TP.CITY], Measure("sum", TP.FARE))
    ref = TP.run_legacy(orc, q, hbs)
    for zm in (None, [synth.zone_map(hb) for hb in hbs]):
        got = TP.run_fused(eng, q, hbs, zone_maps=zm)
        assert got.groups == ref.groups < 2 * 24 * 31, (got.groups, ref.groups)
        assert got.measures.tobytes() == ref.measures.tobytes()      # merged sums, hash-ascending order
        # dims: a member of the run (first-in-stable-order is the reference's rule; the fused path keeps the member
        # its table slot order yields — DESIGN.md 4, deviation (2), probability g^2 / 2^65 without the seam)
print("ok")
"""


def _run_child(backends, fused, mask=0xFF):
    root = Path(__file__).resolve().parent.parent
    code = CHILD.format(tests=str(root / "tests"), root=str(root), mask=mask, backends=backends, fused=fused)
    env = dict(os.environ, ARESDB_B200_TEST_HASH64_MASK=f"{mask:x}")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


def test_sort_reduce_merges_runs_of_equal_hashes_oracle():
    _run_child(["oracle"], False)


@pytest.mark.gpu
def test_sort_reduce_merges_runs_of_equal_hashes_b200():
    _run_child(["oracle", "b200"], True)
