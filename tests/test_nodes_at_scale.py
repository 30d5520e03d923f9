"""The per-node entry points (Unary/BinaryFilter, Sort, Reduce, HashReduce, HyperLogLog) at the sizes where their
multi-tile machinery runs, against plain numpy restatements that share no code with the engine or the oracle.

What only shows at scale:
* filter compaction: more 1024-row tiles than resident CTAs, dynamic tile tickets, RecordID vectors moved in lockstep;
* radix sort: blocks capped at 4 x SMs, each owning a chunk of several 2048-key tiles (the digit carry between them);
* Reduce: runs longer than kLongRun (one block each), more of them than longRunKernel has blocks, the short-run
  path handing long runs on twice, run heads over many 2048-element tiles;
* HashReduce: one slot under millions of atomics, the table capacity at its doubling edge, the extraction look-back
  over thousands of tiles, and MIN / MAX / AVG (identity fill, float CAS loops).

Integer results and orders match bit for bit.  Float results match bit for bit too, because the data keeps every
partial sum exact in any association order: f32 sums add small integers whose partial sums stay below 2^24, f64 sums
add multiples of 1/64 whose partial sums stay below 2^47.  Two exceptions: AVG (a rolling float32 average whose
rounding depends on the order rows meet) is compared to 2e-5 relative, as tests/test_pipeline_parity.assert_same_avg
does; and within one float MIN / MAX group -0.0 and +0.0 compare as values, because the combine keeps whichever of
two equal operands it already holds, so the atomic or tree order decides which zero wins.

The engine's tile sizes and grid caps are not exported; they are restated below with the line that sets them, and
every case asserts from its own input that it reaches the path it targets.  The filter's look-back passing its first
32-tile window depends on timing and cannot be forced: the largest filter cases run ~1.3e5 tiles to give it the
chance, which is not a claim that it was covered.

The CPU tests pin each restatement to the oracle (and to the reference's HOST build when oracle/_ref is built, else to
the digest recorded from it) on small inputs of the same shapes.
"""
from __future__ import annotations

import ctypes as C
import gc

import numpy as np
import pytest

import harness as H
import hashes
from aresdb_b200 import cabi as A

FILTER_TILE = 1024          # kFilterTile = 256 threads x 4 items, aresdb_b200/csrc/legacy_nodes.cu:331-333
FILTER_CTAS_PER_SM = 8      # 256-thread CTAs resident per SM (2048 threads per SM on sm_90)
HEAD_TILE = 2048            # kHeadTile, aresdb_b200/csrc/sort_reduce.cu:29-31
LONG_RUN = 1 << 15          # kLongRun, aresdb_b200/csrc/sort_reduce.cu:73
LONG_RUN_BLOCKS_PER_SM = 2  # longRunKernel grid = min(n / kLongRun + 1, 2 x SMs), aresdb_b200/csrc/sort_reduce.cu:236
SORT_TILE = 2048            # kSortTile, aresdb_b200/csrc/radix_sort.cuh:22
SORT_BLOCKS_PER_SM = 4      # planGrid's block cap, aresdb_b200/csrc/radix_sort.cu:16
EXT_TILE = 2048             # kExtTile, aresdb_b200/csrc/hash_reduce.cu:52-54
HASH_MIN_CAPACITY = 64      # HashReduce table: smallest power of two >= 2 x length, at least 64, hash_reduce.cu:120-121

F32_EXACT = 1 << 24
FLT_MAX, FLT_MIN = np.float32(3.402823466e38), np.float32(1.175494351e-38)

# every (aggregate, valueBytes) pair aggOpOf accepts (aresdb_b200/csrc/agg.cuh:18-35)
AGGS = [(A.AGGR_SUM_UNSIGNED, 4), (A.AGGR_SUM_UNSIGNED, 8), (A.AGGR_SUM_SIGNED, 4), (A.AGGR_SUM_SIGNED, 8),
        (A.AGGR_SUM_FLOAT, 4), (A.AGGR_SUM_FLOAT, 8), (A.AGGR_MIN_UNSIGNED, 4), (A.AGGR_MIN_SIGNED, 4),
        (A.AGGR_MIN_FLOAT, 4), (A.AGGR_MAX_UNSIGNED, 4), (A.AGGR_MAX_SIGNED, 4), (A.AGGR_MAX_FLOAT, 4),
        (A.AGGR_AVG_FLOAT, 8)]
AGG_NAME = {A.AGGR_SUM_UNSIGNED: "sum_u", A.AGGR_SUM_SIGNED: "sum_s", A.AGGR_SUM_FLOAT: "sum_f",
            A.AGGR_MIN_UNSIGNED: "min_u", A.AGGR_MIN_SIGNED: "min_s", A.AGGR_MIN_FLOAT: "min_f",
            A.AGGR_MAX_UNSIGNED: "max_u", A.AGGR_MAX_SIGNED: "max_s", A.AGGR_MAX_FLOAT: "max_f", A.AGGR_AVG_FLOAT: "avg"}
MEASURE_TYPE = {A.AGGR_MIN_UNSIGNED: np.uint32, A.AGGR_MAX_UNSIGNED: np.uint32, A.AGGR_MIN_SIGNED: np.int32,
                A.AGGR_MAX_SIGNED: np.int32, A.AGGR_MIN_FLOAT: np.float32, A.AGGR_MAX_FLOAT: np.float32}
# the identity a DEVICE-side hash map starts every slot from (the reference's get_identity_value, query/utils.hpp:169-184;
# MAX_FLOAT really is FLT_MIN there); pinned below against the oracle's NULL -> identity measure sink
IDENTITY = {A.AGGR_MIN_UNSIGNED: np.uint32(0xFFFFFFFF), A.AGGR_MIN_SIGNED: np.int32(2**31 - 1),
            A.AGGR_MIN_FLOAT: FLT_MAX, A.AGGR_MAX_UNSIGNED: np.uint32(0), A.AGGR_MAX_SIGNED: np.int32(-2**31),
            A.AGGR_MAX_FLOAT: FLT_MIN}


def agg_id(p):
    return f"{AGG_NAME[p[0]]}{p[1]}"


def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def _free_device_memory():
    """Each case releases its device buffers before the next starts (the GPU may be shared)."""
    yield
    gc.collect()
    try:
        import torch
        if torch.cuda.is_available() and torch.cuda.is_initialized():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    except ImportError:
        pass


# ---- dimension blocks --------------------------------------------------------------------------------------------
def dim_block(rng, nd, cap, n, card):
    """Column-major DimensionVector block of n rows drawn from `card` distinct prototype rows (card=None: every row
    drawn independently, so nearly all distinct).  NULL dims store value 0, as the transform sinks leave them."""
    offs, nulls, widths, total = H.dim_layout(nd, cap)
    block = np.zeros(total, np.uint8)
    pick = None if card is None else rng.integers(0, card, n)
    for o, no, w in zip(offs, nulls, widths):
        m = n if card is None else card
        vals = rng.integers(0, 256, (m, w), dtype=np.uint8)
        valid = (rng.random(m) >= 0.05).astype(np.uint8)
        vals *= valid[:, None]
        if pick is not None:
            vals, valid = vals[pick], valid[pick]
        block[o:o + n * w] = vals.reshape(-1)
        block[no:no + n] = valid
    return block


def packed_rows(block, nd, cap, idx):
    """uint8[len(idx), rowBytes]: the dims of rows idx in layout order, then one validity byte per dim."""
    offs, nulls, widths, _ = H.dim_layout(nd, cap)
    parts = [block[o:o + cap * w].reshape(cap, w)[idx] for o, w in zip(offs, widths)]
    parts += [block[no:no + cap][idx][:, None] for no in nulls]
    return np.hstack(parts)


# ---- measures and the restated folds -----------------------------------------------------------------------------
def measures(rng, agg, vb, n, max_group):
    """Measure vector for (agg, vb) whose every partial sum over at most `max_group` rows is exact (see the module
    docstring).  Integer sums use the full range, so 32-bit sums wrap."""
    if agg in (A.AGGR_SUM_UNSIGNED, A.AGGR_SUM_SIGNED):
        if vb == 4:
            return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        return rng.integers(0, np.iinfo(np.uint64).max, n, dtype=np.uint64, endpoint=True)
    if agg == A.AGGR_SUM_FLOAT and vb == 4:
        b = min(100, (F32_EXACT - 1) // max_group)
        if b >= 1:
            return rng.integers(-b, b + 1, n).astype(np.float32)
        v = (rng.random(n) < 0.5 * F32_EXACT / n).astype(np.float32)   # 0 / 1: partial sums <= the count of ones
        assert v.sum() < F32_EXACT
        return v
    if agg == A.AGGR_SUM_FLOAT:
        assert max_group * 100 < 2 ** 47
        return rng.integers(-6400, 6401, n) / 64.0
    if agg == A.AGGR_AVG_FLOAT:
        v = (rng.integers(64, 128, n) / 64.0).astype(np.float32)        # one row each: count 1
        return (np.uint64(1) << np.uint64(32)) | v.view(np.uint32).astype(np.uint64)
    t = MEASURE_TYPE[agg]
    if t == np.float32:
        v = (rng.standard_normal(n) * 1000).astype(np.float32)
        z = rng.random(n)
        v[z < 0.02] = 0.0
        v[z > 0.98] = -0.0
        return v
    return rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(t)


def fold(agg, vb, v, starts, start_from=None):
    """Per-group result of the values v (already in group order) whose groups begin at `starts`.
    start_from: None (fold the group's own values, as Reduce does), "identity" (a hash map slot filled with the
    aggregate's identity first) or "zero" (a slot default-constructed to zero)."""
    if agg in (A.AGGR_SUM_UNSIGNED, A.AGGR_SUM_SIGNED):
        if vb == 4:
            return (np.add.reduceat(v.view(np.uint32).astype(np.uint64), starts) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        with np.errstate(over="ignore"):
            return np.add.reduceat(v.view(np.uint64), starts)
    if agg == A.AGGR_SUM_FLOAT:
        s = np.add.reduceat(v.astype(np.float64), starts)
        return s.astype(np.float32) if vb == 4 else s
    if agg == A.AGGR_AVG_FLOAT:
        cnt = np.add.reduceat(v >> np.uint64(32), starts)
        tot = np.add.reduceat((v & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.float32).astype(np.float64), starts)
        return cnt, tot / cnt
    t = MEASURE_TYPE[agg]
    is_min = agg in (A.AGGR_MIN_UNSIGNED, A.AGGR_MIN_SIGNED, A.AGGR_MIN_FLOAT)
    r = (np.minimum if is_min else np.maximum).reduceat(v.view(t), starts)
    if start_from == "identity":
        r = (np.minimum if is_min else np.maximum)(r, IDENTITY[agg])
    elif start_from == "zero":
        r = (np.minimum if is_min else np.maximum)(r, t(0))
    return r.astype(t)


def assert_measures(agg, vb, got_bytes, exp, ctx):
    """Bit-exact, except AVG (2e-5 relative, counts exact) and the sign of a float MIN / MAX zero."""
    if agg == A.AGGR_AVG_FLOAT:
        cnt, avg = exp
        got = np.frombuffer(got_bytes, np.uint64)
        assert (got >> np.uint64(32) == cnt).all(), f"{ctx}: AVG counts differ"
        gv = (got & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.float32)
        np.testing.assert_allclose(gv, avg, rtol=2e-5, atol=1e-6, err_msg=ctx)
        return
    exp = np.ascontiguousarray(exp)
    got = np.frombuffer(got_bytes, exp.dtype)
    same = got.view(np.uint8).reshape(len(got), -1) == exp.view(np.uint8).reshape(len(exp), -1)
    ok = same.all(axis=1)
    if agg in (A.AGGR_MIN_FLOAT, A.AGGR_MAX_FLOAT):
        ok |= (got == 0) & (exp == 0)
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, f"{ctx}: {bad.size} measures differ; first at {bad[0]}: got {got[bad[0]]!r}, expected {exp[bad[0]]!r}"


def measure_width(agg, vb):
    return 8 if agg == A.AGGR_AVG_FLOAT else (vb if agg in (A.AGGR_SUM_UNSIGNED, A.AGGR_SUM_SIGNED, A.AGGR_SUM_FLOAT) else 4)


# ---- calls into the C ABI ----------------------------------------------------------------------------------------
def run_filter(be, keep_rows, index, recs, binary):
    """One filter node over index positions: the predicate of position i is keep_rows[index[i]].  Binary: Equal of a
    Uint8 column and the constant 1; unary: Noop of a Bool column.  Returns (count, index, predicate, RecordIDs)."""
    n = len(index)
    keep = []
    if binary:
        vals = keep_rows.astype(np.uint8)
        vals[::3][~keep_rows[::3]] = 2
        buf, vp = H.make_column(be, A.Uint8, vals)
        keep.append(buf)
        ins = [A.vp_input(vp), A.const_input(1, True)]
    else:
        buf, vp = H.make_column(be, A.Bool, keep_rows.astype(np.uint8))
        keep.append(buf)
        ins = [A.vp_input(vp)]
    idx = be.put(np.asarray(index, np.uint32))
    pred = be.zeros(n)
    rbufs = [be.put(r) for r in recs]
    ptrs = (C.c_void_p * max(len(recs), 1))(*[b.ptr for b in rbufs])
    rp = C.cast(ptrs, C.c_void_p).value if recs else None
    s, d = be.space.stream, be.device
    if binary:
        m = be.lib.BinaryFilter(ins[0], ins[1], idx.ptr, pred.ptr, n, rp, len(recs), None, 0, A.Equal, s, d)
    else:
        m = be.lib.UnaryFilter(ins[0], idx.ptr, pred.ptr, n, rp, len(recs), None, 0, A.Noop, s, d)
    return m, idx.get(np.uint32, n), pred.get(np.uint8, n), [b.get(np.uint64, n) for b in rbufs]


def expected_filter(keep_rows, index, recs):
    """Stable in-place compaction: survivors move to the front in order; positions past the count keep their values."""
    pred = keep_rows[index]
    sel = np.flatnonzero(pred)
    m = sel.size
    idx = np.array(index, np.uint32)
    idx[:m] = idx[sel]
    out = []
    for r in recs:
        r = r.copy()
        r[:m] = r[sel]
        out.append(r)
    return m, idx, pred.astype(np.uint8), out


def run_sort(be, block, nd, cap, index):
    n = len(index)
    db, hv, idx = be.put(block), be.zeros(8 * cap), be.put(np.asarray(index, np.uint32))
    be.lib.Sort(A.make_dimension_vector(db.ptr, hv.ptr, idx.ptr, nd, cap), n, be.space.stream, be.device)
    return hv.get(np.uint64, n), idx.get(np.uint32, n)


def expected_sort(block, nd, cap, index):
    """murmur3-x64-128 low word of each packed row, then a stable sort by it (ties keep index-vector order)."""
    h = hashes.murmur3_128_lo(packed_rows(block, nd, cap, index))
    order = np.argsort(h, kind="stable")
    return h[order], np.asarray(index, np.uint32)[order]


def run_reduce(be, block, nd, cap, hv, index, meas, vb, agg):
    n = len(index)
    w = measure_width(agg, vb)
    db, hb, ib, mb = be.put(block), be.put(hv), be.put(np.asarray(index, np.uint32)), be.put(meas)
    od, oh, oi, om = be.zeros(len(block)), be.zeros(8 * cap), be.zeros(4 * cap), be.zeros(w * cap)
    g = be.lib.Reduce(A.make_dimension_vector(db.ptr, hb.ptr, ib.ptr, nd, cap), mb.ptr,
                      A.make_dimension_vector(od.ptr, oh.ptr, oi.ptr, nd, cap), om.ptr, vb, n, agg,
                      be.space.stream, be.device)
    return g, oh.get(np.uint64, g), oi.get(np.uint32, g), om.get(np.uint8, g * w), od.get(np.uint8)


def run_hash_reduce(be, block, nd, cap, n, meas, vb, agg):
    w = measure_width(agg, vb)
    db, mb = be.put(block), be.put(meas)
    od, om = be.zeros(len(block)), be.zeros(w * cap)
    g = be.lib.HashReduce(A.make_dimension_vector(db.ptr, None, None, nd, cap), mb.ptr,
                          A.make_dimension_vector(od.ptr, None, None, nd, cap), om.ptr, vb, n, agg,
                          be.space.stream, be.device)
    return g, om.get(np.uint8, g * w), od.get(np.uint8)


# ---- case builders -----------------------------------------------------------------------------------------------
PATTERNS = ["all", "none", "first", "last", "tile_edge", "alternate", "random50", "random1e-4", "last_tile"]


def pattern(name, n, rng):
    """Survivor mask over n index positions."""
    k = np.zeros(n, bool)
    if name == "all":
        k[:] = True
    elif name == "first":
        k[0] = True
    elif name == "last":
        k[-1] = True
    elif name == "tile_edge":        # one survivor per tile: the first row of even tiles, the last row of odd ones
        t = np.arange((n + FILTER_TILE - 1) // FILTER_TILE)
        pos = np.minimum(t * FILTER_TILE + np.where(t % 2 == 1, FILTER_TILE - 1, 0), n - 1)
        k[pos] = True
    elif name == "alternate":
        k[::2] = True
    elif name == "random50":
        k = rng.random(n) < 0.5
    elif name == "random1e-4":
        k = rng.random(n) < 1e-4
    elif name == "last_tile":
        k[(n - 1) // FILTER_TILE * FILTER_TILE:] = True
    return k


def filter_case(rng, name, n, sparse, num_recs):
    """(keep_rows, index, recs): with sparse=True the index vector is ascending with gaps, as a later filter sees it."""
    if sparse:
        index = (np.cumsum(1 + (rng.random(n) < 0.3)) - 1).astype(np.uint32)
        rows = int(index[-1]) + 1 + 5
    else:
        index = np.arange(n, dtype=np.uint32)
        rows = n
    keep_rows = rng.random(rows) < 0.5            # rows the index vector skips: arbitrary
    keep_rows[index] = pattern(name, n, rng)
    recs = [((np.uint64(f + 1) << np.uint64(32)) | np.arange(n, dtype=np.uint64)) for f in range(num_recs)]
    return keep_rows, index, recs


def check_filter(be, keep_rows, index, recs, binary, ctx):
    m, idx, pred, out = run_filter(be, keep_rows, index, recs, binary)
    em, eidx, epred, eout = expected_filter(keep_rows, index, recs)
    assert m == em, f"{ctx}: count {m}, expected {em}"
    assert np.array_equal(pred, epred), f"{ctx}: predicate vector differs"
    bad = np.flatnonzero(idx != eidx)
    assert bad.size == 0, f"{ctx}: index vector differs at {bad.size} positions, first {bad[0]}"
    for f, (a, b) in enumerate(zip(out, eout)):
        assert np.array_equal(a, b), f"{ctx}: RecordID vector {f} differs"
    return m


SORT_CASES = {   # name -> (dims per width, prototype rows or None, permuted index)
    "equal": ((0, 1, 0, 0, 0), 1, True),           # one hash value: output order = index-vector order
    "two": ((1, 1, 1, 0, 0), 2, False),            # 31-byte rows: a 16-byte body block and a 15-byte tail
    "distinct": ((1, 1, 1, 0, 0), None, False),
    "permuted": ((0, 0, 1, 1, 0), 1000, True),     # ties keep the order of a permuted index vector
}


def sort_case(rng, name, n):
    nd, card, perm = SORT_CASES[name]
    cap = n + 3
    block = dim_block(rng, nd, cap, n, card)
    index = rng.permutation(n).astype(np.uint32) if perm else np.arange(n, dtype=np.uint32)
    return nd, cap, block, index


def check_sort(be, nd, cap, block, index, ctx):
    gh, gi = run_sort(be, block, nd, cap, index)
    eh, ei = expected_sort(block, nd, cap, index)
    assert np.array_equal(gh, eh), f"{ctx}: sorted hashes differ"
    bad = np.flatnonzero(gi != ei)
    assert bad.size == 0, f"{ctx}: sorted index differs at {bad.size} positions, first {bad[0]}"


def runs_case(rng, lengths):
    """Hand-built Reduce input: ascending distinct hashes repeated by run length, a permuted index vector."""
    lengths = np.asarray(lengths, np.int64)
    g, n = len(lengths), int(lengths.sum())
    h = np.unique(rng.integers(0, np.iinfo(np.uint64).max, g + 64, dtype=np.uint64, endpoint=True))[:g]
    assert len(h) == g
    hv = np.repeat(h, lengths)
    index = rng.permutation(n).astype(np.uint32)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    return hv, index, starts


def check_reduce(be, rng, lengths, aggs, ctx, nd=(0, 1, 1, 0, 1)):
    hv, index, starts = runs_case(rng, lengths)
    n, g = len(index), len(lengths)
    cap = n + 1
    block = dim_block(rng, nd, cap, n, 50)
    max_run = int(np.max(lengths))
    exp_rows = packed_rows(block, nd, cap, index[starts])
    for agg, vb in aggs:
        c = f"{ctx} {agg_id((agg, vb))}"
        meas = measures(rng, agg, vb, n, max_run)
        got_g, oh, oi, om, od = run_reduce(be, block, nd, cap, hv, index, meas, vb, agg)
        assert got_g == g, f"{c}: {got_g} runs, expected {g}"
        assert not oh.any(), f"{c}: Reduce wrote outputKeys.HashValues (the reference discards the run keys)"
        assert np.array_equal(oi, index[starts]), f"{c}: output index (first entry of each run) differs"
        assert np.array_equal(packed_rows(od, nd, cap, np.arange(g)), exp_rows), f"{c}: gathered dimension rows differ"
        assert_measures(agg, vb, om.tobytes(), fold(agg, vb, meas[index], starts), c)


def hash_classes(block, nd, cap, n):
    """Rows grouped by murmur3-32 of the packed row: (order grouping the rows class by class, class starts, the
    smallest row index of each class)."""
    h = hashes.murmur3_32(packed_rows(block, nd, cap, np.arange(n)))
    order = np.argsort(h, kind="stable")
    hs = h[order]
    starts = np.flatnonzero(np.r_[True, hs[1:] != hs[:-1]])
    return h, order, starts, order[starts]


def check_hash_reduce(be, rng, block, nd, cap, n, aggs, ctx, start_from="identity"):
    h, order, starts, rep = hash_classes(block, nd, cap, n)
    sizes = np.diff(np.r_[starts, n])
    exp_rows = packed_rows(block, nd, cap, rep)
    for agg, vb in aggs:
        c = f"{ctx} {agg_id((agg, vb))}"
        meas = measures(rng, agg, vb, n, int(sizes.max()))
        g, om, od = run_hash_reduce(be, block, nd, cap, n, meas, vb, agg)
        assert g == len(starts), f"{c}: {g} groups, expected {len(starts)}"
        got_rows = packed_rows(od, nd, cap, np.arange(g))
        gh = hashes.murmur3_32(got_rows)
        go = np.argsort(gh, kind="stable")         # output order is unspecified: compare class by class
        assert np.array_equal(gh[go], h[rep]), f"{c}: group hashes differ"
        assert np.array_equal(got_rows[go], exp_rows), f"{c}: a group is not named by its smallest row index"
        w = measure_width(agg, vb)
        gm = np.frombuffer(om.tobytes(), np.uint8).reshape(g, w)[go].tobytes()
        assert_measures(agg, vb, gm, fold(agg, vb, meas[order], starts, start_from), c)


def hash_capacity(length):
    cap = HASH_MIN_CAPACITY
    while cap < 2 * length:
        cap <<= 1
    return cap


# =================================================================================================================
# CPU: the restatements against the oracle (and the reference's HOST build, or the digest recorded from it)
# =================================================================================================================
def _pin(key, outputs, run_ref):
    """outputs: the restatement's results of a pin test; run_ref(): the same from oracle/_ref."""
    H.assert_matches_reference(f"nodes_at_scale/{key}", H.digest(outputs),
                               (lambda: H.digest(run_ref())) if H.reference_built() else None)


def test_filter_restatement_matches_the_oracle():
    orc = H.get_backend("oracle")
    rng = np.random.default_rng(71)
    outputs, cases = [], []
    for k, name in enumerate(PATTERNS):
        for n in (3 * FILTER_TILE - 1, 3 * FILTER_TILE, 3 * FILTER_TILE + 1):
            for sparse, nrec, binary in ((False, 0, k % 2 == 0), (True, 1, k % 2 == 1), (True, 8, False)):
                kr, idx, recs = filter_case(rng, name, n, sparse, nrec)
                exp = expected_filter(kr, idx, recs)
                got = run_filter(orc, kr, idx, recs, binary)
                ctx = f"{name} n={n} sparse={sparse} recs={nrec}"
                assert got[0] == exp[0] and np.array_equal(got[1], exp[1]) and np.array_equal(got[2], exp[2]), ctx
                assert all(np.array_equal(a, b) for a, b in zip(got[3], exp[3])), ctx
                outputs.append([exp[0], exp[1], exp[2], exp[3]])
                cases.append((kr, idx, recs, binary))

    def ref():
        out = []
        for kr, idx, recs, binary in cases:
            m, i, p, r = run_filter(H.get_backend("ref"), kr, idx, recs, binary)
            out.append([m, i, p, r])
        return out
    _pin("filter", outputs, ref)


def test_sort_restatement_matches_the_oracle():
    orc = H.get_backend("oracle")
    rng = np.random.default_rng(72)
    outputs, cases = [], []
    for name in SORT_CASES:
        for n in (1, 2, 700, 5000):
            nd, cap, block, index = sort_case(rng, name, n)
            eh, ei = expected_sort(block, nd, cap, index)
            gh, gi = run_sort(orc, block, nd, cap, index)
            assert np.array_equal(gh, eh) and np.array_equal(gi, ei), f"{name} n={n}"
            outputs.append([eh, ei])
            cases.append((block, nd, cap, index))
    _pin("sort", outputs, lambda: [list(run_sort(H.get_backend("ref"), *c)) for c in cases])


def _small_run_shapes(rng):
    """The Reduce shapes of the GPU tests with a run threshold of 40 instead of kLongRun."""
    return {
        "one_long": [120],
        "edge": [5, 40, 7, 41, 1],
        "many_long": [45] * 12,
        "handoff": list(rng.permutation([1] * 300 + [3] * 20 + [60])),
        "g4_eq": [4] * 50,
        "g4_below": [4] * 49 + [3],
        "g4_above": [4] * 49 + [5],
        "tile_cross": list(rng.integers(1, 90, 60)),
    }


def test_reduce_restatement_matches_the_oracle():
    orc = H.get_backend("oracle")
    rng = np.random.default_rng(73)
    nd = (0, 1, 1, 0, 1)
    outputs, cases = [], []
    for shape, lengths in _small_run_shapes(rng).items():
        hv, index, starts = runs_case(rng, lengths)
        n = len(index)
        cap = n + 1
        block = dim_block(rng, nd, cap, n, 50)
        for agg, vb in AGGS:
            meas = measures(rng, agg, vb, n, int(max(lengths)))
            if agg in (A.AGGR_MIN_FLOAT, A.AGGR_MAX_FLOAT):
                meas[meas == 0] = 0.5     # a sequential fold and numpy may keep different zeros
            ctx = f"{shape} {agg_id((agg, vb))}"
            g, oh, oi, om, od = run_reduce(orc, block, nd, cap, hv, index, meas, vb, agg)
            exp = fold(agg, vb, meas[index], starts)
            assert g == len(lengths) and not oh.any() and np.array_equal(oi, index[starts]), ctx
            assert np.array_equal(packed_rows(od, nd, cap, np.arange(g)), packed_rows(block, nd, cap, index[starts])), ctx
            assert_measures(agg, vb, om.tobytes(), exp, ctx)
            if agg != A.AGGR_AVG_FLOAT:          # AVG is compared to 2e-5, so it stays out of the digest
                outputs.append([g, index[starts], np.ascontiguousarray(exp)])
                cases.append((block, nd, cap, hv, index, meas, vb, agg, exp.dtype))

    def ref():
        out = []
        for block, nd_, cap, hv, index, meas, vb, agg, dt in cases:
            g, oh, oi, om, _ = run_reduce(H.get_backend("ref"), block, nd_, cap, hv, index, meas, vb, agg)
            out.append([g, oi, np.frombuffer(om.tobytes(), dt)])
        return out
    _pin("reduce", outputs, ref)


def test_hash_reduce_identities_match_the_oracle():
    """The identity table of the restatement is the reference's: the value a NULL measure becomes in the measure sink."""
    import parity_cases as P
    orc = H.get_backend("oracle")
    sink_type = {np.uint32: A.Uint32, np.int32: A.Int32, np.float32: A.Float32}
    for agg, ident in IDENTITY.items():
        t = MEASURE_TYPE[agg]
        null = P.InputSpec("const", const=0, const_valid=False)
        got = P.run_transform(orc, [null], A.Noop, ("measure", sink_type[t], agg), 1)["values"]
        assert got.tobytes() == np.asarray(ident, t).tobytes(), AGG_NAME[agg]


def test_hash_reduce_restatement_matches_the_oracle():
    """The oracle restates the reference's HOST map, which default-constructs a slot to zero before folding; the
    engine's table starts from the identity, as the reference's DEVICE map does.  The fold and the choice of the
    representative are pinned here with start_from="zero"; the identities by the test above."""
    orc = H.get_backend("oracle")
    rng = np.random.default_rng(74)
    for nd in ((0, 0, 1, 1, 0), (0, 1, 0, 1, 0)):
        for n, card in ((1, 1), (3000, 1), (3000, 40), (1 << 11, None), ((1 << 11) + 1, None)):
            block = dim_block(rng, nd, n + 2, n, card)
            check_hash_reduce(orc, rng, block, nd, n + 2, n, AGGS, f"nd={nd} n={n}", start_from="zero")


# =================================================================================================================
# GPU: the engine at scale
# =================================================================================================================
BIG_TILES = 127_000            # ~1.3e8 index positions


@pytest.mark.gpu
@pytest.mark.parametrize("name", PATTERNS)
def test_filter_compaction_at_scale(name):
    """Every survivor pattern at k x 1024 - 1, k x 1024 and k x 1024 + 1 index positions (k = 127,000 tiles, far more
    than the resident CTAs); unary Noop and binary Equal alternate; and the sparse ascending index vector a later
    filter sees."""
    eng = H.get_backend("b200")
    assert BIG_TILES > 8 * FILTER_CTAS_PER_SM * sm_count() and BIG_TILES >= 100_000
    rng = np.random.default_rng(60 + PATTERNS.index(name))
    for j, n in enumerate((BIG_TILES * FILTER_TILE - 1, BIG_TILES * FILTER_TILE, BIG_TILES * FILTER_TILE + 1)):
        kr, idx, recs = filter_case(rng, name, n, sparse=j == 2, num_recs=0)
        check_filter(eng, kr, idx, recs, binary=j == 1, ctx=f"{name} n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("num_recs", [1, 8])
def test_filter_moves_record_ids_at_scale(num_recs):
    """RecordID vectors of joined tables are compacted in lockstep with the index vector over thousands of tiles."""
    eng = H.get_backend("b200")
    tiles = 20_000 if num_recs == 1 else 3_000
    assert tiles > FILTER_CTAS_PER_SM * sm_count()
    rng = np.random.default_rng(80 + num_recs)
    for name in ("random50", "tile_edge", "last_tile"):
        kr, idx, recs = filter_case(rng, name, tiles * FILTER_TILE + 1, sparse=True, num_recs=num_recs)
        m = check_filter(eng, kr, idx, recs, binary=name == "random50", ctx=f"{name} recs={num_recs}")
        assert m > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SORT_CASES))
def test_sort_at_scale(name):
    """Sort from below one tile through the 4 x SMs x 2048 block cap (+-1: one tile per block, then two) to ~3e7 keys
    (several tiles per block: the digit carry between the tiles of one chunk)."""
    eng = H.get_backend("b200")
    cap_keys = SORT_BLOCKS_PER_SM * sm_count() * SORT_TILE
    rng = np.random.default_rng(90 + len(name))
    sizes = [1000, cap_keys - 1, cap_keys, cap_keys + 1] + ([30_000_000] if name in ("distinct", "permuted") else [])
    multi = False
    for n in sizes:
        tiles = -(-n // SORT_TILE)
        tiles_per_block = -(-tiles // (SORT_BLOCKS_PER_SM * sm_count()))
        multi |= tiles_per_block >= 2
        nd, cap, block, index = sort_case(rng, name, n)
        check_sort(eng, nd, cap, block, index, f"{name} n={n}")
    assert multi, "no size gave a block more than one tile"


def _reduce_shapes(rng, sms):
    handoff = np.array([1] * 400_000 + [3] * 2_000 + [LONG_RUN + 17_000])
    heads = [HEAD_TILE - 1, 1, HEAD_TILE, HEAD_TILE + 1, 2 * HEAD_TILE - 1] + list(rng.integers(1, 5000, 2000))
    return {
        "one_long": [3, 200_000, 2],
        "edge": [5, LONG_RUN, 7, LONG_RUN + 1, 1, LONG_RUN - 1],
        "many_long": [40_000] * 300,
        "handoff": list(rng.permutation(handoff)),
        "g4_eq": [4] * 100_000,
        "g4_below": [4] * 99_999 + [3],
        "g4_above": [4] * 99_999 + [5],
        "tile_cross": heads,
    }


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_long", "edge", "many_long", "handoff", "g4_eq", "g4_below", "g4_above", "tile_cross"])
def test_reduce_at_scale(shape):
    """Reduce over hand-built sorted runs, every aggregate: the long-run kernel (runs > kLongRun, and more of them than
    its 2 x SMs blocks), the kLongRun boundary, the short path (g x 4 > n) handing a long run on through the warp
    kernel, both sides of g x 4 == n, and runs across the 2048-element head tiles."""
    eng = H.get_backend("b200")
    sms = sm_count()
    rng = np.random.default_rng(100 + len(shape))
    lengths = np.asarray(_reduce_shapes(rng, sms)[shape])
    n, g = int(lengths.sum()), len(lengths)
    long = int((lengths > LONG_RUN).sum())
    if shape == "one_long":
        assert long == 1
    elif shape == "edge":
        assert LONG_RUN in lengths and LONG_RUN + 1 in lengths and long == 1
    elif shape == "many_long":
        assert long > LONG_RUN_BLOCKS_PER_SM * sms
    elif shape == "handoff":
        assert g * 4 > n and long == 1 and (lengths == 3).any()
    elif shape == "g4_eq":
        assert g * 4 == n
    elif shape == "g4_below":
        assert g * 4 == n + 1
    elif shape == "g4_above":
        assert g * 4 == n - 1
    else:
        ends = np.cumsum(lengths)
        starts = ends - lengths
        assert (starts // HEAD_TILE != (ends - 1) // HEAD_TILE).sum() > 100 and (ends % HEAD_TILE == 0).any()
        assert -(-n // HEAD_TILE) > 1000
    check_reduce(eng, rng, lengths, AGGS, shape)


HASH_CASES = {   # name -> (dims per width, rows, prototype rows or None, aggregates)
    "one_group": ((0, 0, 1, 1, 0), 50_000_000, 1, [a for a in AGGS if a[0] != A.AGGR_AVG_FLOAT]),
    "one_group_avg": ((0, 0, 1, 1, 0), 20_000, 1, [(A.AGGR_AVG_FLOAT, 8)]),
    "groups_1e6": ((0, 1, 0, 1, 0), 20_000_000, 1_000_000, AGGS),
    "distinct_2^22": ((0, 0, 1, 1, 0), 1 << 22, None, AGGS),
    "distinct_2^22+1": ((0, 1, 0, 1, 0), (1 << 22) + 1, None, AGGS),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(HASH_CASES))
def test_hash_reduce_at_scale(case):
    """HashReduce, every aggregate: 5e7 rows on one slot, ~1e6 groups over 2e7 rows, nearly all distinct rows at a
    length of 2^22 and 2^22 + 1 (the table doubles between them).  Groups are murmur3-32 classes of the packed row
    (colliding rows merge), each named by its smallest row index; slots start from the aggregate's identity."""
    eng = H.get_backend("b200")
    nd, n, card, aggs = HASH_CASES[case]
    rng = np.random.default_rng(110 + len(case))
    cap = n + 5
    block = dim_block(rng, nd, cap, n, card)
    if case.startswith("distinct"):
        k = n.bit_length() - 1
        assert hash_capacity(n) == (2 << k if n == 1 << k else 4 << k)
        assert hash_capacity(n) // EXT_TILE > 1000
    if case.startswith("one_group"):
        assert len(np.unique(hashes.murmur3_32(packed_rows(block, nd, cap, np.arange(min(n, 1000)))))) == 1
    check_hash_reduce(eng, rng, block, nd, cap, n, aggs, case)


# ---- the legacy per-node sequence end to end at BASELINE sizes --------------------------------------------------
def _legacy(name, rows, days, reduce_mode=None, hll=False):
    import torch
    import independent as I
    import test_at_size as S
    from aresdb_b200 import synth
    from aresdb_b200.executor import Batch, LegacyBatchExecutor
    eng = H.get_backend("b200")
    dev = torch.device("cuda:0")
    q = S._queries(days)[name]
    t0 = synth.BASE_TS
    exp = I.Expected({"cfg4_sort": "cfg4"}.get(name, name), days, dev, t0, t0 + 1800, t0 + days * 86400 - 1800)
    ex = LegacyBatchExecutor(eng.lib, eng.space, q)
    group_rows = None
    for d in range(days):
        bufs, voff, cols = S._batch(d, rows, dev)
        ex.process_batch(Batch(cols, rows), is_last=d == days - 1)
        exp.add_batch(bufs, voff, rows)
        if name == "cfg2":         # rows per city among the survivors: the runs Reduce sees
            (_, city, status, _), (_, vcity, vstatus, _) = I.decode_columns(bufs, voff, rows)
            keep = vstatus & (status == 1)
            cidx = torch.where(vcity, city, torch.full_like(city, I.CITY_SPACE - 1))[keep]
            group_rows = torch.bincount(cidx, minlength=I.CITY_SPACE).cpu().numpy()
        del bufs, cols
    return ex, exp, group_rows


@pytest.mark.gpu
def test_legacy_cfg2_1e8_rows():
    """1e8 rows, ~2.5e5 surviving rows per city: Reduce's long-run kernel on real data."""
    ex, exp, group_rows = _legacy("cfg2", 100_000_000, 1)
    assert (group_rows > LONG_RUN).sum() > 50
    out = exp.check(ex.result())
    assert out["groups"] == 101


@pytest.mark.gpu
def test_legacy_cfg3_sum_one_full_batch():
    """cfg3 SUM on one 1.25e8-row batch: five filters (the first over ~1.2e5 tiles), then Sort + Reduce."""
    ex, exp, _ = _legacy("cfg3", 125_000_000, 1)
    out = exp.check(ex.result())
    assert out["groups"] == 24 * 100 and out["rows_kept"] > 0.2 * 125_000_000


@pytest.mark.gpu
def test_legacy_cfg4_sort_mode_carried_results():
    """cfg4 in sort mode, 8 x 1.25e7 rows: each batch re-reduces the carried groups with its own rows (1.16e6 groups)."""
    ex, exp, _ = _legacy("cfg4_sort", 12_500_000, 8)
    out = exp.check(ex.result())
    assert out["groups"] > 1_150_000


@pytest.mark.gpu
def test_legacy_cfg4_hash_mode_carried_results():
    """cfg4 in hash mode, 8 x 1.25e7 rows.  Rows whose murmur3-32 collide are one group; once a group has been carried
    any member may name it (the carried row is re-inserted ahead of the batch's rows), and its measure is the class sum."""
    import independent as I
    from aresdb_b200 import synth
    ex, exp, _ = _legacy("cfg4", 12_500_000, 8)
    res = ex.result()
    rows = res.packed_rows()
    h = hashes.murmur3_32(rows)
    assert len(np.unique(h)) == res.groups, "two output groups share a hash"
    present, vals = exp.present.cpu().numpy(), exp.vals.cpu().numpy()
    gidx = np.nonzero(present)[0]
    tidx, cidx = gidx // I.CITY_SPACE, gidx % I.CITY_SPACE
    tnull, cnull = tidx == exp.tn - 1, cidx == I.CITY_SPACE - 1
    erow = np.zeros((gidx.size, 8), np.uint8)
    erow[:, 0:4] = np.where(tnull, 0, synth.BASE_TS + tidx * 60).astype("<u4").view(np.uint8).reshape(-1, 4)
    erow[:, 4:6] = np.where(cnull, 0, cidx).astype("<u2").view(np.uint8).reshape(-1, 2)
    erow[:, 6] = ~tnull
    erow[:, 7] = ~cnull
    eh = hashes.murmur3_32(erow)
    order = np.argsort(eh, kind="stable")
    uniq, start = np.unique(eh[order], return_index=True)
    sums = np.add.reduceat(vals[gidx][order], start)
    assert res.groups == uniq.size and gidx.size - uniq.size > 0, "no 32-bit collision among 1.16e6 groups?"
    pos = np.searchsorted(uniq, h)
    assert (uniq[pos] == h).all()
    assert (res.measures.view(np.uint64) == sums[pos].view(np.uint64)).all()
    assert {r.tobytes() for r in rows} <= {r.tobytes() for r in erow}


@pytest.mark.gpu
def test_legacy_cfg4_hll_two_batches():
    """HyperLogLog over 2 x 2.5e7 rows through the per-node call, registers built on the second (last) batch from the
    carried results; GetHLLValue with the CUDA int-shift semantics (tests/independent.hll_value)."""
    ex, exp, _ = _legacy("cfg4_hll", 25_000_000, 2)
    out = exp.check_hll(ex.hll)
    assert out["groups"] >= 2 * 100
