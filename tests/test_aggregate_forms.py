"""Every aggregate of the fused kernel in every accumulation form it can take, on an edge table, against a numpy
restatement of the reference's semantics.

How the kernel accumulates a measure depends on the aggregate, the measure's type, the zone map, the batch size and
AggSpec.ExpectedGroups (jit.cu: jitAnalyzeDense / generate, batch_plan.cu: layoutStages).  The forms, and what selects
them in the generated text:

  cta     CTA-resident slots                 JIT_DENSE 1; JIT_DENSE_ACC 1 (4-byte atomics: count, integer min / max) or
                                             2 (rows 0-1 of a quad in shared memory, 2-3 on the CTA's L2 slice: sums,
                                             AVG, float min / max); JIT_DENSE_FLAGS 0 for count(*) only
  fx      exact-integer float sum            JIT_DENSE 1, JIT_DENSE_ACC 4 (sum of a Float32 column that a filter proves
                                             non-NULL, zone map on the measure)
  global  one slot array for the grid        JIT_DENSE 2 (more slots than a CTA holds), JIT_DENSE_CHECK 1: no flags, a
                                             row equal to the neutral element takes the hash path (count: CHECK 0)
  hash    CTA hash table, then global table  JIT_DENSE 0, JIT_BYPASS 0 (no zone map)
  bypass  straight to the global table       JIT_DENSE 0, JIT_BYPASS 1 (ExpectedGroups > 32,768)
  tail    one-CTA launch                     a batch without a full tile: JIT_DENSE 0 whatever the zone map says
  shared  several measures, one kernel       kMeasAcc / kMeasFlags / kMeasCheck: each member keeps its solo form

Matrix (aggregate x column type x form x reduce mode); every cell names its test, or why the engine does not allow it:

  aggregate      types                         cta   fx    global  hash  bypass  tail  rle        shared
  sum            i8 i16 i32 u8 u16 u32         S     -(1)  -(2)    S3    S3      S3    S(i16)     S, X
  sum            f32                           S     S     S       S     S       S     S          S, X
  min / max      i8 i16 i32 u8 u16 u32         S     -(1)  S3      S3    S3      S3    S(i16)     S, X
  min / max      f32                           S     -(1)  S       S     S       S     S          S, X
  avg            every type                    S     -(1)  S3      S3    S3      S3    S(i16,f32) S, X
  count          -                             S     -(1)  S       S     S       S     S          S, X
  hash mode      one case per form             H     -     H       H     H       -     -          -

  S  test_solo_forms_on_gpu (cta, fx, global: exact, too narrow and stale zone maps; the global and bypass cases group
     by w x hour, ~90,000 groups, so they also run the >32,768-group finalize); S3: the cta form takes all seven column types, the
     other forms Int16, Uint32 and Float32 (one each of signed, unsigned and float); H: test_solo_forms_on_gpu, hash-reduce
     cases; rle: test_rle_batches_on_gpu (the measure as a first-class RLE column and as an unsorted column);
     shared: test_shared_form_on_gpu (with and without member filters), X: test_exchange_of_shared_requests_on_gpu.
  (1) the exact-integer form is a sum of a Float32 column only.
  (2) the global slot array has no flags; an integer column's sum can return to 0, so it keeps the hash table
      (test_form_of_every_case asserts JIT_DENSE 0 for each of them).

The restatement (`restate`): rows pass the filter, group by the packed dimension row, a NULL measure becomes the
aggregate's identity (the reference's get_identity_value: MIN 0xFFFFFFFF / INT32_MAX / FLT_MAX, MAX 0 / INT32_MIN /
FLT_MIN, sums 0), AVG takes a NULL as (0, count 0), integer sums wrap in 64 bits, SUM / COUNT / AVG of an RLE batch count
run lengths and MIN / MAX do not; sort mode orders groups by the 64-bit murmur3 of the row, hash mode keys them by its
32-bit murmur3 (colliding rows are one group) and starts float sums from +0.0.  Float sums keep every partial sum exact
(each group holds one edge value, or small integers), so they compare bit for bit.  Float MIN / MAX compare by value
(-0.0 == +0.0: which zero wins depends on order, in the reference too).  AVG: counts exact, averages to 2e-5 of the
largest magnitude in the group (the rolling float average rounds at every combine); groups holding values of 2^127 or
more are checked by count only, because the rolling combine of such values overflows to inf or not depending on order.
The CPU tests pin the restatement to the oracle's per-node call sequence and to the reference's HOST build (stored
digests), and check with the generator's dry run that every GPU case reaches the form it targets.
"""
from __future__ import annotations

import ctypes as C
import functools
import gc

import numpy as np
import pytest

import harness as H
import hashes
import test_pipeline_parity as T
import test_shared_scan as S
import test_sharded_request as SR
from aresdb_b200 import cabi as A
from aresdb_b200 import columns, expr as E
from aresdb_b200.executor import Batch, FusedBatchExecutor, FusedRequestExecutor, LegacyBatchExecutor, query_result
from aresdb_b200.query import AggQuery, Measure

# ---- the edge table -----------------------------------------------------------------------------------------------
T0 = 1_700_006_400                      # an hour boundary
HOURS = 150                             # hours one batch spans: w x hour = 301 x 151 slots, more than a CTA holds
NK, NW = 4, 300                         # k in [0, 4), w in [0, 300)
W_NULL, W_CANCEL, W_DROPPED, W_HOT = 250, 252, 298, 299
TYPES = [A.Int8, A.Int16, A.Int32, A.Uint8, A.Uint16, A.Uint32, A.Float32]
NAME = {A.Int8: "i8", A.Int16: "i16", A.Int32: "i32", A.Uint8: "u8", A.Uint16: "u16", A.Uint32: "u32", A.Float32: "f32"}
NP = {A.Int8: np.int8, A.Int16: np.int16, A.Int32: np.int32, A.Uint8: np.uint8, A.Uint16: np.uint16, A.Uint32: np.uint32,
      A.Float32: np.float32}
COL = {dt: 3 + i for i, dt in enumerate(TYPES)}
COLUMN_TYPES = [A.Uint32, A.Uint8, A.Uint16] + TYPES
TS, KC, WC = E.Col(0, A.Uint32, "ts"), E.Col(1, A.Uint8, "k"), E.Col(2, A.Uint16, "w")
SIGNED = (A.Int8, A.Int16, A.Int32)
THREE = [A.Int16, A.Uint32, A.Float32]   # one signed, one unsigned, one float column

F32_MAX, F32_MIN = float(np.finfo(np.float32).max), float(np.finfo(np.float32).tiny)
DENORM_MIN, DENORM_MAX = float(np.float32(2.0 ** -149)), float(np.uint32(0x007FFFFF).view(np.float32))


def MC(dt):
    return E.Col(COL[dt], dt, NAME[dt])


def edge_values(dt):
    """One value per edge group w = 0 .. len - 1: type extremes, +-1 off them, 0, +-1, the neutral elements of the
    engine's accumulators (0xFFFFFFFF, INT32_MAX / MIN, +-inf, -0.0) and the reference's identities (FLT_MAX, FLT_MIN)."""
    if dt == A.Float32:
        return [np.inf, -np.inf, -0.0, 0.0, F32_MAX, -F32_MAX, F32_MIN, -F32_MIN, DENORM_MIN, -DENORM_MIN, DENORM_MAX,
                1.0, -1.0, 0.5, 100.0, 2.0 ** -20]
    info = np.iinfo(NP[dt])
    vals = [info.min, info.max, info.min + 1, info.max - 1, 0, 1, 100]
    return vals + ([-1, -100] if dt in SIGNED else [])


EDGE_GROUPS = 16     # the longest edge list
BLOCK_W = list(range(EDGE_GROUPS)) + [W_NULL, W_CANCEL]


def _cancel_value(dt):
    return F32_MAX if dt == A.Float32 else int(np.iinfo(NP[dt]).max) if dt in SIGNED else 0


def edge_batch(seed, rows, hour0=0):
    """Host arrays of one batch.  Group (k, w): w < 16 holds one edge value per column (no NULLs when k == 0), W_NULL
    only NULLs, W_CANCEL +x and -x in equal numbers (signed and float columns: its sum is exactly 0), W_HOT (k = 1) 40 %
    of the rows; the others random values (float columns: small integers, so that every partial sum is exact).  Blocks
    of every edge group, four rows each (every position of a quad), open the batch and sit at the end of the last full
    tile and in the tail of every tile size the engine picks.  Garbage under NULL in the Int16, Uint32 and Float32
    columns."""
    rng = np.random.default_rng(seed)
    hot = rng.random(rows) < 0.4
    w = np.where(hot, W_HOT, rng.integers(0, NW - 1, rows)).astype(np.uint16)
    k = np.where(hot, 1, rng.integers(0, NK, rows)).astype(np.uint8)
    block = np.repeat(np.asarray(BLOCK_W, np.uint16), 4)
    starts = {0, rows - len(block)}
    for tr in (3968, 1920, 896):
        tail = max(rows - 128, 0) // tr * tr
        starts |= {tail - len(block), tail}
    for s in sorted(starts):
        s = max(0, min(s - s % 4, rows - len(block)))
        if s >= 0:
            w[s:s + len(block)] = block[:rows - s]
            k[s:s + len(block)] = (np.arange(len(block)) // 4 % NK)[:rows - s].astype(np.uint8)
    ts = (T0 + (hour0 + rng.integers(0, HOURS, rows)) * 3600 + rng.integers(0, 3600, rows)).astype(np.uint32)
    hb = {"ts": ts, "k": k, "w": w, "rows": rows}
    for dt in TYPES:
        npt = NP[dt]
        edges = edge_values(dt)
        if dt == A.Float32:
            vals = rng.integers(-100, 101, rows).astype(np.float32)
        else:
            info = np.iinfo(npt)
            vals = rng.integers(int(info.min), int(info.max) + 1, rows, dtype=np.int64).astype(npt)
        ok = rng.random(rows) >= 0.1
        e = w < len(edges)
        vals[e] = np.asarray(edges, np.float64 if dt == A.Float32 else np.int64)[w[e]].astype(npt)
        ok[e & (k == 0)] = True
        ok[w == W_NULL] = False
        c = np.flatnonzero(w == W_CANCEL)
        x = _cancel_value(dt)
        for kk in range(NK):
            pos = c[k[c] == kk]
            ok[pos] = True
            vals[pos[0::2]] = npt(x)
            vals[pos[1::2]] = npt(-x) if dt in SIGNED or dt == A.Float32 else npt(x)
            if len(pos) % 2:
                ok[pos[-1]] = False
        if dt in (A.Int16, A.Uint32, A.Float32):
            vals[~ok] = npt(-F32_MAX) if dt == A.Float32 else np.iinfo(npt).min if dt in SIGNED else np.iinfo(npt).max
        hb[dt] = (vals, ok)
    return hb


@functools.lru_cache(maxsize=None)
def edge_batches(kind="solo"):
    if kind == "tail":          # no full tile: the whole batch is the tail, folded by one CTA
        return [edge_batch(31, 3001), edge_batch(32, 1999, HOURS)]
    if kind == "cpu":
        return [edge_batch(41, 30011), edge_batch(42, 20003, HOURS)]
    return [edge_batch(11, 300_003), edge_batch(12, 150_001, HOURS)]


def zone_map(hb, how="exact"):
    """Ranges of the dimension columns: exact, too narrow (upper half cut off) or stale (another batch's)."""
    lo = int(hb["ts"].min())
    zm = {0: (lo, int(hb["ts"].max())), 1: (0, NK - 1), 2: (0, NW - 1)}
    if how == "narrow":
        zm = {c: (a, a + (b - a) // 2) for c, (a, b) in zm.items()}
    elif how == "stale":
        zm = {0: (lo + HOURS * 3600, int(hb["ts"].max()) + HOURS * 3600), 1: (2, NK + 1), 2: (150, NW + 149)}
    return zm


def upload(be, hb, ranges=None):
    cols, keep = [], []
    for c, dt in enumerate(COLUMN_TYPES):
        if c < 3:
            buf, vp = columns.make_column(be.space, dt, hb[("ts", "k", "w")[c]])
        else:
            v, ok = hb[dt]
            buf, vp = columns.make_column(be.space, dt, v, valid=ok)
        cols.append(vp)
        keep.append(buf)
    return Batch(cols, hb["rows"], keep=keep, ranges=ranges)


# ---- queries -----------------------------------------------------------------------------------------------------
# filters are (op, column, literal) triples: the same triple builds the AggQuery filter and the restatement's mask
BASE_FILTER = ("ne", "w", W_DROPPED)
FX_FILTER = ("ge", A.Float32, -1.0e30)        # proves the Float32 measure non-NULL: the exact-integer form
FX_RANGE = (0, int(np.float32(100.0).view(np.uint32)))
OPS = {"ne": (E.ne, np.not_equal), "eq": (E.eq, np.equal), "ge": (E.ge, np.greater_equal), "gt": (E.gt, np.greater),
       "lt": (E.lt, np.less)}


def filter_expr(f):
    op, col, lit = f
    c = {"w": WC, "k": KC, "ts": TS}.get(col) if isinstance(col, str) else MC(col)
    return OPS[op][0](c, E.Lit(lit))


def filter_mask(hb, f):
    """NULL never passes; integers compare in the int32 class (a ConstInt literal), floats in float32."""
    op, col, lit = f
    if isinstance(col, str):
        v, ok = hb[col].astype(np.int64), np.ones(hb["rows"], bool)
    else:
        v, ok = hb[col]
        v = v.astype(np.float32) if col == A.Float32 else v.astype(np.int64).astype(np.uint32).view(np.int32).astype(np.int64)
        lit = np.float32(lit) if col == A.Float32 else lit
    return ok & OPS[op][1](v, lit)


DIMS = {"kw": [KC, WC], "wh": [WC, E.floor(TS, E.Lit(3600))]}


def make_query(kind, dt, dims="kw", filters=(BASE_FILTER,), mode=A.ARES_REDUCE_SORT):
    m = Measure("count") if kind == "count" else Measure(kind, MC(dt))
    return AggQuery([filter_expr(f) for f in filters], DIMS[dims], m, reduce_mode=mode)


# ---- the restatement ---------------------------------------------------------------------------------------------
IDENTITY = {("min", "u"): 0xFFFFFFFF, ("min", "s"): 2 ** 31 - 1, ("min", "f"): F32_MAX,
            ("max", "u"): 0, ("max", "s"): -2 ** 31, ("max", "f"): F32_MIN}


def _cls(dt):
    return "f" if dt == A.Float32 else "s" if dt in SIGNED else "u"


def packed_rows(hb, dims):
    """uint8[n, rowBytes]: dimension values in layout order (widest first), then one validity byte each."""
    n = hb["rows"]
    w = hb["w"].astype("<u2").view(np.uint8).reshape(n, 2)
    one = np.ones((n, 1), np.uint8)
    if dims == "kw":
        return np.hstack([w, hb["k"].reshape(n, 1), one, one])
    hour = (hb["ts"] - hb["ts"] % 3600).astype("<u4").view(np.uint8).reshape(n, 4)
    return np.hstack([hour, w, one, one])


class Expected:
    """rows (packed bytes, in the reference's order) and per group the measure (and the AVG count); `loose`: AVG groups
    compared by count only, `scale`: the largest magnitude that met in an AVG group."""

    def __init__(self, rows, meas, counts=None, scale=None):
        self.rows, self.meas, self.counts, self.scale = rows, meas, counts, scale


def restate(hbs, kind, dt, dims="kw", filters=(BASE_FILTER,), mode=A.ARES_REDUCE_SORT):
    keys, vals, oks, mult = [], [], [], []
    for hb in hbs:
        alive = np.ones(hb["rows"], bool)
        for f in filters:
            alive &= filter_mask(hb, f)
        keys.append(packed_rows(hb, dims)[alive])
        v, ok = hb[dt] if dt is not None else (np.zeros(hb["rows"], np.int8), np.ones(hb["rows"], bool))
        vals.append(v[alive])
        oks.append(ok[alive])
        mult.append(hb.get("mult", np.ones(hb["rows"], np.int64))[alive])
    rows = np.vstack(keys)
    v, ok, mult = np.concatenate(vals), np.concatenate(oks), np.concatenate(mult).astype(np.int64)
    if mode == A.ARES_REDUCE_SORT:
        key = np.zeros(len(rows), np.uint64)
        for b in range(rows.shape[1]):
            key |= rows[:, b].astype(np.uint64) << np.uint64(8 * b)
    else:
        key = hashes.murmur3_32(rows)
    uniq, first, inv = np.unique(key, return_index=True, return_inverse=True)
    g = len(uniq)
    counts = scale = None
    if kind == "count":
        meas = np.zeros(g, np.int64)
        np.add.at(meas, inv, mult)
        meas = (meas & 0xFFFFFFFF).astype(np.uint32)
    elif kind == "sum" and dt != A.Float32:
        meas = np.zeros(g, np.int64)
        np.add.at(meas, inv, np.where(ok, v.astype(np.int64), 0) * mult)
        meas = meas.view(np.uint64) if dt not in SIGNED else meas
    elif kind == "sum":
        meas = np.full(g, -0.0)
        np.add.at(meas, inv, np.where(ok, v.astype(np.float64), 0.0) * mult)
        if mode == A.ARES_REDUCE_HASH:
            meas = meas + 0.0        # the hash-reduce mode's slots start at +0.0
    elif kind in ("min", "max"):
        cl = _cls(dt)
        ident = IDENTITY[(kind, cl)]
        fold = np.minimum if kind == "min" else np.maximum
        if cl == "f":
            meas = np.full(g, np.inf if kind == "min" else -np.inf, np.float32)
            x = np.where(ok, v, np.float32(ident)).astype(np.float32)
        else:
            npt = np.int64
            meas = np.full(g, 2 ** 40 if kind == "min" else -2 ** 40, npt)
            x = np.where(ok, v.astype(np.int64), ident)
        fold.at(meas, inv, x)
        if cl != "f":
            meas = meas.astype(np.uint32) if cl == "u" else meas.astype(np.int32)
    else:   # avg: (float average, count); an integer value is converted to float32 first
        cnt = np.zeros(g, np.int64)
        np.add.at(cnt, inv, np.where(ok, mult, 0))
        x = np.where(ok, v.astype(np.float32).astype(np.float64), 0.0)
        s = np.zeros(g)
        np.add.at(s, inv, x * mult)
        scale = np.zeros(g)
        np.maximum.at(scale, inv, np.abs(x))
        with np.errstate(invalid="ignore", divide="ignore"):
            meas = np.where(cnt > 0, s / np.maximum(cnt, 1), 0.0)
        counts = cnt
    if mode == A.ARES_REDUCE_SORT:
        grows = rows[first]
        order = np.argsort(hashes.murmur3_128_lo(grows), kind="stable")
        out = Expected([r.tobytes() for r in grows[order]], meas[order], None if counts is None else counts[order],
                       None if scale is None else scale[order])
    else:
        out = Expected(uniq.tolist(), meas, counts, scale)
    return out


def _by_hash(got):
    keys = hashes.murmur3_32(got.packed_rows()) if got.groups else np.zeros(0, np.uint32)
    order = np.argsort(keys, kind="stable")
    return keys[order].tolist(), order


def assert_matches(got, exp, kind, dt, mode=A.ARES_REDUCE_SORT, ctx=""):
    """got: a QueryResult.  The comparison rules of the module docstring."""
    assert got.groups == len(exp.rows), f"{ctx}: {got.groups} groups, expected {len(exp.rows)}"
    if mode == A.ARES_REDUCE_SORT:
        assert got.rows == exp.rows, f"{ctx}: dimension rows / order differ"
        gm, gc_ = got.measures, got.counts
    else:
        keys, order = _by_hash(got)
        assert keys == exp.rows, f"{ctx}: group hashes differ"
        gm, gc_ = got.measures[order], None if got.counts is None else got.counts[order]
    if kind == "avg":
        assert gc_.tolist() == exp.counts.tolist(), f"{ctx}: counts differ"
        tight = exp.scale < 2.0 ** 127
        with np.errstate(invalid="ignore"):
            err = np.abs(gm.astype(np.float64) - exp.meas)
        bad = tight & ~(err <= 2e-5 * exp.scale + 1e-6)
        assert not bad.any(), f"{ctx}: averages differ: {list(zip(gm[bad][:5], exp.meas[bad][:5]))}"
    elif kind in ("min", "max") and dt == A.Float32:
        bad = gm != exp.meas
        assert not bad.any(), f"{ctx}: float {kind} differs: {list(zip(gm[bad][:5], exp.meas[bad][:5]))}"
    else:
        assert gm.dtype == exp.meas.dtype, f"{ctx}: {gm.dtype} vs {exp.meas.dtype}"
        if gm.tobytes() != exp.meas.tobytes():
            diff = [i for i in range(len(gm)) if gm[i:i + 1].tobytes() != exp.meas[i:i + 1].tobytes()]
            raise AssertionError(f"{ctx}: measures differ at {len(diff)} groups, e.g. {[(gm[i], exp.meas[i]) for i in diff[:5]]}")


# ---- the matrix --------------------------------------------------------------------------------------------------
AGGS = ["sum", "min", "max", "avg"]


def matrix():
    """name -> (kind, column type, form, dims, filters, reduce mode)."""
    cases = {}

    def add(kind, dt, form, dims="kw", filters=(BASE_FILTER,), mode=A.ARES_REDUCE_SORT):
        name = f"{form}/{kind}" + (f"_{NAME[dt]}" if dt is not None else "") + ("/hash" if mode == A.ARES_REDUCE_HASH else "")
        cases[name] = (kind, dt, form, dims, filters, mode)

    for kind in AGGS:
        for dt in TYPES:
            add(kind, dt, "cta")
    add("count", None, "cta")
    add("sum", A.Float32, "fx", filters=(FX_FILTER,))
    for form, dims in (("global", "wh"), ("hash", "kw"), ("bypass", "wh"), ("tail", "kw")):
        for kind in AGGS:
            for dt in THREE:
                if form == "global" and kind == "sum" and dt != A.Float32:
                    continue        # (2): integer sums keep the hash table
                add(kind, dt, form, dims)
        add("count", None, form, dims)
    add("max", A.Int16, "cta", mode=A.ARES_REDUCE_HASH)
    add("sum", A.Float32, "fx", filters=(FX_FILTER,), mode=A.ARES_REDUCE_HASH)
    add("min", A.Float32, "global", "wh", mode=A.ARES_REDUCE_HASH)
    add("avg", A.Uint32, "hash", mode=A.ARES_REDUCE_HASH)
    add("sum", A.Int16, "bypass", "wh", mode=A.ARES_REDUCE_HASH)
    return cases


CASES = matrix()
BYPASS_GROUPS = 100_000


def _expected_groups(form):
    return BYPASS_GROUPS if form == "bypass" else 0


def _zone_map_modes(form):
    return {"cta": ("exact", "narrow", "stale"), "fx": ("exact", "narrow", "stale"), "global": ("exact", "narrow", "stale"),
            "hash": (None,), "bypass": (None,), "tail": ("exact",)}[form]


def _ranges(hb, form, how):
    if how is None:
        return None
    zm = zone_map(hb, how)
    if form == "fx":
        zm[COL[A.Float32]] = FX_RANGE
    return zm


# ---- CPU: the form every GPU case reaches --------------------------------------------------------------------------
def _plan(insts, rows, ranges=None, base_counts=None):
    p = A.BatchPlan()
    p.NumInsts = len(insts)
    for i, pi in enumerate(insts):
        p.Insts[i] = pi
    p.NumColumns = len(COLUMN_TYPES)
    for i, dt in enumerate(COLUMN_TYPES):   # fake, aligned device addresses: nothing is dereferenced
        p.Columns[i] = columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, rows, 0, 64 * 200 * 4, 1 if i < 3 else 2, 0)
    p.NumRows = rows
    if base_counts is not None:
        p.BaseCounts = base_counts
    for col, (lo, hi) in (ranges or {}).items():
        p.Ranges[col].Known, p.Ranges[col].Min, p.Ranges[col].Max = 1, lo, hi
    return p


def _dry_run(q, rows, ranges=None, expected_groups=0):
    """The generated text of `q` over a batch of the edge table's columns (ARESDB_B200_JIT_GENERATE_ONLY)."""
    fn = A.load_engine().alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    p = _plan(q.plan_instructions(), rows, ranges)
    src = C.c_char_p()
    h = fn(q.agg_spec(expected_groups), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return (src.value or b"").decode()


def _macro(src, name):
    for line in src.splitlines():
        if line.startswith(f"#define {name} "):
            return int(line.split()[2])
    raise AssertionError(f"{name} not in the generated text")


def expected_form(kind, dt, form):
    """The macros a case must generate."""
    if form in ("hash", "tail"):
        return {"JIT_DENSE": 0, "JIT_BYPASS": 0}
    if form == "bypass":
        return {"JIT_DENSE": 0, "JIT_BYPASS": 1}
    if form == "fx":
        return {"JIT_DENSE": 1, "JIT_DENSE_ACC": 4, "JIT_DENSE_FLAGS": 0}
    if form == "global":
        return {"JIT_DENSE": 2, "JIT_DENSE_CHECK": 0 if kind == "count" else 1, "JIT_DENSE_FLAGS": 0 if kind == "count" else 1}
    four_byte = kind == "count" or (kind in ("min", "max") and dt != A.Float32)
    return {"JIT_DENSE": 1, "JIT_DENSE_ACC": 1 if four_byte else 2, "JIT_DENSE_FLAGS": 0 if kind == "count" else 1}


def case_form_source(name):
    kind, dt, form, dims, filters, mode = CASES[name]
    hb = edge_batches("tail" if form == "tail" else "solo")[0]
    how = _zone_map_modes(form)[0]
    q = make_query(kind, dt, dims, filters, mode)
    return _dry_run(q, hb["rows"], _ranges(hb, form, how), _expected_groups(form))


def test_form_of_every_case(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    texts = set()
    for name, (kind, dt, form, dims, filters, mode) in CASES.items():
        src = case_form_source(name)
        for macro, want in expected_form(kind, dt, form).items():
            assert _macro(src, macro) == want, f"{name}: {macro}"
        texts.add(src)
    # (2) an integer column's sum over more slots than a CTA holds keeps the hash table
    hb = edge_batches()[0]
    for dt in TYPES[:-1]:
        src = _dry_run(make_query("sum", dt, "wh"), hb["rows"], zone_map(hb))
        assert _macro(src, "JIT_DENSE") == 0, NAME[dt]
    # the integer form needs the filter that proves the measure non-NULL
    assert _macro(_dry_run(make_query("sum", A.Float32), hb["rows"], _ranges(hb, "fx", "exact")), "JIT_DENSE_ACC") == 2
    # the zone-map variants of a case run the same kernel: the ranges are runtime parameters
    for name in ("cta/min_i32", "global/max_f32"):
        kind, dt, form, dims, filters, mode = CASES[name]
        q = make_query(kind, dt, dims, filters, mode)
        srcs = {_dry_run(q, hb["rows"], _ranges(hb, form, how)) for how in _zone_map_modes(form)}
        assert len(srcs) == 1, name
    print(f"{len(CASES)} solo cases, {len(texts)} distinct kernel texts")


SHARED_REQUESTS = {
    # i16 min (ACC 1), f32 max (ACC 2), i32 sum (ACC 2, flags), avg u8 (ACC 2)
    "mixed": ([("min", A.Int16), ("max", A.Float32), ("sum", A.Int32), ("avg", A.Uint8)], (BASE_FILTER,),
              [("ne", A.Int16, 0), ("gt", A.Float32, -1.0), ("ge", A.Int32, 0), ("ne", A.Uint8, 255)],
              {"kMeasAcc": "{1, 2, 2, 2}", "kMeasFlags": "{true, true, true, true}", "kMeasCheck": "{true, true, false, true}"}),
    # exact-integer sum(f32) (ACC 4), count (flag-less), u32 max (ACC 1), f32 min (ACC 2)
    "exact": ([("sum", A.Float32), ("count", None), ("max", A.Uint32), ("min", A.Float32)], (FX_FILTER,),
              [("lt", A.Float32, 50.0), ("ge", A.Int16, 0), ("ne", A.Uint32, 0), ("ne", A.Float32, 1.0)],
              {"kMeasAcc": "{4, 1, 1, 2}", "kMeasFlags": "{false, false, true, true}", "kMeasCheck": "{true, false, true, true}"}),
}


def shared_queries(name, member_filters):
    """The request's queries and, per query, its filter triples."""
    ms, common, own, _ = SHARED_REQUESTS[name]
    out = []
    for (kind, dt), f in zip(ms, own):
        fs = tuple(common) + ((f,) if member_filters else ())
        out.append((make_query(kind, dt, "kw", fs), kind, dt, fs))
    return out


def test_shared_form_of_every_request(monkeypatch):
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    lib = A.load_engine()
    hb = edge_batches()[0]
    for name, (_, _, _, tables) in SHARED_REQUESTS.items():
        for mf in (False, True):
            qs = [q for q, *_ in shared_queries(name, mf)]
            from aresdb_b200.executor import shared_scan_groups
            assert shared_scan_groups(qs, member_filters=True) == [[0, 1, 2, 3]]
            _, src = S.dry_run_multi(lib, qs, _plan(qs[0].plan_instructions(measures=qs), hb["rows"], _ranges(hb, "fx", "exact")))
            assert "#define JIT_NMEAS 4" in src and "#define JIT_DENSE 1" in src, name
            for t, want in tables.items():
                assert f"{t}[JIT_NMEAS] = {want};" in src, (name, mf, t)
            assert ("JIT_LIVE_ARG" in src) == mf


# ---- CPU: the restatement equals the oracle's call sequence and the reference's HOST build -------------------------
def _legacy(be, q, hbs):
    ex = LegacyBatchExecutor(be.lib, be.space, q)
    for hb in hbs:
        ex.process_batch(upload(be, hb))
    return ex.result()


@pytest.mark.parametrize("kind", AGGS + ["count"])
def test_restatement_matches_oracle_and_reference(kind):
    """Sort mode, every column type, the edge table (NULLs, garbage under NULL, type extremes, neutral elements)."""
    orc = H.get_backend("oracle")
    hbs = edge_batches("cpu")
    dts = [None] if kind == "count" else TYPES
    results = []
    for dt in dts:
        q = make_query(kind, dt)
        got = _legacy(orc, q, hbs)
        assert_matches(got, restate(hbs, kind, dt), kind, dt, ctx=f"oracle {kind} {NAME.get(dt)}")
        results.append(got)
    H.assert_matches_reference(f"aggregate_forms/{kind}", H.digest(results),
                               lambda: H.digest([_legacy(H.get_backend("ref"), make_query(kind, dt), hbs) for dt in dts]))


def test_hash_mode_restatement_matches_oracle():
    """Hash-reduce mode: groups keyed by the 32-bit murmur3 of the (5-byte) row, float sums from +0.0.  MIN / MAX are not
    pinned here: the HOST map starts them from zero where the DEVICE map starts from the identity (DESIGN §4)."""
    orc = H.get_backend("oracle")
    hbs = edge_batches("cpu")
    for kind, dt in (("sum", A.Int16), ("sum", A.Float32), ("count", None), ("avg", A.Uint32)):
        got = _legacy(orc, make_query(kind, dt, mode=A.ARES_REDUCE_HASH), hbs)
        assert_matches(got, restate(hbs, kind, dt, mode=A.ARES_REDUCE_HASH), kind, dt, A.ARES_REDUCE_HASH,
                       ctx=f"oracle hash mode {kind} {NAME.get(dt)}")


def test_restatement_quirks():
    """The reference's identities on the edge table: a NULL row in a group of negative floats makes its MAX FLT_MIN, a
    group of NULLs is MIN 0xFFFFFFFF / INT32_MAX / FLT_MAX, AVG (0, count 0); the cancelling groups sum to 0."""
    hbs = edge_batches("cpu")
    neg = [i for i, v in enumerate(edge_values(A.Float32)) if v < 0]

    def by_w(exp, k):
        return {(r[2], r[0] | r[1] << 8): m for r, m in zip(exp.rows, exp.meas)}.get

    mx = by_w(restate(hbs, "max", A.Float32), 0)
    assert all(mx((1, w)) == np.float32(F32_MIN) for w in neg) and mx((0, 1)) == -np.inf
    for dt, ident in ((A.Uint8, 0xFFFFFFFF), (A.Int32, 2 ** 31 - 1), (A.Float32, np.float32(F32_MAX))):
        mn = by_w(restate(hbs, "min", dt), 0)
        assert all(mn((k, W_NULL)) == ident for k in range(NK))
    avg = restate(hbs, "avg", A.Int16)
    nulls = [i for i, r in enumerate(avg.rows) if r[0] | r[1] << 8 == W_NULL]
    assert nulls and all(avg.counts[i] == 0 and avg.meas[i] == 0 for i in nulls)
    for dt in (A.Int8, A.Int32, A.Float32):
        s = by_w(restate(hbs, "sum", dt), 0)
        assert all(s((k, W_CANCEL)) == 0 for k in range(NK))
    s = by_w(restate(hbs, "sum", A.Float32), 0)
    assert np.signbit(s((0, 2))) and not np.signbit(s((1, 2)))   # -0.0 alone stays -0.0; a NULL adds +0.0


# ---- GPU ---------------------------------------------------------------------------------------------------------
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


def _run(eng, q, batches, expected_groups=0):
    ex = FusedBatchExecutor(eng.lib, eng.space, q, expected_groups)
    for b in batches:
        ex.process_batch(b)
    r = ex.result()
    ex.close()
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_solo_forms_on_gpu(name):
    eng = H.get_backend("b200")
    kind, dt, form, dims, filters, mode = CASES[name]
    hbs = edge_batches("tail" if form == "tail" else "solo")
    q = make_query(kind, dt, dims, filters, mode)
    exp = restate(hbs, kind, dt, dims, filters, mode)
    if form in ("global", "bypass"):
        assert len(exp.rows) > 32768, "the >32,768-group finalize"
    for how in _zone_map_modes(form):
        before = T.dense_launches(eng)
        got = _run(eng, q, [upload(eng, hb, _ranges(hb, form, how)) for hb in hbs], _expected_groups(form))
        assert_matches(got, exp, kind, dt, mode, ctx=f"{name}/{how}")
        dense = T.dense_launches(eng) - before
        assert dense == (len(hbs) if form in ("cta", "fx", "global") else 0), f"{name}/{how}: {dense} direct-indexed launches"


def rle_batch(be, hb, measure_rle, seed):
    """An archive-style batch over the index positions of edge batch `hb`: k is the first sort column (run-length
    encoded, its counts are the batch's base counts; one index position per run), ts and w one value per index position;
    the measures one value per index position, or (measure_rle) first-class RLE columns with their own, finer runs.
    Returns the Batch and the host arrays per index position (with `mult`, the run lengths) for the restatement."""
    rng = np.random.default_rng(seed)
    n = hb["rows"]
    lens = rng.integers(1, 9, n)
    base = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    total = int(base[-1])
    order = np.argsort(hb["k"], kind="stable")            # k sorted: its runs are the index positions
    idx = {c: hb[c][order] for c in ("ts", "k", "w")}
    view = {"rows": n, "mult": lens.astype(np.int64), **idx}
    cols, keep = [], []
    for c, dt in enumerate(COLUMN_TYPES[:3]):
        counts = base if c == 1 else None
        buf, vp = columns.make_column(be.space, dt, idx[("ts", "k", "w")[c]], counts=counts)
        cols.append(vp)
        keep.append(buf)
    for dt in TYPES:
        v, ok = (a[order] for a in hb[dt])
        if measure_rle:
            # finer runs: cut points include every index position's first row, so each position starts a run whose
            # value is that position's
            extra = np.sort(rng.choice(np.setdiff1d(np.arange(1, total), base), size=min(n, total - n - 1), replace=False))
            cuts = np.union1d(base, extra).astype(np.uint32)
            run_of = np.searchsorted(base, cuts[:-1], side="right") - 1
            rv, rok = v[run_of].copy(), ok[run_of].copy()
            inner = ~np.isin(cuts[:-1], base)                     # runs that start inside a position: never read
            rv[inner] = v[::-1][run_of[inner] % n]
            buf, vp = columns.make_column(be.space, dt, rv, valid=rok, counts=cuts)
        else:
            buf, vp = columns.make_column(be.space, dt, v, valid=ok)
        view[dt] = (v, ok)
        cols.append(vp)
        keep.append(buf)
    bc = be.put(base)
    return Batch(cols, n, base_counts=bc, start_count=0, keep=keep, ranges={1: (0, NK - 1), 2: (0, NW - 1)}), view


RLE_CASES = [(k, dt) for k in AGGS for dt in (A.Int16, A.Float32)] + [("count", None)]


@pytest.mark.gpu
@pytest.mark.parametrize("measure_rle", [True, False], ids=["rle_measure", "unsorted_measure"])
def test_rle_batches_on_gpu(measure_rle):
    """SUM / COUNT / AVG count run lengths, MIN / MAX do not, in the CTA form (the dimension columns' zone map)."""
    import ctypes
    eng = H.get_backend("b200")
    hbs = [edge_batch(51, 60_001), edge_batch(52, 40_003)]
    batches, views = zip(*[rle_batch(eng, hb, measure_rle, 60 + i) for i, hb in enumerate(hbs)])
    out = (ctypes.c_ulonglong * 2)()
    for kind, dt in RLE_CASES:
        q = make_query(kind, dt)
        eng.lib.alg.AresJitStats(out)
        before, dense = int(out[1]), T.dense_launches(eng)
        got = _run(eng, q, batches)
        eng.lib.alg.AresJitStats(out)
        assert int(out[1]) - before == len(batches) and T.dense_launches(eng) - dense == len(batches)
        assert_matches(got, restate(views, kind, dt), kind, dt, ctx=f"rle {kind} {NAME.get(dt)}")


def _shared_batches(eng, how="exact"):
    return [upload(eng, hb, _ranges(hb, "fx", how)) for hb in edge_batches()]


@pytest.mark.gpu
@pytest.mark.parametrize("member_filters", [False, True], ids=["common", "member_filters"])
@pytest.mark.parametrize("request_name", list(SHARED_REQUESTS))
def test_shared_form_on_gpu(request_name, member_filters):
    """Four members of different forms in one kernel per batch, each against the restatement."""
    eng = H.get_backend("b200")
    qspecs = shared_queries(request_name, member_filters)
    qs = [q for q, *_ in qspecs]
    for how in ("exact", "narrow", "stale"):
        req = FusedRequestExecutor(eng.lib, eng.space, qs)
        for b in _shared_batches(eng, how):
            k0, d0 = eng.lib.kernel_launch_count(), T.dense_launches(eng)
            req.process_batch(b)
            assert (eng.lib.kernel_launch_count() - k0, T.dense_launches(eng) - d0) == (1, 1), "one launch per batch"
        for got, (q, kind, dt, fs) in zip(req.results(), qspecs):
            assert_matches(got, restate(edge_batches(), kind, dt, "kw", fs), kind, dt, ctx=f"{request_name}/{how}/{kind}")
        req.close()


@pytest.mark.gpu
@pytest.mark.parametrize("request_name", list(SHARED_REQUESTS))
def test_exchange_of_shared_requests_on_gpu(request_name):
    """Batch i on simulated rank i mod 2; the merged parts (mergePartsKernel: signed and float MIN / MAX, AVG, sums)
    equal the restatement over all batches on every rank."""
    eng = H.get_backend("b200")
    qspecs = shared_queries(request_name, True)
    qs = [q for q, *_ in qspecs]
    locals_ = [FusedRequestExecutor(eng.lib, eng.space, qs) for _ in range(2)]
    for i, b in enumerate(_shared_batches(eng)):
        locals_[i % 2].process_batch(b)
    xqs, out = SR._exchange_on_one_device(eng, locals_, 32768, (1,))
    for r, (merged, res, claimed) in enumerate(out[0]):
        for j, (q, kind, dt, fs) in enumerate(qspecs):
            assert not isinstance(res[j], Exception), f"rank {r} query {j}: {res[j]}"
            assert_matches(query_result(xqs[j], *res[j]), restate(edge_batches(), kind, dt, "kw", fs), kind, dt,
                           ctx=f"{request_name}/rank{r}/{kind}")
        for m in merged:
            m.close()
    for ex in locals_:
        ex.close()
