"""Dimension-table joins at their edges, against an independent numpy restatement of a join.

What a join is (the reference: HashLookupFunctor query/functor.hpp:1173-1266, RecordIDJoinIterator query/iterator.hpp:
846-931; here `joins.py`, `csrc/join.cuh` and the gather stage `jit.cu` generates), stated one rule per line in
`restate_lookup` / `restate_foreign`:

  key bytes   the key is the low keyBytes bytes of the main-table value widened to 32 bits (a Bool is 0 / 1, a signed
              value is sign-extended): Int8 -1 matches the primary key 0xFF, Uint32 65541 joined to a Uint16 key finds 5
  misses      a NULL key or a key that is not in the index gives RecordID {0, 0}; every foreign column then reads NULL
  bounds      batch = batchID - BaseBatchID; an index >= NumRecordsInLastBatch is NULL in the last batch only
  mode 0      a foreign batch without vectors yields the COLUMN's default (ForeignColumnVector.DefaultValue), not the
              batch slice's own
  time zone   the enum -> offset table applies to the raw stored value, valid or not, and keeps its validity:
              table[e] if e < size else 0; a Float32 enum is truncated to int; a Bool column's result is off != 0
  NULLs       a NULL foreign value fails every comparison, is a NULL dimension and adds the aggregate's identity

Two documented departures, where the reference reads out of bounds: a batchID outside [BaseBatchID, BaseBatchID +
NumBatches) and a negative (signed) enum give NULL and offset 0.  Those cases are checked against the restatement, the
oracle and the engine only, never against the reference's HOST build.

The query on top is evaluated with numpy and grouped by test_aggregate_forms.restate (the reference's row identity and
order).  The CPU tests pin the restatement to the oracle's per-node call sequence and to the reference's HOST build
(stored digests where it is not built); the GPU tests run the per-node HashLookup and every form of the fused kernel
that carries the gather, and each GPU case asserts the form it reached.

Combinations the engine refuses, asserted as refusals: a countdistincthll measure over a foreign column (the measure of
an HLL query is a main-table column), keys of 8 and 16 bytes on the fused path (an Int64 / UUID key column when the plan
compiles, an index of such keys in `uploadJoin`), a dimension table of more than 8 batches (`makeForeignDesc`, both
engine paths) and a fifth joined table (`_BatchPlans`).
"""
from __future__ import annotations

import ctypes as C
import functools
import gc

import numpy as np
import pytest

import harness as H
import hashes
import test_aggregate_forms as AF
import test_pipeline_parity as T
from aresdb_b200 import cabi as A
from aresdb_b200 import columns, expr as E, joins as J
from aresdb_b200.executor import Batch, FusedBatchExecutor, FusedRequestExecutor, LegacyBatchExecutor
from aresdb_b200.query import AggQuery, Join, Measure

BACKENDS = [pytest.param("ref", id="ref"), pytest.param("oracle", id="oracle"), pytest.param("b200", marks=pytest.mark.gpu, id="b200")]
NP = {A.Bool: np.uint8, A.Int8: np.int8, A.Int16: np.int16, A.Int32: np.int32, A.Uint8: np.uint8, A.Uint16: np.uint16,
      A.Uint32: np.uint32, A.Float32: np.float32, A.Int64: np.int64}
SIGNED = (A.Int8, A.Int16, A.Int32, A.Int64)
FUSED_KEY_ERROR = "fused path: keys of at most 4 bytes"                 # uploadJoin: the index's key width
FUSED_KEY_COLUMN_ERROR = "join keys of the fused path are 1-, 2- or 4-byte columns"   # compilePlan: the key column
BATCHES_ERROR = "a joined dimension table may hold at most 8 batches"


@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    gc.collect()
    try:
        import torch
        if torch.cuda.is_available() and torch.cuda.is_initialized():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    except ImportError:
        pass


# ---- an index placed by hand ---------------------------------------------------------------------------------------
def key_bytes_of(value: int, kb: int) -> bytes:
    return (int(value) & ((1 << (8 * kb)) - 1)).to_bytes(kb, "little")


class IndexWriter:
    """The memstore's cuckoo layout (per bucket RecordID[8] | signature[8] | key[8], numBuckets buckets, then the stash
    bucket), with every key put where the test says."""

    def __init__(self, kb, num_buckets, num_hashes=4, seeds=J.DEFAULT_SEEDS):
        self.kb, self.nb, self.nh, self.seeds = kb, num_buckets, num_hashes, tuple(seeds)
        self.cell = 8 + kb + 1
        self.raw = np.zeros(8 * self.cell * (num_buckets + 1), np.uint8)

    def hash(self, key: bytes, t: int) -> int:
        return J.murmur3_32(key, self.seeds[t])

    def bucket_of(self, key: bytes, t: int) -> int:
        return self.hash(key, t) % self.nb

    def signature(self, key: bytes, t: int) -> int:
        return max(self.hash(key, t) >> 24, 1)

    def put(self, bucket: int, cell: int, key: bytes, rid, sig: int):
        base = bucket * 8 * self.cell
        self.raw[base + 8 * cell: base + 8 * cell + 8] = np.frombuffer(np.array([rid[0]], "<i4").tobytes() + np.array([rid[1]], "<u4").tobytes(), np.uint8)
        self.raw[base + 64 + cell] = sig
        self.raw[base + 72 + cell * self.kb: base + 72 + (cell + 1) * self.kb] = np.frombuffer(key, np.uint8)

    def put_hashed(self, key: bytes, rid, t: int, cell: int):
        self.put(self.bucket_of(key, t), cell, key, rid, self.signature(key, t))

    def put_stash(self, key: bytes, rid, cell: int, sig: int = 1):
        self.put(self.nb, cell, key, rid, sig)

    def index(self, be, num_hashes=None):
        buf = be.put(self.raw)
        h = A.CuckooHashIndex()
        h.buckets = buf.ptr
        for i in range(4):
            h.seeds[i] = self.seeds[i]
        h.keyBytes, h.numHashes, h.numBuckets = self.kb, self.nh if num_hashes is None else num_hashes, self.nb
        return h, buf


def place_all(keys: np.ndarray, kb: int, rids: np.ndarray, num_hashes=4, seeds=J.DEFAULT_SEEDS):
    """Vectorised first-free placement of many keys (uint32 values, their low kb bytes; rids int64[n, 2]): hash t of the
    keys not yet placed, a key takes the next free cell of its bucket, the rest go on to hash t + 1, then the stash.
    Returns (raw bytes, num_buckets)."""
    n = len(keys)
    kbytes = np.ascontiguousarray(keys.astype("<u4").view(np.uint8).reshape(n, 4)[:, :kb])
    nb = max(3, n // 4 + 1)
    cell = 8 + kb + 1
    while True:
        raw = np.zeros((nb + 1, 8 * cell), np.uint8)
        used = np.zeros(nb + 1, np.int64)
        todo = np.arange(n)
        for t in range(num_hashes):
            if not len(todo):
                break
            h = hashes.murmur3_32(kbytes[todo], seeds[t]).astype(np.int64)
            b = h % nb
            order = np.argsort(b, kind="stable")
            sb = b[order]
            rank = np.arange(len(sb)) - np.searchsorted(sb, sb, side="left")
            c = used[sb] + rank
            ok = c < 8
            _write_cells(raw, sb[ok], c[ok], kbytes[todo[order[ok]]], rids[todo[order[ok]]], np.maximum(h[order[ok]] >> 24, 1), kb)
            used += np.bincount(sb[ok], minlength=nb + 1)
            todo = todo[order[~ok]]
        if len(todo) <= 4:
            h0 = hashes.murmur3_32(kbytes[todo], seeds[0]).astype(np.int64)
            _write_cells(raw, np.full(len(todo), nb), np.arange(len(todo)), kbytes[todo], rids[todo], np.maximum(h0 >> 24, 1), kb)
            return raw.reshape(-1), nb
        nb = nb * 3 // 2 + 1


def _write_cells(raw, bucket, cell, kbytes, rids, sig, kb):
    rb = np.zeros((len(bucket), 8), np.uint8)
    rb[:, :4] = rids[:, 0].astype("<i4").view(np.uint8).reshape(-1, 4)
    rb[:, 4:] = rids[:, 1].astype("<u4").view(np.uint8).reshape(-1, 4)
    for i in range(8):
        raw[bucket, 8 * cell + i] = rb[:, i]
    raw[bucket, 64 + cell] = sig.astype(np.uint8)
    for i in range(kb):
        raw[bucket, 72 + cell * kb + i] = kbytes[:, i]


# ---- the restatement ---------------------------------------------------------------------------------------------
def widen(values, dt):
    """The 32-bit pattern the reference hashes: a Bool is 0 / 1, signed values sign-extend."""
    v = np.asarray(values)
    if dt == A.Bool:
        return (v != 0).astype(np.int64)
    return v.astype(np.int64) & 0xFFFFFFFF


def restate_lookup(pk: dict, kb: int, values, valid, dt):
    """RecordIDs (batchID int64[n], index int64[n]) of a main-table key column; pk: key (int, its kb bytes) -> rid."""
    key = widen(values, dt) & ((1 << (8 * kb)) - 1)          # the low keyBytes bytes of the widened value
    pks = np.array(sorted(pk), np.int64)                     # a sorted-array lookup of the primary keys
    rids = np.array([pk[k] for k in pks.tolist()], np.int64).reshape(-1, 2)
    at = np.clip(np.searchsorted(pks, key), 0, len(pks) - 1)
    found = np.asarray(valid, bool) & (pks[at] == key)       # a NULL key or a miss is RecordID {0, 0}
    return np.where(found, rids[at, 0], 0), np.where(found, rids[at, 1], 0)


class DimData:
    """A dimension table on the host: per column the values and validity of every physical slot [batch, row], the mode
    of every batch, the column default, the Bool columns' start bits."""

    def __init__(self, types, vals, ok, modes, defaults, nlast, base, start_bits=None, slice_defaults=None):
        self.types, self.vals, self.ok, self.modes, self.defaults = types, vals, ok, modes, defaults
        self.nb, self.rows = vals[0].shape
        self.nlast, self.base = nlast, base
        self.start_bits = start_bits or [[0] * self.nb for _ in types]
        self.slice_defaults = slice_defaults


def restate_foreign(d: DimData, c: int, bid, idx, tz=None):
    """(values, valid) of foreign column c at RecordIDs (bid, idx); tz: the enum -> offset table (int16 array)."""
    n = len(bid)
    dt = d.types[c]
    v = np.zeros(n, np.float32 if dt == A.Float32 else np.int64)
    ok = np.zeros(n, bool)
    b = bid - d.base                                          # batch = batchID - BaseBatchID
    hit = bid != 0                                            # RecordID {0, 0}: NULL
    hit &= (b < d.nb - 1) | (idx < d.nlast)                   # index >= NumRecordsInLastBatch: NULL in the last batch only
    hit &= (b >= 0) & (b < d.nb)                              # departure: the reference reads outside the batch array
    bi, ri = np.where(hit, b, 0), np.where(hit, np.minimum(idx, d.rows - 1), 0)
    const = hit & (np.asarray(d.modes[c])[bi] == 0)          # mode 0: the column's default, not the slice's ...
    mapped = hit & ~const                                     # ... and not mapped through the time-zone table
    v[mapped], ok[mapped] = d.vals[c][bi[mapped], ri[mapped]], d.ok[c][bi[mapped], ri[mapped]]
    ok[const], v[const] = d.defaults[c]
    if tz is not None and np.any(mapped):
        keep = v.copy()
        e = np.trunc(v).astype(np.int64) if dt == A.Float32 else v.astype(np.int64)   # Float32 enums truncate
        inside = (e >= 0) & (e < len(tz))                     # departure: a negative enum is outside the table
        off = np.where(inside, np.asarray(tz, np.int64)[np.clip(e, 0, len(tz) - 1)], 0)
        off = np.where(hit, off, 0)
        if dt == A.Float32:
            v = off.astype(np.float32)
        elif dt == A.Bool:
            v = (off != 0).astype(np.int64)                   # a Bool column's result is off != 0
        else:
            v = off if dt in SIGNED else off & 0xFFFFFFFF     # the offset as a 32-bit value; validity is kept
        v = np.where(mapped | ~hit, v, keep).astype(v.dtype)
    return v, ok


class Env:
    """One fact batch and the joins of one query: evaluates expressions with numpy."""

    def __init__(self, hb, q: AggQuery, dims: list, tzs: list):
        self.hb, self.q, self.cache = hb, q, {}
        self.rids = []
        for j, (d, pk, kb) in zip(q.joins, dims):
            kv, kok = hb[j.on.index]
            self.rids.append(restate_lookup(pk, kb, kv, kok, j.on.data_type))
        self.dims, self.tzs = dims, tzs

    def value(self, e):
        """(values, valid, data type) of a leaf or a bucketizer; values int64 / float32."""
        if isinstance(e, E.Col):
            v, ok = self.hb[e.index]
            return (v.astype(np.float32) if e.data_type == A.Float32 else widen_signed(v, e.data_type)), np.asarray(ok, bool), e.data_type
        if isinstance(e, E.ForeignCol):
            key = (e.table, e.index, e.timezone)
            if key not in self.cache:
                bid, idx = self.rids[e.table]
                self.cache[key] = restate_foreign(self.dims[e.table][0], e.index, bid, idx, self.tzs[e.table] if e.timezone else None)
            v, ok = self.cache[key]
            if e.data_type in SIGNED and not e.timezone:
                v = widen_signed(v, e.data_type)
            return v, ok, e.data_type
        if isinstance(e, E.Bucket):                           # manual partitions: the count of partitions <= x
            v, ok, _ = self.value(e.expr)
            x = v.astype(np.float64)
            nan = np.isnan(x)
            ordinal = np.searchsorted(np.asarray(e.bounds), np.where(nan, 0, x), side="right")
            ok = ok & ~nan                                    # NULL and NaN give NULL, ordinal 0
            return np.where(ok, ordinal, 0).astype(np.int64), ok, A.Uint8
        if isinstance(e, E.Binary) and e.op == A.Floor:       # floor(unsigned column, literal): v - v % literal
            v, ok, _ = self.value(e.lhs)
            return v - v % int(e.rhs.value), ok, A.Uint32
        raise TypeError(e)

    def mask(self, f):
        """A filter: comparison of a leaf with a literal, IsNull / IsNotNull; NULL fails every comparison."""
        if isinstance(f, E.Unary):
            _, ok, _ = self.value(f.expr)
            return ~ok if f.op == A.IsNull else ok
        v, ok, dt = self.value(f.lhs)
        lit = f.rhs.value
        if dt == A.Float32:
            v, lit = v.astype(np.float32), np.float32(lit)
        elif dt in SIGNED or f.rhs.type == E.Type.Signed:
            v = v.astype(np.int64)
        op = {A.Equal: np.equal, A.NotEqual: np.not_equal, A.LessThan: np.less, A.LessThanOrEqual: np.less_equal,
              A.GreaterThan: np.greater, A.GreaterThanOrEqual: np.greater_equal}[f.op]
        with np.errstate(invalid="ignore"):
            return ok & op(v, lit)


def widen_signed(v, dt):
    v = np.asarray(v)
    if dt in SIGNED:
        return v.astype(NP[dt]).astype(np.int64)
    return v.astype(np.int64)


def dim_bytes(v, ok, dt):
    w = max(A.DATA_TYPE_BYTES[dt], 1)
    if dt == A.Float32:
        raw = np.asarray(v, np.float32).view(np.uint32).astype(np.int64)
    else:
        raw = np.asarray(v).astype(np.int64) & ((1 << (8 * w)) - 1)
    # a NULL dimension keeps the bytes of the value read (a miss reads 0): NULL groups differ by what lies under them
    return raw.astype("<u8").view(np.uint8).reshape(-1, 8)[:, :w]


def restate_query(q: AggQuery, hbs, dims, tzs):
    """The restatement's groups of `q` over the host batches: an AF.Expected (rows in the reference's order)."""
    views = []
    mdt = None
    for hb in hbs:
        env = Env(hb, q, dims, tzs)
        alive = np.ones(hb["rows"], bool)
        for f in q.filters:
            alive &= env.mask(f)
        cols = [env.value(q.dimensions[qi]) for qi in q.dim_order]
        packed = np.hstack([dim_bytes(v, ok, dt) for v, ok, dt in cols] + [ok.astype(np.uint8).reshape(-1, 1) for _, ok, _ in cols]) \
            if cols else np.zeros((hb["rows"], 0), np.uint8)
        view = {"rows": int(alive.sum()), "packed": packed[alive], "mult": hb.get("mult", np.ones(hb["rows"], np.int64))[alive]}
        if q.measure_kind != "count":
            v, ok, mdt = env.value(q.measure)
            if mdt == A.Float32:
                v = v.astype(np.float32)
            view[mdt] = (v[alive], ok[alive])
        views.append(view)
    return AF.restate(views, q.measure_kind, mdt, dims=None, filters=(), mode=q.reduce_mode)


# ---- the edge dimension table --------------------------------------------------------------------------------------
FLAG, I8, I16, F32, TZ8, TZF, U16, F32S, TZB = range(9)
DIM_TYPES = [A.Bool, A.Int8, A.Int16, A.Float32, A.Uint8, A.Float32, A.Uint16, A.Float32, A.Bool]
NB_DIM, ROWS_DIM, NLAST = 8, 40, 25
BASE = 1000                                       # a non-default BaseBatchID
TZ = np.array([-3600, 1800, 0, 7200, -1800, 3600, 19800, -7200, 0, 5400, -600, 1200], np.int16)   # TZ[0] != 0
TZ_SENTINEL = 30000                               # the entry after the table: read only by e <= size
MISS_KEYS = range(400, 480)


def f32_edges():
    return np.array([0.0, -0.0, 2.0 ** -149, -(2.0 ** -149), float(np.uint32(0x007FFFFF).view(np.float32)), np.nan, 1.5,
                     -2.5, 100.0, 3.0e38], np.float32)


@functools.lru_cache(maxsize=None)
def dim_data(seed=5) -> DimData:
    rng = np.random.default_rng(seed)
    shape = (NB_DIM, ROWS_DIM)
    vals = [None] * 9
    vals[FLAG] = rng.integers(0, 2, shape)
    vals[I8] = rng.choice(np.array([-128, -1, -2, 0, 1, 127, 5, -77]), shape)
    vals[I16] = rng.choice(np.array([-32768, -1, -300, 0, 1, 32767, 12, -6]), shape)
    f = f32_edges()
    f[5] = np.uint32(0x7FC00000).view(np.float32)
    vals[F32] = rng.choice(f, shape)
    vals[F32][0, :4] = np.array([0xFFC00001, 0x80000000, 0x00000001, 0x7FC00000], np.uint32).view(np.float32)
    vals[TZ8] = rng.choice(np.array([0, len(TZ) - 1, len(TZ), 255, 3, 6]), shape)
    vals[TZF] = rng.choice(np.array([2.9, 0.0, 11.99, 12.0, 250.0, 5.5], np.float32), shape)
    vals[U16] = rng.integers(0, 10, shape)
    # (the values that are not tiny are positive: every order of summation absorbs the denormals the same way)
    vals[F32S] = rng.choice(np.array([0.0, -0.0, 2.0 ** -149, 2.0 ** -140, 1.0, 3.0, 0.5], np.float32), shape)
    vals[TZB] = rng.integers(0, 2, shape)
    ok = [rng.random(shape) > 0.15 for _ in range(9)]
    for c in (I16, F32, U16):                          # garbage under NULL: values that would change the answer
        vals[c] = np.where(ok[c], vals[c], {I16: -32768, F32: -1.0, U16: 9}[c])
    # batch modes: 0 in batch 2 (column default valid) and 5 (... NULL for the columns without a default), 1 in batch 3
    modes = [[0 if b in (2, 5) else 1 if b == 3 else 2 for b in range(NB_DIM)] for _ in range(9)]
    for c in range(9):
        ok[c][3] = True
    defaults = [(True, 1), (True, -3), (False, 0), (True, -0.0), (True, len(TZ) - 1), (False, 0), (True, 7), (True, 2.0 ** -149),
                (False, 0)]
    # Bool columns: the batches that hold vectors start at bits 1..6 (FLAG) and 7, 0..4 (TZB)
    start_bits = [[0] * NB_DIM for _ in range(9)]
    for c, first in ((FLAG, 1), (TZB, 7)):
        for i, b in enumerate(b for b in range(NB_DIM) if modes[c][b] != 0):
            start_bits[c][b] = (first + i) % 8
    # each mode-0 slice carries a default of its own that the reads must ignore
    slice_defaults = [(True, 0), (True, 99), (True, 42), (True, 123.0), (True, 1), (True, 3.0), (True, 3), (True, 1.0), (True, 1)]
    return DimData(DIM_TYPES, [np.asarray(v) for v in vals], ok, modes, defaults, NLAST, BASE, start_bits, slice_defaults)


def make_table(be, d: DimData, columns_subset=None):
    """The dimension table's column batches in `be` (J.DimensionTable without an index)."""
    batches, keep = [], []
    for b in range(d.nb):
        cols = []
        for c, dt in enumerate(d.types):
            if d.modes[c][b] == 0:
                sv, sd = d.slice_defaults[c] if d.slice_defaults else (False, 0)
                cols.append(columns.constant_column(dt, sd, sv))
                continue
            v = d.vals[c][b].astype(NP[dt])
            buf, vp = columns.make_column(be.space, dt, v, valid=None if d.modes[c][b] == 1 else d.ok[c][b].astype(np.uint8),
                                          start_bit=d.start_bits[c][b])
            keep.append(buf)
            cols.append(vp)
        batches.append(cols)
    defaults = [A.make_default_value(valid, val, dt) for (valid, val), dt in zip(d.defaults, d.types)]
    return batches, defaults, keep


def joined_table(be, d: DimData, pk: dict, kb: int, made=None):
    """J.DimensionTable of `d` whose primary-key index (placed by place_all) maps pk: key -> (batchID, index)."""
    batches, defaults, keep = made or make_table(be, d)
    keys = np.array(sorted(pk), np.int64)
    rids = np.array([pk[k] for k in keys], np.int64).reshape(-1, 2)
    raw, nb = place_all(keys.astype(np.uint32), kb, rids)
    ibuf = be.put(raw)
    return J.DimensionTable(list(d.types), batches, d.nlast, ibuf, J.DEFAULT_SEEDS, kb, 4, nb, defaults, d.base, [keep])


def slots(d: DimData, rng, n):
    """n RecordIDs over the physical slots the table holds (rows past NumRecordsInLastBatch only in earlier batches)."""
    live = np.arange((d.nb - 1) * d.rows + d.nlast)
    live = live[(live < (d.nb - 1) * d.rows) | (live % d.rows < d.nlast)]
    flat = rng.choice(live, n, replace=n > len(live))
    return [(d.base + int(s) // d.rows, int(s) % d.rows) for s in flat]


@functools.lru_cache(maxsize=None)
def key_maps(departures=False):
    """Primary key -> RecordID per index width.  kb 2 also serves Int16 and (masked) Uint32 keys; kb 1 Int8 and Bool."""
    d = dim_data()
    rng = np.random.default_rng(17)
    k2 = list(range(0, 300)) + [65535, 65534, 32768, 65236]
    k1 = [0xFF, 0x80, 0x7F, 0xFE, 1, 5, 0xB3, 0x00]
    k4 = [5, 2 ** 31, 2 ** 32 - 1, 65541, 2 ** 31 + 7, 123456789] + list(range(1, 200))
    m = {2: dict(zip(k2, slots(d, rng, len(k2)))), 1: dict(zip(k1, slots(d, rng, len(k1)))), 4: dict(zip(k4, slots(d, rng, len(k4))))}
    # rows past NumRecordsInLastBatch: in the last batch NULL (the batch holds a value there), in an earlier one a value
    m[2][1], m[2][2] = (BASE + NB_DIM - 1, NLAST), (BASE + NB_DIM - 1, ROWS_DIM - 1)
    m[2][3] = (BASE + 1, NLAST + 3)
    m[2][4], m[2][5] = (BASE + 2, 0), (BASE + 5, 7)                                    # mode-0 batches
    if departures:                                      # batches outside the table: the reference reads out of bounds
        m[2][6], m[2][7], m[2][8] = (BASE - 1, 0), (BASE + NB_DIM, 0), (BASE + NB_DIM + 100, NLAST - 1)
    return m


# ---- fact batches --------------------------------------------------------------------------------------------------
TS, KC, WC, K16, K8, K16S, K32, KB_, FARE = range(9)
FACT_TYPES = [A.Uint32, A.Uint8, A.Uint16, A.Uint16, A.Int8, A.Int16, A.Uint32, A.Bool, A.Float32]
T0, HOURS, NW, W_DROP = 1_700_006_400, 40, 200, 199


def col(i):
    return E.Col(i, FACT_TYPES[i], f"c{i}")


def fcol(t, c, tz=False):
    return E.ForeignCol(t, c, DIM_TYPES[c], f"f{t}_{c}", timezone=tz)


def fact_batch(seed, rows, key_mode=None):
    """Host arrays {column: (values, valid), 'rows': n}.  Keys: ~10 % misses, ~5 % NULL with a present key stored under
    the NULL; quads of every hit / miss / NULL / filtered pattern at the start, the end of the last full tile and in the
    tail of every tile size; key_mode: the K16 key as a mode-0 column ('valid' / 'null')."""
    rng = np.random.default_rng(seed)
    km = key_maps()
    hb = {"rows": rows}
    ts = (T0 + rng.integers(0, HOURS, rows) * 3600 + rng.integers(0, 3600, rows)).astype(np.uint32)
    hb[TS] = (ts, np.ones(rows, bool))
    hb[KC] = (rng.integers(0, 4, rows).astype(np.uint8), np.ones(rows, bool))
    hb[WC] = (rng.integers(0, NW, rows).astype(np.uint16), np.ones(rows, bool))

    def keys(present, misses, dt):
        v = np.where(rng.random(rows) < 0.9, rng.choice(np.asarray(present, np.int64), rows), rng.choice(np.asarray(misses, np.int64), rows))
        ok = rng.random(rows) >= 0.05
        v = np.where(ok, v, present[0])                    # garbage under NULL: a key that is present
        return v.astype(np.int64).astype(NP[dt]) if dt not in (A.Bool,) else (v != 0).astype(np.uint8), ok

    hb[K16] = keys(list(km[2]), list(MISS_KEYS), A.Uint16)
    hb[K8] = keys([-1, -128, 127, -2, 1, 5, -77, 0], [2, 3, -3, 100], A.Int8)
    hb[K16S] = keys([-1, -2, -32768, 0, 7, 299, -300], [-5, 1000, -1000], A.Int16)
    hb[K32] = keys([5, 2 ** 31, 2 ** 32 - 1, 65541, 2 ** 31 + 7, 123456789, 65536 + 7, 3 * 65536 + 250] + list(range(1, 200)),
                   [2 ** 31 + 1, 999999, 2 ** 32 - 2], A.Uint32)
    hb[KB_] = keys([1], [0], A.Bool)
    hb[FARE] = (rng.integers(-50, 200, rows).astype(np.float32) / 4, rng.random(rows) > 0.05)
    # alive-mask quads: each row of a quad is hit / miss / NULL key / filtered (W_DROP); all 256 patterns
    pat = np.arange(256)
    state = np.stack([(pat >> (2 * r)) & 3 for r in range(4)], axis=1).reshape(-1)
    block = len(state)
    starts = {0, rows - block}
    for tr in (3968, 1920, 896):
        tail = max(rows - 128, 0) // tr * tr
        starts |= {tail - block, tail}
    k16, ok16 = hb[K16][0].copy(), hb[K16][1].copy()
    w = hb[WC][0].copy()
    for s in sorted(starts) if rows >= block else ():
        s = max(0, min(s - s % 4, rows - block))
        sl = slice(s, s + block)
        present = rng.permutation(np.array(sorted(km[2]), np.int64))   # hits: every primary key, in random positions
        k16[sl] = np.where(state == 1, MISS_KEYS[0], np.resize(present, block))
        ok16[sl] = state != 2
        w[sl] = np.where(state == 3, W_DROP, np.arange(block) % W_DROP)
    hb[K16], hb[WC] = (k16, ok16), (w, np.ones(rows, bool))
    if key_mode is not None:
        hb[K16] = (np.full(rows, 10, np.uint16), np.full(rows, key_mode == "valid"))
        hb["const_key"] = key_mode
    return hb


def upload_fact(be, hb, ranges=None):
    cols, keep = [], []
    for c, dt in enumerate(FACT_TYPES):
        v, ok = hb[c]
        if c == K16 and "const_key" in hb:
            cols.append(columns.constant_column(dt, int(v[0]), bool(ok[0])))
            continue
        buf, vp = columns.make_column(be.space, dt, v, valid=None if ok.all() else ok.astype(np.uint8))
        cols.append(vp)
        keep.append(buf)
    return Batch(cols, hb["rows"], keep=keep, ranges=ranges)


def fact_ranges(hb, how="exact"):
    zm = {KC: (0, 3), WC: (0, NW - 1), TS: (int(hb[TS][0].min()), int(hb[TS][0].max()))}
    if how == "narrow":
        zm = {c: (a, a + (b - a) // 2) for c, (a, b) in zm.items()}
    return zm


# ---- the joins of a backend ----------------------------------------------------------------------------------------
class Joins:
    """Per index width a J.DimensionTable of the edge table in one backend, and the time-zone table."""

    def __init__(self, be, departures=False):
        d = dim_data()
        made = make_table(be, d)
        km = key_maps(departures)
        self.tables = {kb: joined_table(be, d, km[kb], kb, made) for kb in (1, 2, 4)}
        self.specs = {kb: (d, km[kb], kb) for kb in (1, 2, 4)}
        tz = np.concatenate([TZ, [TZ_SENTINEL]]).astype(np.int16)
        self.tzbuf = be.put(tz)
        self.keep = made

    def join(self, kb, on):
        return Join(self.tables[kb], col(on), self.tzbuf.ptr, len(TZ))


JOIN_ON = {"k16": (2, K16), "k8": (1, K8), "k16s": (2, K16S), "k32_2": (2, K32), "k32_4": (4, K32), "kb": (1, KB_)}


def edge_queries(jn: Joins):
    """name -> AggQuery over the edge table (one join each unless the name says otherwise)."""
    j = {n: jn.join(*v) for n, v in JOIN_ON.items()}
    KD, WD, F = col(KC), col(WC), fcol
    not_dropped = E.ne(WD, E.Lit(W_DROP))
    qs = {
        "i8_dim": AggQuery([not_dropped], [KD, F(0, I8)], Measure("count"), joins=[j["k16"]]),
        "f32_dim": AggQuery([], [F(0, F32)], Measure("count"), joins=[j["k16"]]),
        "f32_filter": AggQuery([E.gt(F(0, F32), E.Lit(0.0))], [KD], Measure("sum", col(FARE)), joins=[j["k16"]]),
        "f32_sum": AggQuery([], [KD, F(0, FLAG)], Measure("sum", F(0, F32S)), joins=[j["k16"]]),
        "i16_min": AggQuery([E.lt(F(0, I16), E.Lit(-1))], [KD], Measure("min", F(0, I16)), joins=[j["k16"]]),
        "i16_sum_hash": AggQuery([], [F(0, U16)], Measure("sum", F(0, I16)), reduce_mode=A.ARES_REDUCE_HASH, joins=[j["k16"]]),
        "bool_dim": AggQuery([], [F(0, FLAG), F(0, U16)], Measure("count"), joins=[j["k16"]]),
        "unmatched": AggQuery([E.Unary(A.IsNull, F(0, U16))], [KD], Measure("count"), joins=[j["k16"]]),
        "tz_u8": AggQuery([], [KD], Measure("sum", F(0, TZ8, True)), joins=[j["k16"]]),
        "tz_f32": AggQuery([], [KD], Measure("sum", F(0, TZF, True)), joins=[j["k16"]]),
        "tz_bool": AggQuery([], [F(0, TZB, True), KD], Measure("count"), joins=[j["k16"]]),
        "key_i8": AggQuery([], [F(0, U16), F(0, I8)], Measure("count"), joins=[j["k8"]]),
        "key_i16": AggQuery([], [F(0, U16)], Measure("sum", F(0, I16)), joins=[j["k16s"]]),
        "key_u32_masked": AggQuery([], [F(0, U16), KD], Measure("count"), joins=[j["k32_2"]]),
        "key_u32": AggQuery([], [F(0, U16)], Measure("sum", F(0, F32S)), joins=[j["k32_4"]]),
        "key_bool": AggQuery([], [F(0, U16), KD], Measure("count"), joins=[j["kb"]]),
        # two tables joined on different columns: each gather probes with its own key
        "two_tables": AggQuery([], [F(0, U16), F(1, I8)], Measure("count"), joins=[j["k16"], j["k8"]]),
    }
    return qs


DEPARTURE_QUERIES = {"tz_i8_negative", "outside_batches"}


def departure_queries(jn: Joins):
    j = jn.join(2, K16)
    return {
        "tz_i8_negative": AggQuery([], [col(KC)], Measure("sum", fcol(0, I8, True)), joins=[j]),
        "outside_batches": AggQuery([], [fcol(0, U16), fcol(0, I8)], Measure("count"), joins=[j]),
    }


def cpu_batches():
    return [fact_batch(71, 3001), fact_batch(72, 1203), fact_batch(73, 64, "valid"), fact_batch(74, 64, "null")]


def legacy(be, q, hbs, upload=upload_fact):
    ex = LegacyBatchExecutor(be.lib, be.space, q)
    for hb in hbs:
        ex.process_batch(upload(be, hb))
    return ex.result()


def expected(q, hbs, jn: Joins):
    dims = [jn.specs[{id(t): kb for kb, t in jn.tables.items()}[id(j.table)]] for j in q.joins]
    tzs = [TZ for _ in q.joins]
    return restate_query(q, hbs, dims, tzs)


def assert_query(got, q, exp, ctx):
    AF.assert_matches(got, exp, q.measure_kind, _measure_dt(q), q.reduce_mode, ctx=ctx)


def _measure_dt(q):
    if q.measure_kind == "count":
        return None
    return q.measure.data_type


# ---- CPU: the restatement against the oracle and the reference -----------------------------------------------------
EDGE_NAMES = ["i8_dim", "f32_dim", "f32_filter", "f32_sum", "i16_min", "i16_sum_hash", "bool_dim", "unmatched", "tz_u8",
              "tz_f32", "tz_bool", "key_i8", "key_i16", "key_u32_masked", "key_u32", "key_bool", "two_tables"]


def test_restatement_rules():
    """The rules, each on one value."""
    d = dim_data()
    km = key_maps()
    # key bytes: Int8 -1 is the byte 0xFF, Uint32 65541 joined to a 2-byte key is 5, a Bool is 1
    assert restate_lookup({0xFF: (7, 1)}, 1, np.array([-1], np.int8), [True], A.Int8)[0].tolist() == [7]
    assert restate_lookup({5: (7, 2)}, 2, np.array([65541], np.uint32), [True], A.Uint32)[1].tolist() == [2]
    assert restate_lookup({0xFFFFFFFF: (7, 3)}, 4, np.array([-1], np.int8), [True], A.Int8)[1].tolist() == [3]
    assert restate_lookup({1: (7, 4)}, 1, np.array([1], np.uint8), [True], A.Bool)[1].tolist() == [4]
    assert restate_lookup({5: (7, 2)}, 2, np.array([5], np.uint16), [False], A.Uint16)[0].tolist() == [0]   # NULL key
    # bounds: the last batch's rows past NumRecordsInLastBatch are NULL, an earlier batch's are values
    bid = np.array([km[2][k][0] for k in (1, 2, 3)])
    idx = np.array([km[2][k][1] for k in (1, 2, 3)])
    _, ok = restate_foreign(d, U16, bid, idx)
    assert ok.tolist() == [False, False, bool(d.ok[U16][1, NLAST + 3])]
    # Bool columns: the batches with vectors start at every bit 0..7
    assert {d.start_bits[c][b] for c in (FLAG, TZB) for b in range(NB_DIM) if d.modes[c][b] != 0} == set(range(8))
    # mode 0: the column default, valid or NULL
    v, ok = restate_foreign(d, I8, np.array([BASE + 2, BASE + 5]), np.array([0, 7]))
    assert v.tolist() == [-3, -3] and ok.tolist() == [True, True]
    _, ok = restate_foreign(d, I16, np.array([BASE + 2]), np.array([0]))
    assert ok.tolist() == [False]
    # time zones: table[e] below the size, else 0; Float32 truncates; Bool is off != 0; validity kept
    e = np.array([0, len(TZ) - 1, len(TZ), 255])
    d8 = DimData([A.Uint8], [e.reshape(1, -1)], [np.array([[True, True, True, False]])], [[2]], [(False, 0)], 4, BASE)
    v, ok = restate_foreign(d8, 0, np.full(4, BASE), np.arange(4), TZ)
    assert v.tolist() == [int(TZ[0]) & 0xFFFFFFFF, int(TZ[-1]) & 0xFFFFFFFF, 0, 0] and ok.tolist() == [True, True, True, False]
    df = DimData([A.Float32], [np.array([[2.9]], np.float32)], [np.array([[True]])], [[2]], [(False, 0)], 1, BASE)
    assert restate_foreign(df, 0, np.array([BASE]), np.array([0]), TZ)[0].tolist() == [float(TZ[2])]
    db = DimData([A.Bool], [np.array([[0, 1]])], [np.array([[True, True]])], [[2]], [(False, 0)], 2, BASE)
    assert restate_foreign(db, 0, np.array([BASE, BASE]), np.array([0, 1]), TZ)[0].tolist() == [1, 1]   # TZ[0], TZ[1] != 0
    # a mode-0 batch of an enum column yields its default unmapped
    assert restate_foreign(d, TZ8, np.array([BASE + 2]), np.array([3]), TZ)[0].tolist() == [len(TZ) - 1]
    # departures: outside the batches is NULL, a negative enum is offset 0
    assert restate_foreign(d, U16, np.array([BASE - 1, BASE + NB_DIM]), np.array([0, 0]))[1].tolist() == [False, False]
    di = DimData([A.Int8], [np.array([[-1]])], [np.array([[True]])], [[2]], [(False, 0)], 1, BASE)
    assert restate_foreign(di, 0, np.array([BASE]), np.array([0]), TZ)[0].tolist() == [0]


@pytest.mark.parametrize("name", EDGE_NAMES)
def test_restatement_matches_oracle_and_reference(name):
    hbs = cpu_batches()
    orc = H.get_backend("oracle")
    jn = Joins(orc)
    q = edge_queries(jn)[name]
    got = legacy(orc, q, hbs)
    assert got.groups > 0
    assert_query(got, q, expected(q, hbs, jn), f"oracle {name}")

    def reference():
        ref = H.get_backend("ref")
        rj = Joins(ref)
        return legacy(ref, edge_queries(rj)[name], hbs)
    H.assert_matches_reference(f"join_edges/{name}", H.digest(canonical(got)), lambda: H.digest(canonical(reference())))


def canonical(r):
    """A result with the value bytes of its NULL dimensions zeroed and the groups that merges folded together, sorted by
    row.  The reference reads a missed or out-of-bounds RecordID into an uninitialised variable (RecordIDJoinIterator::
    dereference), so the bytes under such a NULL dimension are unspecified there; the engine and the oracle write 0.
    What the reference does specify — every group's identity apart from those bytes and every measure — is compared."""
    rows = r.packed_rows().copy()
    widths = r.query.layout_widths
    off = 0
    for p, w in enumerate(widths):
        rows[rows[:, sum(widths) + p] == 0, off:off + w] = 0
        off += w
    kind = r.query.measure_kind
    out = {}
    for row, m in zip((x.tobytes() for x in rows), r.measures.tolist()):
        if row not in out:
            out[row] = m
        elif kind in ("count", "sum"):
            out[row] = out[row] + m
        else:
            out[row] = (min if kind == "min" else max)(out[row], m)
    if kind in ("count", "sum") and r.measures.dtype.kind in "ui":
        out = {k: v % 2 ** (8 * r.measures.dtype.itemsize) for k, v in out.items()}
    return sorted((k, repr(v)) for k, v in out.items())


@pytest.mark.parametrize("name", sorted(DEPARTURE_QUERIES))
def test_departures_restatement_matches_oracle(name):
    """A batchID outside the table and a negative enum: the reference reads out of bounds, so the reference is not asked;
    the restatement and the oracle give NULL and offset 0."""
    hbs = cpu_batches()
    orc = H.get_backend("oracle")
    jn = Joins(orc, departures=True)
    q = departure_queries(jn)[name]
    got = legacy(orc, q, hbs)
    assert got.groups > 0
    assert_query(got, q, expected(q, hbs, jn), f"oracle {name}")


# ---- per-node HashLookup on indexes placed by hand ------------------------------------------------------------------
def _find(pred, start=0, dt_kb=4, limit=2_000_000):
    for v in range(start, start + limit):
        if pred(key_bytes_of(v, dt_kb), v):
            return v
    raise AssertionError("no such key")


def probe_cases():
    """name -> (IndexWriter, key column type, probe values, probe validity, expected (batchID, index) per probe, numHashes
    overrides {numHashes: expected}).  RecordIDs use batch ids that are never 0."""
    cases = {}
    # every cell of one bucket (a bucket count that is not a power of two), every stash cell, absent keys
    w = IndexWriter(4, 7)
    b0 = 3
    in_b0 = []
    v = 1000
    while len(in_b0) < 8:
        if w.bucket_of(key_bytes_of(v, 4), 0) == b0:
            in_b0.append(v)
        v += 1
    exp = {}
    for j, k in enumerate(in_b0):
        w.put_hashed(key_bytes_of(k, 4), (BASE, j), 0, j)
        exp[k] = (BASE, j)
    stash = [77, 2 ** 31 + 5, 2 ** 32 - 1, 65541]
    for j, k in enumerate(stash):
        w.put_stash(key_bytes_of(k, 4), (BASE, 10 + j), j, sig=j * 60 + 1)
        exp[k] = (BASE, 10 + j)
    probes = in_b0 + stash + [5, 6, 2 ** 31, 12345]
    cases["cells_and_stash"] = (w, A.Uint32, probes, [True] * len(probes), [exp.get(p, (0, 0)) for p in probes], {})
    # numHashes 1..4: a key only in the bucket of its last hash function (found with numHashes = t + 1, not with t)
    for t in range(4):
        w = IndexWriter(4, 11, num_hashes=t + 1)
        k = _find(lambda kb, v: len({w.bucket_of(kb, i) for i in range(t + 1)}) == t + 1, 500 + 100 * t)
        w.put_hashed(key_bytes_of(k, 4), (BASE, 20 + t), t, 5)
        cases[f"num_hashes_{t + 1}"] = (w, A.Uint32, [k, k + 1], [True, True], [(BASE, 20 + t), (0, 0)],
                                       {t: [(0, 0), (0, 0)]} if t else {})
    # a key whose hash has a top byte of 0: its signature is clamped to 1
    w = IndexWriter(2, 5)
    k = _find(lambda kb, v: w.hash(kb, 0) >> 24 == 0, 0, 2)
    w.put_hashed(key_bytes_of(k, 2), (BASE, 10), 0, 2)
    assert w.signature(key_bytes_of(k, 2), 0) == 1
    cases["signature_clamp"] = (w, A.Uint16, [k], [True], [(BASE, 10)], {})
    # two keys of one bucket with one signature: the key compare decides
    w = IndexWriter(2, 3)
    first = key_bytes_of(40, 2)
    k2 = _find(lambda kb, v: v != 40 and w.bucket_of(kb, 0) == w.bucket_of(first, 0) and w.signature(kb, 0) == w.signature(first, 0), 41, 2, 65000)
    w.put_hashed(first, (BASE, 11), 0, 0)
    w.put_hashed(key_bytes_of(k2, 2), (BASE, 12), 0, 1)
    cases["same_signature"] = (w, A.Uint16, [k2, 40], [True, True], [(BASE, 12), (BASE, 11)], {})
    # an empty stash cell (signature 0) holding the bytes of a probed absent key, a RecordID, and a NULL probe of a key
    w = IndexWriter(1, 2)
    w.put_stash(key_bytes_of(0xAB, 1), (BASE, 13), 0, sig=0)
    w.put_stash(key_bytes_of(0xFF, 1), (BASE, 14), 1, sig=9)
    cases["empty_stash_cell"] = (w, A.Int8, [np.int8(-85), -1, -1], [True, True, False], [(0, 0), (BASE, 14), (0, 0)], {})
    # key masking: a Uint32 column against 1- and 2-byte keys, Int8 / Int16 negatives, Bool
    w = IndexWriter(2, 3)
    w.put_hashed(key_bytes_of(5, 2), (BASE, 15), 1, 7)
    w.put_hashed(key_bytes_of(0xFFFE, 2), (BASE, 16), 0, 0)
    cases["mask_u32_to_2"] = (w, A.Uint32, [65541, 5, 2 ** 32 - 2, 0xFFFE, 6], [True] * 5,
                              [(BASE, 15), (BASE, 15), (BASE, 16), (BASE, 16), (0, 0)], {})
    cases["i16_negative"] = (w, A.Int16, [-2, 5, -1], [True] * 3, [(BASE, 16), (BASE, 15), (0, 0)], {})
    w = IndexWriter(1, 2)
    w.put_hashed(key_bytes_of(1, 1), (BASE, 17), 2, 3)
    w.put_hashed(key_bytes_of(0x80, 1), (BASE, 18), 3, 4)
    cases["bool_key"] = (w, A.Bool, [1, 0], [True, True], [(BASE, 17), (0, 0)], {})
    cases["i8_negative"] = (w, A.Int8, [-128, 1, -1], [True] * 3, [(BASE, 18), (BASE, 17), (0, 0)], {})
    w = IndexWriter(4, 5)
    w.put_hashed(key_bytes_of(-1, 4), (BASE, 19), 1, 1)
    cases["i8_against_4_bytes"] = (w, A.Int8, [-1, 127], [True, True], [(BASE, 19), (0, 0)], {})
    return cases


PROBES = list(probe_cases())


def test_probe_cases_point_into_the_probe_table():
    """Every RecordID a hand-placed index holds is a row of the one-batch probe table (batch BASE, index below
    PAYLOAD_ROWS), so the fused gather reads a value for every key it finds and NULL for every miss; every case has a key
    to find."""
    for name, (w, dt, vals, valid, exp, overrides) in probe_cases().items():
        hits = [r for r in exp if r != (0, 0)]
        assert hits and all(r[0] == BASE and r[1] < PAYLOAD_ROWS for r in hits), name
WIDE_PROBES = ["int64_key", "uuid_key"]


def wide_probe(name):
    """8- and 16-byte keys (per-node path only)."""
    kb = 8 if name == "int64_key" else 16
    w = IndexWriter(kb, 3)
    keys = [(2 ** 63 - 1, 0), (2 ** 40 + 5, 7)] if kb == 8 else [(1, 2), (2 ** 64 - 1, 5)]
    kbytes = [k[0].to_bytes(8, "little") + (k[1].to_bytes(8, "little") if kb == 16 else b"") for k in keys]
    w.put_hashed(kbytes[0], (BASE, 1), 0, 6)
    w.put_stash(kbytes[1], (BASE, 2), 3, sig=4)
    if kb == 8:
        vals = np.array([keys[0][0], keys[1][0], 12345], np.uint64).view(np.int64)
    else:
        vals = np.array([[1, 2], [2 ** 64 - 1, 5], [2, 1]], np.uint64).reshape(-1)
    return w, (A.Int64 if kb == 8 else A.UUID), vals, [True, True, True], [(BASE, 1), (BASE, 2), (0, 0)]


def _hash_lookup(be, h, dt, values, valid):
    n = len(valid)
    vals = np.asarray(values) if dt in (A.Int64, A.UUID) else np.asarray(values).astype(np.int64).astype(NP[dt])
    buf, vp = columns.make_column(be.space, dt, vals, valid=np.asarray(valid, np.uint8))
    if dt == A.UUID:
        vp.Length = n
    idx = be.put(np.arange(n, dtype=np.uint32))
    out = be.zeros(8 * n)
    be.lib.HashLookup(A.vp_input(vp), out.ptr, idx.ptr, n, None, 0, h, be.space.stream, be.device)
    got = out.get(np.uint8, 8 * n).reshape(n, 8)
    return list(zip(got[:, :4].copy().view(np.int32).reshape(-1).tolist(), got[:, 4:].copy().view(np.uint32).reshape(-1).tolist()))


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("name", PROBES + WIDE_PROBES)
def test_hash_lookup_hand_placed(name, backend):
    be = H.get_backend(backend)
    if name in WIDE_PROBES:
        w, dt, vals, valid, exp = wide_probe(name)
        overrides = {}
    else:
        w, dt, vals, valid, exp, overrides = probe_cases()[name]
    h, keep = w.index(be)
    assert _hash_lookup(be, h, dt, vals, valid) == [tuple(e) for e in exp], name
    for nh, exp2 in overrides.items():
        h2, keep2 = w.index(be, num_hashes=nh)
        assert _hash_lookup(be, h2, dt, vals, valid) == [tuple(e) for e in exp2], f"{name} numHashes {nh}"


# ---- the fused gather on the same indexes ---------------------------------------------------------------------------
PAYLOAD_ROWS = 40


def probe_table(be, w: IndexWriter, num_hashes=None):
    """A one-batch dimension table (payload of row r = 7r + 3, NumRecordsInLastBatch = 40) behind index `w`."""
    payload = (np.arange(PAYLOAD_ROWS) * 7 + 3).astype(np.uint32)
    buf, vp = columns.make_column(be.space, A.Uint32, payload)
    ibuf = be.put(w.raw)
    return J.DimensionTable([A.Uint32], [[vp]], PAYLOAD_ROWS, ibuf, w.seeds, w.kb, w.nh if num_hashes is None else num_hashes, w.nb,
                            [A.make_default_value(False, 0, A.Uint32)], BASE, [buf])


def probe_query(table, dt):
    """Group by (row number, payload): one group per probe row."""
    pay = E.ForeignCol(0, 0, A.Uint32, "payload")
    return AggQuery([], [E.Col(1, A.Uint32, "row"), pay], Measure("count"), joins=[Join(table, E.Col(0, dt, "key"))])


def probe_expected(exp, rows):
    """The payload every probe row must read: 7 * index + 3 for a hit of batch BASE, else NULL."""
    out = []
    for r, (bid, idx) in enumerate(exp):
        hit = bid == BASE and idx < PAYLOAD_ROWS
        out.append((r, 7 * idx + 3 if hit else None))
    return out


def _fused_probe(eng, w, dt, vals, valid, num_hashes=None, tile=False):
    """Runs probe_query with the probes repeated to a full tile and a tail (`tile`)."""
    table = probe_table(eng, w, num_hashes)
    q = probe_query(table, dt)
    reps = 1000 if tile else 1
    n = len(valid) * reps
    v = np.tile(np.asarray(vals).astype(np.int64).astype(NP[dt]), reps)
    ok = np.tile(np.asarray(valid, np.uint8), reps)
    kb_, kvp = columns.make_column(eng.space, dt, v, valid=ok)
    rb, rvp = columns.make_column(eng.space, A.Uint32, (np.arange(n) % len(valid)).astype(np.uint32))
    ex = FusedBatchExecutor(eng.lib, eng.space, q)
    ex.process_batch(Batch([kvp, rvp], n, keep=[kb_, rb]))
    r = ex.result()
    ex.close()
    rows, pay = r.decoded_dims()
    return sorted(zip(rows, pay)), r


@pytest.mark.gpu
@pytest.mark.parametrize("name", PROBES)
def test_fused_gather_hand_placed(name):
    eng = H.get_backend("b200")
    w, dt, vals, valid, exp, overrides = probe_cases()[name]
    assert any(p is not None for _, p in probe_expected(exp, len(valid))), f"{name}: no probe that the gather must find"
    for tile in (False, True):
        got, _ = _fused_probe(eng, w, dt, vals, valid, tile=tile)
        assert got == probe_expected(exp, len(valid)), f"{name} tile={tile}"
    for nh, exp2 in overrides.items():
        got, _ = _fused_probe(eng, w, dt, vals, valid, num_hashes=nh)
        assert got == probe_expected(exp2, len(valid)), f"{name} numHashes {nh}"


def golden_index_with_batch_ids():
    """The reference's own CheckLookup index (keys 0..17 -> RecordID {0, i}) with batch id BASE written into its occupied
    cells, so that the fused gather can read what it finds (batch id 0 means 'no record')."""
    g = np.load(H.ROOT / "tests" / "golden" / "hash_lookup.npz")
    kb, nh, nb = g["lookup_params"].tolist()
    w = IndexWriter(kb, nb, nh, tuple(int(s) for s in g["lookup_seeds"].tolist()))
    w.raw = g["lookup_buckets"].copy()
    cell = 8 + kb + 1
    for b in range(nb + 1):
        for j in range(8):
            base = b * 8 * cell
            if w.raw[base + 64 + j]:
                w.raw[base + 8 * j: base + 8 * j + 4] = np.frombuffer(np.array([BASE], "<i4").tobytes(), np.uint8)
    return w


@pytest.mark.gpu
def test_fused_gather_golden_index():
    eng = H.get_backend("b200")
    w = golden_index_with_batch_ids()
    probes = list(range(18)) + [18, 100, 2 ** 31]
    exp = [(BASE, i) if i < 18 else (0, 0) for i in probes]
    h, keep = w.index(eng)
    assert _hash_lookup(eng, h, A.Uint32, probes, [True] * len(probes)) == exp
    got, _ = _fused_probe(eng, w, A.Uint32, probes, [True] * len(probes))
    assert got == probe_expected(exp, len(probes))


@pytest.mark.parametrize("backend", ["oracle", pytest.param("ref", id="ref")])
def test_golden_index_with_batch_ids_on_checkers(backend):
    be = H.get_backend(backend)
    w = golden_index_with_batch_ids()
    probes = list(range(18)) + [18, 100, 2 ** 31]
    h, keep = w.index(be)
    assert _hash_lookup(be, h, A.Uint32, probes, [True] * len(probes)) == [(BASE, i) if i < 18 else (0, 0) for i in probes]


@pytest.mark.gpu
@pytest.mark.parametrize("name", WIDE_PROBES)
def test_fused_path_refuses_wide_keys(name):
    """An 8- or 16-byte key column is refused when the plan compiles; a 4-byte column against an index of 8- or 16-byte
    keys when the join is uploaded."""
    eng = H.get_backend("b200")
    w, dt, vals, valid, exp = wide_probe(name)
    table = probe_table(eng, w)
    rb, rvp = columns.make_column(eng.space, A.Uint32, np.arange(len(valid), dtype=np.uint32))
    buf, vp = columns.make_column(eng.space, dt, vals, valid=np.asarray(valid, np.uint8))
    if dt == A.UUID:
        vp.Length = len(valid)
    for key_type, key_vp, message in ((dt, vp, FUSED_KEY_COLUMN_ERROR), (A.Uint32, rvp, FUSED_KEY_ERROR)):
        ex = FusedBatchExecutor(eng.lib, eng.space, probe_query(table, key_type))
        with pytest.raises(A.AresError, match=message):
            ex.process_batch(Batch([key_vp, rvp], len(valid), keep=[buf, rb]))
        ex.close()


def nine_batch_table(be):
    """A dimension table of 9 one-row batches: more than a join may read."""
    vals = np.arange(9, dtype=np.uint16)
    return J.DimensionTable.build(be.space, [A.Uint16], [vals], None, pk_column=0, rows_per_batch=1)


@pytest.mark.gpu
def test_nine_batches_refused_on_both_engine_paths():
    eng = H.get_backend("b200")
    t = nine_batch_table(eng)
    q = AggQuery([], [E.ForeignCol(0, 0, A.Uint16, "pk")], Measure("count"), joins=[Join(t, E.Col(0, A.Uint16, "key"))])
    buf, vp = columns.make_column(eng.space, A.Uint16, np.arange(9, dtype=np.uint16))
    batch = Batch([vp], 9, keep=[buf])
    ex = FusedBatchExecutor(eng.lib, eng.space, q)
    with pytest.raises(A.AresError, match=BATCHES_ERROR):
        ex.process_batch(batch)
    ex.close()
    with pytest.raises(A.AresError, match=BATCHES_ERROR):
        LegacyBatchExecutor(eng.lib, eng.space, q).process_batch(batch)


# ---- GPU: the edge queries on the fused path -------------------------------------------------------------------------
def fused(eng, q, hbs, ranges=None, expected_groups=0, upload=upload_fact):
    ex = FusedBatchExecutor(eng.lib, eng.space, q, expected_groups)
    batches = [upload(eng, hb, ranges(hb) if ranges else None) for hb in hbs]
    for b in batches:
        ex.process_batch(b)
    r = ex.result()
    ex.close()
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DEPARTURE_QUERIES) + ["two_tables", "tz_u8"] + [n for n in EDGE_NAMES if n not in ("two_tables", "tz_u8")])
def test_edge_queries_on_gpu(name):
    """Each edge query on the per-node engine sequence and the fused kernel (full tiles and a tail) against the
    restatement."""
    _edge_query_on_gpu(name, [fact_batch(81, 20011), fact_batch(82, 1203)])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["outside_batches", "i8_dim", "tz_u8"])
def test_mode0_keys_on_gpu(name):
    """Batches whose join key is a mode-0 column, valid and NULL: the gather probes the batch's constant key (a kernel of
    its own per validity, so a few queries only)."""
    _edge_query_on_gpu(name, [fact_batch(83, 64, "valid"), fact_batch(84, 64, "null"), fact_batch(85, 4000, "valid")])


def _edge_query_on_gpu(name, hbs):
    eng = H.get_backend("b200")
    dep = name in DEPARTURE_QUERIES
    jn = Joins(eng, departures=dep)
    q = (departure_queries(jn) if dep else edge_queries(jn))[name]
    exp = expected(q, hbs, jn)
    assert_query(fused(eng, q, hbs), q, exp, f"fused {name}")
    assert_query(legacy(eng, q, hbs), q, exp, f"per-node {name}")


# ---- every fused form that carries the gather ------------------------------------------------------------------------
PARTITIONS = (-300.0, -2.0, 0.0, 12.0)


def partitions_of(expr, be=None):
    """A manual-partition bucketizer over `expr`; its bounds in `be` (or a fake address for a dry run)."""
    if be is None:
        return E.Bucket(expr, ("partitions",) + PARTITIONS, PARTITIONS, 0x7D0000000000)
    keep = be.space.put(np.array(PARTITIONS, np.float64))
    return E.Bucket(expr, ("partitions",) + PARTITIONS, PARTITIONS, keep.ptr, keep)


def form_cases():
    """name -> (query builder(joins, be), batches, zone map, expected groups, macros the kernel must generate, direct-
    indexed launches per batch)."""
    F, KD, WD = fcol, col(KC), col(WC)
    hour = E.floor(col(TS), E.Lit(3600))
    nd = E.ne(WD, E.Lit(W_DROP))
    hashed = {"JIT_DENSE": 0, "JIT_BYPASS": 0}
    cta = {"JIT_DENSE": 1}
    return {
        "hash/foreign_dim": (lambda j, be: AggQuery([nd], [KD, F(0, U16)], Measure("sum", col(FARE)), joins=[j]), "tiles", None, 0, hashed, 0),
        "hash/foreign_dim/hash_mode": (lambda j, be: AggQuery([nd], [KD, F(0, U16)], Measure("count"), reduce_mode=A.ARES_REDUCE_HASH,
                                                           joins=[j]), "tiles", None, 0, hashed, 0),
        "bypass": (lambda j, be: AggQuery([nd], [WD, F(0, I16), KD], Measure("count"), joins=[j]), "tiles", None, 100_000,
                   {"JIT_DENSE": 0, "JIT_BYPASS": 1}, 0),
        "tail": (lambda j, be: AggQuery([nd], [KD, F(0, I8)], Measure("sum", F(0, F32S)), joins=[j]), "tail", "exact", 0, hashed, 0),
        "direct/main_dims": (lambda j, be: AggQuery([nd, E.gt(F(0, I16), E.Lit(-32768))], [KD, WD], Measure("sum", F(0, F32S)), joins=[j]),
                             "tiles", "exact", 0, cta, 1),
        "direct/foreign_bool": (lambda j, be: AggQuery([nd], [KD, F(0, FLAG)], Measure("count"), joins=[j]), "tiles", "exact", 0, cta, 1),
        "direct/foreign_partitions": (lambda j, be: AggQuery([nd], [KD, partitions_of(F(0, I16), be)], Measure("count"), joins=[j]),
                                      "tiles", "exact", 0, cta, 1),
        "global": (lambda j, be: AggQuery([nd], [WD, hour], Measure("max", F(0, I16)), joins=[j]), "tiles", "exact", 0,
                   {"JIT_DENSE": 2}, 1),
        "cold/narrow_zone_map": (lambda j, be: AggQuery([nd, E.gt(F(0, I16), E.Lit(-32768))], [KD, WD], Measure("sum", F(0, F32S)),
                                                        joins=[j]), "tiles", "narrow", 0, cta, 1),
    }


FORMS = list(form_cases())


def form_batches(kind):
    if kind == "tail":
        return [fact_batch(91, 3001), fact_batch(92, 1999)]
    return [fact_batch(93, 200_003), fact_batch(94, 61_447)]


def _dry_run_of(q, hb, ranges, expected_groups):
    fn = A.load_engine().alg.AresJitDryRun
    fn.argtypes = [A.AggSpec, C.POINTER(A.BatchPlan), C.POINTER(C.c_char_p)]
    fn.restype = A.CGoCallResHandle
    from aresdb_b200.executor import _BatchPlans
    plans = _BatchPlans(q, lambda tf, co: q.plan_instructions(time_filters=tf, cutoff=co))
    cols = [columns.slice_of(0x7F0000000000 + i * (1 << 30), dt, hb["rows"], 0, 64 * 200 * 4, 2, 0) for i, dt in enumerate(FACT_TYPES)]
    p = plans.plan_for(Batch(cols, hb["rows"], ranges=ranges), True, 0)
    src = C.c_char_p()
    h = fn(q.agg_spec(expected_groups), C.byref(p), C.byref(src))
    if h.pStrErr:
        raise A.AresError(C.string_at(h.pStrErr).decode())
    return (src.value or b"").decode()


def test_form_of_every_fused_case(monkeypatch):
    """Each GPU case generates the kernel of the form it targets, with the gather in it."""
    monkeypatch.setenv("ARESDB_B200_JIT_GENERATE_ONLY", "1")
    orc = H.get_backend("oracle")
    jn = Joins(orc)
    for name, (make, kind, how, eg, macros, _) in form_cases().items():
        hb = form_batches(kind)[0]
        src = _dry_run_of(make(jn.join(2, K16), None), hb, fact_ranges(hb, how) if how else None, eg)
        for m, want in macros.items():
            assert AF._macro(src, m) == want, f"{name}: {m}"
        assert "cuckooLookup(P.join->tables[0]" in src and "foreignLoad(P.join->cols[0]" in src, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", FORMS)
def test_fused_forms_on_gpu(name):
    eng = H.get_backend("b200")
    make, kind, how, eg, macros, dense = form_cases()[name]
    jn = Joins(eng)
    q = make(jn.join(2, K16), eng)
    hbs = form_batches(kind)
    exp = expected(q, hbs, jn)
    before = T.dense_launches(eng)
    got = fused(eng, q, hbs, (lambda hb: fact_ranges(hb, how)) if how else None, eg)
    assert T.dense_launches(eng) - before == dense * len(hbs), f"{name}: direct-indexed launches"
    assert_query(got, q, exp, name)


# the fused path refuses a countdistincthll measure over a foreign column: the measure of an HLL query is a column
def test_hll_of_a_foreign_column_is_refused():
    with pytest.raises(ValueError, match="expect 1 argument to be a column"):
        AggQuery([], [col(KC)], Measure("countdistincthll", fcol(0, U16)), joins=[])


@pytest.mark.gpu
@pytest.mark.parametrize("expected_groups", [0, 100_000], ids=["dense", "entries"])
def test_hll_grouped_by_a_foreign_dimension_on_gpu(expected_groups):
    """countdistincthll(w) by a foreign dimension: the registers of every group equal the oracle's call sequence."""
    eng, orc = H.get_backend("b200"), H.get_backend("oracle")
    hbs = form_batches("tiles")

    def query(be):
        jn = Joins(be)
        return AggQuery([], [fcol(0, U16)], Measure("countdistincthll", col(WC)), joins=[jn.join(2, K16)]), jn

    q, keep = query(orc)
    ex = LegacyBatchExecutor(orc.lib, orc.space, q)
    for i, hb in enumerate(hbs):
        ex.process_batch(upload_fact(orc, hb), is_last=i == len(hbs) - 1)
    exp = ex.hll.dense_registers()
    q2, keep2 = query(eng)
    fx = FusedBatchExecutor(eng.lib, eng.space, q2, expected_groups)
    for hb in hbs:
        fx.process_batch(upload_fact(eng, hb))
    got = fx.hll_result().dense_registers()
    fx.close()
    assert set(got) == set(exp) and all(np.array_equal(got[k], exp[k]) for k in exp)


@pytest.mark.gpu
def test_shared_scan_with_foreign_member_filters_and_dimensions_on_gpu():
    """One pass: member filters that read foreign columns, and a foreign member dimension."""
    eng = H.get_backend("b200")
    jn = Joins(eng)
    j = jn.join(2, K16)
    nd = E.ne(col(WC), E.Lit(W_DROP))
    qs = [AggQuery([nd, E.gt(fcol(0, I16), E.Lit(0))], [col(KC)], Measure("count"), joins=[j]),
          AggQuery([nd, E.lt(fcol(0, F32), E.Lit(1.0))], [col(KC)], Measure("sum", fcol(0, F32S)), joins=[j]),
          AggQuery([nd], [col(KC), fcol(0, U16)], Measure("count"), joins=[j])]
    hbs = form_batches("tiles")
    req = FusedRequestExecutor(eng.lib, eng.space, qs)
    assert req.passes == [[0, 1, 2]]
    for hb in hbs:
        k0 = req.calls
        req.process_batch(upload_fact(eng, hb, fact_ranges(hb)))
        assert req.calls - k0 == 1, "one ExecuteBatchPlanMulti call per batch"
    for i, (got, q) in enumerate(zip(req.results(), qs)):
        assert_query(got, q, expected(q, hbs, jn), f"member {i}")
    req.close()


@pytest.mark.gpu
def test_four_tables_and_eight_foreign_columns_on_gpu():
    """The plan limits: four joined tables (on four key columns) and eight foreign columns in one plan."""
    eng = H.get_backend("b200")
    jn = Joins(eng)
    joins = [jn.join(2, K16), jn.join(1, K8), jn.join(2, K16S), jn.join(4, K32)]
    F = fcol
    q = AggQuery([E.ne(F(1, I8), E.Lit(0)), E.Unary(A.IsNotNull, F(2, FLAG)), E.lt(F(3, F32), E.Lit(50.0))],
                 [F(0, U16), F(1, I8), F(2, FLAG), F(3, U16), F(0, TZ8, True), F(2, TZB, True)],
                 Measure("sum", F(3, F32S)), joins=joins)
    assert len(q.plan_instructions()) and len(q.foreign_columns) == 8
    hbs = form_batches("tail")
    assert_query(fused(eng, q, hbs), q, expected(q, hbs, jn), "four tables")


def test_fifth_table_is_refused():
    orc = H.get_backend("oracle")
    jn = Joins(orc)
    joins = [jn.join(2, K16)] * 5
    q = AggQuery([], [fcol(4, U16)], Measure("count"), joins=joins)
    q.plan_instructions()
    from aresdb_b200.executor import _BatchPlans
    with pytest.raises(ValueError, match="too many joined tables / foreign columns for one plan"):
        _BatchPlans(q, lambda tf, co: q.plan_instructions(time_filters=tf, cutoff=co))


def rle_fact(be, hb, seed):
    """An archive batch over hb's index positions: KC sorted and run-length encoded with the base counts; K16 first-class
    RLE (four RLE columns in all: K8, K16S, KB_, K16) or the fifth RLE column, which the engine expands."""
    rng = np.random.default_rng(seed)
    n = hb["rows"]
    lens = rng.integers(1, 6, n)
    base = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    order = np.argsort(hb[KC][0], kind="stable")
    view = {"rows": n, "mult": lens.astype(np.int64)}
    for c in range(len(FACT_TYPES)):
        view[c] = tuple(a[order] for a in hb[c])
    cols, keep = [], []
    for c, dt in enumerate(FACT_TYPES):
        v, ok = view[c]
        counts = base if c in (KC, K16, K8, K16S, KB_, K32) else None
        buf, vp = columns.make_column(be.space, dt, v, valid=None if ok.all() else ok.astype(np.uint8), counts=counts)
        cols.append(vp)
        keep.append(buf)
    return Batch(cols, n, base_counts=be.put(base), start_count=0, keep=keep, ranges={KC: (0, 3)}), view


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["first_class", "expanded"])
def test_rle_archive_batches_on_gpu(key):
    """The join key read from its runs (first-class RLE input) and expanded (the fifth RLE column of the plan)."""
    eng = H.get_backend("b200")
    jn = Joins(eng)
    on = K16 if key == "first_class" else K32
    if key == "first_class":
        q = AggQuery([], [col(KC), fcol(0, U16)], Measure("sum", fcol(0, F32S)), joins=[jn.join(2, on)])
    else:   # four other RLE columns come first
        q = AggQuery([E.ne(col(K8), E.Lit(100)), E.ne(col(K16S), E.Lit(1000)), E.Unary(A.IsNotNull, col(KB_)),
                      E.ne(col(K16), E.Lit(MISS_KEYS[0]))], [col(KC), fcol(0, U16)], Measure("sum", fcol(0, F32S)),
                     joins=[jn.join(2, on)])
    hbs = [fact_batch(95, 30_011), fact_batch(96, 8_003)]
    batches, views = zip(*[rle_fact(eng, hb, 97 + i) for i, hb in enumerate(hbs)])
    ex = FusedBatchExecutor(eng.lib, eng.space, q)
    for b in batches:
        ex.process_batch(b)
    got = ex.result()
    ex.close()
    assert_query(got, q, expected(q, views, jn), f"rle {key}")


# ---- one case at size ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["hash", "direct"])
def test_join_at_size_on_gpu(form):
    """2e5 keys in 8 batches, 5e7 fact rows with Zipf keys and ~10 % misses, against a torch restatement: a dense
    key -> (value, valid) array and index_add."""
    import torch
    eng = H.get_backend("b200")
    nkeys, per = 200_000, 25_000
    rng = np.random.default_rng(101)
    keys = rng.permutation(np.arange(1, 2 ** 22))[:nkeys].astype(np.uint32)
    val = rng.integers(0, 1000, nkeys).astype(np.float32)
    vok = rng.random(nkeys) > 0.05
    grp = rng.integers(0, 16, nkeys).astype(np.uint8)
    batches, keep = [], []
    for b in range(8):
        sl = slice(b * per, (b + 1) * per)
        vb, vvp = columns.make_column(eng.space, A.Float32, val[sl], valid=vok[sl].astype(np.uint8))
        gb, gvp = columns.make_column(eng.space, A.Uint8, grp[sl])
        batches.append([vvp, gvp])
        keep += [vb, gb]
    rids = np.stack([BASE + np.arange(nkeys) // per, np.arange(nkeys) % per], axis=1)
    raw, nb = place_all(keys, 4, rids)
    table = J.DimensionTable([A.Float32, A.Uint8], batches, per, eng.put(raw), J.DEFAULT_SEEDS, 4, 4, nb,
                             [A.make_default_value(False, 0, A.Float32), A.make_default_value(False, 0, A.Uint8)], BASE, keep)
    KEY, K4 = E.Col(0, A.Uint32, "key"), E.Col(1, A.Uint8, "k")
    # hash table: by k and the foreign g; direct-indexed: by k (its zone map), the foreign column only in the measure
    dims = [K4, E.ForeignCol(0, 1, A.Uint8, "g")] if form == "hash" else [K4]
    q = AggQuery([], dims, Measure("sum", E.ForeignCol(0, 0, A.Float32, "v")), joins=[Join(table, KEY)])
    dense_key = torch.full((2 ** 22,), -1, dtype=torch.int64, device="cuda")
    dense_key[torch.from_numpy(keys.astype(np.int64)).cuda()] = torch.arange(nkeys, device="cuda")
    tval = torch.from_numpy(np.where(vok, val, 0).astype(np.float64)).cuda()
    tgrp = torch.from_numpy(grp.astype(np.int64)).cuda()
    sums = torch.zeros(4 * 17, dtype=torch.float64, device="cuda")
    seen = torch.zeros(4 * 17, dtype=torch.int64, device="cuda")
    ex = FusedBatchExecutor(eng.lib, eng.space, q)
    before = T.dense_launches(eng)
    n_batches, rows = 10, 5_000_000
    for i in range(n_batches):
        z = np.minimum(rng.zipf(1.3, rows), nkeys) - 1
        k = np.where(rng.random(rows) < 0.1, 2 ** 22 + rng.integers(0, 1000, rows), keys[z].astype(np.int64)).astype(np.uint32)
        k4 = rng.integers(0, 4, rows).astype(np.uint8)
        kb_, kvp = columns.make_column(eng.space, A.Uint32, k)
        k4b, k4vp = columns.make_column(eng.space, A.Uint8, k4)
        ex.process_batch(Batch([kvp, k4vp], rows, keep=[kb_, k4b], ranges={1: (0, 3)} if form == "direct" else None))
        tk = torch.from_numpy(k.astype(np.int64)).cuda()
        row = torch.where(tk < 2 ** 22, dense_key[tk.clamp(max=2 ** 22 - 1)], torch.full_like(tk, -1))
        hit = row >= 0
        g = torch.where(hit, tgrp[row.clamp(min=0)], torch.full_like(row, 16))       # 16: the NULL group
        slot = torch.from_numpy(k4.astype(np.int64)).cuda() * 17 + g
        sums.index_add_(0, slot, torch.where(hit, tval[row.clamp(min=0)], torch.zeros_like(tval[:1]).expand_as(row)))
        seen.index_add_(0, slot, torch.ones_like(slot))
    got = ex.result()
    ex.close()
    assert T.dense_launches(eng) - before == (n_batches if form == "direct" else 0)
    exp = {}
    s, c = sums.cpu().numpy(), seen.cpu().numpy()
    for slot in np.flatnonzero(c):
        k4, g = divmod(int(slot), 17)
        key = (k4, None if g == 16 else g) if form == "hash" else (k4,)
        exp[key] = exp.get(key, 0.0) + s[slot]
    have = {k: m for k, m in zip(zip(*got.decoded_dims()), got.measures.tolist())}
    assert have.keys() == exp.keys()
    assert all(have[k] == exp[k] for k in exp), "sums differ"     # integer-valued float sums below 2^53: exact
