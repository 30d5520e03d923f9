"""ctypes view of the engine's C ABI (include/aresdb_b200/*.h).

Field-exact mirrors of the structs the Go side builds in query/time_series_aggregate.go:166-360
(makeVectorPartySlice, makeConstantInput, makeScratchSpaceInput/Output,
makeDimensionVectorOutput, makeMeasureVectorOutput, makeDimensionVector) so that host code
written against them reads like the reference's cgo glue.  The same bindings load

  * aresdb_b200/lib/libalgorithm.so  - the B200 engine (product),
  * any other library exporting the same symbols (tests bind the reference's own HOST build
    and the C restatement under oracle/ through this module to act as checkers).

There is no CPU implementation behind these bindings: if the CUDA library is missing,
`load_engine()` raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

# ---- limits / enums (aql_abi.h) -----------------------------------------------------------
NUM_DIM_WIDTH = 5
MAX_DIMENSION_BYTES = 32
HLL_BITS = 14
HLL_DENSE_SIZE = 1 << HLL_BITS
HLL_DENSE_THRESHOLD = HLL_DENSE_SIZE // 4
DIM_WIDTHS = (16, 8, 4, 2, 1)

(AGGR_SUM_UNSIGNED, AGGR_SUM_SIGNED, AGGR_SUM_FLOAT, AGGR_MIN_UNSIGNED, AGGR_MIN_SIGNED,
 AGGR_MIN_FLOAT, AGGR_MAX_UNSIGNED, AGGR_MAX_SIGNED, AGGR_MAX_FLOAT, AGGR_HLL,
 AGGR_AVG_FLOAT) = range(1, 12)

(Bool, Int8, Uint8, Int16, Uint16, Int32, Uint32, Float32, Int64, Uint64, Float64, GeoPoint,
 UUID) = range(13)
DATA_TYPE_BYTES = {Bool: 0, Int8: 1, Uint8: 1, Int16: 2, Uint16: 2, Int32: 4, Uint32: 4, Float32: 4,
                   Int64: 8, Uint64: 8, Float64: 8, GeoPoint: 8, UUID: 16}

ConstInt, ConstFloat, ConstGeoPoint, ConstUUID = range(4)

(Negate, Not, BitwiseNot, IsNull, IsNotNull, Noop, GetWeekStart, GetMonthStart, GetQuarterStart,
 GetYearStart, GetDayOfMonth, GetDayOfYear, GetMonthOfYear, GetQuarterOfYear, GetHLLValue,
 ArrayLength) = range(16)

(And, Or, Equal, NotEqual, LessThan, LessThanOrEqual, GreaterThan, GreaterThanOrEqual, Plus, Minus,
 Multiply, Divide, Mod, BitwiseAnd, BitwiseOr, BitwiseXor, Floor, ArrayContains,
 ArrayElementAt) = range(19)

VectorPartyInput, ScratchSpaceInput, ConstantInput, ForeignColumnInput, ArrayVectorPartyInput = range(5)
ScratchSpaceOutput, MeasureOutput, DimensionOutput = range(3)

PLAN_OPERAND_NONE, PLAN_OPERAND_COLUMN, PLAN_OPERAND_CONST, PLAN_OPERAND_STACK, PLAN_OPERAND_FOREIGN = range(5)
PLAN_SINK_STACK, PLAN_SINK_FILTER, PLAN_SINK_DIMENSION, PLAN_SINK_MEASURE, PLAN_SINK_MEASURE_FILTER, PLAN_SINK_MEMBER_DIMENSION = range(6)
ARES_REDUCE_SORT, ARES_REDUCE_HASH = range(2)
ARES_MAX_PLAN_COLUMNS = 32
ARES_MAX_PLAN_INSTS = 64

DEVICE_MEMORY_IMPLEMENTATION_FLAG = 1
POOLED_MEMORY_FLAG = 2
HASH_REDUCTION_SUPPORT = 4


# ---- structs ---------------------------------------------------------------------------------
class CGoCallResHandle(C.Structure):
    _fields_ = [("res", C.c_void_p), ("pStrErr", C.c_void_p)]


class RecordID(C.Structure):
    _fields_ = [("batchID", C.c_int32), ("index", C.c_uint32)]


class CuckooHashIndex(C.Structure):
    _fields_ = [("buckets", C.c_void_p), ("seeds", C.c_uint32 * 4), ("keyBytes", C.c_int),
                ("numHashes", C.c_int), ("numBuckets", C.c_int)]


class GeoPointT(C.Structure):
    _fields_ = [("Lat", C.c_float), ("Long", C.c_float)]


class UUIDT(C.Structure):
    _fields_ = [("p1", C.c_uint64), ("p2", C.c_uint64)]


class _DefaultValueU(C.Union):
    _fields_ = [("BoolVal", C.c_bool), ("Int32Val", C.c_int32), ("Uint32Val", C.c_uint32),
                ("FloatVal", C.c_float), ("Int64Val", C.c_int64), ("GeoPointVal", GeoPointT),
                ("UUIDVal", UUIDT)]


class DefaultValue(C.Structure):
    _fields_ = [("HasDefault", C.c_bool), ("Value", _DefaultValueU)]


class VectorPartySlice(C.Structure):
    _fields_ = [("BasePtr", C.c_void_p), ("NullsOffset", C.c_uint32), ("ValuesOffset", C.c_uint32),
                ("StartingIndex", C.c_uint8), ("DataType", C.c_int), ("DefaultValue", DefaultValue),
                ("Length", C.c_uint32)]


class ScratchSpaceVector(C.Structure):
    _fields_ = [("Values", C.c_void_p), ("NullsOffset", C.c_uint32), ("DataType", C.c_int)]


class _ConstU(C.Union):
    _fields_ = [("IntVal", C.c_int32), ("FloatVal", C.c_float), ("GeoPointVal", GeoPointT),
                ("UUIDVal", UUIDT)]


class ConstantVector(C.Structure):
    _fields_ = [("Value", _ConstU), ("IsValid", C.c_bool), ("DataType", C.c_int)]


class ForeignColumnVector(C.Structure):
    _fields_ = [("RecordIDs", C.c_void_p), ("Batches", C.c_void_p), ("BaseBatchID", C.c_int32),
                ("NumBatches", C.c_int32), ("NumRecordsInLastBatch", C.c_int32),
                ("TimezoneLookup", C.c_void_p), ("TimezoneLookupSize", C.c_int16),
                ("DataType", C.c_int), ("DefaultValue", DefaultValue)]


class ArrayVectorPartySlice(C.Structure):
    _fields_ = [("OffsetLengthVector", C.c_void_p), ("ValueOffsetAdj", C.c_uint32),
                ("DataType", C.c_int), ("Length", C.c_uint32)]


class _InputU(C.Union):
    _fields_ = [("Constant", ConstantVector), ("VP", VectorPartySlice),
                ("ScratchSpace", ScratchSpaceVector), ("ForeignVP", ForeignColumnVector),
                ("ArrayVP", ArrayVectorPartySlice)]


class InputVector(C.Structure):
    _fields_ = [("Vector", _InputU), ("Type", C.c_int)]


class DimensionVector(C.Structure):
    _fields_ = [("DimValues", C.c_void_p), ("HashValues", C.c_void_p), ("IndexVector", C.c_void_p),
                ("VectorCapacity", C.c_int), ("NumDimsPerDimWidth", C.c_uint8 * NUM_DIM_WIDTH)]


class DimensionOutputVector(C.Structure):
    _fields_ = [("DimValues", C.c_void_p), ("DimNulls", C.c_void_p), ("DataType", C.c_int)]


class MeasureOutputVector(C.Structure):
    _fields_ = [("Values", C.c_void_p), ("DataType", C.c_int), ("AggFunc", C.c_int)]


class _OutputU(C.Union):
    _fields_ = [("ScratchSpace", ScratchSpaceVector), ("Dimension", DimensionOutputVector),
                ("Measure", MeasureOutputVector)]


class OutputVector(C.Structure):
    _fields_ = [("Vector", _OutputU), ("Type", C.c_int)]


class GeoShapeBatch(C.Structure):
    _fields_ = [("LatLongs", C.c_void_p), ("TotalNumPoints", C.c_int32), ("TotalWords", C.c_uint8)]


class _PlanConstU(C.Union):
    _fields_ = [("IntVal", C.c_int32), ("FloatVal", C.c_float)]


class PlanOperand(C.Structure):
    _fields_ = [("Kind", C.c_uint8), ("Column", C.c_uint8), ("ConstType", C.c_uint8),
                ("ConstValid", C.c_uint8), ("Const", _PlanConstU)]


class PlanInst(C.Structure):
    _fields_ = [("NumOperands", C.c_uint8), ("Functor", C.c_uint8), ("Sink", C.c_uint8),
                ("SinkArg", C.c_uint8), ("SinkDataType", C.c_uint8), ("Bucket", C.c_uint8), ("Reserved", C.c_uint8 * 2),
                ("A", PlanOperand), ("B", PlanOperand)]


class ColumnRange(C.Structure):
    """Zone-map hint of one column of one batch (batch_plan.h): valid values lie in [Min, Max]."""
    _fields_ = [("Known", C.c_uint8), ("Reserved", C.c_uint8 * 3), ("Min", C.c_uint32), ("Max", C.c_uint32)]


ARES_MAX_FOREIGN_TABLES, ARES_MAX_FOREIGN_COLUMNS = 4, 8

# plan-only unary functor: the numeric bucketizer BatchPlan.Bucketizers[PlanInst.Bucket] (batch_plan.h)
PLAN_FN_NUMERIC_BUCKET = 200
PLAN_BUCKET_WIDTH, PLAN_BUCKET_LOG, PLAN_BUCKET_PARTITIONS = 1, 2, 3
ARES_MAX_PLAN_BUCKETIZERS = 4


class PlanBucketizer(C.Structure):
    _fields_ = [("Kind", C.c_uint8), ("Reserved", C.c_uint8 * 3), ("LogMin", C.c_int32), ("Param", C.c_double),
                ("Bounds", C.c_void_p), ("NumBounds", C.c_uint32), ("Reserved2", C.c_uint32)]


class PlanForeignTable(C.Structure):
    _fields_ = [("JoinColumn", C.c_int32), ("Index", CuckooHashIndex)]


class PlanForeignColumn(C.Structure):
    _fields_ = [("Table", C.c_int32), ("Column", ForeignColumnVector)]


class BatchPlan(C.Structure):
    _fields_ = [("Columns", VectorPartySlice * ARES_MAX_PLAN_COLUMNS), ("NumColumns", C.c_int32),
                ("Insts", PlanInst * ARES_MAX_PLAN_INSTS), ("NumInsts", C.c_int32),
                ("BaseCounts", C.c_void_p), ("StartCount", C.c_uint32), ("NumRows", C.c_uint32),
                ("Ranges", ColumnRange * ARES_MAX_PLAN_COLUMNS),
                ("ForeignTables", PlanForeignTable * ARES_MAX_FOREIGN_TABLES), ("NumForeignTables", C.c_int32),
                ("ForeignColumns", PlanForeignColumn * ARES_MAX_FOREIGN_COLUMNS), ("NumForeignColumns", C.c_int32),
                ("Bucketizers", PlanBucketizer * ARES_MAX_PLAN_BUCKETIZERS), ("NumBucketizers", C.c_int32)]


class AggSpec(C.Structure):
    _fields_ = [("NumDimsPerDimWidth", C.c_uint8 * NUM_DIM_WIDTH), ("Reserved", C.c_uint8 * 3),
                ("AggFunc", C.c_int32), ("MeasureDataType", C.c_int32), ("ReduceMode", C.c_int32),
                ("ExpectedGroups", C.c_uint32)]


EXPECTED_SIZES = {DefaultValue: 24, VectorPartySlice: 56, ScratchSpaceVector: 16, ConstantVector: 24,
                  ForeignColumnVector: 72, ArrayVectorPartySlice: 24, InputVector: 80, OutputVector: 32,
                  DimensionVector: 40, CGoCallResHandle: 16}


# ---- constructors mirroring the Go helpers -------------------------------------------------
def make_default_value(valid: bool = False, value=0, data_type: int = Uint32) -> DefaultValue:
    dv = DefaultValue()
    dv.HasDefault = bool(valid)
    if valid:
        if data_type == Bool:
            dv.Value.BoolVal = bool(value)
        elif data_type in (Int8, Int16, Int32):
            dv.Value.Int32Val = int(value)
        elif data_type in (Uint8, Uint16, Uint32):
            dv.Value.Uint32Val = int(value)
        elif data_type == Float32:
            dv.Value.FloatVal = float(value)
        elif data_type == Int64:
            dv.Value.Int64Val = int(value)
        elif data_type == UUID:
            dv.Value.UUIDVal.p1, dv.Value.UUIDVal.p2 = value
        else:
            dv.HasDefault = False
    return dv


def make_vp_slice(base_ptr: int | None, nulls_offset: int, values_offset: int, starting_index: int,
                  data_type: int, length: int, default: DefaultValue | None = None) -> VectorPartySlice:
    vp = VectorPartySlice()
    vp.BasePtr = base_ptr
    vp.NullsOffset = nulls_offset
    vp.ValuesOffset = values_offset
    vp.StartingIndex = starting_index
    vp.DataType = data_type
    vp.DefaultValue = default if default is not None else DefaultValue()
    vp.Length = length
    return vp


def vp_input(vp: VectorPartySlice) -> InputVector:
    iv = InputVector()
    iv.Vector.VP = vp
    iv.Type = VectorPartyInput
    return iv


def const_input(value, is_valid: bool = True, is_float: bool | None = None) -> InputVector:
    """makeConstantInput (query/time_series_aggregate.go:239-270): float -> ConstFloat, else ConstInt."""
    iv = InputVector()
    if is_float is None:
        is_float = isinstance(value, float)
    if is_float:
        iv.Vector.Constant.Value.FloatVal = float(value)
        iv.Vector.Constant.DataType = ConstFloat
    else:
        iv.Vector.Constant.Value.IntVal = int(value)
        iv.Vector.Constant.DataType = ConstInt
    iv.Vector.Constant.IsValid = bool(is_valid)
    iv.Type = ConstantInput
    return iv


def scratch_input(values_ptr: int, nulls_offset: int, data_type: int) -> InputVector:
    iv = InputVector()
    iv.Vector.ScratchSpace.Values = values_ptr
    iv.Vector.ScratchSpace.NullsOffset = nulls_offset
    iv.Vector.ScratchSpace.DataType = data_type
    iv.Type = ScratchSpaceInput
    return iv


def scratch_output(values_ptr: int, nulls_offset: int, data_type: int) -> OutputVector:
    ov = OutputVector()
    ov.Vector.ScratchSpace.Values = values_ptr
    ov.Vector.ScratchSpace.NullsOffset = nulls_offset
    ov.Vector.ScratchSpace.DataType = data_type
    ov.Type = ScratchSpaceOutput
    return ov


def dimension_output(values_ptr: int, nulls_ptr: int, data_type: int) -> OutputVector:
    ov = OutputVector()
    ov.Vector.Dimension.DimValues = values_ptr
    ov.Vector.Dimension.DimNulls = nulls_ptr
    ov.Vector.Dimension.DataType = data_type
    ov.Type = DimensionOutput
    return ov


def measure_output(values_ptr: int, data_type: int, agg_func: int) -> OutputVector:
    ov = OutputVector()
    ov.Vector.Measure.Values = values_ptr
    ov.Vector.Measure.DataType = data_type
    ov.Vector.Measure.AggFunc = agg_func
    ov.Type = MeasureOutput
    return ov


def make_dimension_vector(values_ptr, hash_ptr, index_ptr, num_dims_per_width, capacity: int) -> DimensionVector:
    dv = DimensionVector()
    dv.DimValues = values_ptr
    dv.HashValues = hash_ptr
    dv.IndexVector = index_ptr
    dv.VectorCapacity = capacity
    for i in range(NUM_DIM_WIDTH):
        dv.NumDimsPerDimWidth[i] = num_dims_per_width[i]
    return dv


# ---- library loading ---------------------------------------------------------------------------
class AresError(RuntimeError):
    """What the Go side turns into a panic (cgoutils/utils.go:25-33)."""


_VP = C.c_void_p
_ALGO_SIGS = {
    "InitIndexVector": [_VP, C.c_uint32, C.c_int, _VP, C.c_int],
    "UnaryTransform": [InputVector, OutputVector, _VP, C.c_int, _VP, C.c_uint32, C.c_int, _VP, C.c_int],
    "BinaryTransform": [InputVector, InputVector, OutputVector, _VP, C.c_int, _VP, C.c_uint32, C.c_int, _VP,
                        C.c_int],
    "UnaryFilter": [InputVector, _VP, _VP, C.c_int, _VP, C.c_int, _VP, C.c_uint32, C.c_int, _VP, C.c_int],
    "BinaryFilter": [InputVector, InputVector, _VP, _VP, C.c_int, _VP, C.c_int, _VP, C.c_uint32, C.c_int, _VP,
                     C.c_int],
    "Sort": [DimensionVector, C.c_int, _VP, C.c_int],
    "Reduce": [DimensionVector, _VP, DimensionVector, _VP, C.c_int, C.c_int, C.c_int, _VP, C.c_int],
    "HashReduce": [DimensionVector, _VP, DimensionVector, _VP, C.c_int, C.c_int, C.c_int, _VP, C.c_int],
    "Expand": [DimensionVector, DimensionVector, _VP, _VP, C.c_int, C.c_int, _VP, C.c_int],
    "HyperLogLog": [DimensionVector, DimensionVector, _VP, _VP, C.c_int, C.c_int, C.c_bool,
                    C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_void_p), _VP, C.c_int],
    "HashLookup": [InputVector, _VP, _VP, C.c_int, _VP, C.c_uint32, CuckooHashIndex, _VP, C.c_int],
    "GeoBatchIntersects": [GeoShapeBatch, InputVector, _VP, C.c_int, C.c_uint32, _VP, C.c_int, _VP, C.c_bool,
                           _VP, C.c_int],
    "WriteGeoShapeDim": [C.c_int, DimensionOutputVector, C.c_int, _VP, _VP, C.c_int],
    "BootstrapDevice": [],
}
_PLAN_SIGS = {
    "AggStateCreate": [AggSpec, _VP, C.c_int],
    "ExecuteBatchPlan": [_VP, C.POINTER(BatchPlan), _VP, C.c_int],
    "ExecuteBatchPlanMulti": [C.POINTER(C.c_void_p), C.c_int, C.POINTER(BatchPlan), _VP, C.c_int],
    "AggStateMerge": [_VP, DimensionVector, _VP, C.c_int, _VP, C.c_int],
    "AggStateGroupCount": [_VP, _VP, C.c_int],
    "AggStateFinalize": [_VP, DimensionVector, _VP, _VP, C.c_int],
    "AggStateExport": [_VP, DimensionVector, _VP, _VP, C.c_int],
    "AggStateFinalizeHLL": [_VP, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_void_p),
                            _VP, C.c_int],
    "AggStateFinalizeHLLEstimate": [_VP, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), _VP, C.c_int],
    "AggStateReset": [_VP, _VP, C.c_int],
    "AggStateDestroy": [_VP, C.c_int],
    "AggStatesFinalize": [C.POINTER(C.c_void_p), C.c_int, C.POINTER(DimensionVector), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _VP,
                          C.c_int],
    "AggStatesExportPartsToPeers": [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, C.c_int,
                                    C.c_size_t, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t),
                                    C.c_uint32, _VP, C.c_int],
    "AggStatesMergeParts": [C.POINTER(C.c_void_p), C.c_int, _VP, C.c_int, C.c_size_t, C.c_int, C.POINTER(C.c_size_t),
                            C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), _VP, C.c_uint32, _VP, C.c_int],
    "ComputeColumnRanges": [C.POINTER(VectorPartySlice), C.c_int, C.POINTER(ColumnRange), _VP, C.c_int],
}
_MEM_SIGS = {
    "HostAlloc": [C.c_size_t], "HostFree": [_VP], "HostMemCpy": [_VP, _VP, C.c_size_t],
    "CreateCudaStream": [C.c_int], "WaitForCudaStream": [_VP, C.c_int], "DestroyCudaStream": [_VP, C.c_int],
    "DeviceAllocate": [C.c_size_t, C.c_int], "DeviceFree": [_VP, C.c_int],
    "AsyncCopyHostToDevice": [_VP, _VP, C.c_size_t, _VP, C.c_int],
    "AsyncCopyDeviceToDevice": [_VP, _VP, C.c_size_t, _VP, C.c_int],
    "AsyncCopyDeviceToHost": [_VP, _VP, C.c_size_t, _VP, C.c_int],
    "GetDeviceCount": [], "GetDeviceGlobalMemoryInMB": [C.c_int], "CudaProfilerStart": [],
    "CudaProfilerStop": [], "GetDeviceMemoryInfo": [C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_int],
    "deviceMalloc": [C.POINTER(C.c_void_p), C.c_size_t], "deviceFree": [_VP], "deviceMemset": [_VP, C.c_int, C.c_size_t],
    "asyncCopyHostToDevice": [_VP, _VP, C.c_size_t, _VP], "asyncCopyDeviceToHost": [_VP, _VP, C.c_size_t, _VP],
    "waitForCudaStream": [_VP],
}
MEM_EXTRA_SIGS = {"DeviceMemoryPoolTrim": [C.c_int]}

ALGORITHM_SYMBOLS = tuple(_ALGO_SIGS)
PLAN_SYMBOLS = tuple(_PLAN_SIGS)
MEMORY_SYMBOLS = tuple(_MEM_SIGS) + ("GetFlags",)

_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


class Library:
    """A loaded (libmem, libalgorithm) pair; `lib.Sort(...)` returns int(res) or raises AresError."""

    def __init__(self, algorithm_path: str | os.PathLike, mem_path: str | os.PathLike | None = None,
                 has_plan_api: bool = True, name: str = ""):
        self.name = name or Path(algorithm_path).parent.name
        # RTLD_LOCAL: several implementations of the same symbols may live in one process (tests);
        # each libalgorithm must bind to ITS OWN libmem through DT_NEEDED, never through the global scope.
        self.mem = C.CDLL(str(mem_path)) if mem_path else None
        self.alg = C.CDLL(str(algorithm_path))
        self.has_plan_api = has_plan_api
        self._fns = {}
        for nm, args in _ALGO_SIGS.items():
            self._bind(self.alg, nm, args, required=False)
        if has_plan_api:
            for nm, args in _PLAN_SIGS.items():
                self._bind(self.alg, nm, args, required=True)
        if self.mem is not None:
            for nm, args in {**_MEM_SIGS, **MEM_EXTRA_SIGS}.items():
                self._bind(self.mem, nm, args, required=False)
            try:
                self.mem.GetFlags.restype = C.c_uint32
                self.mem.GetFlags.argtypes = []
            except AttributeError:
                pass

    def _bind(self, dll, nm, args, required):
        try:
            fn = getattr(dll, nm)
        except AttributeError:
            if required:
                raise
            return
        fn.argtypes = args
        fn.restype = CGoCallResHandle
        self._fns[nm] = fn

    def has(self, nm: str) -> bool:
        return nm in self._fns

    def __getattr__(self, nm):
        fns = self.__dict__.get("_fns", {})
        if nm not in fns:
            raise AttributeError(nm)
        fn = fns[nm]

        def call(*args):
            h = fn(*args)
            if h.pStrErr:
                msg = C.string_at(h.pStrErr).decode(errors="replace")
                _libc.free(h.pStrErr)
                raise AresError(msg.strip())
            return int(h.res or 0)

        call.__name__ = nm
        return call

    def get_flags(self) -> int:
        return int(self.mem.GetFlags())

    def kernel_launch_count(self) -> int:
        fn = self.alg.AresKernelLaunchCount
        fn.restype = C.c_ulonglong
        fn.argtypes = []
        return int(fn())


PACKAGE_DIR = Path(__file__).resolve().parent
ENGINE_LIB_DIR = PACKAGE_DIR / "lib"
_engine: Library | None = None


def load_engine() -> Library:
    """Loads the CUDA engine.  Fails loudly when it has not been built: there is no fallback."""
    global _engine
    if _engine is None:
        alg, mem = ENGINE_LIB_DIR / "libalgorithm.so", ENGINE_LIB_DIR / "libmem.so"
        if not alg.exists() or not mem.exists():
            raise RuntimeError(
                f"aresdb_b200: {alg} is missing. Build the CUDA extension first "
                "(python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback.")
        _engine = Library(alg, mem, has_plan_api=True, name="b200")
    return _engine
