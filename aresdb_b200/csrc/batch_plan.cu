// batch_plan.cu — the fused whole-batch engine behind include/aresdb_b200/batch_plan.h.
//
// ExecuteBatchPlan = ONE persistent kernel per batch, specialised for the plan's shape (jit.cu,
// jit_kernel_head.cuh / jit_kernel_tail.cuh):
//   * column slices are staged tile by tile into shared memory by the TMA engine
//     (cp.async.bulk global->shared, completion on an mbarrier, kStages-deep ring), so HBM is
//     read exactly once, fully coalesced, with no LSU issue slots or registers spent on it;
//     the rows after the last full tile are copied by the kernel itself;
//   * every thread owns quads of 4 consecutive rows and evaluates the plan's instructions in
//     registers: filters clear bits of an alive mask, dimension roots pack the row key, the
//     measure root yields the value (NULL -> identity, x RLE count);
//   * surviving rows are aggregated into a CTA-private table (or direct-indexed slots when the
//     zone map bounds every dimension), which is flushed into the L2-resident global group table
//     when the CTA retires; rows that do not fit it go to the global table directly.
// Here: the plan's device form (compilePlan), its inputs made stageable (describeInputs / materialiseInputs:
// run-length columns, unaligned parts), the stage layout (layoutStages), the kernels a batch runs (scheduleBatch) and
// the launch / resume protocol (executePlan).
// The global table lives in an AggState across batches.  AggStateFinalize compacts it, hashes
// each group's packed dimension row with the reference's murmur3, sorts the g groups by hash,
// merges equal hashes and writes the reference's output layout — the observable result of the
// reference's Sort+Reduce (ARES_REDUCE_SORT) or HashReduce (ARES_REDUCE_HASH) over all batches.
#include <cooperative_groups.h>
#include <algorithm>
#include <memory>
#include <vector>

#include "agg.cuh"
#include "column.cuh"
#include "dimrow.cuh"
#include "fused_device.cuh"
#include "plan_device.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "small_sort.cuh"

namespace cg = cooperative_groups;

namespace aresb {

// from legacy_nodes.cu
ForeignDesc makeForeignDesc(const ForeignColumnVector &f);
// from sort_reduce.cu
void gatherDims(const uint8_t *in, const DimLayout &Lin, const uint32_t *rows, int g, uint8_t *out,
                const DimLayout &Lout, cudaStream_t s);
int hllRegisterVectors(const uint64_t *hash, const uint32_t *values, uint32_t *index, int R, uint8_t **hllVectorPtr,
                       size_t *hllVectorSizePtr, uint16_t **hllDimRegIDCountPtr, cudaStream_t s);
int reduceByHash(const uint64_t *hash, const uint32_t *index, const uint8_t *measures, int width, AggOp op, int n,
                 uint32_t *outIndex, uint8_t *outValues, cudaStream_t s, uint64_t *outHash = nullptr);
// from hll_estimate.cu
void hllEstimates(const uint8_t *vec, const uint16_t *counts, int groups, double *out, cudaStream_t s);


// status word of the single-launch finalize / of an exchange part
enum SmallFinalizeStatus : uint32_t { SF_OK = 0, SF_TOO_MANY = 1, SF_TABLE_OVERFLOW = 2, SF_OUTPUT_TOO_SMALL = 3, SF_PART_TRUNCATED = 4, SF_UNSETTLED = 5, SF_PEER_LATE = 6 };

// Group key of a packed dimension row: the row itself (KEY_PACKED), or the reference's hash of it.
__device__ __forceinline__ unsigned long long rowKey(const uint64_t *w, uint8_t keyMode, uint8_t hashBits, int rowBytes) {
  if (keyMode == KEY_PACKED) return w[0];
  return hashBits == 64 ? murmur3_128_lo(w, rowBytes, 0) : (unsigned long long)murmur3_32(w, rowBytes, 0);
}

// ---------------------------------------------------------------------------------------
// merge of already-reduced rows, finalize
// ---------------------------------------------------------------------------------------
// Folds already-reduced row i (dimension block + measures) into the group table; `hll`: 0, 1 (entries), 2 (dense registers).
__device__ __forceinline__ void foldRow(const uint8_t *__restrict__ block, const DimLayout &L, const uint8_t *__restrict__ measures,
                                        uint32_t i, int width, AggOp op, uint8_t keyMode, uint8_t hashBits, int hll, const DevTable &G) {
  uint64_t w[4];
  packRow(block, L, i, w);
  unsigned long long key = rowKey(w, keyMode, hashBits, L.rowBytes);
  const uint64_t v = loadMeasure(measures, i, width);
  if (hll == 2) { hllDenseUpdate(G, nullptr, key, keyMode == KEY_HASHED ? w : nullptr, (uint32_t)v); return; }
  if (hll == 1) key = (key & 0xFFFFFFFFFFFF0000ull) | (v & 0x3FFFu);
  globalUpdate(G, op, key, keyMode == KEY_HASHED ? w : nullptr, v);
}

__global__ void __launch_bounds__(256)
mergeRowsKernel(const uint8_t *__restrict__ block, DimLayout L, const uint8_t *__restrict__ measures, int width,
                AggOp op, int n, uint8_t keyMode, uint8_t hashBits, int hll, DevTable G) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < (uint32_t)n; i += stride)
    foldRow(block, L, measures, i, width, op, keyMode, hashBits, hll, G);
}

// States one exchange / finalize launch serves (AggStates*), and the flag stride of one state: a state's arrival flags are
// 16 consecutive words (one per sending rank), the flags of state k start 16 * k words after those of state 0.
constexpr int kMaxLaunchStates = 16;
constexpr int kMaxPeers = 16;

// Exchange step of a sharded request, receiving side: every state's N gathered parts ([groups, status, rows | dimension
// block of `L.capacity` rows | measures]) are folded by ONE launch; blockIdx.y is the state, and the row counts are read
// from the parts' headers on the device, so the host never waits for them.  Part p of state k lies at
// slots + p * slotStride + partOff[k].  A part whose sender could not fit its rows raises counters[2] of ITS state only.
// Parts carry no HLL state (the export side refuses it).
// `flags` != nullptr (exchange over peer memory): the parts are written into this GPU's memory by the PEERS' export
// kernels, each of which then stores `epoch` into flags[16 * k + its rank] with release semantics at system scope; every
// CTA of state k waits for that state's numParts flags (acquire, system scope) before it reads a part, so no state waits
// for another.  The wait is bounded (a peer that never arrives: counters[2] = 2, reported by finalize), so the kernel
// cannot hang the GPU.
struct MergeStateArgs {
  DevTable G;
  DimLayout L;
  size_t partOff, dimOff, valOff;
  int32_t width;
  uint8_t op, keyMode, hashBits;
};

struct MergePartsArgs {
  MergeStateArgs S[kMaxLaunchStates];
  const uint8_t *slots;
  size_t slotStride;
  const uint32_t *flags;
  int32_t numParts;
  uint32_t epoch;
};

__global__ void __launch_bounds__(256) mergePartsKernel(const __grid_constant__ MergePartsArgs M) {
  const MergeStateArgs &S = M.S[blockIdx.y];
  const DevTable &G = S.G;
  const uint32_t stride = gridDim.x * blockDim.x;
  if (M.flags != nullptr) {
    const uint32_t *flags = M.flags + kMaxPeers * blockIdx.y;
    __shared__ uint32_t sLate;
    if (threadIdx.x == 0) {
      uint32_t late = 0;
      const long long t0 = clock64();
      for (int p = 0; p < M.numParts && !late; p++) {
        for (;;) {
          uint32_t seen;
          asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(flags + p) : "memory");
          if ((int32_t)(seen - M.epoch) >= 0) break;
          if (clock64() - t0 > 4000000000ll) { late = 1; break; }   // ~2 s at 2 GHz
          __nanosleep(100);
        }
      }
      sLate = late;
      if (late) atomicExch(&G.counters[2], 2u);
    }
    __syncthreads();
    if (sLate) return;
  }
  for (int p = 0; p < M.numParts; p++) {
    const uint8_t *part = M.slots + (size_t)p * M.slotStride + S.partOff;
    const uint32_t *hdr = reinterpret_cast<const uint32_t *>(part);
    if (hdr[1] != SF_OK) {
      if (blockIdx.x == 0 && threadIdx.x == 0) atomicExch(&G.counters[2], 1u);
      continue;
    }
    const uint32_t n = hdr[0];
    const uint8_t *block = part + S.dimOff, *measures = part + S.valOff;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
      foldRow(block, S.L, measures, i, S.width, (AggOp)S.op, S.keyMode, S.hashBits, 0, G);
  }
}

// ---------------------------------------------------------------------------------------
// dense HLL mode: registers -> the carried (key, value) rows of query/hll.cu, already in key order
// ---------------------------------------------------------------------------------------
// one CTA per group (d-th in hash order): number of registers that were hit
__global__ void __launch_bounds__(256)
hllDenseCountKernel(const uint32_t *__restrict__ regs, const unsigned long long *__restrict__ acc, const uint32_t *__restrict__ slotOf, const uint32_t *__restrict__ order,
                    uint32_t *__restrict__ counts) {
  __shared__ uint32_t sWarp[256 / 32 + 1];
  const uint32_t *r = regs + (size_t)((uint32_t)acc[slotOf[order[blockIdx.x]]] - 1u) * kHllRegisters;   // (claim ordinal: hllRegArray)
  uint32_t c = 0;
  for (uint32_t i = threadIdx.x; i < kHllRegisters; i += 256) c += r[i] != 0;
  uint32_t total;
  blockExclusiveScan<256>(c, sWarp, &total);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// exclusive prefix of n <= 8192 counts by one CTA; offsets[n] = total
__global__ void __launch_bounds__(1024) hllDenseOffsetsKernel(const uint32_t *__restrict__ counts, int n, uint32_t *__restrict__ offsets) {
  __shared__ uint32_t sWarp[1024 / 32 + 1];
  __shared__ uint32_t sCarry;
  if (threadIdx.x == 0) sCarry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t x = i < n ? counts[i] : 0;
    uint32_t total;
    const uint32_t excl = blockExclusiveScan<1024>(x, sWarp, &total);
    if (i < n) offsets[i] = sCarry + excl;
    __syncthreads();
    if (threadIdx.x == 0) sCarry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[n] = sCarry;
}

// one CTA per group: its hit registers in ascending register order -> (key, value, group ordinal)
__global__ void __launch_bounds__(256)
hllDenseEmitKernel(const uint32_t *__restrict__ regs, const unsigned long long *__restrict__ acc, const uint32_t *__restrict__ slotOf, const uint32_t *__restrict__ order,
                   const uint64_t *__restrict__ sortedHash, const uint32_t *__restrict__ offsets,
                   uint64_t *__restrict__ outHash, uint32_t *__restrict__ outVals, uint32_t *__restrict__ outIndex) {
  __shared__ uint32_t sWarp[256 / 32 + 1];
  const uint32_t d = blockIdx.x;
  const uint32_t *r = regs + (size_t)((uint32_t)acc[slotOf[order[d]]] - 1u) * kHllRegisters;
  const uint64_t hi = sortedHash[d] & 0xFFFFFFFFFFFF0000ull;
  uint32_t pos = offsets[d];
  for (uint32_t base = 0; base < kHllRegisters; base += 256) {
    const uint32_t reg = base + threadIdx.x;
    const uint32_t v = r[reg];
    uint32_t total;
    const uint32_t excl = blockExclusiveScan<256>(v != 0, sWarp, &total);
    if (v != 0) {
      outHash[pos + excl] = hi | reg;
      outVals[pos + excl] = v - 1u;
      outIndex[pos + excl] = d;
    }
    pos += total;
    __syncthreads();
  }
}

// Dense registers -> the reference's register vectors directly (AggStateFinalizeHLL; query/hll.cu:262-290 semantics without
// the detour through (key, value) entries: 13M entries = 212 MB for 808 groups).  Layout pass, one CTA: per group d in hash
// order with counts[d] hit registers — its output ordinal among the groups that have any, the byte offset of its vector
// (4 bytes per hit register below HLL_DENSE_THRESHOLD, else HLL_DENSE_SIZE), totals[0] = dims, totals[1] = bytes.
__global__ void __launch_bounds__(1024)
hllVectorLayoutKernel(const uint32_t *__restrict__ counts, int n, uint32_t *__restrict__ outIdx, uint32_t *__restrict__ byteOff,
                      uint32_t *__restrict__ rowsOf, unsigned long long *__restrict__ totals) {
  __shared__ uint32_t sWarp[1024 / 32 + 1];
  __shared__ uint32_t sCarryP, sCarryB;
  if (threadIdx.x == 0) { sCarryP = 0; sCarryB = 0; }
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t c = i < n ? counts[i] : 0;
    const uint32_t p = c != 0, sz = c == 0 ? 0u : (c < (uint32_t)HLL_DENSE_THRESHOLD ? c * 4u : (uint32_t)HLL_DENSE_SIZE);
    uint32_t totP, totB;
    const uint32_t exP = blockExclusiveScan<1024>(p, sWarp, &totP);
    __syncthreads();
    const uint32_t exB = blockExclusiveScan<1024>(sz, sWarp, &totB);
    if (i < n) {
      outIdx[i] = sCarryP + exP;
      byteOff[i] = sCarryB + exB;
      if (p) rowsOf[sCarryP + exP] = (uint32_t)i;
    }
    __syncthreads();
    if (threadIdx.x == 0) { sCarryP += totP; sCarryB += totB; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { totals[0] = sCarryP; totals[1] = sCarryB; }
}

// one CTA per group: its vector (sparse: (rho << 16 | register) entries in ascending register order; dense: one rho byte
// per register) and its register count
__global__ void __launch_bounds__(256)
hllVectorEmitKernel(const uint32_t *__restrict__ regs, const unsigned long long *__restrict__ acc, const uint32_t *__restrict__ slotOf,
                    const uint32_t *__restrict__ order, const uint32_t *__restrict__ counts, const uint32_t *__restrict__ outIdx,
                    const uint32_t *__restrict__ byteOff, uint8_t *__restrict__ vec, uint16_t *__restrict__ regCount) {
  __shared__ uint32_t sWarp[256 / 32 + 1];
  const uint32_t d = blockIdx.x, c = counts[d];
  if (c == 0) return;
  if (threadIdx.x == 0) regCount[outIdx[d]] = (uint16_t)c;
  const uint32_t *r = regs + (size_t)((uint32_t)acc[slotOf[order[d]]] - 1u) * kHllRegisters;
  uint8_t *dst = vec + byteOff[d];
  // a register holds value + 1, value = rho << 16 | register (0: never hit); the vectors carry rho + 1
  if (c < (uint32_t)HLL_DENSE_THRESHOLD) {
    uint32_t pos = 0;
    for (uint32_t base = 0; base < kHllRegisters; base += 256) {
      const uint32_t reg = base + threadIdx.x, v = r[reg];
      uint32_t total;
      const uint32_t excl = blockExclusiveScan<256>(v != 0, sWarp, &total);
      if (v != 0) reinterpret_cast<uint32_t *>(dst)[pos + excl] = (((((v - 1u) >> 16) & 0xFFu) + 1u) << 16) | reg;
      pos += total;
      __syncthreads();
    }
  } else {
    for (uint32_t q = threadIdx.x; q < kHllRegisters / 4; q += 256) {
      const uint4 v = reinterpret_cast<const uint4 *>(r)[q];
      auto rho = [](uint32_t x) { return x ? ((((x - 1u) >> 16) & 0xFFu) + 1u) : 0u; };
      reinterpret_cast<uint32_t *>(dst)[q] = rho(v.x) | (rho(v.y) << 8) | (rho(v.z) << 16) | (rho(v.w) << 24);
    }
  }
}


constexpr int kCmpThreads = 256;
constexpr int kCmpItems = 8;
constexpr int kCmpTile = kCmpThreads * kCmpItems;

// Reference hash of the group whose table key is `key` (a packed key is its row; a hashed key already is the hash).
__device__ __forceinline__ uint64_t groupHash(unsigned long long key, uint8_t keyMode, uint8_t hashBits, int rowBytes, uint64_t mask) {
  uint64_t h = key;
  if (keyMode == KEY_PACKED) {
    const uint64_t w[4] = {key, 0, 0, 0};
    h = rowKey(w, KEY_HASHED, hashBits, rowBytes);
  }
  return hashBits == 64 ? h & mask : h;
}

// Packed dimension row of the group in `slot`.
__device__ __forceinline__ void slotRow(const DevTable &G, uint8_t keyMode, uint32_t slot, uint64_t (&w)[4]) {
  if (keyMode == KEY_PACKED) { w[0] = G.keys[slot]; w[1] = w[2] = w[3] = 0; return; }
#pragma unroll
  for (int i = 0; i < 4; i++) w[i] = G.rows[(size_t)slot * 4 + i];
}

// Compacts occupied slots: slotOf[g] = slot index, hash[g] = reference hash of the group's row,
// vals[g] = accumulator (tight `width`-byte elements).
__global__ void __launch_bounds__(kCmpThreads)
compactGroupsKernel(DevTable G, size_t cap, uint8_t keyMode, uint8_t hashBits, uint64_t hashMask, int rowBytes, int width, ScanTileState st,
                    uint32_t *__restrict__ slotOf, uint64_t *__restrict__ hash, uint8_t *__restrict__ vals,
                    uint32_t *__restrict__ outCount) {
  __shared__ uint32_t sTile, sPrefix;
  __shared__ uint32_t sWarp[kCmpThreads / 32 + 1];
  if (threadIdx.x == 0) sTile = atomicAdd(st.ticket, 1u);
  __syncthreads();
  const uint32_t tile = sTile;
  const size_t base = (size_t)tile * kCmpTile + (size_t)threadIdx.x * kCmpItems;
  uint32_t mask = 0;
#pragma unroll
  for (int k = 0; k < kCmpItems; k++) {
    size_t i = base + k;
    if (i < cap && G.keys[i] != kEmptyKey) mask |= 1u << k;
  }
  uint32_t blockTotal;
  const uint32_t excl = blockExclusiveScan<kCmpThreads>(__popc(mask), sWarp, &blockTotal);
  if (threadIdx.x < 32) {
    uint32_t p = decoupledLookback(st, tile, blockTotal);
    if (threadIdx.x == 0) {
      sPrefix = p;
      if (((size_t)tile + 1) * kCmpTile >= cap) *outCount = p + blockTotal;
    }
  }
  __syncthreads();
  uint32_t pos = sPrefix + excl;
#pragma unroll
  for (int k = 0; k < kCmpItems; k++) {
    if (!(mask & (1u << k))) continue;
    size_t i = base + k;
    const uint64_t h = groupHash(G.keys[i], keyMode, hashBits, rowBytes, hashMask);
    slotOf[pos] = (uint32_t)i;
    hash[pos] = h;
    storeMeasure(vals, pos, width, G.acc[i]);
    pos++;
  }
}

// Large results: the claim list replaces the table scan — slotOf / hash / vals of the n claimed groups, claim order.
__global__ void __launch_bounds__(256)
gatherClaimedKernel(DevTable G, uint32_t n, uint8_t keyMode, uint8_t hashBits, uint64_t hashMask, int rowBytes, int width,
                    uint32_t *__restrict__ slotOf, uint64_t *__restrict__ hash, uint8_t *__restrict__ vals) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t slot = G.claimed[i];
    const uint64_t h = groupHash(G.keys[slot], keyMode, hashBits, rowBytes, hashMask);
    slotOf[i] = slot;
    hash[i] = h;
    storeMeasure(vals, i, width, G.acc[slot]);
  }
}

__global__ void __launch_bounds__(256)
emitGroupsKernel(DevTable G, uint8_t keyMode, const uint32_t *__restrict__ slotOf, const uint32_t *__restrict__ repIndex,
                 uint32_t g, uint8_t *__restrict__ outBlock, DimLayout L, uint32_t *__restrict__ outIndex) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < g; s += stride) {
    uint64_t w[4];
    slotRow(G, keyMode, slotOf[repIndex[s]], w);
    unpackRow(outBlock, L, s, w);
    if (outIndex) outIndex[s] = s;
  }
}

__global__ void iotaKernel(uint32_t *p, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256)
fillTableKernel(unsigned long long *keys, unsigned long long *acc, size_t cap, unsigned long long neutral) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride) {
    keys[i] = kEmptyKey;
    acc[i] = neutral;
  }
}

// out[i] = in[i] + (+0.0): float sums of the hash-reduce mode (see finalize())
__global__ void __launch_bounds__(256) copyPlusZeroKernel(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, int n, int width) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (width == 8) reinterpret_cast<double *>(out)[i] = reinterpret_cast<const double *>(in)[i] + 0.0;
  else reinterpret_cast<float *>(out)[i] = reinterpret_cast<const float *>(in)[i] + 0.0f;
}

// Global dense slots (DevPlan::denseGlobal): after the batch, every reached slot of the state's accumulator array is
// folded into the group table under the packed dimension row its index decodes to, and reset to the neutral element.
struct DenseFold {
  uint32_t lo[8], cnt[8], step[8], stride[8];
  uint8_t rowOff[8], width[8], nullOff[8];
  uint32_t nd, total, reps;
  uint8_t keyMode, hashBits, rowBytes, op;
  unsigned long long neutral;
};

__global__ void __launch_bounds__(256)
denseFoldKernel(unsigned long long *__restrict__ acc, DenseFold F, DevTable G) {
  const uint32_t strideAll = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < F.total; i += strideAll) {
    unsigned long long v = F.neutral;
    for (uint32_t c = 0; c < F.reps; c++) {   // the copies the CTA groups accumulated into
      const unsigned long long x = acc[(size_t)c * F.total + i];
      if (x == F.neutral) continue;
      acc[(size_t)c * F.total + i] = F.neutral;
      v = v == F.neutral ? x : aggCombine((AggOp)F.op, v, x);
    }
    if (v == F.neutral) continue;
    uint64_t row[4] = {0, 0, 0, 0};
    uint8_t *rb = reinterpret_cast<uint8_t *>(row);
    uint32_t rem = i;
    for (int k = (int)F.nd - 1; k >= 0; k--) {
      const uint32_t ix = rem / F.stride[k];
      rem -= ix * F.stride[k];
      const bool valid = ix != F.cnt[k];
      const uint32_t val = valid ? (F.lo[k] + ix) * F.step[k] : 0u;
      for (int b = 0; b < F.width[k]; b++) rb[F.rowOff[k] + b] = (uint8_t)(val >> (8 * b));
      rb[F.nullOff[k]] = valid ? 1 : 0;
    }
    globalUpdate(G, (AggOp)F.op, rowKey(row, F.keyMode, F.hashBits, F.rowBytes), F.keyMode == KEY_PACKED ? nullptr : row, v);
  }
}

// ---------------------------------------------------------------------------------------
// single-launch finalize for results of up to kSmallFinalizeMax groups
// ---------------------------------------------------------------------------------------
// One thread-block cluster of kFinCtas CTAs walks the claim list (no table scan, no compaction), hashes each group's
// packed row with the reference's murmur3, sorts the (hash, claim ordinal) pairs — one bucketing pass over the top 12 hash
// bits (histogram in L2, every CTA scans it into its own shared memory), then every element ranks itself inside its
// bucket —, merges runs of equal hashes with the aggregate's rule — the member claimed first names the run — and writes
// the reference's DimensionVector block + measure vector.  The phases are chains of two or three dependent loads per
// element: 8192 threads give every thread at most four elements, so a phase costs a few memory latencies, and the
// phases are separated by the hardware cluster barrier (one CTA of 1024 threads would serialise those latencies).
// The group count goes to a mapped pinned host word, so the
// host's only interaction is one stream synchronise.  `ordered == 0` is the exchange form of AggStateExport: the
// claimed slots as they are, no sort, no merge.
constexpr int kSmallFinalizeMax = kSmallSortMax;
constexpr int kFinCtas = 8;                          // portable cluster maximum
constexpr uint32_t kFinThreads = kFinCtas * 1024u;
constexpr size_t kFinHistWords = 2 * kSmallBuckets + 64;   // bucket counts | scatter cursors | per-CTA run-head totals

struct SmallFinalizeArgs {
  DevTable G;
  DimLayout L;              // output block layout (capacity = outputKeys.VectorCapacity)
  uint64_t hashMask;
  uint64_t *hashA, *tmpK;   // scratch: kSmallFinalizeMax entries each
  uint32_t *idxA, *tmpI;
  uint32_t *hist;           // scratch: kFinHistWords
  uint8_t *outBlock, *outValues;
  uint64_t *outHash;
  uint32_t *outIndex;
  uint32_t *resultDev;      // [0] groups, [1] status, [2] claimed slots
  volatile uint32_t *resultHost;
  int32_t rowBytes, width, outCapacity;
  uint8_t keyMode, hashBits, op, plusZero, ordered;
};

// The exchange form: the n claimed slots as they are, in claim order, no sort and no merge.
__device__ __forceinline__ void exportClaimed(const SmallFinalizeArgs &A, uint32_t n, uint32_t gtid) {
  for (uint32_t i = gtid; i < n; i += kFinThreads) {
    const uint32_t slot = A.G.claimed[i];
    uint64_t w[4];
    slotRow(A.G, A.keyMode, slot, w);
    unpackRow(A.outBlock, A.L, i, w);
    storeMeasure(A.outValues, i, A.width, A.G.acc[slot]);
    if (A.outIndex) A.outIndex[i] = i;
  }
}

// One launch serves several states: cluster c (CTAs c * kFinCtas ..) works on S[c] alone, with its own scratch and result
// words, so clusters never wait for each other.
struct SmallFinalizeBatch {
  SmallFinalizeArgs S[kMaxLaunchStates];
};

__global__ void __cluster_dims__(kFinCtas, 1, 1) __launch_bounds__(1024, 1) finalizeSmallKernel(const __grid_constant__ SmallFinalizeBatch B) {
  __shared__ uint32_t off[kSmallBuckets + 1];
  __shared__ uint32_t sWarp[1024 / 32 + 1];
  cg::cluster_group cluster = cg::this_cluster();
  const uint32_t ctaRank = cluster.block_rank(), gtid = ctaRank * 1024u + threadIdx.x;
  const SmallFinalizeArgs &A = B.S[blockIdx.x / kFinCtas];
  const DevTable &G = A.G;
  const uint32_t n = G.counters[0];
  uint32_t status = SF_OK;
  if (G.counters[1]) status = SF_TABLE_OVERFLOW;
  else if (G.counters[2] == 2u) status = SF_PEER_LATE;   // AggStatesMergeParts gave up waiting for a peer's flag
  else if (G.counters[2]) status = SF_PART_TRUNCATED;   // AggStatesMergeParts met a part that did not hold all its rows
  else if (G.counters[3] || G.counters[4]) status = SF_UNSETTLED;   // stopped at the growth threshold / rows parked: the host settles first
  else if (n > (uint32_t)kSmallFinalizeMax) status = SF_TOO_MANY;
  else if (!A.ordered && n > (uint32_t)A.outCapacity) status = SF_OUTPUT_TOO_SMALL;
  auto publish = [&](uint32_t groups, uint32_t st, uint32_t claimedSlots) {
    A.resultDev[0] = groups; A.resultDev[1] = st; A.resultDev[2] = claimedSlots;
    A.resultHost[0] = groups; A.resultHost[1] = st; A.resultHost[2] = claimedSlots;
  };
  if (status != SF_OK || n == 0) {   // (uniform over the cluster: nobody waits at a barrier below)
    if (gtid == 0) publish(0, status, n);
    return;
  }
  if (!A.ordered) {
    exportClaimed(A, n, gtid);
    if (gtid == 0) publish(n, SF_OK, n);
    return;
  }
  uint32_t *cnt = A.hist, *cur = A.hist + kSmallBuckets, *ctaHeads = A.hist + 2 * kSmallBuckets;
  const int shift = A.hashBits - kSmallBits;
  for (uint32_t b = gtid; b < (uint32_t)kSmallBuckets; b += kFinThreads) { cnt[b] = 0; cur[b] = 0; }
  cluster.sync();
  // 1. reference hash of every group's row; histogram of the top hash bits
  for (uint32_t i = gtid; i < n; i += kFinThreads) {
    const uint64_t h = groupHash(G.keys[G.claimed[i]], A.keyMode, A.hashBits, A.rowBytes, A.hashMask);
    A.hashA[i] = h;
    atomicAdd(&cnt[(uint32_t)(h >> shift) & (kSmallBuckets - 1)], 1u);
  }
  cluster.sync();
  // 2. bucket offsets: every CTA scans the histogram for itself (no barrier, and the offsets are in shared memory)
  {
    constexpr int kPer = kSmallBuckets / 1024;
    uint32_t c[kPer], sum = 0, total;
#pragma unroll
    for (int j = 0; j < kPer; j++) { c[j] = cnt[threadIdx.x * kPer + j]; sum += c[j]; }
    uint32_t excl = blockExclusiveScan<1024>(sum, sWarp, &total);
#pragma unroll
    for (int j = 0; j < kPer; j++) { off[threadIdx.x * kPer + j] = excl; excl += c[j]; }
    if (threadIdx.x == 0) off[kSmallBuckets] = total;
  }
  __syncthreads();
  // 3. unordered scatter into the buckets
  for (uint32_t i = gtid; i < n; i += kFinThreads) {
    const uint64_t h = A.hashA[i];
    const uint32_t d = (uint32_t)(h >> shift) & (kSmallBuckets - 1);
    const uint32_t p = off[d] + atomicAdd(&cur[d], 1u);
    A.tmpK[p] = h;
    A.tmpI[p] = i;
  }
  cluster.sync();
  // 4. every element finds its rank among its bucket's members by (hash, claim ordinal): 4.7 members on average for
  // 19,200 groups; a degenerate bucket only costs time
  for (uint32_t i = gtid; i < n; i += kFinThreads) {
    const uint64_t k = A.tmpK[i];
    const uint32_t v = A.tmpI[i];
    const uint32_t d = (uint32_t)(k >> shift) & (kSmallBuckets - 1);
    const uint32_t lo = off[d], hi = off[d + 1];
    uint32_t rank = 0;
    for (uint32_t j = lo; j < hi; j++) {
      const uint64_t kj = A.tmpK[j];
      rank += (kj < k) || (kj == k && A.tmpI[j] < v);
    }
    A.hashA[lo + rank] = k;
    A.idxA[lo + rank] = v;
  }
  cluster.sync();
  // 5. runs of equal hashes: every thread owns a contiguous chunk, counts the run heads in it ...
  const uint32_t per = (n + kFinThreads - 1) / kFinThreads;
  const uint32_t begin = gtid * per < n ? gtid * per : n, end = begin + per < n ? begin + per : n;
  uint32_t heads = 0;
  for (uint32_t j = begin; j < end; j++) heads += j == 0 || A.hashA[j] != A.hashA[j - 1];
  uint32_t ctaTotal;
  uint32_t pos = blockExclusiveScan<1024>(heads, sWarp, &ctaTotal);
  if (threadIdx.x == 0) ctaHeads[ctaRank] = ctaTotal;
  cluster.sync();
  uint32_t g = 0;
#pragma unroll
  for (int r = 0; r < kFinCtas; r++) {
    const uint32_t t = ctaHeads[r];
    if ((uint32_t)r < ctaRank) pos += t;
    g += t;
  }
  if (g > (uint32_t)A.outCapacity) {
    if (gtid == 0) publish(0, SF_OUTPUT_TOO_SMALL, g);
    return;
  }
  // ... 6. and folds + emits the runs that start in its chunk (a run may extend into the next chunks)
  for (uint32_t j = begin; j < end; j++) {
    const uint64_t h = A.hashA[j];
    if (!(j == 0 || h != A.hashA[j - 1])) continue;
    const uint32_t slot = G.claimed[A.idxA[j]];
    uint64_t acc = G.acc[slot];
    for (uint32_t k = j + 1; k < n && A.hashA[k] == h; k++) acc = aggCombine((AggOp)A.op, acc, G.acc[G.claimed[A.idxA[k]]]);
    if (A.plusZero) {   // hash-reduce float sums start from +0.0 (see finalize())
      if (A.width == 8) acc = (uint64_t)__double_as_longlong(__longlong_as_double((long long)acc) + 0.0);
      else acc = __float_as_uint(__uint_as_float((uint32_t)acc) + 0.0f);
    }
    uint64_t w[4];
    slotRow(G, A.keyMode, slot, w);
    unpackRow(A.outBlock, A.L, pos, w);
    storeMeasure(A.outValues, pos, A.width, acc);
    if (A.outHash) A.outHash[pos] = h;
    if (A.outIndex) A.outIndex[pos] = pos;
    pos++;
  }
  if (gtid == 0) publish(g, SF_OK, n);
}

// Exchange over peer memory, sending side: ONE kernel writes this rank's rows of every state as parts ([rows, status,
// claimed | dimension block | measures], AggStatesExportPartsToPeers' sub-part) into its own slot of its receive buffer —
// cluster c (kFinCtas CTAs) exports state c into sub-part c —, copies each sub-part into the same place in every peer's
// receive buffer with 16-byte stores over NVLink, and then stores `epoch` into state c's flag for this rank on every peer
// (release, system scope) — export, all-gather and the "it has arrived" signal in one launch, no collective library and
// no host in between.  peerFlag[0] == nullptr: the local export only (the parts then travel by a collective all-gather).
struct PeerExportArgs {
  SmallFinalizeArgs F[kMaxLaunchStates];   // the exports (ordered = 0); outBlock / outValues / resultDev lie in the local sub-part
  size_t partOffset[kMaxLaunchStates];     // sub-part of state c inside a slot
  size_t partBytes[kMaxLaunchStates];      // its size, a multiple of 16
  uint8_t *peerSlot[kMaxPeers];            // this rank's slot in every peer's receive buffer (peerSlot[myRank]: the local one)
  uint32_t *peerFlag[kMaxPeers];           // &flags[state 0][myRank] on every peer; state c's flag lies kMaxPeers * c words further
  uint32_t numPeers, myRank, epoch;
};

__global__ void __cluster_dims__(kFinCtas, 1, 1) __launch_bounds__(1024) exportToPeersKernel(const __grid_constant__ PeerExportArgs E) {
  cg::cluster_group cluster = cg::this_cluster();
  const uint32_t gtid = cluster.block_rank() * 1024u + threadIdx.x;
  const uint32_t c = blockIdx.x / kFinCtas;
  const SmallFinalizeArgs &A = E.F[c];
  const DevTable &G = A.G;
  const uint32_t n = G.counters[0];
  uint32_t status = SF_OK;
  if (G.counters[1]) status = SF_TABLE_OVERFLOW;
  else if (G.counters[3] || G.counters[4]) status = SF_UNSETTLED;
  else if (n > (uint32_t)A.outCapacity) status = SF_OUTPUT_TOO_SMALL;
  if (status == SF_OK) exportClaimed(A, n, gtid);
  if (gtid == 0) { A.resultDev[0] = status == SF_OK ? n : 0u; A.resultDev[1] = status; A.resultDev[2] = n; }
  if (E.peerFlag[0] == nullptr) return;
  cluster.sync();   // the local part is complete (and visible to the cluster)
  // the part travels as it lies: header, the used prefix of every section would save bytes, but a part is 0.5 MB and the
  // copy is a few microseconds of NVLink time
  const uint4 *src = reinterpret_cast<const uint4 *>(E.peerSlot[E.myRank] + E.partOffset[c]);
  const uint32_t words = (uint32_t)(E.partBytes[c] / 16);
  for (uint32_t p = 0; p < E.numPeers; p++) {
    if (p == E.myRank) continue;
    uint4 *dst = reinterpret_cast<uint4 *>(E.peerSlot[p] + E.partOffset[c]);
    for (uint32_t i = gtid; i < words; i += kFinThreads) dst[i] = src[i];
  }
  __threadfence_system();
  cluster.sync();   // every thread's stores are ordered before the flags
  if (gtid < E.numPeers)
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(E.peerFlag[gtid] + kMaxPeers * c), "r"(E.epoch) : "memory");
}

// AggStateReset: only the claimed slots are emptied (and, for dense HLL states, only their register arrays).
__global__ void __launch_bounds__(256)
resetClaimedKernel(DevTable G, unsigned long long neutral) {
  const uint32_t n = G.counters[0];
  if (G.regs != nullptr) {   // one CTA per claimed group at a time: 16384 registers
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
      if (i >= kHllDenseMaxGroups) break;   // (claims past the register arrays were turned away)
      uint4 *r = reinterpret_cast<uint4 *>(G.regs + (size_t)i * kHllRegisters);   // register arrays go by claim ordinal
      for (uint32_t k = threadIdx.x; k < kHllRegisters / 4; k += blockDim.x) r[k] = make_uint4(0, 0, 0, 0);
    }
  }
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t slot = G.claimed[i];
    G.keys[slot] = kEmptyKey;
    G.acc[slot] = neutral;
  }
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct AggState {
  AggSpec spec;
  int device;
  DimLayout rowLayout;     // capacity-independent parts (rowOff / width / numDims)
  KeyMode keyMode;
  int hashBits;
  AggOp op;
  int measWidth;
  ValClass measClass;
  uint64_t accNeutral;
  bool hll;
  bool hllDense;           // HLL with one dense register array per group (few groups) instead of (group, register) entries
  size_t capacity;
  DevTable table;
  void *mem;               // single allocation behind the table
  unsigned long long *ctaAcc;  // [kMaxGridCtas][8192] private accumulator slices of the fused kernel's CTAs
  unsigned long long *denseAcc = nullptr;  // [kGlobalDenseMaxSlots] shared accumulators of the global dense form (lazy)
  uint64_t occUpper = 0;                   // host-side upper bound of the occupied slots (exact after a synchronise)
  uint32_t unchecked = 0;                  // hash-table batches launched since the last check of the STOP flag
  bool everChecked = false;                // a batch of this query has been waited for (its occupancy is known)
  uint8_t *smallScratch = nullptr;         // single-launch finalize: hash / index ping-pong arrays (in `mem`)
  uint32_t *resultDev = nullptr;           // [0] groups, [1] status, [2] claimed slots of the last single-launch finalize
  uint32_t *resultHost = nullptr;          // the same three words in mapped pinned host memory
  uint32_t *resultHostDev = nullptr;       // device alias of resultHost
};

constexpr size_t kHllDenseSlots = 8192;

// DevPlan::hll and mergeRowsKernel's `hll`: 0 no HLL, 1 (group, register) entries, 2 dense register arrays
static uint8_t hllMode(const AggState *st) { return st->hll ? (st->hllDense ? 2 : 1) : 0; }

static void *deviceAllocOrThrow(size_t bytes) {
  void *mem = nullptr;
  CGoCallResHandle h = deviceMalloc(&mem, bytes);
  if (h.pStrErr) { std::string m(h.pStrErr); free((void *)h.pStrErr); throw EngineError(m); }
  return mem;
}

static uint64_t neutralOf(AggOp op) {
  switch (op) {
    case OP_SUM_F32: return 0x80000000ull;                // -0.0f: (-0) + x == x for every x
    case OP_SUM_F64: return 0x8000000000000000ull;        // -0.0
    case OP_MIN_U32: return 0xFFFFFFFFull;
    case OP_MIN_I32: return 0x7FFFFFFFull;
    case OP_MAX_I32: return 0x80000000ull;
    case OP_MIN_F32: return 0x7F800000ull;                // +inf
    case OP_MAX_F32: return 0xFF800000ull;                // -inf
    default: return 0;                                     // integer sums, unsigned max
  }
}

static ValClass measureClassOf(int dt) {
  switch (dt) {
    case Int32: return VC_I32;
    case Uint32: return VC_U32;
    case Float32: return VC_F32;
    case Int64: return VC_I64;
    case Float64: return VC_F64;
    default: throw EngineError("Unsupported data type for MeasureOutput");
  }
}

static void allocTable(AggState *st, size_t cap, cudaStream_t s) {
  const bool rows = st->keyMode == KEY_HASHED;
  const size_t ctaAccBytes = (size_t)kMaxGridCtas * 8192 * sizeof(unsigned long long);
  const size_t regBytes = st->hllDense ? (size_t)kHllDenseMaxGroups * kHllRegisters * sizeof(uint32_t) : 0;   // by claim ordinal
  const size_t claimedBytes = (cap * 4 + 255) / 256 * 256;
  const size_t smallBytes = (size_t)kSmallFinalizeMax * (8 + 8 + 4 + 4) + kFinHistWords * 4;
  const size_t progressBytes = ((size_t)(kProgressTail + 1) * 4 + 255) / 256 * 256;
  const size_t spillBytes = (size_t)kSpillCap * sizeof(SpillEntry);
  size_t bytes = cap * 16 + (rows ? cap * 32 : 0) + 256 + ctaAccBytes + regBytes + claimedBytes + smallBytes + progressBytes + spillBytes;
  void *mem = deviceAllocOrThrow(bytes);
  st->mem = mem;
  st->capacity = cap;
  uint8_t *p = static_cast<uint8_t *>(mem);
  st->table.counters = reinterpret_cast<uint32_t *>(p);
  st->table.keys = reinterpret_cast<unsigned long long *>(p + 256);
  st->table.acc = st->table.keys + cap;
  st->table.rows = rows ? reinterpret_cast<uint64_t *>(st->table.acc + cap) : nullptr;
  st->ctaAcc = reinterpret_cast<unsigned long long *>(p + 256 + cap * 16 + (rows ? cap * 32 : 0));
  st->table.mask = (uint32_t)(cap - 1);
  st->table.regs = st->hllDense ? reinterpret_cast<uint32_t *>(p + 256 + cap * 16 + (rows ? cap * 32 : 0) + ctaAccBytes) : nullptr;
  uint8_t *tail = p + 256 + cap * 16 + (rows ? cap * 32 : 0) + ctaAccBytes + regBytes;
  st->table.claimed = reinterpret_cast<uint32_t *>(tail);
  st->smallScratch = tail + claimedBytes;
  st->table.progress = reinterpret_cast<uint32_t *>(tail + claimedBytes + smallBytes);
  st->table.spill = reinterpret_cast<SpillEntry *>(tail + claimedBytes + smallBytes + progressBytes);
  // half full = time to grow (the dense HLL directory does not grow: its register arrays are sized with it)
  st->table.growAt = st->hllDense ? 0xFFFFFFFFu : (uint32_t)(cap / 2);
  st->resultDev = st->table.counters + 8;   // inside the 256-byte header
  if (!st->resultHost) {
    ARES_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&st->resultHost), 64, cudaHostAllocMapped));
    ARES_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void **>(&st->resultHostDev), st->resultHost, 0));
    memset(st->resultHost, 0, 64);
  }
  st->table.occPublish = st->resultHostDev + 8;
  if (st->hllDense) ARES_CUDA(cudaMemsetAsync(st->table.regs, 0, regBytes, s));
  ARES_CUDA(cudaMemsetAsync(p, 0, 256, s));
  fillTableKernel<<<smCount() * 8, 256, 0, s>>>(st->table.keys, st->table.acc, cap, st->accNeutral);
  checkLastError("fillTable");
}

static void describeState(AggState *st, const AggSpec &spec) {
  st->spec = spec;
  st->rowLayout = makeDimLayout(spec.NumDimsPerDimWidth, 1);
  if (spec.ReduceMode != ARES_REDUCE_SORT && spec.ReduceMode != ARES_REDUCE_HASH) throw EngineError("unknown ReduceMode");
  st->hashBits = spec.ReduceMode == ARES_REDUCE_SORT ? 64 : 32;
  st->keyMode = st->rowLayout.rowBytes <= 8 ? KEY_PACKED : KEY_HASHED;
  st->measClass = measureClassOf(spec.MeasureDataType);
  int bytes = (st->measClass == VC_I64 || st->measClass == VC_F64) ? 8 : 4;
  if (spec.AggFunc == AGGR_AVG_FLOAT && bytes != 8) throw EngineError("an AVG measure is 8 bytes (average, count)");
  st->hll = spec.AggFunc == AGGR_HLL;
  st->hllDense = st->hll && spec.ExpectedGroups <= kHllDenseMaxGroups;
  if (st->hll) {
    if (st->measClass != VC_U32) throw EngineError("an HLL measure is Uint32");
    st->hashBits = 64;
    st->op = OP_MAX_U32;
    st->measWidth = 4;
    // entry mode: group identity = the reference's HLL key (dim-row hash with the register in its low
    // 16 bits, query/functor.hpp:1299-1305), the table keeps the max value (rho << 16 | reg) per key.
    // dense mode (ExpectedGroups <= 4096 groups): the table is the directory of dimension rows and
    // every group owns 16384 registers in DevTable::regs.
    if (!st->hllDense) st->keyMode = KEY_HASHED;
  } else {
    st->op = aggOpOf(spec.AggFunc, bytes, &st->measWidth);
  }
  st->accNeutral = neutralOf(st->op);
}

static AggState *createState(const AggSpec &spec, cudaStream_t s, int device) {
  AggState *st = new AggState();
  try {
    describeState(st, spec);
    st->device = device;
    // global table: 2^21 slots (32 MB, L2-resident) unless the caller expects more groups
    size_t want = (size_t)spec.ExpectedGroups * 2;
    size_t cap = (size_t)1 << 21;
    while (cap < want) cap <<= 1;
    if (const char *e = getenv("ARESDB_B200_TABLE_SLOTS")) {   // tests: start small so that the table has to grow
      const long v = atol(e);
      if (v >= 1024 && (v & (v - 1)) == 0) cap = (size_t)v;
    }
    if (st->hllDense) cap = kHllDenseSlots;
    allocTable(st, cap, s);
  } catch (...) {
    delete st;
    throw;
  }
  return st;
}

static AggState *asState(void *p) {
  if (!p) throw EngineError("null AggState handle");
  return static_cast<AggState *>(p);
}

static uint8_t operandClassOf(const PlanOperand &o, const BatchPlan &bp) {
  switch (o.Kind) {
    case PLAN_OPERAND_COLUMN: {
      if (o.Column >= bp.NumColumns) throw EngineError("plan operand references a column outside BatchPlan.Columns");
      switch (bp.Columns[o.Column].DataType) {
        case Bool: return VC_BOOL;
        case Int8: case Int16: case Int32: return VC_I32;
        case Uint8: case Uint16: case Uint32: return VC_U32;
        case Float32: return VC_F32;
        case Int64: return VC_I64;
        case UUID: return VC_UUID;
        default: throw EngineError("Unsupported data type for VectorPartyInput");
      }
    }
    case PLAN_OPERAND_CONST:
      if (o.ConstType == ConstInt) return VC_I32;
      if (o.ConstType == ConstFloat) return VC_F32;
      throw EngineError("Unsupported constant type in plan");
    case PLAN_OPERAND_FOREIGN: {
      if (o.Column >= bp.NumForeignColumns) throw EngineError("plan operand references a column outside BatchPlan.ForeignColumns");
      switch (bp.ForeignColumns[o.Column].Column.DataType) {
        case Bool: return VC_BOOL;
        case Int8: case Int16: case Int32: return VC_I32;
        case Uint8: case Uint16: case Uint32: return VC_U32;
        case Float32: return VC_F32;
        default: throw EngineError("foreign columns of the fused path are Bool / 1-, 2-, 4-byte integers / Float32");
      }
    }
    default: throw EngineError("plan instruction has a missing operand");
  }
}

static ValClass sinkClassOf(int dt, bool dim) {
  switch (dt) {
    case Bool: if (dim) return VC_BOOL; break;
    case Int8: if (dim) return VC_I8; break;
    case Uint8: if (dim) return VC_U8; break;
    case Int16: if (dim) return VC_I16; break;
    case Uint16: if (dim) return VC_U16; break;
    case Int32: return VC_I32;
    case Uint32: return VC_U32;
    case Float32: return VC_F32;
    case Int64: return VC_I64;
    case Float64: if (!dim) return VC_F64; break;
    case UUID: if (dim) return VC_UUID; break;
    default: break;
  }
  throw EngineError("Unsupported sink data type in plan");
}

static int classWidth(ValClass c) {
  switch (c) {
    case VC_BOOL: case VC_I8: case VC_U8: return 1;
    case VC_I16: case VC_U16: return 2;
    case VC_I32: case VC_U32: case VC_F32: return 4;
    case VC_I64: case VC_F64: return 8;
    default: return 16;
  }
}

// Translates the ABI plan into the device form, resolving value classes by the reference's rules.  `multi` (nmulti
// states, ExecuteBatchPlanMulti): the plan has one measure root per state, SinkArg = the state's ordinal, each checked
// against its own state; everything else is taken from `st` (= multi[0]) and the per-measure fields are left to the caller.
static void compilePlan(const AggState *st, const BatchPlan &bp, DevPlan &P, AggState *const *multi = nullptr, int nmulti = 0) {
  memset(&P, 0, sizeof(P));
  if (bp.NumColumns < 0 || bp.NumColumns > kMaxPlanCols)
    throw EngineError("the fused path stages at most 16 distinct columns per batch");
  if (bp.NumInsts <= 0 || bp.NumInsts > ARES_MAX_PLAN_INSTS) throw EngineError("invalid plan instruction count");
  P.ncols = bp.NumColumns;
  P.ninsts = bp.NumInsts;
  P.baseCounts = bp.BaseCounts;
  P.startCount = bp.StartCount;
  P.numRows = bp.NumRows;
  for (int c = 0; c < bp.NumColumns; c++) {
    P.cols[c].in = makeColumnDesc(bp.Columns[c], /*allowWide=*/true);
    int dt = bp.Columns[c].DataType;
    P.cols[c].width = dt == Bool ? 0 : (dt == Int8 || dt == Uint8) ? 1 : (dt == Int16 || dt == Uint16) ? 2
                    : (dt == Int64 || dt == Uint64) ? 8 : dt == UUID ? 16 : 4;
    P.cols[c].used = 0;      // set below by the instructions that read the column: only those are staged
    const ColumnRange &cr = bp.Ranges[c];
    P.cols[c].rangeKnown = cr.Known && cr.Min <= cr.Max && cr.Max < 0x80000000u && P.cols[c].width <= 4 ? 1 : 0;
    P.cols[c].rangeLo = cr.Min;
    P.cols[c].rangeHi = cr.Max;
    P.cols[c].staged = 0;
    P.cols[c].hasNulls = 0;
  }
  // joined dimension tables
  if (bp.NumForeignTables < 0 || bp.NumForeignTables > kMaxForeignTables || bp.NumForeignColumns < 0 ||
      bp.NumForeignColumns > kMaxForeignCols)
    throw EngineError("invalid number of foreign tables / columns");
  P.numForeignTables = (uint8_t)bp.NumForeignTables;
  P.numForeignCols = (uint8_t)bp.NumForeignColumns;
  for (int t = 0; t < bp.NumForeignTables; t++) {
    const int jc = bp.ForeignTables[t].JoinColumn;
    if (jc < 0 || jc >= bp.NumColumns) throw EngineError("foreign table joins on a column outside BatchPlan.Columns");
    if (P.cols[jc].width > 4) throw EngineError("join keys of the fused path are 1-, 2- or 4-byte columns");
    P.joinCol[t] = (uint8_t)jc;
  }
  for (int k = 0; k < bp.NumForeignColumns; k++) {
    const int t = bp.ForeignColumns[k].Table;
    if (t < 0 || t >= bp.NumForeignTables) throw EngineError("foreign column of a table outside BatchPlan.ForeignTables");
    P.foreignTableOf[k] = (uint8_t)t;
  }
  // numeric bucketizers: the parameters are checked here, the bounds tables (device memory) are the caller's
  if (bp.NumBucketizers < 0 || bp.NumBucketizers > kJitMaxBuckets) throw EngineError("invalid number of numeric bucketizers");
  P.nbuckets = (uint8_t)bp.NumBucketizers;
  for (int j = 0; j < bp.NumBucketizers; j++) {
    const PlanBucketizer &B = bp.Bucketizers[j];
    const double v = B.Param;
    switch (B.Kind) {
      case PLAN_BUCKET_WIDTH:
        if (!(v > 0.0 && v <= kMaxFinite)) throw EngineError("numeric bucketizer " + std::to_string(j) + ": the width must be finite and > 0");
        break;
      case PLAN_BUCKET_LOG:
        if (!(v > 1.0 && v <= kMaxFinite)) throw EngineError("numeric bucketizer " + std::to_string(j) + ": the log base must be finite and > 1");
        if (!B.Bounds || B.NumBounds < 2 || B.NumBounds > 65537)
          throw EngineError("numeric bucketizer " + std::to_string(j) + ": a log table has 2..65537 bounds in device memory");
        break;
      case PLAN_BUCKET_PARTITIONS:
        if (!B.Bounds || B.NumBounds < 1 || B.NumBounds > 255)
          throw EngineError("numeric bucketizer " + std::to_string(j) + ": manual partitions are 1..255 bounds in device memory");
        break;
      default: throw EngineError("numeric bucketizer " + std::to_string(j) + ": unknown kind");
    }
    P.bucketKind[j] = B.Kind;
    P.bucketSlot[j] = 0xFF;
    JitBucket &D = P.buckets[j];
    D.bounds = B.Bounds;
    D.param = v;
    D.n = B.NumBounds;
    D.logMin = B.LogMin;
    D.invLog2 = B.Kind == PLAN_BUCKET_LOG ? (float)(1.0 / log2(v)) : 0.0f;
  }
  int nbucketSlots = 0;
  const DimLayout &RL = st->rowLayout;
  std::vector<int> stack;   // the instructions whose pushed values are on the evaluation stack
  std::vector<bool> dimSeen(RL.numDims, false);
  bool measureSeen = false;
  std::vector<bool> stateFed(nmulti, false);
  P.lastFilter = -1;
  int firstMemberFilter = -1, firstDimOrMeasure = -1, firstMeasure = -1;
  bool plainDims = false;
  std::vector<int> memberDimsOf(nmulti, 0);   // member dimension roots of each state so far
  int nmagic = 0;
  for (int i = 0; i < bp.NumInsts; i++) {
    const PlanInst &pi = bp.Insts[i];
    DevInst &I = P.insts[i];
    if (pi.NumOperands != 1 && pi.NumOperands != 2) throw EngineError("plan instruction must have 1 or 2 operands");
    I.nops = pi.NumOperands; I.fn = pi.Functor; I.sink = pi.Sink; I.sinkArg = pi.SinkArg;
    // Each stack operand is linked to the instruction that pushed its value (the right operand pops first when both come
    // from the stack); a stack operand's class is its producer's sink class.  The later passes follow the links and
    // resolve operand a, then b: resolving a stack operand has no side effect (the generator emits no load for it and
    // takes no JitParams::consts slot), so the order they read the links in changes neither the kernel text nor its
    // parameters.
    auto pop = [&]() -> int {
      if (stack.empty()) throw EngineError("plan pops an empty evaluation stack");
      const int j = stack.back();
      stack.pop_back();
      return j;
    };
    I.bsrc = (int8_t)(pi.NumOperands == 2 && pi.B.Kind == PLAN_OPERAND_STACK ? pop() : -1);
    I.asrc = (int8_t)(pi.A.Kind == PLAN_OPERAND_STACK ? pop() : -1);
    const uint8_t acls = I.asrc >= 0 ? P.insts[I.asrc].oclass : operandClassOf(pi.A, bp);
    const uint8_t bcls = pi.NumOperands != 2 ? (uint8_t)VC_NONE : I.bsrc >= 0 ? P.insts[I.bsrc].oclass : operandClassOf(pi.B, bp);
    auto fill = [&](const PlanOperand &o, uint8_t &kind, uint8_t &col, uint8_t &valid, uint32_t &k) {
      kind = o.Kind; col = o.Column; valid = o.ConstValid;
      if (o.Kind == PLAN_OPERAND_COLUMN) P.cols[o.Column].used = 1;
      if (o.Kind == PLAN_OPERAND_FOREIGN) P.cols[P.joinCol[P.foreignTableOf[o.Column]]].used = 1;   // the join key is staged
      if (o.Kind == PLAN_OPERAND_CONST) {
        if (o.ConstType == ConstFloat) memcpy(&k, &o.Const.FloatVal, 4); else k = (uint32_t)o.Const.IntVal;
      }
    };
    fill(pi.A, I.akind, I.acol, I.avalid, I.aconst);
    if (pi.NumOperands == 2) fill(pi.B, I.bkind, I.bcol, I.bvalid, I.bconst);
    I.aclass = acls; I.bclass = bcls;

    const bool wideIn = acls == VC_I64 || acls == VC_UUID || bcls == VC_I64 || bcls == VC_UUID;
    if (wideIn) {
      // only "dimension = 8/16-byte column" is meaningful (what UnaryTransform Noop to a
      // DimensionOutput of the same type does)
      // (a wide member dimension never reaches the kernel as one: the direct-indexed form the member form needs has none)
      const bool dimSink = pi.Sink == PLAN_SINK_DIMENSION || pi.Sink == PLAN_SINK_MEMBER_DIMENSION;
      ValClass oc = dimSink ? sinkClassOf(pi.SinkDataType, true) : VC_NONE;
      if (pi.NumOperands != 1 || pi.Functor != Noop || !dimSink || pi.A.Kind != PLAN_OPERAND_COLUMN ||
          oc != (ValClass)acls)
        throw EngineError("int64/UUID columns are only supported as verbatim dimensions on the fused path");
      I.wide = 1;
    } else if (pi.NumOperands == 2) {
      I.tclass = commonClass((ValClass)acls, (ValClass)bcls);
      Cell z; z.v = 0; z.valid = true;
      ValClass rc;
      evalBinary(pi.Functor, z, z, (ValClass)I.tclass, &rc);
      I.rclass = rc;
    } else if (pi.Functor == PLAN_FN_NUMERIC_BUCKET) {
      // a dimension root over a 32-bit (or Bool) value whose sink type is the ordinal type of the bucketizer's kind
      if (pi.NumOperands != 1) throw EngineError("PLAN_FN_NUMERIC_BUCKET is a unary functor");
      if (pi.Bucket >= bp.NumBucketizers) throw EngineError("PLAN_FN_NUMERIC_BUCKET names a bucketizer outside BatchPlan.Bucketizers");
      if (pi.Sink != PLAN_SINK_DIMENSION && pi.Sink != PLAN_SINK_MEMBER_DIMENSION) throw EngineError("a numeric bucketizer is a dimension root");
      if (acls != VC_BOOL && acls != VC_I32 && acls != VC_U32 && acls != VC_F32)
        throw EngineError("a numeric bucketizer's operand is a Bool, 1-, 2-, 4-byte integer or Float32 value");
      const uint8_t kind = P.bucketKind[pi.Bucket];
      const int dt = kind == PLAN_BUCKET_WIDTH ? Int32 : kind == PLAN_BUCKET_LOG ? Uint16 : Uint8;
      if (pi.SinkDataType != dt)
        throw EngineError("a numeric bucketizer's dimension is Int32 (width), Uint16 (log base) or Uint8 (manual partitions)");
      if (kind == PLAN_BUCKET_PARTITIONS && P.bucketSlot[pi.Bucket] == 0xFF) P.bucketSlot[pi.Bucket] = (uint8_t)nbucketSlots++;
      I.bucket = pi.Bucket;
      I.tclass = acls;
      I.rclass = sinkClassOf(dt, true);
    } else {
      I.tclass = acls;
      Cell z; z.v = 0; z.valid = true;
      ValClass rc;
      evalUnary(pi.Functor, z, (ValClass)acls, &rc);
      I.rclass = rc;
    }
    // the first kJitMaxMagic fast divisions of the plan take a magic slot each; the others run the functor
    I.magic = (int8_t)(isFastDiv(I) && nmagic < kJitMaxMagic ? nmagic++ : -1);
    switch (pi.Sink) {
      case PLAN_SINK_STACK: {
        ValClass oc = sinkClassOf(pi.SinkDataType, false);
        if (oc != VC_I32 && oc != VC_U32 && oc != VC_F32) throw EngineError("stack temporaries are Int32/Uint32/Float32");
        if ((int)stack.size() >= ARES_PLAN_STACK_DEPTH) throw EngineError("plan exceeds the evaluation stack depth");
        I.oclass = oc;
        stack.push_back(i);
        break;
      }
      case PLAN_SINK_FILTER:
        if (firstMemberFilter >= 0) throw EngineError("member filter roots must follow the last PLAN_SINK_FILTER root");
        I.oclass = VC_BOOL;
        P.lastFilter = i;
        break;
      case PLAN_SINK_MEASURE_FILTER:   // (ExecuteBatchPlanMulti: a filter of state SinkArg alone)
        if (!multi) throw EngineError("PLAN_SINK_MEASURE_FILTER (member filter) roots need ExecuteBatchPlanMulti");
        if (pi.SinkArg >= nmulti)
          throw EngineError("member filter root with SinkArg " + std::to_string(pi.SinkArg) + ": there are " + std::to_string(nmulti) + " states");
        if (firstDimOrMeasure >= 0) throw EngineError("member filter roots must precede the first dimension root");
        if (firstMemberFilter < 0) firstMemberFilter = i;
        I.oclass = VC_BOOL;
        break;
      case PLAN_SINK_MEMBER_DIMENSION: {   // (ExecuteBatchPlanMulti: a dimension of the states in mask SinkArg)
        if (!multi) throw EngineError("PLAN_SINK_MEMBER_DIMENSION (member dimension) roots need ExecuteBatchPlanMulti");
        if (pi.SinkArg == 0) throw EngineError("member dimension root with an empty state mask");
        if (pi.SinkArg >> nmulti)
          throw EngineError("member dimension root with state mask " + std::to_string(pi.SinkArg) + ": there are " + std::to_string(nmulti) + " states");
        if (plainDims) throw EngineError("a plan has PLAN_SINK_DIMENSION or PLAN_SINK_MEMBER_DIMENSION roots, not both");
        if (firstMeasure >= 0) throw EngineError("member dimension roots must precede the measure roots");
        if (firstDimOrMeasure < 0) firstDimOrMeasure = i;
        const ValClass oc = sinkClassOf(pi.SinkDataType, true);
        const int u = P.memberDims++;   // this root is member dimension u (dense dimension u of the shared form)
        if (u >= kJitMaxDenseDims * kJitMaxMeasures) throw EngineError("too many member dimension roots");
        for (int k = 0; k < nmulti; k++) {
          if (!((pi.SinkArg >> k) & 1)) continue;
          const DimLayout &L = multi[k]->rowLayout;
          const int j = memberDimsOf[k]++;
          if (j >= L.numDims || classWidth(oc) != L.width[j])
            throw EngineError("member dimension roots of state " + std::to_string(k) + " do not match its NumDimsPerDimWidth");
          if (u < kJitMaxDenseDims) {
            P.meas[k].dims |= (uint8_t)(1u << u);
            P.meas[k].rowOff[u] = L.rowOff[j];
            P.meas[k].nullOff[u] = (uint8_t)(L.valueBytes + j);
          }
        }
        I.oclass = oc;
        I.width = (uint8_t)classWidth(oc);
        break;
      }
      case PLAN_SINK_DIMENSION: {
        if (P.memberDims) throw EngineError("a plan has PLAN_SINK_DIMENSION or PLAN_SINK_MEMBER_DIMENSION roots, not both");
        plainDims = true;
        if (pi.SinkArg >= RL.numDims) throw EngineError("dimension ordinal outside AggSpec.NumDimsPerDimWidth");
        ValClass oc = sinkClassOf(pi.SinkDataType, true);
        if (classWidth(oc) != RL.width[pi.SinkArg]) throw EngineError("dimension data type does not match its layout width");
        if (dimSeen[pi.SinkArg]) throw EngineError("dimension written twice");
        dimSeen[pi.SinkArg] = true;
        if (firstDimOrMeasure < 0) firstDimOrMeasure = i;
        I.oclass = oc;
        I.rowOff = RL.rowOff[pi.SinkArg];
        I.width = RL.width[pi.SinkArg];
        I.nullOff = (uint8_t)(RL.valueBytes + pi.SinkArg);
        break;
      }
      case PLAN_SINK_MEASURE: {
        const AggState *fed = st;
        if (multi) {
          if (pi.SinkArg >= nmulti)
            throw EngineError("measure root with SinkArg " + std::to_string(pi.SinkArg) + ": there are " + std::to_string(nmulti) + " states");
          if (stateFed[pi.SinkArg]) throw EngineError("two measure roots feed state " + std::to_string(pi.SinkArg) + " (duplicate SinkArg)");
          stateFed[pi.SinkArg] = true;
          fed = multi[pi.SinkArg];
        } else if (measureSeen) {
          throw EngineError("only one measure per plan");
        }
        P.meas[multi ? pi.SinkArg : 0].inst = (int8_t)i;
        measureSeen = true;
        if (firstDimOrMeasure < 0) firstDimOrMeasure = i;
        if (firstMeasure < 0) firstMeasure = i;
        ValClass oc = sinkClassOf(pi.SinkDataType, false);
        if (oc != fed->measClass) throw EngineError("measure data type differs from AggSpec.MeasureDataType");
        I.oclass = oc;
        break;
      }
      default: throw EngineError("unknown plan sink");
    }
  }
  if (!stack.empty()) throw EngineError("plan leaves values on the evaluation stack");
  P.bucketSmem = (uint32_t)nbucketSlots * kBucketSmemBytes;
  for (int d = 0; d < RL.numDims && !P.memberDims; d++)
    if (!dimSeen[d]) throw EngineError("plan does not produce every dimension of AggSpec");
  for (int k = 0; k < nmulti && P.memberDims; k++)
    if (memberDimsOf[k] != multi[k]->rowLayout.numDims)
      throw EngineError("member dimension roots of state " + std::to_string(k) + " do not match its NumDimsPerDimWidth");
  if (!measureSeen) throw EngineError("plan has no measure instruction");
  for (int k = 0; k < nmulti; k++)
    if (!stateFed[k]) throw EngineError("no measure root feeds state " + std::to_string(k) + " (missing SinkArg)");
  P.hasMeasure = 1;
  P.keyMode = st->keyMode;
  P.rowBytes = (uint8_t)RL.rowBytes;
  P.valueBytes = (uint8_t)RL.valueBytes;
  P.hashBits = (uint8_t)st->hashBits;
  P.aggOp = st->op;
  {  // can a reached accumulator return to the neutral element?  (global dense slots carry no "reached" flags)
    bool safe = st->op != OP_SUM_I32 && st->op != OP_SUM_I64;   // float sums (-0.0), min / max (extreme), AVG (count 0)
    for (int i = 0; i < P.ninsts; i++) safe = safe || positiveLiteralSum(P.insts[i], st->op);   // integer sums: count(*)
    P.neutralSafe = safe && !st->hll;
  }
  P.measWidth = (uint8_t)st->measWidth;
  P.measClass = st->measClass;
  P.hll = hllMode(st);
  P.denseSlots = st->hllDense ? (uint32_t)st->capacity : 0;
  const int agg = st->spec.AggFunc;
  P.skipCount = !((agg >= AGGR_SUM_UNSIGNED && agg <= AGGR_SUM_FLOAT) || agg == AGGR_AVG_FLOAT);
  P.measureIdentity = aggIdentity(agg, st->measClass);
  P.accNeutral = st->accNeutral;
}

// ---------------------------------------------------------------------------------------
// archive batches: run-length encoded (mode-3) columns that the kernel does not decode from their runs
// are expanded once per batch into plain mode-2 scratch columns (one value + one validity bit per
// index position), see describeInputs.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
expandRleKernel(InputDesc d, const uint32_t *__restrict__ baseCounts, uint32_t startCount, uint32_t n, int width, bool direct,
                uint8_t *__restrict__ outValues, uint32_t *__restrict__ outNulls) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warpsPerGrid = gridDim.x * (blockDim.x >> 5);
  const uint32_t *counts = reinterpret_cast<const uint32_t *>(d.base);
  const uint8_t *vals = d.base + d.valuesOff, *nulls = d.base + d.nullsOff;
  for (uint32_t w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w * 32 < n; w += warpsPerGrid) {
    const uint32_t i = w * 32 + lane;
    bool valid = false, bit = false;
    if (i < n) {
      // index position i stands for row baseCounts[i] (or startCount + i); `direct`: this column's own
      // count vector IS the batch's base counts, so its run number is i
      const uint32_t p = direct ? i : rlePosition(counts, d.length, baseCounts ? baseCounts[i] : startCount + i);
      valid = bitAt(nulls, p + d.startBit);
      switch (width) {
        case 0: bit = bitAt(vals, p + d.startBit); break;
        case 1: outValues[i] = vals[p]; break;
        case 2: reinterpret_cast<uint16_t *>(outValues)[i] = reinterpret_cast<const uint16_t *>(vals)[p]; break;
        case 4: reinterpret_cast<uint32_t *>(outValues)[i] = reinterpret_cast<const uint32_t *>(vals)[p]; break;
        case 8: reinterpret_cast<uint64_t *>(outValues)[i] = reinterpret_cast<const uint64_t *>(vals)[p]; break;
        default:   // UUID (8-byte aligned, as wide columns are)
          reinterpret_cast<uint64_t *>(outValues)[2 * (size_t)i] = reinterpret_cast<const uint64_t *>(vals)[2 * (size_t)p];
          reinterpret_cast<uint64_t *>(outValues)[2 * (size_t)i + 1] = reinterpret_cast<const uint64_t *>(vals)[2 * (size_t)p + 1];
          break;
      }
    }
    const uint32_t vword = __ballot_sync(0xFFFFFFFFu, valid), bword = __ballot_sync(0xFFFFFFFFu, bit);
    if (lane == 0) {
      outNulls[w] = vword;
      if (width == 0) reinterpret_cast<uint32_t *>(outValues)[w] = bword;
    }
  }
}

// First-class RLE columns: run that holds the first index position of every tile (and of the batch's last position), so
// that the kernel searches a window of a few runs per quad instead of the whole count vector per row.
__global__ void __launch_bounds__(256)
rleTileRunsKernel(const uint32_t *__restrict__ counts, uint32_t length, const uint32_t *__restrict__ baseCounts, uint32_t startCount,
                  uint32_t numRows, uint32_t tileRows, uint32_t entries, uint32_t *__restrict__ out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= entries) return;
  uint64_t pos = (uint64_t)t * tileRows;
  if (pos > numRows - 1) pos = numRows - 1;
  const uint32_t row = baseCounts ? baseCounts[pos] : startCount + (uint32_t)pos;
  out[t] = rlePosition(counts, length, row);
}

// SUM / AVG need the run lengths of an archive batch, and RLE columns the row numbers of its index positions: the base
// counts are then staged with the columns.
static bool stagesBaseCounts(const DevPlan &P) {
  if (P.baseCounts == nullptr) return false;
  bool anyRle = false;
  for (int c = 0; c < P.ncols; c++) anyRle = anyRle || (P.cols[c].used && P.cols[c].rle);
  return !P.skipCount || anyRle;
}

// What a laid-out single-measure plan decided for its measure (denseFx: it takes the exact-integer form), as the kernel's
// per-measure code takes it: for the plan itself, or for a state's measure in a shared plan (scheduleStates).
static void describeMeasure(const DevPlan &Q, DevMeasure &M) {
  M.aggOp = Q.aggOp; M.measWidth = Q.measWidth; M.skipCount = Q.skipCount; M.neutralSafe = Q.neutralSafe;
  M.denseFx = Q.denseFx; M.fxShift = Q.fxShift; M.measureIdentity = Q.measureIdentity; M.accNeutral = Q.accNeutral;
}

// Member dimensions: the slots of each measure's region when `avail` bytes of shared memory hold them, false when they do
// not.  Each region holds at least the measure's own slots; the rest of `avail` is shared in proportion to them (for
// lane-private copies of few slots).
static bool memberSlots(DevPlan &P, size_t avail) {
  size_t need = 0, sb[kJitMaxMeasures], r16[kJitMaxMeasures];
  for (int m = 0; m < P.nmeas; m++) {
    DevMeasure &M = P.meas[m];
    uint64_t total = 1;
    for (int j = 0; j < P.denseNd && total <= kDenseMaxSlots; j++)
      if ((M.dims >> j) & 1u) total *= (uint64_t)P.denseCnt[j] + 1;
    if (total > kDenseMaxSlots) return false;
    M.total = (uint32_t)total;
    sb[m] = denseSlotBytes(M.denseFx);
    r16[m] = (total + 15) / 16 * 16;
    need += r16[m] * sb[m];
  }
  if (avail < 128u * P.nmeas + need) return false;
  avail -= 128u * P.nmeas;   // (each region starts on a 128-byte boundary)
  for (int m = 0; m < P.nmeas; m++) {
    const size_t cap = r16[m] * avail / need / 16 * 16;
    P.meas[m].slots = (uint32_t)(cap < kDenseMaxSlots ? cap : kDenseMaxSlots);
  }
  return true;
}

// Decides the tile size, the stage layout, the TMA ring depth and the shared table size.  The shared table gets what the
// workload needs first (a table that overflows sends rows to contended L2 atomics, tools/microbench/agg_microbench.cu),
// the ring takes the rest.  Staged parts must start on a 16-byte boundary (materialiseInputs copies those that do not).
// A single-measure plan describes its measure in meas[0].
static size_t layoutStages(DevPlan &P, uint32_t expectedGroups) {
  const bool stageBc = stagesBaseCounts(P);
  // (partition tables of numeric bucketizers sit after the stages)
  const size_t budget = (size_t)kSmemBudget - P.bucketSmem;
  // The shared table takes 8192 slots (128 KB) whenever a ring of >= 2 stages still fits beside
  // it: measured on cfg3 (2,400 groups per batch) 8192 slots beat 4096 by 1.5x because fewer
  // probe iterations are paid per warp; a plan with very wide rows falls back to fewer slots.
  uint32_t slots = 8192;
  // The caller expects far more groups than the shared table holds (or HLL, whose entries are
  // (group, register) pairs): compile the kernel with the direct-to-global mode it can switch to.
  P.bypassOk = (P.hll || expectedGroups > 4 * slots) ? 1 : 0;
  // zone map known for every dimension: no key table, slots addressed by dimension value (jit.cu)
  P.denseGlobal = 0;
  jitAnalyzeDense(P);
  auto stageBytesFor = [&](uint32_t tr) {
    size_t stage = 0;
    for (int c = 0; c < P.ncols; c++) {
      const DevColumn &col = P.cols[c];
      if (col.in.mode == 0 || !col.used || col.width > 4 || col.rle) continue;
      stage += ((col.width ? (size_t)tr * col.width : tr / 8 + 16) + 15) / 16 * 16;
      if (col.in.mode == 2) stage += (tr / 8 + 16 + 15) / 16 * 16;
    }
    if (stageBc) stage += ((size_t)tr + 4) * 4;
    return stage;
  };
  // stages of tiles of `tr` rows that fit in `avail` bytes (a plan that stages nothing has empty stages: any number fits)
  auto stagesIn = [&](size_t avail, uint32_t tr) -> uint32_t {
    const size_t bytes = stageBytesFor(tr), n = bytes ? avail / bytes : (size_t)kMaxStages;
    return n > (size_t)kMaxStages ? (uint32_t)kMaxStages : (uint32_t)n;
  };
  // keep >= 128 rows for the tail so that the last full tile's 16-byte bitmap over-read stays inside the column
  auto fullTiles = [&](uint32_t tr) { return P.numRows > 128 ? (P.numRows - 128) / tr : 0u; };
  uint32_t tileRows = 0, stages = 0;
  if (P.denseNd != 0) {
    // Dense slots cost 9 bytes each (flag + 8-byte accumulator).  Give the ring as many stages as possible
    // and the slots the rest: the capacity (part of the kernel text) then depends on the stage layout only,
    // not on the batch's ranges.
    for (uint32_t tr : {3968u, 1920u, 896u}) {
      for (uint32_t n = kMaxStages; n >= 2 && !tileRows; n--) {
        // (several measures: one 128-byte aligned region of accumulators each)
        const size_t need = 128 + n * stageBytesFor(tr) + (P.nmeas > 1 && !P.memberDims ? 128 * P.nmeas : 0);
        if (need >= budget) continue;
        if (P.memberDims) {   // (only with several measures: scheduleStates)
          if (memberSlots(P, budget - need)) {
            tileRows = tr; stages = n; slots = 16;
            for (int m = 0; m < P.nmeas; m++) slots = P.meas[m].slots > slots ? P.meas[m].slots : slots;
          }
          continue;
        }
        size_t slotBytes = denseSlotBytes(P.denseFx, P.hll);
        if (P.nmeas > 1) {
          slotBytes = 0;
          for (int m = 0; m < P.nmeas; m++) slotBytes += denseSlotBytes(P.meas[m].denseFx);
        }
        uint32_t cap = (uint32_t)((budget - need) / slotBytes / 16 * 16);
        if (cap > kDenseMaxSlots) cap = kDenseMaxSlots;
        if (cap >= P.denseTotal) { tileRows = tr; stages = n; slots = cap; }
      }
      if (tileRows) break;
    }
    if (!tileRows && !P.hll && P.nmeas <= 1 && P.neutralSafe && P.denseTotal <= kGlobalDenseMaxSlots) {
      // more slots than a CTA holds: one accumulator array in global memory for the whole grid; shared memory is all ring
      for (uint32_t tr : {3968u, 1920u, 896u}) {
        const uint32_t n = stagesIn(budget - 128 - 256, tr);
        if (n >= 2) {
          tileRows = tr; stages = n; slots = 16; P.denseGlobal = 1; P.denseFx = 0;
          // L2 atomics saturate at >= ~1M distinct addresses and contend below (tools/microbench/agg_microbench.cu):
          // replicate the slot array until it has about that many
          uint32_t reps = 1;
          while (reps < 8 && (uint64_t)P.denseTotal * reps * 2 <= kGlobalDenseMaxSlots && (uint64_t)P.denseTotal * reps < (1u << 20)) reps *= 2;
          P.denseGlobalReps = (uint8_t)reps;
          break;
        }
      }
    }
    // no layout holds the slots, or a batch without a full tile (all of it is the tail, which one CTA folds): hash table
    if (tileRows && fullTiles(tileRows) == 0) { tileRows = 0; slots = 8192; }
    if (!tileRows) { P.denseNd = 0; P.denseGlobal = 0; P.denseFx = 0; }
  }
  if (!tileRows && P.nmeas > 1) { P.denseNd = 0; return 0; }   // several measures share only the CTA's direct-indexed slots
  if (!tileRows) {
    for (uint32_t sl : {slots, slots / 2, slots / 4}) {
      for (uint32_t tr : {3968u, 1920u, 896u}) {  // 128 rows x (31 | 15 | 7) consumer warps
        const uint32_t n = stagesIn(budget - 128 - (size_t)sl * 8, tr);
        if (n >= 2) { tileRows = tr; stages = n; break; }
      }
      if (tileRows) { slots = sl; break; }
    }
    // (sixteen 4-byte columns with null bitmaps and the base counts take 62 KB per 896-row stage: two fit beside 8192 slots)
    if (!tileRows) throw EngineError("no stage layout fits the plan's columns into shared memory");
  }
  size_t stageBytes = 0;
  for (int c = 0; c < P.ncols; c++) {
    DevColumn &col = P.cols[c];
    if (col.in.mode == 0 || !col.used || col.width > 4 || col.rle) continue;
    col.staged = 1;
    col.smemValues = (uint32_t)stageBytes;
    // bit-packed bools and bitmaps copy one 16-byte chunk beyond the tile so that a non-zero
    // StartingIndex can read across the tile's last byte; full tiles always have those bytes.
    col.tileValueBytes = col.width ? tileRows * col.width : tileRows / 8 + 16;
    stageBytes += (col.tileValueBytes + 15) / 16 * 16;
    if (col.in.mode == 2) {
      col.hasNulls = 1;
      col.smemNulls = (uint32_t)stageBytes;
      col.tileNullBytes = tileRows / 8 + 16;
      stageBytes += (col.tileNullBytes + 15) / 16 * 16;
    }
  }
  P.smemBc = 0;
  P.tileBcBytes = 0;
  if (stageBc) {
    P.smemBc = (uint32_t)stageBytes;
    P.tileBcBytes = (tileRows + 4) * 4;   // one count more than rows (run length = difference), padded to 16 bytes
    stageBytes += P.tileBcBytes;
  }
  P.tileRows = tileRows;
  P.numStages = stages;
  P.numFullTiles = fullTiles(tileRows);
  P.stageBytes = (uint32_t)stageBytes;
  P.smemSlots = slots;
  P.tableBytes = P.denseNd != 0 ? (slots * denseSlotBytes(P.denseFx, P.hll) + 127) / 128 * 128 : slots * 8;
  if (P.nmeas > 1) {
    P.tableBytes = 0;
    for (int m = 0; m < P.nmeas; m++) P.tableBytes += measureRegionBytes(P, m);
  } else {
    describeMeasure(P, P.meas[0]);
  }
  return 128 + (size_t)P.tableBytes + stageBytes * P.numStages + P.bucketSmem;
}

// ---------------------------------------------------------------------------------------
// growth of the group table
// ---------------------------------------------------------------------------------------
// The reference sizes its hash map at 2 x rows for every batch and so never runs out (query/hash_reduction.cu:211-292);
// here the table starts L2-sized and doubles when it is half full.  Kernels notice on the device (DevTable::growAt
// raises the STOP flag at claim time): tile kernels whose launch the host waits for drain and are resumed after the
// growth; kernels the host does not wait for (direct-indexed ones) park new groups in the spill list; launches that
// cannot be resumed (merges, folds, the direct path) get their room up front.
__global__ void __launch_bounds__(256) rehashKernel(DevTable oldG, uint32_t n, DevTable newG) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t slot = oldG.claimed[i];
    const uint32_t to = globalFindOrClaim(newG, oldG.keys[slot], oldG.rows ? &oldG.rows[(size_t)slot * 4] : nullptr);
    if (to != 0xFFFFFFFFu) newG.acc[to] = oldG.acc[slot];
  }
}

__global__ void __launch_bounds__(256) mergeSpillKernel(DevTable G, uint32_t n, AggOp op) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const SpillEntry e = G.spill[i];
    globalUpdate(G, op, e.key, G.rows ? e.row : nullptr, e.val);
  }
}

struct TableCounters { uint32_t occupied, overflow, truncated, stop, spilled, spillOverflow; };

// Throws when the table's overflow counter is set.
static void checkOverflow(const AggState *st, uint32_t overflow) {
  if (!overflow) return;
  if (st->hllDense)
    throw EngineError("dense HLL state: more than " + std::to_string(kHllDenseMaxGroups) +
                      " dimension groups; recreate the AggState with AggSpec.ExpectedGroups > 4096 (entry mode) and replay the batches");
  throw EngineError("group table overflow: more than " + std::to_string(st->capacity) +
                    " slots needed; recreate the AggState with a larger AggSpec.ExpectedGroups and replay the batches");
}

static TableCounters readCounters(AggState *st, cudaStream_t s) {
  TableCounters c;
  uint32_t *pinned = st->resultHost + 10;   // (pinned: a pageable target costs a staging copy and ~100 us)
  ARES_CUDA(cudaMemcpyAsync(pinned, st->table.counters, sizeof(c), cudaMemcpyDeviceToHost, s));
  ARES_CUDA(cudaStreamSynchronize(s));
  memcpy(&c, pinned, sizeof(c));
  st->occUpper = c.occupied;
  st->resultHost[8] = c.occupied;
  return c;
}

// New table of `newCap` slots holding the groups of the old one; STOP flag cleared.
static void growTable(AggState *st, size_t newCap, cudaStream_t s) {
  if (st->hllDense) throw EngineError("dense HLL state: more than " + std::to_string(st->capacity) + " dimension groups");
  if (newCap > ((size_t)1 << 31)) throw EngineError("group table cannot grow beyond 2^31 slots");
  void *oldMem = st->mem;
  const DevTable oldG = st->table;
  uint32_t header[64];
  ARES_CUDA(cudaMemcpyAsync(header, oldG.counters, sizeof(header), cudaMemcpyDeviceToHost, s));
  ARES_CUDA(cudaStreamSynchronize(s));
  const uint32_t n = header[0];
  allocTable(st, newCap, s);   // fresh table (keys empty, counters 0), new claim list / progress / spill areas
  if (n) {
    int blocks = divUp(n, 256);
    if (blocks > smCount() * 8) blocks = smCount() * 8;
    rehashKernel<<<blocks, 256, 0, s>>>(oldG, n, st->table);
    checkLastError("rehash");
  }
  // progress of a stopped launch and parked rows survive the move
  ARES_CUDA(cudaMemcpyAsync(st->table.progress, oldG.progress, (size_t)(kProgressTail + 1) * 4, cudaMemcpyDeviceToDevice, s));
  const uint32_t spilled = header[4] < kSpillCap ? header[4] : kSpillCap;
  if (spilled) ARES_CUDA(cudaMemcpyAsync(st->table.spill, oldG.spill, (size_t)spilled * sizeof(SpillEntry), cudaMemcpyDeviceToDevice, s));
  uint32_t keep[2] = {header[4], header[5]};
  ARES_CUDA(cudaMemcpyAsync(st->table.counters + 4, keep, sizeof(keep), cudaMemcpyHostToDevice, s));
  ARES_CUDA(cudaMemcpyAsync(st->table.counters + 1, header + 1, 2 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));   // overflow / truncated
  ARES_CUDA(cudaStreamSynchronize(s));
  deviceFree(oldMem);
  st->occUpper = n;
}

// Folds parked rows (growing first when needed); loud when more rows were parked than the list holds.
static void settleTable(AggState *st, cudaStream_t s) {
  TableCounters c = readCounters(st, s);
  if (c.spillOverflow)
    throw EngineError("group table: more than " + std::to_string(kSpillCap) + " rows of new groups arrived from direct-indexed batches while the "
                      "table was full (a zone map far off the data); recreate the AggState with a larger AggSpec.ExpectedGroups and replay");
  checkOverflow(st, c.overflow);
  if (c.stop && st->unchecked > 0) {
    const uint32_t n = st->unchecked;
    st->unchecked = 0;
    throw EngineError("the group table reached its growth threshold (" + std::to_string(c.occupied) + " groups) during " + std::to_string(n) +
                      " batch(es) whose launches were not waited for — the number of groups jumped from under an eighth of that threshold; "
                      "rows were NOT folded: recreate the AggState with AggSpec.ExpectedGroups >= " + std::to_string((uint64_t)c.occupied * 4) +
                      " (or set ARESDB_B200_CHECK_EVERY_BATCH=1) and replay the batches");
  }
  if (!c.stop && !c.spilled) return;
  size_t cap = st->capacity;
  while ((uint64_t)c.occupied + c.spilled > cap / 4) cap <<= 1;   // settle at a quarter full at most
  if (cap != st->capacity || c.stop) growTable(st, cap == st->capacity ? cap << 1 : cap, s);
  if (c.spilled) {
    int blocks = divUp(c.spilled, 256);
    mergeSpillKernel<<<blocks, 256, 0, s>>>(st->table, c.spilled, st->op);
    checkLastError("mergeSpill");
    ARES_CUDA(cudaMemsetAsync(st->table.counters + 4, 0, 8, s));
    readCounters(st, s);
  }
}

// Room for a launch that cannot be resumed and inserts at most `bound` new groups.
static void ensureRoom(AggState *st, uint64_t bound, cudaStream_t s) {
  if (st->hllDense) return;
  if (st->occUpper + bound < st->table.growAt) { st->occUpper += bound; return; }
  settleTable(st, s);   // exact occupancy (and nothing parked)
  size_t cap = st->capacity;
  while (st->occUpper + bound >= cap / 2) cap <<= 1;
  if (cap != st->capacity) growTable(st, cap, s);
  st->occUpper += bound;
}

// An RLE column whose count vector IS the batch's base counts: its run p holds index position p.
static bool countsAreBaseCounts(const InputDesc &in, const BatchPlan &bp) {
  return bp.BaseCounts != nullptr && reinterpret_cast<const uint32_t *>(in.base) == bp.BaseCounts;
}

// Describes every input of the plan as the kernel will read it (before layoutStages), without device work.
// Archive batches: run-length encoded (mode 3) columns.
//  * the column whose count vector IS the batch's base counts has one value per index position: it is read like an
//    uncompressed column (values / null bitmap of its runs), no copy;
//  * up to kJitMaxRle other 1- to 4-byte RLE columns are FIRST-CLASS inputs of the kernel: decoded from their runs inside
//    the tile loop (jit_kernel_head.cuh ldrle) with a per-tile run hint computed by executePlan — HBM sees the runs, not
//    the rows;
//  * the others (and 8- / 16-byte ones, which the kernel reads row by row) are expanded once per batch into mode-2
//    scratch columns (one value + one validity bit per index position): described here, made by materialiseInputs.
// The layout and the kernel text depend on these descriptors and never on the addresses materialiseInputs sets:
// layoutStages (with jitAnalyzeDense) does not read DevColumn::in.base, and reads DevPlan::baseCounts only to test it
// for null.  That is what lets a batch's launches be scheduled before any of them runs.
static void describeInputs(DevPlan &P, const BatchPlan &bp) {
  const uint32_t n = P.numRows;
  int nrle = 0;
  for (int c = 0; c < P.ncols; c++) {
    DevColumn &col = P.cols[c];
    if (!col.used || col.in.mode != 3) continue;
    if (countsAreBaseCounts(col.in, bp) && col.in.length >= n) {   // run number == index position
      col.in.mode = 2;
      continue;
    }
    if (col.width <= 4 && nrle < kJitMaxRle && col.in.length > 0) {
      col.rle = 1;
      nrle++;
      continue;
    }
    col.expand = 1;
    col.in.base = nullptr;
    col.in.nullsOff = 0;
    col.in.valuesOff = (uint32_t)(((size_t)(n + 31) / 32 * 4 + 16 + 63) / 64 * 64);   // the null bitmap comes first
    col.in.length = n;
    col.in.mode = 2;
    col.in.startBit = 0;
  }
}

// Makes the inputs describeInputs described readable by the kernel of a laid-out plan: the expanded columns are made
// from the batch's RLE columns, and the first-class ones get their run hints.  Staged parts (values and null bitmaps of
// 1- to 4-byte columns, the base counts) are fetched by the TMA engine, which needs a 16-byte aligned source: a part that
// is not aligned is copied once, byte for byte (same bit offset).
static void materialiseInputs(DevPlan &P, const BatchPlan &bp, cudaStream_t s, std::vector<std::unique_ptr<Scratch>> &scratch) {
  const uint32_t n = P.numRows;
  auto alloc = [&](size_t bytes) {
    scratch.emplace_back(new Scratch(bytes, s));
    return scratch.back()->as<uint8_t>();
  };
  for (int c = 0; c < P.ncols; c++) {
    DevColumn &col = P.cols[c];
    if (!col.expand) continue;
    const InputDesc runs = makeColumnDesc(bp.Columns[c], /*allowWide=*/true);
    const size_t nullBytes = col.in.valuesOff;
    const size_t valueBytes = (col.width ? (size_t)n * col.width : (size_t)(n + 31) / 32 * 4) + 64;
    uint8_t *buf = alloc(nullBytes + valueBytes);
    int blocks = divUp((int64_t)(n + 31) / 32, 8);
    if (blocks > smCount() * 16) blocks = smCount() * 16;
    expandRleKernel<<<blocks, 256, 0, s>>>(runs, bp.BaseCounts, bp.StartCount, n, col.width, countsAreBaseCounts(runs, bp),
                                           buf + nullBytes, reinterpret_cast<uint32_t *>(buf));
    checkLastError("expandRle");
    col.in.base = buf;
  }
  auto misaligned = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; };
  for (int c = 0; c < P.ncols; c++) {
    DevColumn &col = P.cols[c];
    if (!col.used || col.rle || col.width > 4 || (col.in.mode != 1 && col.in.mode != 2)) continue;
    const uint8_t *values = col.in.base + col.in.valuesOff, *nulls = col.in.base + col.in.nullsOff;
    const bool hasNulls = col.in.mode == 2;
    if (!misaligned(values) && !(hasNulls && misaligned(nulls))) continue;
    // (the kernel reads the bytes of the batch's rows: a full tile's 16-byte bitmap over-read stays below row numRows - 1)
    const size_t bitBytes = ((size_t)n + col.in.startBit + 7) / 8;
    const size_t valueBytes = col.width ? (size_t)n * col.width : bitBytes, nullBytes = hasNulls ? (bitBytes + 15) / 16 * 16 : 0;
    uint8_t *buf = alloc(nullBytes + valueBytes);
    if (hasNulls) ARES_CUDA(cudaMemcpyAsync(buf, nulls, bitBytes, cudaMemcpyDefault, s));
    ARES_CUDA(cudaMemcpyAsync(buf + nullBytes, values, valueBytes, cudaMemcpyDefault, s));
    col.in.base = buf;
    col.in.nullsOff = 0;
    col.in.valuesOff = (uint32_t)nullBytes;
  }
  if (stagesBaseCounts(P) && misaligned(P.baseCounts)) {
    uint8_t *buf = alloc(((size_t)n + 1) * 4);
    ARES_CUDA(cudaMemcpyAsync(buf, P.baseCounts, ((size_t)n + 1) * 4, cudaMemcpyDefault, s));
    P.baseCounts = reinterpret_cast<const uint32_t *>(buf);
  }
  for (int c = 0; c < P.ncols; c++) {   // per-tile run hints of the first-class RLE columns (layoutStages sized the tiles)
    DevColumn &col = P.cols[c];
    if (!col.rle) continue;
    const uint32_t entries = (P.numRows + P.tileRows - 1) / P.tileRows + 2;
    uint32_t *hints = reinterpret_cast<uint32_t *>(alloc(sizeof(uint32_t) * entries));
    rleTileRunsKernel<<<divUp(entries, 256), 256, 0, s>>>(reinterpret_cast<const uint32_t *>(col.in.base), col.in.length, bp.BaseCounts,
                                                         bp.StartCount, P.numRows, P.tileRows, entries, hints);
    checkLastError("rleTileRuns");
    col.tileRun = hints;
  }
}

// Joined dimension tables: indexes + foreign-column batches go to device memory for the kernel's lifetime (joinMem).
static void uploadJoin(DevPlan &P, const BatchPlan &bp, cudaStream_t s, std::unique_ptr<Scratch> &joinMem) {
  P.join = nullptr;
  if (P.numForeignCols > 0 || P.numForeignTables > 0) {
    static thread_local DevJoin J;
    memset(&J, 0, sizeof(J));
    for (int t = 0; t < bp.NumForeignTables; t++) {
      const CuckooHashIndex &h = bp.ForeignTables[t].Index;
      if (h.buckets == nullptr || h.numBuckets <= 0 || h.keyBytes <= 0 || h.keyBytes > 4 || h.numHashes < 0 || h.numHashes > 4)
        throw EngineError("invalid CuckooHashIndex in BatchPlan.ForeignTables (fused path: keys of at most 4 bytes)");
      J.tables[t].buckets = h.buckets;
      for (int i = 0; i < 4; i++) J.tables[t].seeds[i] = h.seeds[i];
      J.tables[t].keyBytes = h.keyBytes; J.tables[t].numHashes = h.numHashes; J.tables[t].numBuckets = h.numBuckets;
    }
    for (int k = 0; k < bp.NumForeignColumns; k++) J.cols[k] = makeForeignDesc(bp.ForeignColumns[k].Column);
    joinMem.reset(new Scratch(sizeof(DevJoin), s));
    ARES_CUDA(cudaMemcpyAsync(joinMem->ptr, &J, sizeof(DevJoin), cudaMemcpyHostToDevice, s));
    ARES_CUDA(cudaStreamSynchronize(s));   // J is reused by the next call of this thread
    P.join = joinMem->as<DevJoin>();
  }
}

// one CTA per SM, or per full tile when there are fewer; a batch without a full tile is the tail of one CTA
static int launchGrid(const DevPlan &P) {
  int grid = smCount() < kMaxGridCtas ? smCount() : kMaxGridCtas;
  if ((uint32_t)grid > P.numFullTiles) grid = P.numFullTiles ? (int)P.numFullTiles : 1;
  return grid;
}

// One kernel launch of a batch (see scheduleBatch): the states it feeds, the plan it runs — the batch's plan, a dimension
// set's or one state's (measurePlan) — and that plan's device form, laid out for this batch.
struct Launch {
  AggState *sts[kJitMaxMeasures];
  int n;
  bool set;                // the plan of a dimension set (member dimensions)
  const BatchPlan *plan;
  DevPlan *P;
};

// Runs one launch of a batch: materialises its inputs, launches its kernel and, for a hash-table kernel, checks it and
// resumes it when the table's growth stopped it.
static void executePlan(const Launch &L, cudaStream_t s) {
  DevPlan &P = *L.P;
  AggState *st = L.sts[0];
  P.resume = 0;
  std::vector<std::unique_ptr<Scratch>> scratch;   // expanded / realigned columns, run hints: released in stream order
  materialiseInputs(P, *L.plan, s, scratch);
  std::unique_ptr<Scratch> joinMem;
  uploadJoin(P, *L.plan, s, joinMem);
  // hash-table kernels are checked after the launch and resumed when they stopped (a kernel that feeds several states is
  // direct-indexed)
  const bool resumable = P.denseNd == 0 && !st->hllDense;
  if (P.denseGlobal) {
    if (!st->denseAcc) {   // first use: 16 MB of accumulators at the neutral element (denseFoldKernel leaves them so)
      st->denseAcc = static_cast<unsigned long long *>(deviceAllocOrThrow((size_t)kGlobalDenseMaxSlots * sizeof(unsigned long long)));
      fillTableKernel<<<smCount() * 8, 256, 0, s>>>(st->denseAcc, st->denseAcc, kGlobalDenseMaxSlots, st->accNeutral);
      checkLastError("denseAcc fill");
    }
    P.denseAcc = st->denseAcc;
  }
  for (;;) {
    // Direct-indexed kernels are not waited for (see "growth of the group table"): what their flush may insert (the CTA
    // slots; the global slot array's fold) is reserved in every state's table up front, and their out-of-range rows park.
    for (int k = 0; k < L.n; k++) {
      if (P.denseNd != 0) ensureRoom(L.sts[k], (uint64_t)(P.memberDims ? P.meas[k].total : P.denseTotal), s);
      P.meas[k].G = L.sts[k]->table;      // (after a possible growth: the slices live in the table's allocation)
      P.meas[k].ctaAcc = L.sts[k]->ctaAcc;
    }
    P.ctaAcc = st->ctaAcc;
    jitLaunch(P, st->table, 128 + (size_t)P.tableBytes + (size_t)P.stageBytes * P.numStages + P.bucketSmem, launchGrid(P), s);
    if (P.denseGlobal) {
      DenseFold F;
      memset(&F, 0, sizeof(F));
      uint32_t stride = 1;
      for (int k = 0; k < P.denseNd; k++) {
        const DevInst &I = P.insts[P.denseInst[k]];
        F.lo[k] = P.denseLo[k]; F.cnt[k] = P.denseCnt[k]; F.step[k] = P.denseStep[k]; F.stride[k] = stride;
        F.rowOff[k] = I.rowOff; F.width[k] = I.width; F.nullOff[k] = I.nullOff;
        stride *= P.denseCnt[k] + 1;
      }
      F.nd = P.denseNd; F.total = P.denseTotal; F.reps = P.denseGlobalReps ? P.denseGlobalReps : 1;
      F.keyMode = P.keyMode; F.hashBits = P.hashBits; F.rowBytes = P.rowBytes; F.op = P.aggOp;
      F.neutral = P.accNeutral;
      int blocks = divUp((int64_t)P.denseTotal, 256);
      if (blocks > smCount() * 8) blocks = smCount() * 8;
      denseFoldKernel<<<blocks, 256, 0, s>>>(st->denseAcc, F, st->table);
      checkLastError("denseFold");
    }
    if (!resumable) return;   // a hash-table kernel ran: wait for it and resume it if the table stopped it
    // Waiting for every hash-table batch would cost a launch gap per batch (the host cannot prepare the next one while it
    // waits).  The wait is therefore adaptive: always for the first batch of a query, and from then on whenever the
    // occupancy last seen — read back then, or published by a finishing kernel into mapped pinned memory — is above an
    // eighth of the threshold.  A table that fills from under an eighth of its threshold within unwatched batches is
    // reported loudly at the next synchronising call (settleTable), never folded wrongly.
    static const bool everyBatch = [] { const char *e = getenv("ARESDB_B200_CHECK_EVERY_BATCH"); return e && e[0] == '1'; }();
    const uint64_t seen = st->resultHost[8] > st->occUpper ? st->resultHost[8] : st->occUpper;
    if (P.resume == 0 && st->everChecked && !everyBatch && st->unchecked < 64 && seen * 8 < st->table.growAt) {
      st->unchecked++;
      return;
    }
    const TableCounters c = readCounters(st, s);
    st->everChecked = true;
    checkOverflow(st, c.overflow);
    if (!c.stop && !c.spilled) { st->unchecked = 0; return; }
    if (c.stop && st->unchecked > 0) settleTable(st, s);   // raises: earlier unwatched batches stopped as well
    const bool stopped = c.stop != 0;
    settleTable(st, s);   // grows (a quarter full at most afterwards) and folds the parked groups
    if (!stopped) return;
    P.resume = 1;
  }
}

// ---------------------------------------------------------------------------------------
// the launches of a batch: one plan, or several measures over one scan (ExecuteBatchPlanMulti)
// ---------------------------------------------------------------------------------------
static bool hasSink(const BatchPlan &bp, int sink) {
  for (int i = 0; i < bp.NumInsts && i < ARES_MAX_PLAN_INSTS; i++)
    if (bp.Insts[i].Sink == sink) return true;
  return false;
}

// States that may share a plan: the same reduce mode, no HLL, and the same dimension layout unless the plan gives each
// state its own dimensions (member dimensions, checked by compilePlan).
static void checkSharedStates(AggState *const *sts, int n, const BatchPlan &bp) {
  const bool memberDims = hasSink(bp, PLAN_SINK_MEMBER_DIMENSION);
  for (int k = 0; k < n; k++) {
    if (sts[k]->hll) throw EngineError("AGGR_HLL states cannot share a plan");
    if (!memberDims && memcmp(sts[k]->spec.NumDimsPerDimWidth, sts[0]->spec.NumDimsPerDimWidth, NUM_DIM_WIDTH) != 0)
      throw EngineError("states differ in NumDimsPerDimWidth");
    if (sts[k]->spec.ReduceMode != sts[0]->spec.ReduceMode) throw EngineError("states differ in ReduceMode");
  }
}

// The plan of the states in `set` (bit k = state k): every instruction except the other states' measure, member filter
// and member dimension roots and the sub-expressions only they consume.  The kept states are renumbered in order; their
// member dimensions become PLAN_SINK_DIMENSION roots (ordinals in plan order: the states of a set have the same
// dimensions), and the member filters of a single state become ordinary filters.  `P` is `bp` compiled.
static void measurePlan(const DevPlan &P, const BatchPlan &bp, uint32_t set, BatchPlan &out) {
  bool drop[ARES_MAX_PLAN_INSTS] = {};
  for (int i = 0; i < bp.NumInsts; i++) {
    const PlanInst &pi = bp.Insts[i];
    const bool other = ((pi.Sink == PLAN_SINK_MEASURE || pi.Sink == PLAN_SINK_MEASURE_FILTER) && !((set >> pi.SinkArg) & 1u)) ||
                       (pi.Sink == PLAN_SINK_MEMBER_DIMENSION && (pi.SinkArg & set) == 0);
    if (other) forSubexpression(P, i, [&](int j) { drop[j] = true; });
  }
  const bool single = (set & (set - 1)) == 0;
  auto rank = [&](int k) { return (uint8_t)__builtin_popcount(set & ((1u << k) - 1u)); };
  memcpy(&out, &bp, sizeof(BatchPlan));
  int n = 0, dims = 0;
  for (int i = 0; i < bp.NumInsts; i++) {
    if (drop[i]) continue;
    PlanInst &pi = out.Insts[n++];
    pi = bp.Insts[i];
    if (pi.Sink == PLAN_SINK_MEASURE) pi.SinkArg = rank(pi.SinkArg);
    if (pi.Sink == PLAN_SINK_MEASURE_FILTER) {
      if (single) pi.Sink = PLAN_SINK_FILTER;
      pi.SinkArg = single ? 0 : rank(pi.SinkArg);
    }
    if (pi.Sink == PLAN_SINK_MEMBER_DIMENSION) { pi.Sink = PLAN_SINK_DIMENSION; pi.SinkArg = (uint8_t)dims++; }
  }
  out.NumInsts = n;
}

// The states of a plan with member dimensions grouped by their dimensions: one mask (bit k = state k) per distinct set
// of member dimension roots, in the order of each set's first state.
static std::vector<uint32_t> dimensionSets(int n, const BatchPlan &bp) {
  std::vector<std::vector<bool>> sig(n, std::vector<bool>(bp.NumInsts, false));
  for (int i = 0; i < bp.NumInsts; i++)
    for (int k = 0; k < n; k++)
      sig[k][i] = bp.Insts[i].Sink == PLAN_SINK_MEMBER_DIMENSION && ((bp.Insts[i].SinkArg >> k) & 1u);
  std::vector<uint32_t> sets;
  std::vector<int> lead;
  for (int k = 0; k < n; k++) {
    size_t j = 0;
    while (j < lead.size() && sig[lead[j]] != sig[k]) j++;
    if (j == lead.size()) { lead.push_back(k); sets.push_back(0); }
    sets[j] |= 1u << k;
  }
  return sets;
}

// The launches of one batch in launch order (a state is fed by exactly one), and the plans and device plans they use:
// the batch's plan, each state's own plan at most twice (in the batch and in its dimension set), one per dimension set.
// Thread-local, reused by every batch of the thread (BatchPlan has no default constructor: raw storage).
struct Schedule {
  static constexpr int kMaxPlans = 3 * kJitMaxMeasures;
  int count, nplans, ndev;
  Launch launch[kJitMaxMeasures];
  DevPlan dev[kMaxPlans + 1];
  alignas(BatchPlan) unsigned char planMem[kMaxPlans][sizeof(BatchPlan)];
  BatchPlan &newPlan() { assert(nplans < kMaxPlans); return *reinterpret_cast<BatchPlan *>(planMem[nplans++]); }
  DevPlan &newDevPlan() { assert(ndev <= kMaxPlans); return dev[ndev++]; }
  void add(AggState *const *sts, int n, const BatchPlan &plan, DevPlan &P, bool set) {
    Launch &L = launch[count++];
    std::copy(sts, sts + n, L.sts);
    L.n = n; L.set = set; L.plan = &plan; L.P = &P;
  }
};

// Schedules states sts[0..n) over `bp`, compiled for them into P (with `multi` when n > 1).  One state runs P.  Several
// share one kernel when each state's own plan (measurePlan) takes the CTA's direct-indexed slots and all of them fit a
// CTA together: P is then laid out with every measure in the form its own plan takes.  Otherwise, with member
// dimensions, each set of states with the same dimensions (dimensionSets order) is scheduled the same way, so a batch
// never runs more kernels than states; without, each state runs its own plan, in state order.
static void scheduleStates(Schedule &S, AggState *const *sts, int n, const BatchPlan &bp, DevPlan &P, bool set) {
  if (n == 1) {
    describeInputs(P, bp);
    layoutStages(P, sts[0]->spec.ExpectedGroups);
    S.add(sts, 1, bp, P, set);
    return;
  }
  BatchPlan *own[kJitMaxMeasures];
  DevPlan *Q[kJitMaxMeasures];
  bool shared = true;
  bool skipCount = true;
  uint32_t expected = 0;
  for (int k = 0; k < n; k++) {
    own[k] = &S.newPlan();
    measurePlan(P, bp, 1u << k, *own[k]);
    Q[k] = &S.newDevPlan();
    compilePlan(sts[k], *own[k], *Q[k]);
    describeInputs(*Q[k], *own[k]);
    layoutStages(*Q[k], sts[k]->spec.ExpectedGroups);
    shared = shared && Q[k]->denseNd != 0 && !Q[k]->denseGlobal;
    describeMeasure(*Q[k], P.meas[k]);
    skipCount = skipCount && Q[k]->skipCount;
    expected = sts[k]->spec.ExpectedGroups > expected ? sts[k]->spec.ExpectedGroups : expected;
    // member dimensions: every state packs its rows with the kernel's one key form (JIT_KW / JIT_ROW_BYTES)
    if (P.memberDims && (sts[k]->keyMode != sts[0]->keyMode ||
                         (sts[k]->keyMode == KEY_HASHED && sts[k]->rowLayout.rowBytes != sts[0]->rowLayout.rowBytes)))
      shared = false;
  }
  if (shared) {
    P.nmeas = (uint8_t)n;
    P.skipCount = skipCount;   // base counts are staged when some measure counts run lengths
    describeInputs(P, bp);
    if (layoutStages(P, expected) != 0) {
      S.add(sts, n, bp, P, set);
      return;
    }
  }
  if (!P.memberDims) {
    for (int k = 0; k < n; k++) S.add(&sts[k], 1, *own[k], *Q[k], false);
    return;
  }
  for (uint32_t mask : dimensionSets(n, bp)) {
    AggState *ss[kJitMaxMeasures];
    int m = 0;
    for (int k = 0; k < n; k++)
      if ((mask >> k) & 1u) ss[m++] = sts[k];
    BatchPlan &plan = S.newPlan();
    measurePlan(P, bp, mask, plan);
    DevPlan &Q1 = S.newDevPlan();
    compilePlan(ss[0], plan, Q1, ss, m);
    scheduleStates(S, ss, m, plan, Q1, true);
  }
}

// The one decision of which kernels a batch runs, for ExecuteBatchPlan (multi = false, n = 1), ExecuteBatchPlanMulti
// and the dry runs: validates the plan and schedules its launches (none for an empty batch) without device work;
// executePlan materialises each launch's inputs when it runs.  One state of ExecuteBatchPlanMulti runs the plan with its
// member filters and dimensions turned into plain ones.
static const Schedule &scheduleBatch(AggState *const *sts, int n, const BatchPlan &bp, bool multi) {
  static thread_local Schedule S;
  S.count = S.nplans = S.ndev = 0;
  if (multi) checkSharedStates(sts, n, bp);
  if (bp.NumRows > 0x7FFFFFFFu) throw EngineError("a batch holds at most 2^31-1 rows");
  DevPlan &P = S.newDevPlan();
  compilePlan(sts[0], bp, P, multi ? sts : nullptr, multi ? n : 0);
  if (bp.NumRows == 0) return S;
  const BatchPlan *plan = &bp;
  if (n == 1 && multi && (hasSink(bp, PLAN_SINK_MEASURE_FILTER) || hasSink(bp, PLAN_SINK_MEMBER_DIMENSION))) {
    BatchPlan &one = S.newPlan();
    measurePlan(P, bp, 1u, one);
    compilePlan(sts[0], one, P);
    plan = &one;
  }
  scheduleStates(S, sts, n, *plan, P, false);
  return S;
}

static void executeBatch(AggState *const *sts, int n, const BatchPlan &bp, bool multi, cudaStream_t s) {
  const Schedule &S = scheduleBatch(sts, n, bp, multi);
  for (int i = 0; i < S.count; i++) executePlan(S.launch[i], s);
}

static void mergeRows(AggState *st, const DimensionVector &in, const uint8_t *values, int length, cudaStream_t s) {
  if (length <= 0) return;
  for (int i = 0; i < NUM_DIM_WIDTH; i++)
    if (in.NumDimsPerDimWidth[i] != st->spec.NumDimsPerDimWidth[i]) throw EngineError("dimension layout differs from AggSpec");
  DimLayout L = makeDimLayout(in.NumDimsPerDimWidth, in.VectorCapacity);
  ensureRoom(st, (uint64_t)length, s);
  int blocks = divUp(length, 256);
  if (blocks > smCount() * 8) blocks = smCount() * 8;
  mergeRowsKernel<<<blocks, 256, 0, s>>>(in.DimValues, L, values, st->measWidth, st->op, length, st->keyMode,
                                        (uint8_t)st->hashBits, hllMode(st), st->table);
  checkLastError("AggStateMerge");
}

static int64_t groupCount(AggState *st, cudaStream_t s) {
  TableCounters c = readCounters(st, s);
  if (c.stop || c.spilled || c.spillOverflow) {
    settleTable(st, s);
    c = readCounters(st, s);
  }
  checkOverflow(st, c.overflow);
  return c.occupied;
}

// Dense HLL state -> carried rows.  Fills `block` (one dim row per group, capacity = groups, hash
// order) and, per hit register in (group, register) order, key / value / group ordinal.
struct DenseCarried {
  int groups = 0;
  int64_t entries = 0;
  Scratch block, hash, values, index;
};

// The claimed groups of a dense HLL state in the order of the reference hash of their dim row: the d-th group is in
// directory slot slotOf[order[d]], hash[d] is its hash.
struct DenseGroups {
  int n = 0;
  Scratch slotOf, hash, order;
};

static void denseGroups(AggState *st, cudaStream_t s, DenseGroups &out) {
  uint32_t c[2];
  ARES_CUDA(cudaMemcpyAsync(c, st->table.counters, sizeof(c), cudaMemcpyDeviceToHost, s));
  ARES_CUDA(cudaStreamSynchronize(s));
  checkOverflow(st, c[1]);
  const int n = (int)c[0];
  out.n = n;
  if (n == 0) return;
  const int tiles = divUp((int64_t)st->capacity, kCmpTile);
  Scratch state(scanStateBytes(tiles) + sizeof(uint32_t), s);
  ARES_CUDA(cudaMemsetAsync(state.ptr, 0, state.bytes, s));
  ScanTileState sst = makeScanState(state.ptr, tiles);
  uint32_t *dCount = reinterpret_cast<uint32_t *>(static_cast<uint8_t *>(state.ptr) + scanStateBytes(tiles));
  out.slotOf.reset(sizeof(uint32_t) * (size_t)n, s);
  out.hash.reset(sizeof(uint64_t) * (size_t)n, s);
  out.order.reset(sizeof(uint32_t) * (size_t)n, s);
  Scratch vals(sizeof(uint32_t) * (size_t)n, s);
  compactGroupsKernel<<<tiles, kCmpThreads, 0, s>>>(st->table, st->capacity, st->keyMode, 64, ~0ull, st->rowLayout.rowBytes, 4, sst,
                                                   out.slotOf.as<uint32_t>(), out.hash.as<uint64_t>(), vals.as<uint8_t>(), dCount);
  checkLastError("compactGroups");
  Scratch tmpK(sizeof(uint64_t) * (size_t)n, s), tmpV(sizeof(uint32_t) * (size_t)n, s);
  iotaKernel<<<divUp(n, 256), 256, 0, s>>>(out.order.as<uint32_t>(), n);
  sortKeyIndexPairs(out.hash.as<uint64_t>(), out.order.as<uint32_t>(), tmpK.as<uint64_t>(), tmpV.as<uint32_t>(), n, 64, s);
}

static void denseCarried(AggState *st, cudaStream_t s, DenseCarried &out, bool countOnly) {
  DenseGroups dg;
  denseGroups(st, s, dg);
  const int n = dg.n;
  out.groups = n;
  out.entries = 0;
  if (n == 0) return;
  uint32_t *slotOf = dg.slotOf.as<uint32_t>(), *order = dg.order.as<uint32_t>();
  Scratch counts(sizeof(uint32_t) * (size_t)n, s), offsets(sizeof(uint32_t) * ((size_t)n + 1), s);
  hllDenseCountKernel<<<n, 256, 0, s>>>(st->table.regs, st->table.acc, slotOf, order, counts.as<uint32_t>());
  checkLastError("hllDenseCount");
  hllDenseOffsetsKernel<<<1, 1024, 0, s>>>(counts.as<uint32_t>(), n, offsets.as<uint32_t>());
  checkLastError("hllDenseOffsets");
  uint32_t total = 0;
  ARES_CUDA(cudaMemcpyAsync(&total, offsets.as<uint32_t>() + n, 4, cudaMemcpyDeviceToHost, s));
  ARES_CUDA(cudaStreamSynchronize(s));
  out.entries = total;
  if (countOnly || total == 0) return;
  out.block.reset((size_t)st->rowLayout.rowBytes * n, s);
  out.hash.reset(sizeof(uint64_t) * (size_t)total, s);
  out.values.reset(sizeof(uint32_t) * (size_t)total, s);
  out.index.reset(sizeof(uint32_t) * (size_t)total, s);
  DimLayout L = makeDimLayout(st->spec.NumDimsPerDimWidth, n);
  emitGroupsKernel<<<divUp(n, 256), 256, 0, s>>>(st->table, st->keyMode, slotOf, order, (uint32_t)n, out.block.as<uint8_t>(), L, nullptr);
  checkLastError("emitGroups");
  hllDenseEmitKernel<<<n, 256, 0, s>>>(st->table.regs, st->table.acc, slotOf, order, dg.hash.as<uint64_t>(), offsets.as<uint32_t>(),
                                       out.hash.as<uint64_t>(), out.values.as<uint32_t>(), out.index.as<uint32_t>());
  checkLastError("hllDenseEmit");
  ARES_CUDA(cudaStreamSynchronize(s));  // the locals above are released in stream order; keep it simple
}

// Dense HLL state -> the final outputs of AggStateFinalizeHLL, straight from the register arrays.
static int64_t denseVectors(AggState *st, cudaStream_t s, uint8_t **dimValuesPtr, uint8_t **hllVectorPtr, size_t *hllVectorSizePtr,
                            uint16_t **hllDimRegIDCountPtr) {
  DenseGroups dg;
  denseGroups(st, s, dg);
  const int n = dg.n;
  if (n == 0) return 0;
  uint32_t *slotOf = dg.slotOf.as<uint32_t>(), *order = dg.order.as<uint32_t>();
  Scratch counts(sizeof(uint32_t) * (size_t)n, s), outIdx(sizeof(uint32_t) * (size_t)n, s), byteOff(sizeof(uint32_t) * (size_t)n, s);
  Scratch rowsOf(sizeof(uint32_t) * (size_t)n, s), totalsDev(sizeof(unsigned long long) * 2, s);
  hllDenseCountKernel<<<n, 256, 0, s>>>(st->table.regs, st->table.acc, slotOf, order, counts.as<uint32_t>());
  checkLastError("hllDenseCount");
  hllVectorLayoutKernel<<<1, 1024, 0, s>>>(counts.as<uint32_t>(), n, outIdx.as<uint32_t>(), byteOff.as<uint32_t>(), rowsOf.as<uint32_t>(),
                                          totalsDev.as<unsigned long long>());
  checkLastError("hllVectorLayout");
  // the groups' dim rows in hash order (the groups with registers are picked out of it below)
  Scratch blockAll((size_t)st->rowLayout.rowBytes * n, s);
  DimLayout Lin = makeDimLayout(st->spec.NumDimsPerDimWidth, n);
  emitGroupsKernel<<<divUp(n, 256), 256, 0, s>>>(st->table, st->keyMode, slotOf, order, (uint32_t)n, blockAll.as<uint8_t>(), Lin, nullptr);
  checkLastError("emitGroups");
  unsigned long long totals[2] = {0, 0};
  ARES_CUDA(cudaMemcpyAsync(totals, totalsDev.ptr, sizeof(totals), cudaMemcpyDeviceToHost, s));
  ARES_CUDA(cudaStreamSynchronize(s));
  const int dims = (int)totals[0];
  if (dims == 0) return 0;
  void *vec = deviceAllocOrThrow((size_t)totals[1]), *cnt = nullptr, *out = nullptr;
  try {
    cnt = deviceAllocOrThrow(sizeof(uint16_t) * (size_t)dims);
    out = deviceAllocOrThrow((size_t)st->rowLayout.rowBytes * dims);
  } catch (...) {
    deviceFree(vec);
    if (cnt) deviceFree(cnt);
    throw;
  }
  hllVectorEmitKernel<<<n, 256, 0, s>>>(st->table.regs, st->table.acc, slotOf, order, counts.as<uint32_t>(), outIdx.as<uint32_t>(),
                                        byteOff.as<uint32_t>(), static_cast<uint8_t *>(vec), static_cast<uint16_t *>(cnt));
  checkLastError("hllVectorEmit");
  DimLayout Lout = makeDimLayout(st->spec.NumDimsPerDimWidth, dims);
  gatherDims(blockAll.as<uint8_t>(), Lin, rowsOf.as<uint32_t>(), dims, static_cast<uint8_t *>(out), Lout, s);
  ARES_CUDA(cudaStreamSynchronize(s));
  *dimValuesPtr = static_cast<uint8_t *>(out);
  *hllVectorPtr = static_cast<uint8_t *>(vec);
  *hllVectorSizePtr = (size_t)totals[1];
  *hllDimRegIDCountPtr = static_cast<uint16_t *>(cnt);
  return dims;
}

// Arguments of finalizeSmallKernel / exportToPeersKernel for an output block of `capacity` rows; the exchange form
// (ordered = 0) unless the caller says otherwise.
static SmallFinalizeArgs smallFinalizeArgs(const AggState *st, int capacity, uint8_t *outBlock, uint8_t *outValues, uint32_t *resultDev) {
  SmallFinalizeArgs A;
  memset(&A, 0, sizeof(A));
  A.G = st->table;
  A.L = makeDimLayout(st->spec.NumDimsPerDimWidth, capacity);
  A.outBlock = outBlock; A.outValues = outValues; A.resultDev = resultDev;
  A.rowBytes = st->rowLayout.rowBytes; A.width = st->measWidth; A.outCapacity = capacity;
  A.keyMode = st->keyMode; A.hashBits = (uint8_t)st->hashBits; A.op = st->op;
  return A;
}

// Launches the single-launch finalize / exchange-form export of n states: n clusters, cluster c on args[c].
static void launchSmallFinalize(const SmallFinalizeArgs *args, int n, cudaStream_t s, const char *what) {
  static thread_local SmallFinalizeBatch B;
  for (int c = 0; c < n; c++) B.S[c] = args[c];
  finalizeSmallKernel<<<kFinCtas * n, 1024, 0, s>>>(B);
  checkLastError(what);
}

// The single-launch form takes states that announce at most kSmallFinalizeMax groups (their scratch is sized for it).
static bool smallFinalizeFits(const AggState *st, const DimensionVector &out) {
  return !st->hllDense && st->spec.ExpectedGroups <= (uint32_t)kSmallFinalizeMax && out.VectorCapacity > 0;
}

static SmallFinalizeArgs orderedFinalizeArgs(const AggState *st, const DimensionVector &out, uint8_t *outValues, bool ordered) {
  SmallFinalizeArgs A = smallFinalizeArgs(st, out.VectorCapacity, out.DimValues, outValues, st->resultDev);
  A.hashMask = testHash64Mask();
  A.hashA = reinterpret_cast<uint64_t *>(st->smallScratch);
  A.tmpK = A.hashA + kSmallFinalizeMax;
  A.idxA = reinterpret_cast<uint32_t *>(A.tmpK + kSmallFinalizeMax);
  A.tmpI = A.idxA + kSmallFinalizeMax;
  A.hist = A.tmpI + kSmallFinalizeMax;
  A.outHash = ordered ? out.HashValues : nullptr; A.outIndex = out.IndexVector;
  A.resultHost = st->resultHostDev;
  A.plusZero = st->spec.ReduceMode == ARES_REDUCE_HASH && (st->op == OP_SUM_F64 || st->op == OP_SUM_F32);
  A.ordered = ordered;
  return A;
}

static int64_t finalize(AggState *st, const DimensionVector &out, uint8_t *outValues, cudaStream_t s, bool ordered = true);
static int64_t finalizeLarge(AggState *st, const DimensionVector &out, uint8_t *outValues, cudaStream_t s, bool ordered);

// After the single-launch finalize of `st` and a synchronise: its group count, or the path that completes it.
static int64_t finishSmallFinalize(AggState *st, const DimensionVector &out, uint8_t *outValues, cudaStream_t s, bool ordered) {
  const uint32_t status = st->resultHost[1];
  if (status == SF_UNSETTLED) {   // grow / fold the parked rows, then once more (the table moved: new pointers)
    settleTable(st, s);
    return finalize(st, out, outValues, s, ordered);
  }
  if (status == SF_OK) return st->resultHost[0];
  if (status == SF_TABLE_OVERFLOW) checkOverflow(st, 1);
  if (status == SF_OUTPUT_TOO_SMALL) throw EngineError("output DimensionVector capacity is smaller than the number of groups");
  if (status == SF_PEER_LATE) throw EngineError("exchange over peer memory: a peer's part did not arrive within the wait bound");
  if (status == SF_PART_TRUNCATED) throw EngineError("exchange part truncated: a rank held more rows than the fixed part carries; repeat the exchange with exact sizes");
  // SF_TOO_MANY: more groups than one CTA sorts — the multi-launch path
  return finalizeLarge(st, out, outValues, s, ordered);
}

static void checkOutputLayout(const AggState *st, const DimensionVector &out) {
  for (int i = 0; i < NUM_DIM_WIDTH; i++)
    if (out.NumDimsPerDimWidth[i] != st->spec.NumDimsPerDimWidth[i]) throw EngineError("dimension layout differs from AggSpec");
}

static int64_t finalize(AggState *st, const DimensionVector &out, uint8_t *outValues, cudaStream_t s, bool ordered) {
  checkOutputLayout(st, out);
  if (st->hllDense) {  // carried rows straight from the register arrays (already in key order)
    DenseCarried dc;
    denseCarried(st, s, dc, false);
    if (dc.entries == 0) return 0;
    if (dc.entries > out.VectorCapacity) throw EngineError("output DimensionVector capacity is smaller than the number of rows");
    DimLayout Lin = makeDimLayout(out.NumDimsPerDimWidth, dc.groups), Lout = makeDimLayout(out.NumDimsPerDimWidth, out.VectorCapacity);
    gatherDims(dc.block.as<uint8_t>(), Lin, dc.index.as<uint32_t>(), (int)dc.entries, out.DimValues, Lout, s);
    ARES_CUDA(cudaMemcpyAsync(outValues, dc.values.ptr, sizeof(uint32_t) * (size_t)dc.entries, cudaMemcpyDeviceToDevice, s));
    if (out.HashValues)
      ARES_CUDA(cudaMemcpyAsync(out.HashValues, dc.hash.ptr, sizeof(uint64_t) * (size_t)dc.entries, cudaMemcpyDeviceToDevice, s));
    if (out.IndexVector) iotaKernel<<<divUp(dc.entries, 256), 256, 0, s>>>(out.IndexVector, (int)dc.entries);
    ARES_CUDA(cudaStreamSynchronize(s));
    return dc.entries;
  }
  if (smallFinalizeFits(st, out)) {
    // results of up to 32768 groups: ONE launch (claim list -> hash -> sort -> merge -> emit) and ONE synchronise;
    // the group count comes back through mapped pinned memory
    const SmallFinalizeArgs A = orderedFinalizeArgs(st, out, outValues, ordered);
    launchSmallFinalize(&A, 1, s, "finalizeSmall");
    ARES_CUDA(cudaStreamSynchronize(s));
    return finishSmallFinalize(st, out, outValues, s, ordered);
  }
  return finalizeLarge(st, out, outValues, s, ordered);
}

// AggStatesFinalize: every state that can takes ONE shared launch (one cluster each) and ONE synchronise; the others, and
// those the launch could not finish (parked rows, more than kSmallFinalizeMax groups), complete through finalize's
// paths.  groups[k] = the group count of state k, or -1 when it failed; the error then names every failed state.
static void finalizeStates(AggState *const *sts, int numStates, const DimensionVector *outs, uint8_t *const *outValues, int64_t *groups,
                           cudaStream_t s) {
  SmallFinalizeArgs args[kMaxLaunchStates];
  bool small[kMaxLaunchStates];
  int m = 0;
  for (int k = 0; k < numStates; k++) {
    small[k] = smallFinalizeFits(sts[k], outs[k]);
    if (small[k]) args[m++] = orderedFinalizeArgs(sts[k], outs[k], outValues[k], true);
  }
  if (m > 0) {
    launchSmallFinalize(args, m, s, "AggStatesFinalize");
    ARES_CUDA(cudaStreamSynchronize(s));
  }
  std::string failed;
  for (int k = 0; k < numStates; k++) {
    try {
      groups[k] = small[k] ? finishSmallFinalize(sts[k], outs[k], outValues[k], s, true) : finalize(sts[k], outs[k], outValues[k], s);
    } catch (const std::exception &e) {
      groups[k] = -1;
      failed += (failed.empty() ? "" : "\n") + std::string("state ") + std::to_string(k) + ": " + e.what();
    }
  }
  if (!failed.empty()) throw EngineError(failed);
}

// The multi-launch finalize: results of more than kSmallFinalizeMax groups (or states that announce more).
static int64_t finalizeLarge(AggState *st, const DimensionVector &out, uint8_t *outValues, cudaStream_t s, bool ordered) {
  const int width = st->measWidth;
  const bool plusZero = st->spec.ReduceMode == ARES_REDUCE_HASH && (st->op == OP_SUM_F64 || st->op == OP_SUM_F32);
  const int64_t occupied = groupCount(st, s);
  if (occupied == 0) return 0;
  const int n = (int)occupied;
  // 1. the claimed slots (claim order) with their reference hash and accumulator
  Scratch slotOf(sizeof(uint32_t) * (size_t)n, s), hash(sizeof(uint64_t) * (size_t)n, s), vals((size_t)width * n, s);
  {
    int blocks = divUp(n, 256);
    if (blocks > smCount() * 8) blocks = smCount() * 8;
    gatherClaimedKernel<<<blocks, 256, 0, s>>>(st->table, (uint32_t)n, st->keyMode, (uint8_t)st->hashBits, testHash64Mask(),
                                               st->rowLayout.rowBytes, width, slotOf.as<uint32_t>(), hash.as<uint64_t>(),
                                               vals.as<uint8_t>());
  }
  checkLastError("gatherClaimed");
  // 2. sort the groups by hash (stable), 3. merge equal hashes (reference group identity)
  Scratch order(sizeof(uint32_t) * (size_t)n, s), tmpK(sizeof(uint64_t) * (size_t)n, s), tmpV(sizeof(uint32_t) * (size_t)n, s);
  iotaKernel<<<divUp(n, 256), 256, 0, s>>>(order.as<uint32_t>(), n);
  if (!ordered) {
    // exchange form: the occupied slots as they are (no hash order, no merge of colliding hashes —
    // the receiving state's own finalize does both)
    if (n > out.VectorCapacity) throw EngineError("output DimensionVector capacity is smaller than the number of groups");
    DimLayout Lx = makeDimLayout(out.NumDimsPerDimWidth, out.VectorCapacity);
    emitGroupsKernel<<<divUp(n, 256), 256, 0, s>>>(st->table, st->keyMode, slotOf.as<uint32_t>(), order.as<uint32_t>(), (uint32_t)n,
                                                   out.DimValues, Lx, out.IndexVector);
    checkLastError("emitGroups");
    ARES_CUDA(cudaMemcpyAsync(outValues, vals.ptr, (size_t)width * n, cudaMemcpyDeviceToDevice, s));
    ARES_CUDA(cudaStreamSynchronize(s));
    return n;
  }
  sortKeyIndexPairs(hash.as<uint64_t>(), order.as<uint32_t>(), tmpK.as<uint64_t>(), tmpV.as<uint32_t>(), n, st->hashBits, s);
  Scratch rep(sizeof(uint32_t) * (size_t)n, s);
  Scratch mergedVals((size_t)width * n, s);
  const int g = reduceByHash(hash.as<uint64_t>(), order.as<uint32_t>(), vals.as<uint8_t>(), width, st->op, n,
                             rep.as<uint32_t>(), mergedVals.as<uint8_t>(), s,
                             n <= out.VectorCapacity ? out.HashValues : nullptr);
  if (g > out.VectorCapacity) throw EngineError("output DimensionVector capacity is smaller than the number of groups");
  // 4. emit in the reference's layout
  DimLayout L = makeDimLayout(out.NumDimsPerDimWidth, out.VectorCapacity);
  int blocks = divUp(g, 256);
  emitGroupsKernel<<<blocks, 256, 0, s>>>(st->table, st->keyMode, slotOf.as<uint32_t>(), rep.as<uint32_t>(), (uint32_t)g,
                                          out.DimValues, L, out.IndexVector);
  checkLastError("emitGroups");
  if (plusZero) {
    // The reference's hash map folds every value into a slot that starts at the identity +0.0
    // (query/hash_reduction.cu:246-249 + the map's unused element), so a group whose values are all -0.0 ends
    // at +0.0 there, while its sort-reduce (and this table, whose neutral element is -0.0) keeps -0.0.
    copyPlusZeroKernel<<<divUp(g, 256), 256, 0, s>>>(mergedVals.as<uint8_t>(), outValues, g, width);
    checkLastError("copyPlusZero");
  } else {
    ARES_CUDA(cudaMemcpyAsync(outValues, mergedVals.ptr, (size_t)width * g, cudaMemcpyDeviceToDevice, s));
  }
  ARES_CUDA(cudaStreamSynchronize(s));
  return g;
}

// Folds the exchange parts of numStates non-HLL states (AggStatesMergeParts; with `flags`, each state's CTAs first wait
// for its senders' flags) with one launch.
static void mergeParts(AggState *const *sts, int numStates, const uint8_t *slots, int numParts, size_t slotStride, int capRows,
                       const size_t *partOffset, const size_t *dimOffset, const size_t *valuesOffset, const uint32_t *flags,
                       uint32_t epoch, cudaStream_t s) {
  static thread_local MergePartsArgs M;
  memset(&M, 0, sizeof(M));
  for (int k = 0; k < numStates; k++) {
    AggState *st = sts[k];
    ensureRoom(st, (uint64_t)numParts * (uint64_t)capRows, s);   // (may move the table: read it afterwards)
    MergeStateArgs &S = M.S[k];
    S.G = st->table;
    S.L = makeDimLayout(st->spec.NumDimsPerDimWidth, capRows);
    S.partOff = partOffset[k]; S.dimOff = dimOffset[k]; S.valOff = valuesOffset[k];
    S.width = st->measWidth; S.op = (uint8_t)st->op; S.keyMode = (uint8_t)st->keyMode; S.hashBits = (uint8_t)st->hashBits;
  }
  M.slots = slots; M.slotStride = slotStride; M.flags = flags; M.numParts = numParts; M.epoch = epoch;
  const int perState = smCount() * 2 / numStates;
  mergePartsKernel<<<dim3(perState > 0 ? perState : 1, numStates), 256, 0, s>>>(M);
  checkLastError("mergeParts");
}

// Exchange-form export of numStates states into sub-parts of this rank's slot (peerSlots[myRank]) and, with peerFlags, the
// copy into every peer's slot plus the arrival flags: one launch, asynchronous.
static void exportPartsToPeers(AggState *const *sts, int numStates, uint8_t *const *peerSlots, uint32_t *const *peerFlags, int numPeers,
                               int myRank, const size_t *partBytes, int capRows, const size_t *partOffset, const size_t *dimOffset,
                               const size_t *valuesOffset, uint32_t epoch, cudaStream_t s) {
  static thread_local PeerExportArgs E;
  memset(&E, 0, sizeof(E));
  for (int r = 0; r < numPeers; r++) { E.peerSlot[r] = peerSlots[r]; E.peerFlag[r] = peerFlags ? peerFlags[r] : nullptr; }
  for (int k = 0; k < numStates; k++) {
    uint8_t *part = peerSlots[myRank] + partOffset[k];
    E.F[k] = smallFinalizeArgs(sts[k], capRows, part + dimOffset[k], part + valuesOffset[k], reinterpret_cast<uint32_t *>(part));
    E.partOffset[k] = partOffset[k];
    E.partBytes[k] = partBytes[k];
  }
  E.numPeers = (uint32_t)numPeers; E.myRank = (uint32_t)myRank; E.epoch = epoch;
  exportToPeersKernel<<<kFinCtas * numStates, 1024, 0, s>>>(E);
  checkLastError("exportToPeers");
}

// HLL state -> the reference's final outputs.  AggStateFinalize on such a state already yields the
// carried form (one row per (group, register) entry, key-ascending, value = max rho << 16 | reg);
// this runs it into scratch buffers and then the shared register-vector stage of hll.cu.  The dim
// block (VectorCapacity == number of groups) and the two vectors are allocated with deviceMalloc.
static int64_t finalizeHLL(AggState *st, uint8_t **dimValuesPtr, uint8_t **hllVectorPtr, size_t *hllVectorSizePtr,
                           uint16_t **hllDimRegIDCountPtr, cudaStream_t s) {
  if (!st->hll) throw EngineError("AggStateFinalizeHLL needs a state created with AGGR_HLL");
  if (!dimValuesPtr || !hllVectorPtr || !hllVectorSizePtr || !hllDimRegIDCountPtr) throw EngineError("null output pointer");
  *dimValuesPtr = nullptr; *hllVectorPtr = nullptr; *hllVectorSizePtr = 0; *hllDimRegIDCountPtr = nullptr;
  if (st->hllDense) return denseVectors(st, s, dimValuesPtr, hllVectorPtr, hllVectorSizePtr, hllDimRegIDCountPtr);
  const int64_t entries = groupCount(st, s);
  if (entries == 0) return 0;
  const int n = (int)entries;
  const int rowBytes = st->rowLayout.rowBytes;
  Scratch block((size_t)rowBytes * n, s), hash(sizeof(uint64_t) * (size_t)n, s), index(sizeof(uint32_t) * (size_t)n, s);
  Scratch values(sizeof(uint32_t) * (size_t)n, s);
  DimensionVector carried;
  carried.DimValues = block.as<uint8_t>();
  carried.HashValues = hash.as<uint64_t>();
  carried.IndexVector = index.as<uint32_t>();
  carried.VectorCapacity = n;
  for (int i = 0; i < NUM_DIM_WIDTH; i++) carried.NumDimsPerDimWidth[i] = st->spec.NumDimsPerDimWidth[i];
  const int64_t g = finalize(st, carried, values.as<uint8_t>(), s);
  if (g != entries) throw EngineError("HLL state: duplicate keys in the group table");
  const int dims = hllRegisterVectors(hash.as<uint64_t>(), values.as<uint32_t>(), index.as<uint32_t>(), n, hllVectorPtr,
                                      hllVectorSizePtr, hllDimRegIDCountPtr, s);
  void *out = nullptr;
  try {
    out = deviceAllocOrThrow((size_t)rowBytes * dims);
  } catch (...) {
    deviceFree(*hllVectorPtr); deviceFree(*hllDimRegIDCountPtr);
    *hllVectorPtr = nullptr; *hllDimRegIDCountPtr = nullptr;
    throw;
  }
  DimLayout Lin = makeDimLayout(carried.NumDimsPerDimWidth, n), Lout = makeDimLayout(carried.NumDimsPerDimWidth, dims);
  gatherDims(block.as<uint8_t>(), Lin, index.as<uint32_t>(), dims, static_cast<uint8_t *>(out), Lout, s);
  ARES_CUDA(cudaStreamSynchronize(s));
  *dimValuesPtr = static_cast<uint8_t *>(out);
  return dims;
}

// HLL state -> the groups of finalizeHLL and HLL.Compute of each (hll_estimate.cu).  The register vectors stay on the
// device and are freed here; the dim block and the estimates are allocated with deviceMalloc.
static int64_t finalizeHLLEstimate(AggState *st, uint8_t **dimValuesPtr, double **estimatesPtr, cudaStream_t s) {
  if (!st->hll) throw EngineError("AggStateFinalizeHLLEstimate needs a state created with AGGR_HLL");
  if (!dimValuesPtr || !estimatesPtr) throw EngineError("null output pointer");
  *dimValuesPtr = nullptr; *estimatesPtr = nullptr;
  uint8_t *dims = nullptr, *vec = nullptr;
  uint16_t *counts = nullptr;
  size_t vecBytes = 0;
  const int64_t g = finalizeHLL(st, &dims, &vec, &vecBytes, &counts, s);
  if (g == 0) return 0;
  void *est = nullptr;
  try {
    est = deviceAllocOrThrow(sizeof(double) * (size_t)g);
    hllEstimates(vec, counts, (int)g, static_cast<double *>(est), s);
    ARES_CUDA(cudaStreamSynchronize(s));
  } catch (...) {
    deviceFree(vec); deviceFree(counts); deviceFree(dims);
    if (est) deviceFree(est);
    throw;
  }
  deviceFree(vec); deviceFree(counts);
  *dimValuesPtr = dims;
  *estimatesPtr = static_cast<double *>(est);
  return g;
}

// The dry runs: schedules `plan` for AggStates described by `specs`, without device memory.  A schedule of one launch for
// all of them is generated and NVRTC-compiled: returns the cubin size, and *sourceOut (optional) gets a malloc'd copy of
// the kernel's shape-specific source.  Any other schedule is reported as an error that says which kernels run instead.
static size_t dryRun(const AggSpec *specs, int n, const BatchPlan &plan, bool multi, char **sourceOut) {
  AggState st[kJitMaxMeasures] = {}, *sts[kJitMaxMeasures];
  for (int k = 0; k < n; k++) {
    describeState(&st[k], specs[k]);
    st[k].capacity = st[k].hllDense ? kHllDenseSlots : 0;
    sts[k] = &st[k];
  }
  const Schedule &S = scheduleBatch(sts, n, plan, multi);
  if (S.count == 0) throw EngineError("the batch is empty: no kernel runs");
  if (S.count == 1 && S.launch[0].n == n) {
    std::string src;
    const size_t size = jitCompileOnly(*S.launch[0].P, &src);
    if (sourceOut) *sourceOut = strdup(src.c_str());
    return size;
  }
  bool perState = true, perSet = true;
  std::string groups;
  for (int i = 0; i < S.count; i++) {
    const Launch &L = S.launch[i];
    const bool direct = L.P->denseNd != 0;
    perState = perState && L.n == 1 && !(L.set && direct);
    perSet = perSet && L.set && direct;
    groups += i ? ", {" : "{";
    for (int j = 0; j < L.n; j++) groups += (j ? ", " : "") + std::to_string(std::find(sts, sts + n, L.sts[j]) - sts);
    groups += direct ? "} direct-indexed" : "}";
  }
  if (perState) throw EngineError("this plan and zone map run one kernel per state (no shared direct-indexed form)");
  if (perSet)
    throw EngineError("this plan and zone map run one kernel per dimension set (" + std::to_string(S.count) + " sets, each direct-indexed)");
  throw EngineError("this plan and zone map run " + std::to_string(S.count) + " kernels, one kernel per group of states: " + groups);
}

}  // namespace aresb

using namespace aresb;

extern "C" {

CGoCallResHandle AggStateCreate(AggSpec spec, void *cudaStream, int device) {
  CGoCallResHandle h = {nullptr, nullptr};
  try {
    ARES_CUDA(cudaSetDevice(device));
    h.res = createState(spec, (cudaStream_t)cudaStream, device);
  } catch (const std::exception &e) {
    h.pStrErr = strdup((std::string("AggStateCreate: ") + e.what()).c_str());
  }
  return h;
}

CGoCallResHandle ExecuteBatchPlan(void *state, const BatchPlan *plan, void *cudaStream, int device) {
  return guarded("ExecuteBatchPlan", device, [&]() -> int64_t {
    if (!plan) throw EngineError("null plan");
    AggState *st = asState(state);
    executeBatch(&st, 1, *plan, false, (cudaStream_t)cudaStream);
    return 0;
  });
}

CGoCallResHandle ExecuteBatchPlanMulti(void *const *states, int numStates, const BatchPlan *plan, void *cudaStream, int device) {
  return guarded("ExecuteBatchPlanMulti", device, [&]() -> int64_t {
    if (!plan) throw EngineError("null plan");
    if (!states || numStates < 1 || numStates > kJitMaxMeasures) throw EngineError("numStates must be 1.." + std::to_string(kJitMaxMeasures));
    AggState *sts[kJitMaxMeasures];
    for (int k = 0; k < numStates; k++) sts[k] = asState(states[k]);
    executeBatch(sts, numStates, *plan, true, (cudaStream_t)cudaStream);
    return 0;
  });
}

CGoCallResHandle AggStateMerge(void *state, DimensionVector inputKeys, uint8_t *inputValues, int length,
                               void *cudaStream, int device) {
  return guarded("AggStateMerge", device, [&]() -> int64_t {
    mergeRows(asState(state), inputKeys, inputValues, length, (cudaStream_t)cudaStream);
    return 0;
  });
}

CGoCallResHandle AggStateGroupCount(void *state, void *cudaStream, int device) {
  return guarded("AggStateGroupCount", device, [&]() -> int64_t {
    AggState *st = asState(state);
    if (st->hllDense) {  // rows of the carried form = registers that were hit
      DenseCarried dc;
      denseCarried(st, (cudaStream_t)cudaStream, dc, true);
      return dc.entries;
    }
    return groupCount(st, (cudaStream_t)cudaStream);
  });
}

CGoCallResHandle AggStateFinalize(void *state, DimensionVector outputKeys, uint8_t *outputValues, void *cudaStream,
                                  int device) {
  return guarded("AggStateFinalize", device, [&]() -> int64_t {
    return finalize(asState(state), outputKeys, outputValues, (cudaStream_t)cudaStream);
  });
}

CGoCallResHandle AggStateExport(void *state, DimensionVector outputKeys, uint8_t *outputValues, void *cudaStream,
                                int device) {
  return guarded("AggStateExport", device, [&]() -> int64_t {
    return finalize(asState(state), outputKeys, outputValues, (cudaStream_t)cudaStream, false);
  });
}

// ---- several states per launch (the queries of one request) ----
// The states of one call: 1..kMaxLaunchStates distinct, non-HLL AggStates.
static void requestStates(void *const *states, int numStates, AggState **sts) {
  if (states == nullptr) throw EngineError("states is null");
  if (numStates < 1 || numStates > kMaxLaunchStates) throw EngineError("numStates must be 1.." + std::to_string(kMaxLaunchStates));
  for (int k = 0; k < numStates; k++) {
    sts[k] = asState(states[k]);
    if (sts[k]->hll) throw EngineError("state " + std::to_string(k) + " is AGGR_HLL: HLL states exchange through AggStateExport");
    for (int j = 0; j < k; j++)
      if (sts[j] == sts[k]) throw EngineError("state " + std::to_string(k) + " appears twice");
  }
}

// Checks the per-state sub-part layout of an exchange slot: 16-byte aligned offsets, the header in front of the dimension
// block, the dimension block in front of the measures, every sub-part inside the slot and no two overlapping.  Returns
// each sub-part's size (a multiple of 16) in partBytes.
static void checkSlotLayout(AggState *const *sts, int numStates, size_t slotBytes, int capRows, const size_t *partOffset,
                            const size_t *dimOffset, const size_t *valuesOffset, size_t *partBytes) {
  if (!partOffset || !dimOffset || !valuesOffset) throw EngineError("partOffset / dimOffset / valuesOffset must not be null");
  if (capRows <= 0 || capRows > kSmallFinalizeMax) throw EngineError("capRows must be in [1, 32768]");
  if (slotBytes % 16 != 0) throw EngineError("slotBytes must be a multiple of 16");
  for (int k = 0; k < numStates; k++) {
    const std::string who = "state " + std::to_string(k) + ": ";
    if (partOffset[k] % 16 || dimOffset[k] % 16 || valuesOffset[k] % 16) throw EngineError(who + "offsets must be multiples of 16");
    const DimLayout L = makeDimLayout(sts[k]->spec.NumDimsPerDimWidth, capRows);
    size_t dimBytes = 0;
    for (int d = 0; d < L.numDims; d++) dimBytes = std::max<size_t>(dimBytes, (size_t)L.nullOff[d] + (size_t)capRows);
    if (dimOffset[k] < 16 || valuesOffset[k] < dimOffset[k] + dimBytes)
      throw EngineError(who + "the header (16 bytes), the dimension block and the measures must follow each other");
    partBytes[k] = (valuesOffset[k] + (size_t)sts[k]->measWidth * (size_t)capRows + 15) / 16 * 16;
    if (partOffset[k] > slotBytes || partBytes[k] > slotBytes - partOffset[k]) throw EngineError(who + "the sub-part does not fit the slot");
    for (int j = 0; j < k; j++)
      if (partOffset[j] < partOffset[k] + partBytes[k] && partOffset[k] < partOffset[j] + partBytes[j])
        throw EngineError(who + "the sub-part overlaps that of state " + std::to_string(j));
  }
}

CGoCallResHandle AggStatesFinalize(void *const *states, int numStates, const DimensionVector *outputKeys, uint8_t *const *outputValues,
                                   int64_t *groups, void *cudaStream, int device) {
  return guarded("AggStatesFinalize", device, [&]() -> int64_t {
    AggState *sts[kMaxLaunchStates];
    requestStates(states, numStates, sts);
    if (!outputKeys || !outputValues || !groups) throw EngineError("outputKeys / outputValues / groups must not be null");
    for (int k = 0; k < numStates; k++) {
      try {
        checkOutputLayout(sts[k], outputKeys[k]);
      } catch (const EngineError &e) {
        throw EngineError("state " + std::to_string(k) + ": " + e.what());
      }
    }
    finalizeStates(sts, numStates, outputKeys, outputValues, groups, (cudaStream_t)cudaStream);
    return 0;
  });
}

CGoCallResHandle AggStatesExportPartsToPeers(void *const *states, int numStates, uint8_t *const *peerSlots, uint32_t *const *peerFlags,
                                             int numPeers, int myRank, size_t slotBytes, int capRows, const size_t *partOffset,
                                             const size_t *dimOffset, const size_t *valuesOffset, uint32_t epoch, void *cudaStream,
                                             int device) {
  return guarded("AggStatesExportPartsToPeers", device, [&]() -> int64_t {
    AggState *sts[kMaxLaunchStates];
    requestStates(states, numStates, sts);
    if (!peerSlots) throw EngineError("peerSlots is null");
    if (numPeers < 1 || numPeers > kMaxPeers || myRank < 0 || myRank >= numPeers)
      throw EngineError("numPeers must be 1..16 and myRank < numPeers");
    size_t partBytes[kMaxLaunchStates];
    checkSlotLayout(sts, numStates, slotBytes, capRows, partOffset, dimOffset, valuesOffset, partBytes);
    for (int r = 0; r < numPeers; r++)
      if ((r == myRank || peerFlags) && (!peerSlots[r] || (peerFlags && !peerFlags[r]))) throw EngineError("null peer slot or flag");
    exportPartsToPeers(sts, numStates, peerSlots, peerFlags, numPeers, myRank, partBytes, capRows, partOffset, dimOffset, valuesOffset,
                       epoch, (cudaStream_t)cudaStream);
    return 0;
  });
}

CGoCallResHandle AggStatesMergeParts(void *const *states, int numStates, const uint8_t *slots, int numParts, size_t slotStride, int capRows,
                                     const size_t *partOffset, const size_t *dimOffset, const size_t *valuesOffset, const uint32_t *flags,
                                     uint32_t epoch, void *cudaStream, int device) {
  return guarded("AggStatesMergeParts", device, [&]() -> int64_t {
    AggState *sts[kMaxLaunchStates];
    requestStates(states, numStates, sts);
    if (!slots) throw EngineError("slots is null");
    if (numParts < 1 || numParts > kMaxPeers) throw EngineError("numParts must be 1..16");
    size_t partBytes[kMaxLaunchStates];
    checkSlotLayout(sts, numStates, slotStride, capRows, partOffset, dimOffset, valuesOffset, partBytes);
    mergeParts(sts, numStates, slots, numParts, slotStride, capRows, partOffset, dimOffset, valuesOffset, flags, epoch,
               (cudaStream_t)cudaStream);
    return 0;
  });
}

CGoCallResHandle AggStateFinalizeHLL(void *state, uint8_t **dimValuesPtr, uint8_t **hllVectorPtr, size_t *hllVectorSizePtr,
                                     uint16_t **hllDimRegIDCountPtr, void *cudaStream, int device) {
  return guarded("AggStateFinalizeHLL", device, [&]() -> int64_t {
    return finalizeHLL(asState(state), dimValuesPtr, hllVectorPtr, hllVectorSizePtr, hllDimRegIDCountPtr,
                       (cudaStream_t)cudaStream);
  });
}

CGoCallResHandle AggStateFinalizeHLLEstimate(void *state, uint8_t **dimValuesPtr, double **estimatesPtr, void *cudaStream, int device) {
  return guarded("AggStateFinalizeHLLEstimate", device, [&]() -> int64_t {
    return finalizeHLLEstimate(asState(state), dimValuesPtr, estimatesPtr, (cudaStream_t)cudaStream);
  });
}

CGoCallResHandle AggStateReset(void *state, void *cudaStream, int device) {
  return guarded("AggStateReset", device, [&]() -> int64_t {
    AggState *st = asState(state);
    cudaStream_t s = (cudaStream_t)cudaStream;
    // only what was claimed is emptied (claim list): a 2^21-slot table with 19,200 groups resets 0.3 MB, not 32 MB,
    // and a dense HLL state clears the register arrays of its groups, not all 512 MB
    resetClaimedKernel<<<smCount() * 4, 256, 0, s>>>(st->table, st->accNeutral);
    checkLastError("AggStateReset");
    ARES_CUDA(cudaMemsetAsync(st->table.counters, 0, 256, s));
    st->occUpper = 0;
    st->unchecked = 0;
    st->everChecked = false;
    st->resultHost[8] = 0;
    return 0;
  });
}

// Additive diagnostics, usable without a GPU: the kernel ExecuteBatchPlan runs for (spec, plan), generated and compiled;
// res = cubin size.
CGoCallResHandle AresJitDryRun(AggSpec spec, const BatchPlan *plan, char **sourceOut) {
  CGoCallResHandle h = {nullptr, nullptr};
  try {
    h.res = reinterpret_cast<void *>(dryRun(&spec, 1, *plan, false, sourceOut));
  } catch (const std::exception &e) {
    h.pStrErr = strdup((std::string("AresJitDryRun: ") + e.what()).c_str());
  }
  return h;
}

// Additive diagnostics, usable without a GPU: the kernel of a plan whose measure roots feed numSpecs states, when
// ExecuteBatchPlanMulti runs it as one kernel for all of them for this batch's zone map; res = cubin size.  Any other
// schedule (one kernel per state, per dimension set, or a mix) is reported as an error.
CGoCallResHandle AresJitDryRunMulti(const AggSpec *specs, int numSpecs, const BatchPlan *plan, char **sourceOut) {
  CGoCallResHandle h = {nullptr, nullptr};
  try {
    if (!specs || !plan || numSpecs < 1 || numSpecs > kJitMaxMeasures) throw EngineError("numSpecs must be 1.." + std::to_string(kJitMaxMeasures));
    h.res = reinterpret_cast<void *>(dryRun(specs, numSpecs, *plan, true, sourceOut));
  } catch (const std::exception &e) {
    h.pStrErr = strdup((std::string("AresJitDryRunMulti: ") + e.what()).c_str());
  }
  return h;
}

CGoCallResHandle AggStateDestroy(void *state, int device) {
  return guarded("AggStateDestroy", device, [&]() -> int64_t {
    AggState *st = asState(state);
    if (st->mem) deviceFree(st->mem);
    if (st->resultHost) cudaFreeHost(st->resultHost);
    if (st->denseAcc) deviceFree(st->denseAcc);
    delete st;
    return 0;
  });
}

}  // extern "C"
