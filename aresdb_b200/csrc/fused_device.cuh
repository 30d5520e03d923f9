// fused_device.cuh — device building blocks of the NVRTC-specialised fused kernel (jit.cu) and of
// the merge / finalize kernels (batch_plan.cu): TMA bulk copies + mbarriers, the CTA-private
// shared-memory group table and the global (L2-resident) group table.
// NVRTC-clean: no host headers (the JIT prelude provides the fixed-width typedefs).
#pragma once
#include "agg.cuh"

namespace aresb {

constexpr int kMaxStages = 4;
constexpr int kProgressWarps = 32;         // progress slots per CTA (one per warp)
constexpr int kProgressCtas = 160;         // = kMaxGridCtas
constexpr int kProgressTail = kProgressCtas * kProgressWarps;   // index of the "tail rows done" flag
constexpr uint32_t kSmemProbeLimit = 8;
constexpr uint32_t kGlobalProbeLimit = 8192;
constexpr unsigned long long kEmptyKey = ~0ull;
constexpr uint64_t kMix = 0x9E3779B97F4A7C15ull;

// A row (already reduced to key + measure) that arrived while the table was at its growth threshold, from a kernel
// whose launches the host does not wait for (direct-indexed kernels: their flush and their out-of-range rows): folded
// into the table after it has grown, at the state's next synchronising call.
struct SpillEntry { unsigned long long key; uint64_t row[4]; uint64_t val; };
constexpr uint32_t kSpillCap = 1u << 20;   // 48 MB per state: covers the flush of every CTA's shared table (132 x 6144 keys)
constexpr uint32_t kSlotSpill = 0xFFFFFFFEu;

struct DevTable {
  unsigned long long *keys;
  unsigned long long *acc;
  uint64_t *rows;        // [capacity][4] packed rows, wide (hashed) keys only
  uint32_t *counters;    // [0] occupied slots, [1] overflow flag, [2] truncated exchange part, [3] STOP: the table has
                         // reached growAt — consumers finish their tile and drain; the host grows the table and resumes
  uint32_t *progress;    // [kMaxGridCtas * 32 + 1] tile iterations each consumer warp has folded (resume point), tail flag
  uint32_t growAt;       // claim ordinal at which the stop flag is raised (capacity / 2; 0xFFFFFFFF: never)
  volatile uint32_t *occPublish;  // mapped pinned host word: the occupancy a finishing kernel saw (read by the host without
                         // synchronising: decides whether the next batch's launch has to be waited for)
  struct SpillEntry *spill;  // [kSpillCap] rows of kernels that cannot be resumed, parked while the table is full
                         // (counters[4] = entries, counters[5] = spill overflow)
  uint32_t *claimed;     // [capacity] slot index of the i-th claimed group (claim order): finalize / reset / export
                         // walk this list instead of scanning the table
  uint32_t mask;
  uint32_t *regs;        // dense HLL mode: [capacity][16384] registers, value + 1 (0 = never hit); else null
};

constexpr uint32_t kHllRegisters = 1u << 14;   // p = 14
constexpr uint32_t kHllDenseMaxGroups = 4096;  // dense HLL: directory of 8192 slots, register arrays for 4096 groups

// ---------------------------------------------------------------------------------------
// device helpers: TMA bulk copy + mbarrier (sm_90+ PTX; SASS: UBLKCP / SYNCS)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smemAddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbarInit(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(count));
}
__device__ __forceinline__ void mbarExpectTx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarWait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smemAddr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbarArrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smemAddr(bar)) : "memory");
}
__device__ __forceinline__ void tmaLoad1D(void *dstSmem, const void *srcGlobal, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smemAddr(dstSmem)),
               "l"(srcGlobal), "r"(bytes), "r"(smemAddr(bar))
               : "memory");
}

// ---------------------------------------------------------------------------------------
// global group table
// ---------------------------------------------------------------------------------------
// 64 -> 32 bit key mixer (one 32-bit multiply after folding): table positions only, never group identity
__device__ __forceinline__ uint32_t mixKey(unsigned long long key) {
  uint32_t x = (uint32_t)key ^ (uint32_t)(key >> 32) * 0x85EBCA6Bu;
  x *= 0x9E3779B1u;
  return x ^ (x >> 15);
}

__device__ __forceinline__ uint32_t globalHome(const DevTable &G, unsigned long long key) {
  return (mixKey(key) >> 3) & G.mask;
}

// spillWhenStopped: a NEW key is not claimed once the stop flag is up (kSlotSpill: the caller parks the row).
// `Table`: a kernel that feeds several group tables calls one instantiation per table — lanes claiming in different tables
// then run different code, so the warp-aggregated claim counter below only ever combines lanes of one table.
template <int Table = 0>
static __device__ __noinline__ uint32_t globalFindOrClaim(const DevTable &G, unsigned long long key, const uint64_t *roww,
                                                          bool spillWhenStopped = false) {
  uint32_t slot = globalHome(G, key);
#pragma unroll 1
  for (uint32_t probe = 0; probe < kGlobalProbeLimit; probe++) {
    unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(&G.keys[slot]);
    if (k == key) return slot;
    if (k == kEmptyKey) {
      if (spillWhenStopped && *reinterpret_cast<volatile uint32_t *>(&G.counters[3]) != 0u) return kSlotSpill;
      unsigned long long old = atomicCAS(&G.keys[slot], kEmptyKey, key);
      if (old == kEmptyKey) {
        // claim ordinal: the lanes of the warp that claim in the same step share ONE add on the (single-address) counter
        const uint32_t peers = __activemask(), lane = threadIdx.x & 31u, leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(&G.counters[0], (uint32_t)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        const uint32_t ord = base + __popc(peers & ((1u << lane) - 1u));
        G.claimed[ord] = slot;   // every slot is claimed once: the ordinal is < capacity
        // dense HLL directory: the group's register array is addressed by its claim ordinal (see hllRegArray), published
        // in the slot's otherwise unused accumulator word as ordinal + 1
        if (G.regs != nullptr) *reinterpret_cast<volatile unsigned long long *>(&G.acc[slot]) = (unsigned long long)ord + 1ull;
        if (ord >= G.growAt) *reinterpret_cast<volatile uint32_t *>(&G.counters[3]) = 1u;   // filling up: stop consuming tiles
        if (roww != nullptr && G.rows != nullptr) {
#pragma unroll
          for (int i = 0; i < 4; i++) G.rows[(size_t)slot * 4 + i] = roww[i];
        }
        return slot;
      }
      if (old == key) return slot;
    }
    slot = (slot + 1) & G.mask;
  }
  atomicExch(&G.counters[1], 1u);
  return 0xFFFFFFFFu;
}

// parks one row (out of line: it is rare, and globalUpdate is inlined at every aggregation site)
static __device__ __noinline__ void globalPark(const DevTable &G, unsigned long long key, const uint64_t *roww, uint64_t val) {
  const uint32_t i = atomicAdd(&G.counters[4], 1u);
  if (i < kSpillCap) {
    SpillEntry e;
    e.key = key; e.val = val;
#pragma unroll
    for (int w = 0; w < 4; w++) e.row[w] = roww ? roww[w] : 0;
    G.spill[i] = e;
  } else {
    atomicExch(&G.counters[5], 1u);
  }
}

template <int Table = 0>
__device__ __forceinline__ void globalUpdate(const DevTable &G, AggOp op, unsigned long long key, const uint64_t *roww,
                                             uint64_t val, bool spillWhenStopped = false) {
  uint32_t slot = globalFindOrClaim<Table>(G, key, roww, spillWhenStopped);
  if (slot == kSlotSpill) { globalPark(G, key, roww, val); return; }
  if (slot != 0xFFFFFFFFu) aggAtomic(op, &G.acc[slot], val);
}

// ---------------------------------------------------------------------------------------
// dense HLL mode: the table is only the directory of dimension groups; each group owns 16384
// registers in G.regs.  `mirror` (optional) is a shared-memory copy of G.keys with the same
// geometry, filled on demand, so that steady-state lookups never leave the SM.
// ---------------------------------------------------------------------------------------
// Register arrays are addressed by the group's CLAIM ORDINAL, not by its directory slot: the arrays of the groups a batch
// touches are then contiguous (101 groups: 6.6 MB), where slot-addressed arrays are 64 KB chunks scattered over the whole
// 512 MB allocation — and random accesses over that many pages ran at a THIRD of the rate (reductions and plain loads
// alike, tools/microbench/red_lanes.cu; the translation caches, not L2).  The claiming thread
// publishes ordinal + 1 in the slot's accumulator word right after its claim; a thread that finds the key an instant
// earlier waits for it.
__device__ __forceinline__ uint32_t hllRegArray(const DevTable &G, uint32_t slot) {
  unsigned long long o;
  do {
    o = *reinterpret_cast<volatile unsigned long long *>(&G.acc[slot]);
  } while (o == 0ull);
  return (uint32_t)o - 1u;
}

// Register array (claim ordinal) of `key`'s group, claimed on first sight; 0xFFFFFFFF when the directory is full.
__device__ __forceinline__ uint32_t hllDenseLocate(const DevTable &G, unsigned long long *mirror, unsigned long long key,
                                                   const uint64_t *roww) {
  uint32_t slot = globalHome(G, key);
  bool found = false;
  if (mirror != nullptr) {
#pragma unroll 1
    for (uint32_t probe = 0; probe < kSmemProbeLimit; probe++) {
      const unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(&mirror[slot]);
      if (k == key) { found = true; break; }
      if (k == kEmptyKey) break;          // unknown here: ask the global directory
      slot = (slot + 1) & G.mask;
    }
  }
  if (!found) {
    const uint32_t home = globalHome(G, key);
    slot = globalFindOrClaim(G, key, roww);
    if (slot == 0xFFFFFFFFu) return slot;  // directory full: flagged in G.counters[1], reported at finalize
    if (mirror != nullptr) {
      // every directory slot from the key's home up to where it lives is occupied (linear probing):
      // copy them so that the next probe sequence reaches the key without leaving shared memory
      for (uint32_t s2 = home;; s2 = (s2 + 1) & G.mask) {
        mirror[s2] = *reinterpret_cast<volatile unsigned long long *>(&G.keys[s2]);
        if (s2 == slot) break;
      }
    }
  }
  const uint32_t arr = hllRegArray(G, slot);
  if (arr >= kHllDenseMaxGroups) {   // more groups than register arrays: reported like a full directory
    atomicExch(&G.counters[1], 1u);
    return 0xFFFFFFFFu;
  }
  return arr;
}

// Register update: registers only grow, so a (possibly stale) plain read that already shows a value >= ours makes the
// atomic unnecessary — after the first few thousand rows of a group that is the common case (a register sees a new
// maximum H(n) ~ ln n times in n rows), and an L2 read is far cheaper than an L2 atomic.
__device__ __forceinline__ void hllRegisterMax(uint32_t *reg, uint32_t want) {
  if (__ldcg(reg) < want) atomicMax(reg, want);
}

__device__ __forceinline__ void hllDenseUpdate(const DevTable &G, unsigned long long *mirror, unsigned long long key,
                                               const uint64_t *roww, uint32_t value) {
  const uint32_t arr = hllDenseLocate(G, mirror, key, roww);
  if (arr == 0xFFFFFFFFu) return;
  hllRegisterMax(&G.regs[(size_t)arr * kHllRegisters + (value & (kHllRegisters - 1))], value + 1u);
}

// ---------------------------------------------------------------------------------------
// CTA-private shared-memory table
// ---------------------------------------------------------------------------------------
struct SmemTable {
  unsigned long long *keys;
  unsigned long long *acc;
  uint32_t *claims;   // number of occupied slots
  uint32_t mask;
};

__device__ __forceinline__ void smemAtomic(AggOp op, unsigned long long *addr, uint64_t v) {
  switch (op) {
    case OP_SUM_I32: atomicAdd(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); break;
    case OP_SUM_F32: atomicAdd(reinterpret_cast<float *>(addr), __uint_as_float((uint32_t)v)); break;
    case OP_SUM_I64: atomicAdd(addr, (unsigned long long)v); break;
    case OP_SUM_F64: atomicAdd(reinterpret_cast<double *>(addr), __longlong_as_double((long long)v)); break;
    case OP_MIN_U32: atomicMin(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); break;
    case OP_MIN_I32: atomicMin(reinterpret_cast<int *>(addr), (int)(uint32_t)v); break;
    case OP_MAX_U32: atomicMax(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); break;
    case OP_MAX_I32: atomicMax(reinterpret_cast<int *>(addr), (int)(uint32_t)v); break;
    case OP_AVG: aggAtomic(op, addr, v); break;  // 64-bit CAS loop around the rolling-average combine
    default: {  // float min / max
      unsigned int *a = reinterpret_cast<unsigned int *>(addr);
      unsigned int old = *a, assumed;
      do {
        assumed = old;
        unsigned int want = (unsigned int)aggCombine(op, assumed, v);
        if (want == assumed) break;
        old = atomicCAS(a, assumed, want);
      } while (old != assumed);
      break;
    }
  }
}

// Two-choice placement.  A key lives in its first home slot h1 if that was free when the key arrived, else
// in its second home h2, else (both taken: ~2 % of the keys at load 0.3) on the linear run that starts at
// h2.  A lookup therefore costs one probe for ~85 % of the rows and exactly two for nearly all others —
// what matters is that the SECOND step is a fixed short sequence, because with 18 live lanes some lane of
// the warp needs it almost every time.  Slots are addressed by byte offset throughout.
__device__ __forceinline__ uint32_t smemHashWord(unsigned long long key) {
  return ((uint32_t)key ^ (uint32_t)(key >> 32) * 0x85EBCA6Bu) * 0x9E3779B1u;
}
// h1: top bits of the hash word.  h2: h1 XOR a non-zero displacement taken from the word's low bits
// (three instructions, never equal to h1).
__device__ __forceinline__ uint32_t smemHome1(const SmemTable &T, uint32_t x) {
  return (x >> (29 - __popc(T.mask))) & (T.mask << 3);
}
__device__ __forceinline__ uint32_t smemHome2(const SmemTable &T, uint32_t x, uint32_t off1) {
  return off1 ^ (((x << 3) & (T.mask << 3)) | 8u);
}

// Out-of-line insertion of a key the inlined lookup did not find: replays the placement rule with CAS.
// Returns the key's slot, or 0xFFFFFFFF when the row has to go to the global table.
static __device__ __noinline__ uint32_t smemInsert(unsigned long long *keys, uint32_t *claims, uint32_t mask, const DevTable &G,
                                                   unsigned long long key, const uint64_t *roww, uint32_t off1, uint32_t off2) {
  uint32_t slot = off1 >> 3;
#pragma unroll 1
  for (uint32_t step = 0; step < kSmemProbeLimit + 1; step++) {
    unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(&keys[slot]);
    if (k == kEmptyKey) {
      k = atomicCAS(&keys[slot], kEmptyKey, key);
      if (k == kEmptyKey) {
        atomicAdd(claims, 1u);
        // wide keys: the packed row is recorded in the global table once, by whoever claims first
        if (roww != nullptr) globalFindOrClaim(G, key, roww);
        return slot;
      }
    }
    if (k == key) return slot;
    slot = step == 0 ? off2 >> 3 : (slot + 1) & mask;
  }
  return 0xFFFFFFFFu;
}

// Returns false when the row has to go to the global table (no room on the key's probe sequence, or the
// table is closed for new keys).
__device__ __forceinline__ bool smemUpdate(const SmemTable &T, const DevTable &G, AggOp op, unsigned long long key,
                                           const uint64_t *roww, uint64_t val, bool allowClaim) {
  const uint8_t *kb = reinterpret_cast<const uint8_t *>(T.keys);
  const uint32_t x = smemHashWord(key);
  const uint32_t off1 = smemHome1(T, x);
  uint32_t off = off1;
  unsigned long long k = *reinterpret_cast<const volatile unsigned long long *>(kb + off);
  if (k != key) {
    const uint32_t off2 = smemHome2(T, x, off1);
    if (k != kEmptyKey) {
      off = off2;
      k = *reinterpret_cast<const volatile unsigned long long *>(kb + off);
      if (k != key && k != kEmptyKey) {   // both homes taken by other keys: the run behind h2
        uint32_t probe = 1;
#pragma unroll 1
        for (;;) {
          off = (off + 8) & (T.mask << 3);
          k = *reinterpret_cast<const volatile unsigned long long *>(kb + off);
          if (k == key || k == kEmptyKey || ++probe >= kSmemProbeLimit) break;
        }
      }
    }
    if (k != key) {
      if (k != kEmptyKey || !allowClaim) return false;
      const uint32_t slot = smemInsert(T.keys, T.claims, T.mask, G, key, roww, off1, off2);
      if (slot == 0xFFFFFFFFu) return false;
      off = slot << 3;
    }
  }
  smemAtomic(op, reinterpret_cast<unsigned long long *>(reinterpret_cast<uint8_t *>(T.acc) + off), val);
  return true;
}

}  // namespace aresb
