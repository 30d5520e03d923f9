// join.cuh — dimension-table join building blocks (SURVEY.md §8 f4), shared by the legacy HashLookup / ForeignColumnInput
// entry points and the NVRTC-specialised fused kernel (NVRTC-clean: no host headers).
//
//   cuckooLookup   probe of the memstore's primary-key index of a dimension table (reference HashLookupFunctor,
//                  query/functor.hpp:1173-1266; index built by memstore/cuckoo_index.go): numHashes candidate buckets
//                  (murmur3-32 of the key bytes with the index's seeds, bucket = hash % numBuckets, signature = top byte
//                  of the hash, at least 1), 8 cells per bucket laid out RecordID[8] | signature[8] | key[8], then the
//                  4-cell stash bucket behind the last bucket.  RecordID {0, 0} = not found (also for a NULL key).
//   foreignLoad    value of a foreign column at a RecordID (reference RecordIDJoinIterator::dereference,
//                  query/iterator.hpp:846-931): batch = batchID - baseBatchID, bounds check against the last batch's
//                  record count, mode-0 batches yield the column default (not mapped), the others go through the
//                  optional enum -> timezone-offset table; an unmatched row is (unspecified, NULL) — 0 here.
#pragma once
#include "column.cuh"
#include "murmur.cuh"

namespace aresb {

constexpr int kCuckooBucketCells = 8;   // HASH_BUCKET_SIZE
constexpr int kCuckooStashCells = 4;    // HASH_STASH_SIZE
constexpr int kMaxForeignBatches = 8;   // batches of one dimension table (live batches of a small table)

struct CuckooDesc {
  const uint8_t *buckets;
  uint32_t seeds[4];
  int32_t keyBytes, numHashes, numBuckets;
};

struct ForeignDesc {
  const unsigned long long *recordIDs;   // legacy entry points: one RecordID per index position (fused path: unused)
  const int16_t *tzLookup;               // optional enum -> timezone offset table (device memory)
  int32_t numBatches, baseBatchID, numRecordsInLastBatch, tzSize;
  InputDesc batches[kMaxForeignBatches];
};

#ifdef __CUDACC__
// (lo, hi): the key's bytes little-endian (an integer key widened to 32 bits supplies its low keyBytes bytes, exactly what
// reinterpret_cast<uint8_t *>(&v) reads in the reference).  Returns the RecordID as batchID | index << 32.
__device__ __forceinline__ unsigned long long cuckooLookup(const CuckooDesc &H, uint64_t lo, uint64_t hi) {
  const int kb = H.keyBytes;
  if (kb < 16) { if (kb <= 8) { hi = 0; if (kb < 8) lo &= (1ull << (8 * kb)) - 1ull; } else hi &= (1ull << (8 * (kb - 8))) - 1ull; }
  const uint64_t w[4] = {lo, hi, 0, 0};
  const int cellBytes = 8 + kb + 1;
  const size_t bucketBytes = (size_t)kCuckooBucketCells * cellBytes;
  const int offSig = kCuckooBucketCells * 8, offKey = offSig + kCuckooBucketCells;
  auto match = [&](const uint8_t *bucket, int j) -> bool {
    const uint8_t *k = bucket + offKey + j * kb;
    for (int b = 0; b < kb; b++)
      if (k[b] != (uint8_t)((b < 8 ? lo >> (8 * b) : hi >> (8 * (b - 8))) & 0xFF)) return false;
    return true;
  };
  for (int i = 0; i < H.numHashes && i < 4; i++) {
    const uint32_t h = murmur3_32(w, kb, H.seeds[i]);
    const uint8_t *bucket = H.buckets + (size_t)(h % (uint32_t)H.numBuckets) * bucketBytes;
    uint8_t sig = (uint8_t)(h >> 24);
    if (sig < 1) sig = 1;
    // the 8 signatures are one 8-byte word: compare them at once, then check the keys of the matching cells
    unsigned long long sigs = 0;
    for (int b = 0; b < 8; b++) sigs |= (unsigned long long)bucket[offSig + b] << (8 * b);
#pragma unroll 1
    for (int j = 0; j < kCuckooBucketCells; j++)
      if ((uint8_t)(sigs >> (8 * j)) == sig && match(bucket, j)) {
        const uint8_t *r = bucket + 8 * j;
        unsigned long long rid = 0;
        for (int b = 0; b < 8; b++) rid |= (unsigned long long)r[b] << (8 * b);
        return rid;
      }
  }
  const uint8_t *stash = H.buckets + bucketBytes * (size_t)H.numBuckets;
  for (int j = 0; j < kCuckooStashCells; j++)
    if (stash[offSig + j] != 0 && match(stash, j)) {
      const uint8_t *r = stash + 8 * j;
      unsigned long long rid = 0;
      for (int b = 0; b < 8; b++) rid |= (unsigned long long)r[b] << (8 * b);
      return rid;
    }
  return 0ull;
}

__device__ __forceinline__ Cell foreignLoad(const ForeignDesc &F, unsigned long long rid, uint64_t *hi) {
  Cell c; c.v = 0; c.valid = false;
  if (hi) *hi = 0;
  const int32_t batchID = (int32_t)(uint32_t)rid;
  const uint32_t index = (uint32_t)(rid >> 32);
  if (batchID == 0) return c;
  const int32_t b = batchID - F.baseBatchID;
  if (!(b < F.numBatches - 1 || index < (uint32_t)F.numRecordsInLastBatch)) return c;
  if (b < 0 || b >= F.numBatches || b >= kMaxForeignBatches) return c;   // (the reference would read out of bounds)
  const InputDesc &d = F.batches[b];
  c = loadInput(d, index, nullptr, nullptr, 0, hi);
  if (F.tzLookup != nullptr && d.mode != 0 && d.vclass != VC_UUID && d.vclass != VC_I64) {
    // an enum column mapped through the timezone table: (table[enum], valid), 0 beyond the table; a mode-0 batch yields
    // the column default as it is (the reference returns its constant iterator before the lookup)
    const int32_t e = d.vclass == VC_F32 ? (int32_t)__uint_as_float((uint32_t)c.v) : (int32_t)(uint32_t)c.v;
    const int32_t off = e >= 0 && e < F.tzSize ? (int32_t)F.tzLookup[e] : 0;
    c.v = d.vclass == VC_F32 ? (uint64_t)__float_as_uint((float)off) : d.vclass == VC_BOOL ? (uint64_t)(off != 0) : (uint64_t)(uint32_t)off;
  }
  return c;
}
#endif  // __CUDACC__

}  // namespace aresb
