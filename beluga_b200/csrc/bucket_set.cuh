// Open-addressing set of 64-bit spatial-hash keys that keeps, per key, the smallest index inserted with it.  "Index i is
// the first occurrence of its bucket" is then an order-independent fact: the KLD bucket count (kld.cu) and the cell
// numbering of the clusterizer (cluster.cu) both rest on it.  The table is a power of two of slots, cleared to all ones.
#pragma once

#include <cstdint>

namespace bb200 {

namespace {

namespace bucket_set {

/// A free slot's key.
constexpr unsigned long long kEmpty = ~0ull;

/// The key a hash is stored under: the sentinel itself cannot be stored (2^-64 event).
__device__ __forceinline__ unsigned long long key_of(unsigned long long hash) { return hash == kEmpty ? kEmpty - 1 : hash; }

__device__ __forceinline__ uint64_t probe_start(unsigned long long key, uint64_t mask) {
  const unsigned long long h = key * 0x9E3779B97F4A7C15ull;
  return (h ^ (h >> 29)) & mask;
}

/// Claims the slot of `hash` (or finds it, when another index got there first) and lowers the slot's value to `index`.
__device__ __forceinline__ void insert_min(unsigned long long* keys, unsigned int* vals, uint64_t mask, unsigned long long hash, unsigned int index) {
  const unsigned long long key = key_of(hash);
  uint64_t pos = probe_start(key, mask);
  for (;;) {
    const unsigned long long prev = atomicCAS(keys + pos, kEmpty, key);
    if (prev == kEmpty || prev == key) {
      atomicMin(vals + pos, index);
      return;
    }
    pos = (pos + 1) & mask;
  }
}

/// The slot of a hash that has been inserted.
__device__ __forceinline__ uint64_t find(const unsigned long long* keys, uint64_t mask, unsigned long long hash) {
  const unsigned long long key = key_of(hash);
  uint64_t pos = probe_start(key, mask);
  while (keys[pos] != key) pos = (pos + 1) & mask;
  return pos;
}

}  // namespace bucket_set

}  // namespace

}  // namespace bb200
