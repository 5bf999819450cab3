// ---- KLD-adaptive sample size (a12) -----------------------------------------------------------------
// views::take_while_kld (views/take_while_kld.hpp:72-137) keeps drawing while
//   count <= min  ||  count <= target(k),   k = number of distinct spatial-hash buckets so far,
// a sequential early exit over an unordered_set.  Here candidate slots are generated in chunks;
// a device hash set keeps, per bucket, the SMALLEST slot index that produced it, so "slot j is the
// first occurrence of its bucket" is an order-independent fact; a prefix sum of those flags gives
// k after every slot and the first failing count is a min-reduction.
#include "bucket_set.cuh"
#include "cdf.cuh"

namespace bb200 {

namespace {

__global__ void __launch_bounds__(256) kld_insert_kernel(const unsigned long long* __restrict__ hashes, uint64_t n, uint64_t slot_base,
                                                         unsigned long long* keys, unsigned int* vals, uint64_t mask) {
  const uint64_t j = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (j >= n) return;
  bucket_set::insert_min(keys, vals, mask, hashes[j], static_cast<unsigned int>(slot_base + j));
}

__global__ void __launch_bounds__(256) kld_flag_kernel(const unsigned long long* __restrict__ hashes, uint64_t n, uint64_t slot_base,
                                                       const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ vals,
                                                       uint64_t mask, uint32_t* __restrict__ flags) {
  const uint64_t j = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (j >= n) return;
  flags[j] = vals[bucket_set::find(keys, mask, hashes[j])] == static_cast<unsigned int>(slot_base + j) ? 1u : 0u;
}

/// kld_condition target size (views/take_while_kld.hpp:73-80), same operation order as the reference.
__device__ __forceinline__ bool kld_count_allowed(unsigned long long count, unsigned long long k, unsigned long long min_count, double two_epsilon, double z) {
  if (count <= min_count || k <= 2ull) return true;
  const double common = 2. / static_cast<double>(9 * (k - 1));
  const double base = 1. - common + sqrt(common) * z;
  const double result = (static_cast<double>(k - 1) / two_epsilon) * base * base * base;
  const double target = ceil(result);
  return target >= 18446744073709551615.0 || count <= static_cast<unsigned long long>(target);
}

__global__ void __launch_bounds__(256) kld_check_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ exclusive, uint64_t n,
                                                        uint64_t slot_base, unsigned long long k_before, unsigned long long min_count,
                                                        double two_epsilon, double z, Scalars* scalars) {
  const uint64_t j = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  unsigned long long failing = ~0ull;
  if (j < n) {
    const unsigned long long count = slot_base + j + 1;
    const unsigned long long k = k_before + exclusive[j] + flags[j];
    if (!kld_count_allowed(count, k, min_count, two_epsilon, z)) failing = count;
  }
  // Past the cutoff nearly every slot fails: one atomic per warp instead of one per thread on the same word.
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) {
    const unsigned long long o = __shfl_down_sync(0xffffffffu, failing, off);
    failing = o < failing ? o : failing;
  }
  if (threadIdx.x % kWarp == 0 && failing != ~0ull && failing < *reinterpret_cast<volatile unsigned long long*>(&scalars->kld_cutoff))
    atomicMin(&scalars->kld_cutoff, failing);
}

__global__ void kld_reset_kernel(Scalars* scalars) {
  scalars->kld_cutoff = ~0ull;
  scalars->pad[0] = 0;  // tile ticket of the flag scan
  scalars->pad[1] = 0;  // distinct buckets in the chunk
}

}  // namespace

void launch_kld_clear(unsigned long long* keys, unsigned int* vals, uint64_t table_size, cudaStream_t stream) {
  cudaMemsetAsync(keys, 0xFF, table_size * sizeof(unsigned long long), stream);
  cudaMemsetAsync(vals, 0xFF, table_size * sizeof(unsigned int), stream);
}

void launch_kld_chunk(const KldArgs& a, unsigned long long* keys, unsigned int* vals, uint64_t table_size, uint32_t* flags, uint32_t* exclusive,
                      Scalars* scalars, unsigned long long* tile_state, cudaStream_t stream) {
  if (a.n == 0) return;
  const unsigned blocks = static_cast<unsigned>((a.n + 255) / 256);
  const uint32_t tiles = static_cast<uint32_t>((a.n + kScanTile - 1) / kScanTile);
  kld_reset_kernel<<<1, 1, 0, stream>>>(scalars);
  cudaMemsetAsync(tile_state, 0, static_cast<size_t>(tiles) * sizeof(unsigned long long), stream);
  kld_insert_kernel<<<blocks, 256, 0, stream>>>(a.hashes, a.n, a.slot_base, keys, vals, table_size - 1);
  kld_flag_kernel<<<blocks, 256, 0, stream>>>(a.hashes, a.n, a.slot_base, keys, vals, table_size - 1, flags);
  launch_scan_u32_prepared(flags, exclusive, static_cast<uint32_t>(a.n), &scalars->pad[0], tile_state, &scalars->pad[1], stream);
  kld_check_kernel<<<blocks, 256, 0, stream>>>(flags, exclusive, a.n, a.slot_base, a.k_before, a.min_particles, 2 * a.epsilon, a.z, scalars);
}

}  // namespace bb200
