// The fixed-point CDF build: largest weight, exponent, quantise + single-pass decoupled look-back scan; and the u32
// exclusive scan the execution schedule, KLD and the clusterizer count with.
#include "cdf.cuh"

#include <algorithm>

namespace bb200 {

namespace {

__global__ void __launch_bounds__(kMaxThreads) max_weight_kernel(const double* __restrict__ weights, uint64_t n, Scalars* scalars) {
  max_weight_block(weights, n, scalars, blockIdx.x, gridDim.x);
}

__global__ void __launch_bounds__(kMaxThreads) apply_factors_kernel(double* __restrict__ weights, const double* __restrict__ factors, uint64_t n,
                                                                    Scalars* scalars) {
  apply_factors_block(weights, factors, n, scalars, blockIdx.x, gridDim.x);
}

__global__ void prepare_cdf_kernel(Scalars* s, double host_wmax, int ceil_log2_count, unsigned long long* tile_state, uint32_t n_tiles) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += gridDim.x * blockDim.x) tile_state[t] = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const double wmax = host_wmax >= 0.0 ? host_wmax : __longlong_as_double(static_cast<long long>(s->wmax_bits));
    prepare_cdf_scalars(s, wmax, ceil_log2_count);
  }
}

__global__ void __launch_bounds__(kQsThreads) quantize_scan_kernel(const double* __restrict__ weights, uint64_t n,
                                                                   unsigned long long* __restrict__ cdf, Scalars* scalars,
                                                                   unsigned long long* tile_state, int derive_exponent, int ceil_log2_count) {
  // Tiles are taken in blockIdx order (CTAs are dispatched in that order, which is what the look-back's forward progress
  // needs -- the same assumption CUB's decoupled look-back makes): no ticket atomic and no barrier before the loads.
  quantize_scan_tile(weights, n, cdf, scalars, tile_state, blockIdx.x, derive_exponent, ceil_log2_count);
}

/// Exclusive prefix sum of u32 values (bin counters, KLD first-occurrence flags) with the same
/// decoupled look-back machinery; `in` and `out` may alias.
__global__ void __launch_bounds__(kScanThreads) scan_u32_kernel(const uint32_t* in, uint32_t* out, uint32_t n, unsigned long long* ticket,
                                                                unsigned long long* tile_state, unsigned long long* total_out) {
  __shared__ unsigned long long s_warp[kScanThreads / kWarp];
  __shared__ unsigned long long s_prefix;
  (void)ticket;  // tiles in blockIdx order (see quantize_scan_kernel)
  const uint32_t tile = blockIdx.x;
  const uint32_t base = tile * kScanTile + threadIdx.x * kScanItems;
  unsigned long long q[kScanItems];
  unsigned long long local = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    q[k] = base + k < n ? in[base + k] : 0u;
    local += q[k];
  }
  unsigned long long tile_total;
  const unsigned long long inclusive = block_inclusive_scan_u64<kScanThreads>(local, s_warp, tile_total);
  const unsigned long long prefix = lookback_exclusive_prefix(tile_state, tile, tile_total, &s_prefix);
  unsigned long long running = prefix + inclusive - local;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) out[base + k] = static_cast<uint32_t>(running);
    running += q[k];
  }
  if (total_out != nullptr && base <= n - 1 && n - 1 < base + kScanItems) *total_out = prefix + inclusive;
}

}  // namespace

void launch_max_weight(const double* weights, uint64_t n, Scalars* scalars, cudaStream_t stream) {
  if (n == 0) return;
  const unsigned blocks = static_cast<unsigned>(std::min<uint64_t>((n + 511) / 512, kStreamMaxBlocks));
  max_weight_kernel<<<blocks, 512, 0, stream>>>(weights, n, scalars);
}

void launch_apply_factors(double* weights, const double* factors, uint64_t n, Scalars* scalars, cudaStream_t stream) {
  if (n == 0) return;
  const unsigned blocks = static_cast<unsigned>(std::min<uint64_t>((n + kMaxThreads - 1) / kMaxThreads, kStreamMaxBlocks));
  apply_factors_kernel<<<blocks, kMaxThreads, 0, stream>>>(weights, factors, n, scalars);
}

uint32_t scan_tile_count(uint64_t n) { return static_cast<uint32_t>((n + kQsTile - 1) / kQsTile); }

void launch_prepare_cdf(Scalars* scalars, double host_wmax, uint64_t global_count, unsigned long long* tile_state, uint32_t n_tiles,
                        cudaStream_t stream) {
  const unsigned blocks = std::max(1u, std::min((n_tiles + 255u) / 256u, 64u));
  prepare_cdf_kernel<<<blocks, 256, 0, stream>>>(scalars, host_wmax, ceil_log2_count(global_count), tile_state, n_tiles);
}

void launch_quantize_scan(const double* weights, uint64_t n, unsigned long long* cdf, Scalars* scalars, unsigned long long* tile_state,
                          cudaStream_t stream, bool derive_exponent, uint64_t global_count) {
  if (n == 0) return;
  quantize_scan_kernel<<<scan_tile_count(n), kQsThreads, 0, stream>>>(weights, n, cdf, scalars, tile_state, derive_exponent ? 1 : 0,
                                                                     ceil_log2_count(global_count));
}

void launch_scan_u32_prepared(const uint32_t* in, uint32_t* out, uint32_t n, unsigned long long* ticket, unsigned long long* tile_state,
                              unsigned long long* total_out, cudaStream_t stream) {
  const uint32_t tiles = (n + kScanTile - 1) / kScanTile;
  scan_u32_kernel<<<tiles, kScanThreads, 0, stream>>>(in, out, n, ticket, tile_state, total_out);
}

void launch_scan_u32(const uint32_t* in, uint32_t* out, uint32_t n, unsigned long long* ticket, unsigned long long* tile_state,
                     unsigned long long* total_out, cudaStream_t stream) {
  if (n == 0) return;
  const uint32_t tiles = (n + kScanTile - 1) / kScanTile;
  cudaMemsetAsync(ticket, 0, sizeof(unsigned long long), stream);
  cudaMemsetAsync(tile_state, 0, static_cast<size_t>(tiles) * sizeof(unsigned long long), stream);
  launch_scan_u32_prepared(in, out, n, ticket, tile_state, total_out, stream);
}

}  // namespace bb200
