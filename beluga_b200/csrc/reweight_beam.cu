// Beam-model reweight of one filter: the normaliser table, the fused kernel and the two-pass form (walk, mixture).
#include "reweight_beam.cuh"

#include <algorithm>

namespace bb200 {

namespace {

__global__ void __launch_bounds__(256) beam_eta_table_kernel(BeamParams p, double resolution, double2* __restrict__ table, uint32_t entries) {
  const uint32_t k = blockIdx.x * 256 + threadIdx.x;
  if (k >= entries) return;
  const double z_mean = k + 1 == entries ? p.beam_max_range : fmin(sqrt(static_cast<double>(k)) * resolution, p.beam_max_range);
  table[k] = beam_normalisers(p, z_mean);
}

__global__ void __launch_bounds__(kBeamThreads, kBeamBlocksPerSm)
    reweight_beam_kernel(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, const uint32_t* __restrict__ perm,
                         OccupancyView grid, BeamParams params, const double2* __restrict__ points, uint32_t n_points,
                         Scalars* __restrict__ scalars) {
  reweight_beam_block(states, weights, n, perm, grid, params, points, n_points, scalars, blockIdx.x);
}

__global__ void __launch_bounds__(kWalkThreads, kWalkBlocksPerSm)
    beam_walk_kernel(const Pose2* __restrict__ states, uint64_t n, uint64_t slot_base, uint64_t slot_count, const uint32_t* __restrict__ perm,
                     OccupancyView grid, double beam_max_range, const double2* __restrict__ points, uint32_t n_points,
                     uint32_t* __restrict__ hits, uint64_t hit_stride) {
  beam_walk_block(states, n, slot_base, slot_count, perm, grid, beam_max_range, points, n_points, hits, hit_stride, blockIdx.x);
}

__global__ void __launch_bounds__(kMixThreads)
    beam_mixture_kernel(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, uint64_t slot_base, uint64_t slot_count,
                        const uint32_t* __restrict__ perm, OccupancyView grid, BeamParams params, const double2* __restrict__ points,
                        uint32_t n_points, const uint32_t* __restrict__ hits, uint64_t hit_stride, Scalars* __restrict__ scalars) {
  beam_mixture_block(states, weights, n, slot_base, slot_count, perm, grid, params, points, n_points, hits, hit_stride, scalars, blockIdx.x);
}

}  // namespace

uint32_t beam_eta_entries(double beam_max_range, double resolution) {
  const double cells = beam_max_range / resolution + 2.0;
  const double entries = cells * cells + 2.0;
  return (entries > 0.0 && entries < 8.0e6) ? static_cast<uint32_t>(entries) : 0u;  // <= 128 MB; beyond that: per-beam evaluation
}

void launch_beam_eta_table(const BeamParams& params, double resolution, double2* table, uint32_t entries, cudaStream_t stream) {
  if (entries == 0) return;
  beam_eta_table_kernel<<<(entries + 255) / 256, 256, 0, stream>>>(params, resolution, table, entries);
}

uint64_t beam_hit_words(uint64_t particles, uint32_t n_points) {
  const uint64_t stride = (particles + 31) / 32 * 32;
  return stride * n_points;
}

void launch_reweight_beam_two_pass(const Pose2* states, double* weights, uint64_t n, const uint32_t* perm, const OccupancyView& grid,
                                   const BeamParams& params, const double* points_xy_device, uint32_t n_points, uint32_t* hits,
                                   uint64_t pass_particles, Scalars* scalars, cudaStream_t stream) {
  if (n == 0 || n_points == 0 || pass_particles == 0) return;
  const double2* points = reinterpret_cast<const double2*>(points_xy_device);
  const uint64_t stride = (pass_particles + 31) / 32 * 32;
  for (uint64_t base = 0; base < n; base += pass_particles) {
    const uint64_t count = std::min<uint64_t>(pass_particles, n - base);
    const unsigned blocks = static_cast<unsigned>((count + kWalkThreads - 1) / kWalkThreads);
    beam_walk_kernel<<<blocks, kWalkThreads, 0, stream>>>(states, n, base, count, perm, grid, params.beam_max_range, points, n_points, hits, stride);
    beam_mixture_kernel<<<blocks, kMixThreads, 0, stream>>>(states, weights, n, base, count, perm, grid, params, points, n_points, hits, stride, scalars);
  }
}

void launch_reweight_beam(const Pose2* states, double* weights, uint64_t n, const uint32_t* perm, const OccupancyView& grid,
                          const BeamParams& params, const double* points_xy_device, uint32_t n_points, Scalars* scalars, cudaStream_t stream) {
  if (n == 0) return;
  const unsigned blocks = static_cast<unsigned>((n + kBeamThreads - 1) / kBeamThreads);
  reweight_beam_kernel<<<blocks, kBeamThreads, 0, stream>>>(states, weights, n, perm, grid, params,
                                                            reinterpret_cast<const double2*>(points_xy_device), n_points, scalars);
}

}  // namespace bb200
