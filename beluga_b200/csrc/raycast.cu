// Ray casts of one filter's map: Ray2d::cast for many sensor poses and bearings in one launch.
#include "raycast.cuh"

namespace bb200 {

namespace {

__global__ void __launch_bounds__(kRayThreads) cast_rays_kernel(OccupancyView grid, const Pose2* __restrict__ poses, const double2* __restrict__ bearings,
                                                                uint64_t n_bearings, uint64_t n_rays, double max_range, double* __restrict__ ranges) {
  cast_rays_block(grid, poses, bearings, n_bearings, n_rays, max_range, ranges, blockIdx.x);
}

}  // namespace

uint32_t cast_rays_ctas(uint64_t n_rays) { return static_cast<uint32_t>((n_rays + kRayThreads - 1) / kRayThreads); }

void launch_cast_rays(const OccupancyView& grid, const Pose2* poses, const double2* bearings, uint64_t n_bearings, uint64_t n_rays, double max_range,
                      double* ranges, cudaStream_t stream) {
  if (n_rays == 0) return;
  cast_rays_kernel<<<cast_rays_ctas(n_rays), kRayThreads, 0, stream>>>(grid, poses, bearings, n_bearings, n_rays, max_range, ranges);
}

}  // namespace bb200
