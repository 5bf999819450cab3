// Block body of the ray casts (raycast.cu), shared with the batch kernel: Ray2d::cast (algorithm/raycasting.hpp:79-107) for
// given sensor poses and bearings, over the beam model's ray walk (reweight_beam.cuh).
#pragma once

#include <math_constants.h>

#include "reweight_beam.cuh"

namespace bb200 {

namespace {

constexpr int kRayThreads = 256;

/// One CTA of the ray casts: one thread per ray of rays [block * kRayThreads, (block + 1) * kRayThreads) out of n_rays, pose
/// major (ray i * n_bearings + j is pose i, bearing j).  ranges[ray] = min(distance, max_range) on a hit, +inf on a miss.
/// Poses are sensor poses in the map frame; bearings are {cos, sin} pairs taken as given (SO2::raw, not normalised).
__device__ __forceinline__ void cast_rays_block(const OccupancyView& grid, const Pose2* __restrict__ poses, const double2* __restrict__ bearings,
                                                uint64_t n_bearings, uint64_t n_rays, double max_range, double* __restrict__ ranges, uint32_t block) {
  const uint64_t ray = static_cast<uint64_t>(block) * kRayThreads + threadIdx.x;
  if (ray >= n_rays) return;
  const uint64_t i = ray / n_bearings;
  const double2 bearing = bearings[ray - i * n_bearings];
  // Ray2d: source pose in the grid frame and its cell (raycasting.hpp:67-70).
  const Pose2 src = pose_mul(grid.world_to_grid, load_pose(poses + i));
  const int sx = source_cell(src.x, grid.inv_resolution), sy = source_cell(src.y, grid.inv_resolution);
  // far end = r1 * (bearing * max_range) + t1 (raycasting.hpp:81-85)
  const double fx = bearing.x * max_range, fy = bearing.y * max_range;
  const double ex = (src.c * fx - src.s * fy) + src.x;
  const double ey = (src.s * fx + src.c * fy) + src.y;
  RayWalk walk;
  ray_begin(walk, sx, sy, sx + far_span(ex, grid.inv_resolution, sx), sy + far_span(ey, grid.inv_resolution, sy));
  if (!(isfinite(ex) && isfinite(ey))) walk.active = false;  // e.g. a NaN range or heading: the end point lies outside the grid, a miss
  while (walk.active) ray_step(walk, grid);
  unsigned long long d2 = 0;
  const double hit = ray_result(walk, grid, sx, sy, max_range, d2);
  ranges[ray] = walk.hit ? hit : CUDART_INF;  // std::nullopt
}

}  // namespace

}  // namespace bb200
