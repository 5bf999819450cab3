// Per-particle bodies of the motion update and of the free-space state draw, shared by the single-filter kernels
// (propagate.cu), the batch kernels and the recovery injection of the resample.
#pragma once

#include "device_common.cuh"

namespace bb200 {

namespace {

constexpr int kPrThreads = 256;

/// MultivariateUniformDistribution<SE2d, OccupancyGrid> (random/multivariate_uniform_distribution.hpp:143-160): a free
/// cell drawn uniformly, its centroid in the global frame (occupancy_grid.hpp:150-156,166-172), yaw ~ U[-pi, pi).
struct FreeSpace {
  const uint32_t* cells;  // row-major indices of the free cells
  uint64_t n;
  int grid_width;
  double resolution;
  Pose2 origin;
};

__device__ __forceinline__ Pose2 random_free_state(const FreeSpace& fs, const Draw& r) {
  const uint32_t cell = fs.cells[mulhi64(r.a, fs.n)];
  const double pi = 3.14159265358979323846;
  const double yaw = uniform01(r.b) * (pi - (-pi)) + (-pi);
  const double lx = (static_cast<double>(static_cast<int>(cell % static_cast<uint32_t>(fs.grid_width))) + 0.5) * fs.resolution;
  const double ly = (static_cast<double>(static_cast<int>(cell / static_cast<uint32_t>(fs.grid_width))) + 0.5) * fs.resolution;
  const Rot2 rot = rot_exp(yaw);
  return Pose2{rot.c, rot.s, (fs.origin.c * lx - fs.origin.s * ly) + fs.origin.x, (fs.origin.s * lx + fs.origin.c * ly) + fs.origin.y};
}

/// MultivariateUniformDistribution<SE2d, AlignedBox2d> (random/multivariate_uniform_distribution.hpp:43-73) over a
/// landmark map's bounds: yaw ~ U[-pi, pi) first (SO2d::sampleUniform), then x, then y, each a
/// std::uniform_real_distribution: u * (max - min) + min.  Counter stream 6 gives yaw (word a) and x (word b), stream 7 y
/// (word a), both at the index and step of the free-cell draw.
struct BoxSpace {
  double min_x, max_x, min_y, max_y;
};

__device__ __forceinline__ Pose2 random_box_state(const BoxSpace& box, uint64_t seed, uint64_t index, uint32_t step) {
  const Draw r = counter_draw(seed, index, step, kStreamRandomState);
  const Draw q = counter_draw(seed, index, step, kStreamRandomBox);
  const double pi = 3.14159265358979323846;
  const double yaw = uniform01(r.a) * (pi - (-pi)) + (-pi);
  const double x = uniform01(r.b) * (box.max_x - box.min_x) + box.min_x;
  const double y = uniform01(q.a) * (box.max_y - box.min_y) + box.min_y;
  const Rot2 rot = rot_exp(yaw);
  return Pose2{rot.c, rot.s, x, y};
}

__device__ __forceinline__ Pose2 propagate_one(const Pose2& st, const MotionSampling& p, uint64_t seed, uint64_t index, uint32_t step) {
  double z0, z1;
  box_muller_fast(counter_draw(seed, index, step, kStreamMotion0), z0, z1);
  const double z2 = box_muller_first(counter_draw(seed, index, step, kStreamMotion1));
  // std::normal_distribution: ret * stddev + mean (libstdc++ bits/random.tcc:1843)
  const double d0 = z0 * p.stddev[0] + p.mean[0];
  const double d1 = z1 * p.stddev[1] + p.mean[1];
  const double d2 = z2 * p.stddev[2] + p.mean[2];
  return motion_apply_fast(p.model, st, d0, d1, d2, Rot2{p.first_c, p.first_s});
}

}  // namespace

}  // namespace bb200
