// TEST INFRASTRUCTURE ONLY -- the CPU oracle's Ray2d::cast (oracle/beluga_oracle.hpp) with the bearing taken as a raw
// {cos, sin} pair (SO2::raw), so that the device and the oracle cast along identical bits; orc_raycast takes an angle.
// Built by tests/_raycast_oracle.py into a temporary directory; never linked into the product library.
#include <cstdint>
#include <limits>

#include "../../oracle/beluga_oracle.hpp"

using namespace oracle;

extern "C" {

/// ranges[i * n_bearings + j] = Ray2d{grid, poses[i], max_range}.cast(SO2::raw(bearings[j])), +inf for std::nullopt.  Poses
/// and the grid origin are {cos, sin, x, y}.
void orc_raycast_raw(const std::int8_t* cells, int width, int height, double resolution, const double* origin, const double* poses,
                     std::uint64_t n_poses, const double* bearings, std::uint64_t n_bearings, double max_range, double* ranges) {
  OccupancyGrid grid;
  grid.width = width;
  grid.height = height;
  grid.resolution = resolution;
  grid.origin = SE2{SO2::raw(origin[0], origin[1]), origin[2], origin[3]};
  grid.data.assign(cells, cells + static_cast<std::size_t>(width) * static_cast<std::size_t>(height));
  for (std::uint64_t i = 0; i < n_poses; ++i) {
    const double* p = poses + 4 * i;
    const Ray2d ray{grid, SE2{SO2::raw(p[0], p[1]), p[2], p[3]}, max_range};
    for (std::uint64_t j = 0; j < n_bearings; ++j) {
      const auto r = ray.cast(SO2::raw(bearings[2 * j], bearings[2 * j + 1]));
      ranges[i * n_bearings + j] = r.has_value() ? *r : std::numeric_limits<double>::infinity();
    }
  }
}

}  // extern "C"
