// Host-side map preprocessing of the CUDA MCL backend (once per map, not per step).
//
// Computes the per-cell grids the map tables are made from (device_map.hpp lays them out for the kernels):
//   * the likelihood field of LikelihoodFieldModelBase::make_likelihood_field
//     (reference: sensor/likelihood_field_model_base.hpp:130-185), whose brushfire distance map
//     (algorithm/distance_map.hpp:55-98) is order dependent -- the value of a cell depends on which
//     equal-distance parent leaves the std::priority_queue first -- so it is computed with the same
//     queue discipline on the host instead of an exact GPU distance transform;
//   * the free distance of the beam model's ray cast;
//   * the free-cell list of MultivariateUniformDistribution<SE2d, OccupancyGrid>
//     (random/multivariate_uniform_distribution.hpp:158-160).
#pragma once

#include <cstdint>
#include <vector>

#include "../../include/beluga_b200.h"

namespace bb200 {

/// ValueGrid2<float> contents, row-major.
std::vector<float> make_likelihood_field(const bb200_likelihood_field_param& params, const bb200_occupancy_grid& grid);

/// Chebyshev distance (in cells, capped at 255) from every cell to the nearest cell that is not
/// free or lies outside the grid; 0 for non-free cells.  A Bresenham line moves at most one cell
/// per step in each axis, so from a cell with distance d the next d - 1 cells of any ray are free:
/// the beam-model ray cast jumps d steps at a time and still stops at exactly the cell the
/// reference's cell-by-cell walk (algorithm/raycasting.hpp:97-107) stops at.
std::vector<uint8_t> make_free_distance(const bb200_occupancy_grid& grid);

/// Cell indices whose value is free (0), ascending.
std::vector<uint32_t> make_free_cells(const bb200_occupancy_grid& grid);

}  // namespace bb200
