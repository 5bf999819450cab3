// Host pass of the cluster-based estimate: the per-cell flood of
// beluga/algorithm/cluster_based_estimation.hpp (normalize_and_cap_weights :177-192,
// assign_clusters :205-253) and the per-cluster selection of estimate_clusters /
// cluster_based_estimate (:351-432), fed with one record per occupied cell from the device.
#pragma once

#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/beluga_b200.h"

namespace bb200 {

/// Host view of one device CellRecord (cluster.cuh), field for field.
struct HostCell {
  double representative[4];  // cos, sin, x, y
  unsigned long long hash;
  unsigned int first_index;
  unsigned int count;
  double weight;
  double moments[9];
};
static_assert(sizeof(HostCell) == 128, "must match bb200::CellRecord");

struct ClusterSelection {
  std::vector<uint32_t> cluster_of_cell;  // cluster id of every cell (assign_clusters)
  uint32_t clusters{0};                   // number of cluster ids handed out
  bool found{false};                      // a cluster with more than one particle exists
  uint32_t best{0};                       // its id: the heaviest such cluster (first of equals)
  double moments[9]{};                    // raw moments to estimate from: that cluster's, or the whole set's
};

/// cells in first-occurrence order (the insertion order of the reference's unordered_map);
/// n_particles sizes the map's initial reserve like make_cluster_map (:146).
ClusterSelection select_cluster(const HostCell* cells, std::size_t n_cells, std::uint64_t n_particles, double linear_resolution,
                                double angular_resolution, double weight_cap_percentile);

/// Mean and covariance (estimation.hpp:436-475) from the nine raw moments about `pivot` (layout of kMomentCount in
/// kernels.cuh): what every estimate ends with, of the whole set or of the selected cluster.
void estimate_from_moments(const double m[9], const double pivot[2], bb200_estimate* out);

/// Moves the moments' pivot to the estimate's position -- unless that is not finite (a normalising step over weights that
/// sum to 0, NaN or inf), which would make every later estimate NaN.
void pivot_to_estimate(const bb200_estimate& e, double pivot[2]);

}  // namespace bb200
