// Host pass of the cluster-based estimate: the per-cell flood of
// beluga/algorithm/cluster_based_estimation.hpp (normalize_and_cap_weights :177-192,
// assign_clusters :205-253) and the per-cluster selection of estimate_clusters /
// cluster_based_estimate (:351-432), fed with one record per occupied cell from the device.
#pragma once

#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/beluga_b200.h"
#include "cluster_select.cuh"

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

/// Why a cluster estimate refuses `p` (BB200_ERR_INVALID_ARGUMENT), or nullptr when it takes it.
inline const char* cluster_param_error(const bb200_cluster_param& p) {
  if (p.linear_hash_resolution > 0.0 && p.angular_hash_resolution > 0.0 && p.weight_cap_percentile >= 0.0 && p.weight_cap_percentile < 1.0)
    return nullptr;
  return "cluster parameters: resolutions must be positive and the percentile in [0, 1)";
}

/// cells in first-occurrence order (the insertion order of the reference's unordered_map);
/// n_particles sizes the map's initial reserve like make_cluster_map (:146).
ClusterSelection select_cluster(const HostCell* cells, std::size_t n_cells, std::uint64_t n_particles, double linear_resolution,
                                double angular_resolution, double weight_cap_percentile);

/// The bucket counts select_cluster's map passes through, probed from this process's libstdc++: for every
/// want = n_particles / 5 with n_particles <= kSelectMaxCells, start[want] is the first entry of the schedule (RehashStep,
/// cluster_select.cuh) of a map after reserve(want), which covers up to min(5 want + 4, kSelectMaxCells) insertions.
/// Wants whose reserve gives the same bucket count share one schedule.
struct RehashTable {
  std::vector<uint32_t> start;
  std::vector<RehashStep> steps;
};
const RehashTable& rehash_table();
/// Bytes of scratch a member of at most `capacity` particles needs for its selection (select_layout at its largest).
uint64_t select_scratch_bytes(uint64_t capacity);

/// bb200_cluster_merge_host (beluga_b200.h): per-shard cell records, shards in rank order, merged into the cells of the whole
/// particle set in its global first-occurrence order.  merged == nullptr: *n_merged receives the count only.
int merge_cells(const bb200_cluster_cell* const* shard_cells, const uint64_t* shard_counts, const uint64_t* shard_first_index, int shards,
                bb200_cluster_cell* merged, uint64_t capacity, uint64_t* n_merged);

/// Mean and covariance (estimation.hpp:436-475) from the nine raw moments about `pivot` (layout of kMomentCount in
/// kernels.cuh): what every estimate ends with, of the whole set or of the selected cluster.
void estimate_from_moments(const double m[9], const double pivot[2], bb200_estimate* out);

/// Moves the moments' pivot to the estimate's position -- unless that is not finite (a normalising step over weights that
/// sum to 0, NaN or inf), which would make every later estimate NaN.
void pivot_to_estimate(const bb200_estimate& e, double pivot[2]);

}  // namespace bb200
