// One filter over several shards driven by ONE host thread (the shape of beluga_ros's single-process node): shard r is an
// Amcl that holds the contiguous particle range [r * shard, (r + 1) * shard) of the filter, the shards' links are joined
// in this process, and every step runs Amcl::update_group over all of them.
#pragma once

#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "amcl.hpp"

namespace bb200 {

class ShardedAmcl {
 public:
  /// n_shards equal shards of a filter with parameters p, shard r on devices[r].
  ShardedAmcl(const bb200_amcl_param& p, const bb200_motion_param& motion, int n_shards, const int* devices);

  /// The configurations a sharded filter rejects, checked without touching a device (BB200_OK or BB200_ERR_INVALID_ARGUMENT).
  static int validate(const bb200_amcl_param& p, const bb200_motion_param& motion, int n_shards, std::string* error);

  bool ok() const { return created_; }
  int create_status() const { return create_status_; }
  /// The filter's own message, otherwise the first shard's (in rank order) that has one.
  const char* last_error() const;
  void record_error(const std::string& message) const { error_ = message; }  // the C-ABI exception guard
  /// Whether a weighed step is open: update_begin opens it on every shard at once.
  bool step_open() const { return !ranks_.empty() && ranks_[0]->filter().weigh_open(); }

  int shards() const { return static_cast<int>(ranks_.size()); }
  /// Shard r (nullptr when r is out of range).
  Amcl* shard(int r) const { return r >= 0 && r < shards() ? ranks_[static_cast<size_t>(r)] : nullptr; }

  /// Prepares the map's tables once (prepare fills them, or a message) and uploads them to every shard.  A failed
  /// preparation is reported by the first shard, as its own set_*_map call would.
  int set_map(const std::function<int(MapTables*, std::string*)>& prepare);
  /// set_map with the tables of Filter::set_landmark_map: the landmark model (lp) or, with lp null, the bearing model (bp).
  int set_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map);
  int initialize(const double mean[3], const double cov[9]);
  int initialize_from_map();
  void force_update();
  int update(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out);
  /// update() with the landmark map's model weighing the detections: prepared once, uploaded to every shard, then the
  /// step of update().  Null detections with n > 0, n >= 2^32 - 1 and a grid map are refused before any device work; a
  /// step the policies skip launches nothing beyond the uploads.  Atomic as update().
  int update_landmarks(const double control[4], const bb200_landmark_detection* detections, uint64_t n, bb200_update_result* out);
  int update_begin(const double control[4], bb200_weigh_view* views);
  int update_end(bb200_update_result* out);
  int cluster_estimate(const bb200_cluster_param& p, bb200_estimate* out, uint32_t* n_cells, uint32_t* n_clusters);
  int particle_histogram(double linear_resolution, double angular_resolution, bb200_cluster_cell* bins, uint64_t capacity, uint64_t* n_bins,
                         double* max_bin_weight);
  /// The particles in global index order (rank 0's shard first).
  int get_particles(double* states, double* weights, uint64_t capacity);
  int sample_states(uint64_t count, uint32_t step, double* states_out);
  int cast_rays(const double* poses, uint64_t n_poses, const double* bearings_cs, uint64_t n_bearings, double max_range, double* ranges);

 private:
  /// Every shard's cell records (Filter::cell_records, one device pass per shard) merged in rank order (merge_cells): the
  /// cells of the whole particle set in its global first-occurrence order.  BB200_ERR_STATE when no shard holds a particle.
  int merged_cells(double linear_resolution, double angular_resolution, std::vector<bb200_cluster_cell>* merged, uint64_t* n_particles);

  std::vector<std::unique_ptr<Amcl>> shards_;  // in rank order
  std::vector<Amcl*> ranks_;                   // the same shards, as Amcl::update_group takes them
  bool created_{false};
  int create_status_{BB200_OK};
  mutable std::string error_;
};

}  // namespace bb200
