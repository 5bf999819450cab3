// Host control flow of beluga::Amcl (reference: algorithm/amcl_core.hpp:81-233) over the device
// filter: update / resample policies, rolling control window, recovery-probability estimator.
// Only scalars live here; particles never leave the GPU.
#pragma once

#include <memory>
#include <optional>
#include <string>

#include "filter.hpp"

namespace bb200 {

/// DifferentialDriveModel::sampling_fn_2d host part -- motion/differential_drive_model.hpp:129-154.
bb200_diff_drive_sampling diff_drive_sampling(const bb200_diff_drive_param& p, const Pose2& pose, const Pose2& previous_pose);
/// MotionModel::operator()(control) host part for the three motion models.
bb200_motion_sampling motion_sampling(const bb200_motion_param& p, const Pose2& pose, const Pose2& previous_pose);

class Amcl {
 public:
  Amcl(const bb200_amcl_param& p, const bb200_motion_param& motion);
  /// The host half alone (policies, control window, recovery estimator) for a filter whose particles live elsewhere -- a
  /// member of a batch (csrc/batch.hpp).  The owner reports the particle count through set_host_size().
  struct HostOnly {};
  Amcl(const bb200_amcl_param& p, const bb200_motion_param& motion, HostOnly);

  Filter& filter() { return *filter_; }
  bool ok() const { return filter_ && filter_->ok(); }
  int create_status() const { return filter_ ? filter_->create_status() : BB200_ERR_CUDA; }
  const char* last_error() const { return error_.empty() && filter_ ? filter_->last_error() : error_.c_str(); }
  /// Host-only: what initialize*() records after the owner has placed n particles.
  void host_initialized(uint64_t n) {
    host_size_ = n;
    force_update_ = true;
    initialized_ = n > 0;
  }
  /// Host-only: the particle count after a step (a resample sets it to max_particles).
  void set_host_size(uint64_t n) { host_size_ = n; }
  uint64_t host_size() const { return host_size_; }
  void record_error(const std::string& message) const { error_ = message; }  // the C-ABI exception guard

  int initialize(const double mean[3], const double cov[9]);
  int initialize_from_map();
  int initialize_states(const double* states, const double* weights, uint64_t n);
  void force_update() { force_update_ = true; }
  int update(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out);
  /// Host half of update(): policies, control window, recovery estimator -> what to run this step.
  int plan_update(const double control[4], bb200_step_plan* plan);
  /// Closes a planned step (estimator reset after injection, force_update flag).
  void commit_update(int resampled, double random_state_probability);
  bool sharded() const { return params_.shard_capacity != 0; }
  const bb200_amcl_param& params() const { return params_; }
  /// Amcl::update over the `count` shards of ONE filter held by this thread (count == 1: this process drives one shard
  /// and the other ranks call update() themselves, in lock step).  Every phase of the step is enqueued on all shards
  /// before the next one, the exchanges between the shards happen on the devices (csrc/kernels.cuh: ShardMail).
  static int update_group(Amcl* const* ranks, int count, const double control[4], const double* points_xy, uint64_t n_points,
                          bb200_update_result* out);

 private:
  bb200_amcl_param params_;
  bb200_motion_param motion_;
  std::unique_ptr<Filter> filter_;
  mutable std::string error_;

  // policies/on_motion.hpp:121-133
  std::optional<Pose2> latest_pose_;
  // policies/every_n.hpp:47-50
  uint64_t every_n_current_{0};
  // algorithm/thrun_recovery_probability_estimator.hpp:40-94 + exponential_filter.hpp:35-44
  double slow_output_{0.0}, fast_output_{0.0};
  // containers/circular_array.hpp:461-480 RollingWindow<SE2d, 2>
  Pose2 window_[2]{{1, 0, 0, 0}, {1, 0, 0, 0}};
  int window_size_{0};

  bool force_update_{true};
  bool initialized_{false};
  uint32_t step_{0};
  uint64_t host_size_{0};  // particle count of a host-only instance

 public:
  /// Everything plan_update() advances.  The reference's update() is atomic: when the device half of a step
  /// fails, the host half is rolled back so that a retry sees the same motion delta, every_n phase and filters.
  struct HostState {
    std::optional<Pose2> latest_pose;
    uint64_t every_n_current;
    double slow_output, fast_output;
    Pose2 window[2];
    int window_size;
    bool force_update;
    uint32_t step;
  };
  HostState snapshot() const;
  void restore(const HostState& s);

 private:
  int update_device(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out);
};

}  // namespace bb200
