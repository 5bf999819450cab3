// Host control flow of beluga::Amcl (reference: algorithm/amcl_core.hpp:81-233) over the device
// filter: update / resample policies, rolling control window, recovery-probability estimator.
// Only scalars live here; particles never leave the GPU.
#pragma once

#include <optional>
#include <string>

#include "filter.hpp"
#include "state_blob.hpp"

namespace bb200 {

/// DifferentialDriveModel::sampling_fn_2d host part -- motion/differential_drive_model.hpp:129-154.
bb200_diff_drive_sampling diff_drive_sampling(const bb200_diff_drive_param& p, const Pose2& pose, const Pose2& previous_pose);
/// MotionModel::operator()(control) host part for the three motion models.
bb200_motion_sampling motion_sampling(const bb200_motion_param& p, const Pose2& pose, const Pose2& previous_pose);

/// The host half of beluga::Amcl: update and resample policies, rolling control window, recovery-probability estimator.
/// It never touches a device: a bb200_amcl pairs it with a Filter, a member of a batch (csrc/batch.hpp) is one alone.
/// The reference's update() is atomic: when the device half of a step fails, the caller puts back a copy of the policy
/// taken before plan_update(), so that a retry sees the same motion delta, every_n phase and filters.
class AmclPolicy {
 public:
  AmclPolicy(const bb200_amcl_param& p, const bb200_motion_param& motion);

  const bb200_amcl_param& params() const { return params_; }
  const bb200_motion_param& motion() const { return motion_; }
  /// Everything of the policy that decides its later steps, apart from its parameters (a state blob's policy section) ...
  PolicyState save() const;
  /// ... and the policy that saved it, given the same parameters.
  void restore(const PolicyState& state);
  /// The next update runs whether or not the robot moved (amcl_core.hpp:136, after every initialisation).
  void force_update() { force_update_ = true; }
  /// Host half of update() for a filter of n particles (0: not initialised, no update): what to run this step.
  void plan_update(const double control[4], uint64_t n, bb200_step_plan* plan);
  /// Closes a planned step (estimator reset after injection, force_update flag).
  void commit_update(int resampled, double random_state_probability);

 private:
  bb200_amcl_param params_;
  bb200_motion_param motion_;

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
  uint32_t step_{0};
};

/// beluga::Amcl over one device filter (or one shard of a filter).
class Amcl {
 public:
  Amcl(const bb200_amcl_param& p, const bb200_motion_param& motion);

  /// The configurations a filter rejects, checked without touching a device (BB200_OK or BB200_ERR_INVALID_ARGUMENT).
  static int validate(const bb200_amcl_param& p, const bb200_motion_param& motion, std::string* error);

  Filter& filter() { return filter_; }
  bool ok() const { return filter_.ok(); }
  int create_status() const { return filter_.create_status(); }
  const char* last_error() const { return error_.empty() ? filter_.last_error() : error_.c_str(); }
  void record_error(const std::string& message) const { error_ = message; }  // the C-ABI exception guard

  int initialize(const double mean[3], const double cov[9]);
  int initialize_from_map();
  int initialize_states(const double* states, const double* weights, uint64_t n);
  /// This filter's state blob (state_blob.hpp) into out[0, capacity), its size in *size; out == nullptr: the size only.
  /// BB200_ERR_STATE for a shard, BB200_ERR_CAPACITY when capacity is below the size.
  int export_state(void* out, uint64_t capacity, uint64_t* size);
  /// Adopts a decoded state whose params and motion this filter was created with (bb200_amcl_create_from_state).
  int restore_state(const FilterState& s);
  void force_update() { policy_.force_update(); }
  int update(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out);
  /// update() with a landmark or bearing model: the map's model weighs the detections.  Refused on a shard: a sharded
  /// filter takes detection steps through ShardedAmcl::update_landmarks.
  int update_landmarks(const double control[4], const bb200_landmark_detection* detections, uint64_t n, bb200_update_result* out);
  /// AmclPolicy::plan_update over this filter's particle count (a shard: the global count once initialised).
  int plan_update(const double control[4], bb200_step_plan* plan);
  void commit_update(int resampled, double random_state_probability) { policy_.commit_update(resampled, random_state_probability); }
  bool sharded() const { return params().shard_capacity != 0; }
  const bb200_amcl_param& params() const { return policy_.params(); }
  /// Amcl::update over the `count` shards of ONE filter held by this thread (count == 1: this process drives one shard
  /// and the other ranks call update() themselves, in lock step).  Every phase of the step is enqueued on all shards
  /// before the next one, the exchanges between the shards happen on the devices (csrc/kernels.cuh: ShardMail).
  static int update_group(Amcl* const* ranks, int count, const double control[4], const double* points_xy, uint64_t n_points,
                          bb200_update_result* out);
  /// The first half of update() for a sensor model the caller runs: plans the step and, unless the policies skip it,
  /// enqueues the propagate; *view gets the device views the caller weighs.  The step stays open until update_end.
  /// Atomic as update(); refused on shards.
  int update_begin(const double control[4], bb200_weigh_view* view);
  /// The second half: w *= factors and everything update() runs after its sensor model.  Atomic as update().
  int update_end(bb200_update_result* out);
  /// update_begin over the `count` shards of ONE filter held by this thread: views[r] is shard r's slice of the global
  /// particle order (n may be 0 on a KLD-sized shard).  Every shard's step stays open until update_group_end.  Atomic as
  /// update_group.
  static int update_group_begin(Amcl* const* ranks, int count, const double control[4], bb200_weigh_view* views);
  /// The second half: w *= factors on every shard, then everything update_group runs after its sensor model.  No shard's
  /// exchange starts before every shard's factors are applied (stream waits, no host synchronisation).  Atomic as
  /// update_group.
  static int update_group_end(Amcl* const* ranks, int count, bb200_update_result* out);

 private:
  /// The checks and the host half of update_group, the same arithmetic on every shard: the plan, and every rank's policy
  /// before it in weighed_before_.  On failure every policy is put back.
  static int plan_group(Amcl* const* ranks, int count, const double control[4], bb200_step_plan* plan);
  /// Everything update_group runs once the sensor phase is enqueued on every shard: the phases, the KLD window loop, the
  /// selective resampling decision and the commit.  On failure every rank's policy is put back and the step is closed.
  static int finish_group(Amcl* const* ranks, int count, const bb200_step_plan& plan, bb200_update_result* out);
  /// Puts back every rank's policy from weighed_before_ and closes the step on every shard; returns `status`.
  static int rollback_group(Amcl* const* ranks, int count, int status);
  int update_device(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out);
  /// A step that resamples in the fused sequence with one host synchronisation (every_n fired, no ESS test, no KLD).
  bool fused(const bb200_step_plan& plan) const;
  /// What update() runs after the sensor model, up to the result and the policies' commit.
  int finish_update(const bb200_step_plan& plan, bb200_update_result* out);
  int initialized(int status, bool has_particles);  // after initialize*(): the next update is forced

  AmclPolicy policy_;
  Filter filter_;
  mutable std::string error_;
  bool initialized_{false};
  // the open weighed step's plan, and the policy to put back when a step fails (a weighed step, or a step of shards)
  bb200_step_plan weighed_plan_{};
  AmclPolicy weighed_before_{policy_};
};

}  // namespace bb200
