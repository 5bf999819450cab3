#include "amcl.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <initializer_list>
#include <limits>
#include <vector>

namespace bb200 {

namespace {

/// rotation_variance -- differential_drive_model.hpp:167-173: backward and forward motion are
/// treated symmetrically.
double rotation_variance(const Rot2& rotation) {
  static const Rot2 kFlip = rot_exp(3.14159265358979323846);
  const Rot2 flipped = rot_mul(rotation, kFlip);
  const double delta = std::min(std::fabs(rot_log(rotation)), std::fabs(rot_log(flipped)));
  return delta * delta;
}

double exponential_filter(double& output, double alpha, double input) {  // exponential_filter.hpp:41-44
  output += (output == 0.) ? input : alpha * (input - output);
  return output;
}

}  // namespace

bb200_diff_drive_sampling diff_drive_sampling(const bb200_diff_drive_param& p, const Pose2& pose, const Pose2& prev) {
  const double tx = pose.x - prev.x, ty = pose.y - prev.y;
  const double distance = std::sqrt(tx * tx + ty * ty);
  const double distance_variance = distance * distance;
  const Rot2 previous_orientation{prev.c, prev.s};
  const Rot2 current_orientation{pose.c, pose.s};
  const Rot2 heading_rotation = rot_exp(std::atan2(ty, tx));
  const Rot2 first_rotation = distance > p.distance_threshold ? rot_mul(heading_rotation, rot_inverse(previous_orientation)) : Rot2{1.0, 0.0};
  const Rot2 second_rotation = rot_mul(rot_mul(current_orientation, rot_inverse(previous_orientation)), rot_inverse(first_rotation));
  const double v1 = rotation_variance(first_rotation), v2 = rotation_variance(second_rotation);
  bb200_diff_drive_sampling s;
  s.rot1_mean = rot_log(first_rotation);
  s.rot1_std = std::sqrt(p.rotation_noise_from_rotation * v1 + p.rotation_noise_from_translation * distance_variance);
  s.trans_mean = distance;
  s.trans_std = std::sqrt(p.translation_noise_from_translation * distance_variance + p.translation_noise_from_rotation * (v1 + v2));
  s.rot2_mean = rot_log(second_rotation);
  s.rot2_std = std::sqrt(p.rotation_noise_from_rotation * v2 + p.rotation_noise_from_translation * distance_variance);
  return s;
}

bb200_motion_sampling motion_sampling(const bb200_motion_param& p, const Pose2& pose, const Pose2& prev) {
  bb200_motion_sampling out{};
  out.model = p.model;
  out.first_rotation[0] = 1.0;
  out.first_rotation[1] = 0.0;
  if (p.model == BB200_MOTION_STATIONARY) {  // stationary_model.hpp:55: N(0, 0.02) for theta, x, y
    for (int k = 0; k < 3; ++k) {
      out.mean[k] = 0.0;
      out.stddev[k] = 0.02;
    }
    return out;
  }
  if (p.model == BB200_MOTION_OMNIDIRECTIONAL) {  // omnidirectional_drive_model.hpp:101-129
    const double tx = pose.x - prev.x, ty = pose.y - prev.y;
    const double distance = std::sqrt(tx * tx + ty * ty);
    const double distance_variance = distance * distance;
    const Rot2 previous_orientation{prev.c, prev.s};
    const Rot2 current_orientation{pose.c, pose.s};
    const Rot2 rotation = rot_mul(current_orientation, rot_inverse(previous_orientation));
    const Rot2 heading_rotation = rot_exp(std::atan2(ty, tx));
    const Rot2 first_rotation = distance > p.distance_threshold ? rot_mul(heading_rotation, rot_inverse(previous_orientation)) : Rot2{1.0, 0.0};
    const double rv = rotation_variance(rotation);
    out.mean[0] = rot_log(rotation);
    out.stddev[0] = std::sqrt(p.rotation_noise_from_rotation * rv + p.rotation_noise_from_translation * distance_variance);
    out.mean[1] = distance;
    out.stddev[1] = std::sqrt(p.translation_noise_from_translation * distance_variance + p.translation_noise_from_rotation * rv);
    out.mean[2] = 0.0;
    out.stddev[2] = std::sqrt(p.strafe_noise_from_translation * distance_variance + p.translation_noise_from_rotation * rv);
    out.first_rotation[0] = first_rotation.c;
    out.first_rotation[1] = first_rotation.s;
    return out;
  }
  const bb200_diff_drive_param d{p.rotation_noise_from_rotation, p.rotation_noise_from_translation, p.translation_noise_from_translation,
                                 p.translation_noise_from_rotation, p.distance_threshold};
  const bb200_diff_drive_sampling s = diff_drive_sampling(d, pose, prev);
  out.mean[0] = s.rot1_mean, out.stddev[0] = s.rot1_std;
  out.mean[1] = s.trans_mean, out.stddev[1] = s.trans_std;
  out.mean[2] = s.rot2_mean, out.stddev[2] = s.rot2_std;
  return out;
}

AmclPolicy::AmclPolicy(const bb200_amcl_param& p, const bb200_motion_param& motion) : params_(p), motion_(motion) {
  if (params_.resample_interval == 0) params_.resample_interval = 1;
}

PolicyState AmclPolicy::save() const {
  PolicyState s{};
  s.has_latest_pose = latest_pose_.has_value() ? 1 : 0;
  if (latest_pose_) std::memcpy(s.latest_pose, &*latest_pose_, sizeof(s.latest_pose));
  std::memcpy(s.window, window_, sizeof(s.window));
  s.every_n_current = every_n_current_;
  s.slow_output = slow_output_;
  s.fast_output = fast_output_;
  s.step = step_;
  s.window_size = window_size_;
  s.force_update = force_update_ ? 1 : 0;
  return s;
}

void AmclPolicy::restore(const PolicyState& s) {
  latest_pose_.reset();
  if (s.has_latest_pose) latest_pose_ = Pose2{s.latest_pose[0], s.latest_pose[1], s.latest_pose[2], s.latest_pose[3]};
  std::memcpy(window_, s.window, sizeof(window_));
  every_n_current_ = s.every_n_current;
  slow_output_ = s.slow_output;
  fast_output_ = s.fast_output;
  step_ = s.step;
  window_size_ = s.window_size;
  force_update_ = s.force_update != 0;
}

void AmclPolicy::plan_update(const double control[4], uint64_t n, bb200_step_plan* plan) {
  *plan = bb200_step_plan{};
  const Pose2 pose{control[0], control[1], control[2], control[3]};
  if (n == 0) return;  // amcl_core.hpp:166-168 -> std::nullopt

  // update_policy_(control_action) -- on_motion vs the last ACCEPTED pose (on_motion.hpp:121-133)
  bool moved;
  if (!latest_pose_) {
    latest_pose_ = pose;
    moved = true;
  } else {
    const Pose2 delta = pose_mul(pose_inverse(*latest_pose_), pose);
    moved = std::sqrt(delta.x * delta.x + delta.y * delta.y) > params_.update_min_d ||
            std::fabs(rot_log(Rot2{delta.c, delta.s})) > params_.update_min_a;
    if (moved) latest_pose_ = pose;
  }
  if (!moved && !force_update_) return;

  // control_action_window_ << control (circular_array.hpp:473-480); reads clamp to size-1 (:353-361)
  window_[1] = window_[0];
  window_[0] = pose;
  window_size_ = std::min(window_size_ + 1, 2);
  const Pose2& previous = window_[std::min(1, window_size_ - 1)];
  plan->sampling = motion_sampling(motion_, window_[0], previous);
  plan->step = ++step_;

  // random_probability_estimator_(particles_) (thrun_recovery_probability_estimator.hpp:69-89) on the
  // normalised weights, whose total is 1 by construction: average = 1 / N.
  const double average_weight = 1.0 / static_cast<double>(n);
  const double fast_average = exponential_filter(fast_output_, params_.alpha_fast, average_weight);
  const double slow_average = exponential_filter(slow_output_, params_.alpha_slow, average_weight);
  double random_state_probability = 0.0;
  if (!(std::fabs(slow_average) < std::numeric_limits<double>::epsilon())) {
    random_state_probability = std::clamp(1.0 - fast_average / slow_average, 0.0, 1.0);
  }
  if (params_.recovery_probability_override > 0.0) random_state_probability = std::min(params_.recovery_probability_override, 1.0);
  plan->random_state_probability = random_state_probability;

  // resample_policy_: every_n (every_n.hpp:47-50); on_effective_size_drop is applied by the caller
  // once the effective sample size is known (commit_resample_decision).
  every_n_current_ = (every_n_current_ + 1) % params_.resample_interval;
  plan->resample = every_n_current_ == 0 ? 1 : 0;
  plan->needs_ess = (plan->resample && params_.selective_resampling) ? 1 : 0;

  bb200_resample_opts& o = plan->opts;
  o.scheme = params_.resample_scheme;
  o.step = step_;
  o.min_particles = params_.min_particles;
  o.max_particles = params_.max_particles;
  o.kld_epsilon = params_.kld_epsilon;
  o.kld_z = params_.kld_z;
  for (int k = 0; k < 3; ++k) o.spatial_resolution[k] = params_.spatial_resolution[k];
  o.random_state_probability = random_state_probability;
  plan->update = 1;
}

void AmclPolicy::commit_update(int resampled, double random_state_probability) {
  if (resampled && random_state_probability > 0.0) fast_output_ = slow_output_ = 0.0;  // amcl_core.hpp:184-186
  force_update_ = false;
}

// ---------------------------------------------------------------------------------------------------

Amcl::Amcl(const bb200_amcl_param& p, const bb200_motion_param& motion)
    : policy_(p, motion),
      filter_(bb200_filter_config{p.device, p.shard_capacity != 0 ? p.shard_capacity : p.max_particles, p.seed, p.shard_first_index, p.max_particles,
                                  p.record_ancestors}) {
  if (sharded() && p.min_particles < p.max_particles && filter_.ok()) (void)filter_.link().enable_kld();
}

int Amcl::validate(const bb200_amcl_param& p, const bb200_motion_param& motion, std::string* error) {
  auto reject = [&](const char* m) {
    if (error != nullptr) *error = m;
    return static_cast<int>(BB200_ERR_INVALID_ARGUMENT);
  };
  if (motion.model < BB200_MOTION_DIFFERENTIAL || motion.model > BB200_MOTION_STATIONARY) return reject("unknown motion model");
  if (p.shard_capacity != 0 && p.shard_first_index + p.shard_capacity > p.max_particles) return reject("a shard must lie inside [0, max_particles)");
  if (p.max_particles == 0 || p.min_particles > p.max_particles) return reject("need 0 < min_particles <= max_particles");
  if (!(p.alpha_slow >= 0.0) || !(p.alpha_slow <= p.alpha_fast))  // thrun_recovery_probability_estimator.hpp:49-50
    return reject("need 0 <= alpha_slow <= alpha_fast");
  return BB200_OK;
}

int Amcl::initialized(int status, bool has_particles) {
  if (status == BB200_OK) {
    policy_.force_update();  // amcl_core.hpp:136, beluga_ros/include/beluga_ros/amcl.hpp:193-199
    initialized_ = has_particles;
  }
  return status;
}

int Amcl::initialize(const double mean[3], const double cov[9]) {
  error_.clear();
  return initialized(filter_.initialize_normal(mean, cov, sharded() ? params().shard_capacity : params().max_particles), true);
}

int Amcl::initialize_from_map() {
  error_.clear();
  return initialized(filter_.initialize_uniform(sharded() ? params().shard_capacity : params().max_particles), true);
}

int Amcl::initialize_states(const double* states, const double* weights, uint64_t n) {
  error_.clear();
  return initialized(filter_.set_particles(states, weights, n), n > 0);
}

int Amcl::export_state(void* out, uint64_t capacity, uint64_t* size) {
  error_.clear();
  if (sharded() || filter_.link().world() > 1) return filter_.fail_with(BB200_ERR_STATE, "a sharded filter has no state blob");
  FilterState s{};
  s.params = params();
  s.motion = policy_.motion();
  s.policy = policy_.save();
  const bool record = params().record_ancestors != 0;
  if (const int st = filter_.particle_set(&s.set, nullptr, size, record)) return st;
  if (out == nullptr) return BB200_OK;
  if (capacity < *size) return filter_.fail_with(BB200_ERR_CAPACITY, "state blob buffer too small (size has the blob's size)");
  ParticleArrays arrays;
  if (const int st = filter_.particle_set(&s.set, &arrays, size, record)) return st;
  s.states = arrays.states.data();
  s.weights = arrays.weights.data();
  s.cdf = arrays.cdf.data();
  s.ancestors = arrays.ancestors.data();
  write_state_blob(s, out);
  return BB200_OK;
}

int Amcl::restore_state(const FilterState& s) {
  error_.clear();
  const int st = filter_.restore_particle_set(s);
  if (st != BB200_OK) return st;
  policy_.restore(s.policy);
  initialized_ = s.set.n > 0;
  return BB200_OK;
}

int Amcl::plan_update(const double control[4], bb200_step_plan* plan) {
  error_.clear();
  // Sharded filters gate on the GLOBAL particle count, which never drops to zero once initialised.
  const uint64_t n = sharded() ? (initialized_ ? filter_.global_size() : 0u) : filter_.size();
  policy_.plan_update(control, n, plan);
  return BB200_OK;
}

int Amcl::rollback_group(Amcl* const* ranks, int count, int status) {
  for (int r = 0; r < count; ++r) {
    ranks[r]->policy_ = ranks[r]->weighed_before_;
    ranks[r]->filter_.step_abort();
  }
  return status;
}

int Amcl::plan_group(Amcl* const* ranks, int count, const double control[4], bb200_step_plan* plan) {
  Amcl& lead = *ranks[0];
  const bool kld = lead.params().min_particles < lead.params().max_particles;
  if (kld)
    for (int r = 0; r < count; ++r)
      if (!ranks[r]->filter_.link().kld())
        return ranks[r]->filter_.fail_with(BB200_ERR_STATE, "KLD-adaptive resampling on shards: the hash arrays were not exported (create the shards with min_particles < max_particles before joining them)");
  for (int r = 0; r < count; ++r)
    if (ranks[r]->sharded() && ranks[r]->filter_.link().world() <= 1)
      return ranks[r]->filter_.fail_with(BB200_ERR_STATE, "this shard has not joined its peers (bb200_amcl_join_shards / bb200_sharded_amcl_create)");
  for (int r = 0; r < count; ++r) ranks[r]->weighed_before_ = ranks[r]->policy_;
  // The host half is the same arithmetic on every shard (policies, control window, recovery estimator).
  *plan = bb200_step_plan{};
  for (int r = 0; r < count; ++r) {
    bb200_step_plan p{};
    const int st = ranks[r]->plan_update(control, &p);
    if (st != BB200_OK) return rollback_group(ranks, count, st);
    if (r == 0) *plan = p;
    if (p.update != plan->update || p.step != plan->step)
      return rollback_group(ranks, count, lead.filter_.fail_with(BB200_ERR_STATE, "the shards of a filter disagree on the step plan"));
  }
  return BB200_OK;
}

int Amcl::update_group(Amcl* const* ranks, int count, const double control[4], const double* points_xy, uint64_t n_points,
                       bb200_update_result* out) {
  *out = bb200_update_result{};
  if (ranks == nullptr || count < 1 || count > kMaxShards) return BB200_ERR_INVALID_ARGUMENT;
  bb200_step_plan plan{};
  int st = plan_group(ranks, count, control, &plan);
  if (st != BB200_OK || !plan.update) return st;
  const bool resample_now = plan.resample != 0 && plan.needs_ess == 0;
  for (int r = 0; r < count; ++r) {
    st = ranks[r]->filter_.step_begin(plan.sampling, plan.step, points_xy, n_points, plan.opts, resample_now);
    if (st != BB200_OK) return rollback_group(ranks, count, st);
  }
  for (int r = 0; r < count; ++r) {
    st = ranks[r]->filter_.step_phase(Filter::kPhaseReweight);
    if (st != BB200_OK) return rollback_group(ranks, count, st);
  }
  return finish_group(ranks, count, plan, out);
}

int Amcl::finish_group(Amcl* const* ranks, int count, const bb200_step_plan& plan, bb200_update_result* out) {
  Amcl& lead = *ranks[0];
  const bool kld = lead.params().min_particles < lead.params().max_particles;
  out->random_state_probability = plan.random_state_probability;

  auto run_phases = [&](std::initializer_list<int> phases) {
    for (const int phase : phases)
      for (int r = 0; r < count; ++r) {
        const int st = ranks[r]->filter_.step_phase(phase);
        if (st != BB200_OK) return st;
      }
    return static_cast<int>(BB200_OK);
  };
  auto close_batch = [&](double* sum_sq) {
    for (int r = 0; r < count; ++r) {
      bb200_estimate est{};
      double weight_sum = 0.0, sq = 0.0;
      uint64_t n = 0;
      const int st = ranks[r]->filter_.step_end(&est, &weight_sum, &n, &sq);
      if (st != BB200_OK) return st;
      if (r == 0) {  // the exchanged sums are the same bits on every shard
        out->estimate = est;
        out->weight_sum = weight_sum;
        out->n_particles = n;
        if (sum_sq != nullptr) *sum_sq = sq;
      }
    }
    return static_cast<int>(BB200_OK);
  };
  // views::take_while_kld over the shards (take_while_kld.hpp:72-137): the candidate stream is ordered by output slot, and
  // every rank sees the spatial hash of every candidate, so all ranks count distinct buckets over the same stream and
  // stop at the same slot.  Windows of slots double like the single-GPU chunks; one host decision per window.
  auto kld_size = [&](uint64_t* accepted) {
    const uint64_t max = lead.params().max_particles;
    for (int r = 0; r < count; ++r) {
      const int st = ranks[r]->filter_.step_totals();  // on every shard
      if (st != BB200_OK) return st;
    }
    uint64_t begin = 0, k_before = 0;
    uint64_t end = std::min<uint64_t>(max, std::max<uint64_t>(2 * lead.params().min_particles, 65536));
    *accepted = max;
    while (begin < max) {
      for (int r = 0; r < count; ++r) {
        const int st = ranks[r]->filter_.kld_sharded_candidates(begin, end);
        if (st != BB200_OK) return st;
      }
      for (int r = 0; r < count; ++r) {
        const int st = ranks[r]->filter_.kld_sharded_count(begin, end, k_before);
        if (st != BB200_OK) return st;
      }
      uint64_t cutoff = ~0ull, fresh = 0;
      for (int r = 0; r < count; ++r) {
        uint64_t c = 0, f = 0;
        const int st = ranks[r]->filter_.kld_sharded_read(&c, &f);
        if (st != BB200_OK) return st;
        if (r == 0) {
          cutoff = c;
          fresh = f;
        } else if (c != cutoff || f != fresh) {
          return lead.filter_.fail_with(BB200_ERR_STATE, "KLD on shards: the ranks disagree on the count");
        }
      }
      if (cutoff != ~0ull) {
        *accepted = std::min<uint64_t>(cutoff - 1, max);  // take_while drops the first element whose condition fails (:134-136)
        break;
      }
      k_before += fresh;
      begin = end;
      end = std::min<uint64_t>(max, end * 2);
    }
    return static_cast<int>(BB200_OK);
  };

  const bool resample_now = plan.resample != 0 && plan.needs_ess == 0;
  int st = BB200_OK;
  if (resample_now && kld) {
    st = run_phases({Filter::kPhaseCdf});
    uint64_t accepted = 0;
    if (st == BB200_OK) st = kld_size(&accepted);
    if (st == BB200_OK) {
      for (int r = 0; r < count; ++r) ranks[r]->filter_.step_set_kld_accepted(accepted);
      st = run_phases({Filter::kPhaseResample, Filter::kPhaseFinish});
    }
  } else {
    st = resample_now ? run_phases({Filter::kPhaseCdf, Filter::kPhaseResample, Filter::kPhaseFinish})
                      : run_phases({Filter::kPhaseCdf, Filter::kPhaseNormalize, Filter::kPhaseFinish});
  }
  double sum_sq = 0.0;
  if (st == BB200_OK) st = close_batch(&sum_sq);
  if (st != BB200_OK) return rollback_group(ranks, count, st);
  bool resampled = resample_now;
  if (!resample_now && plan.resample != 0) {
    // on_effective_size_drop (on_effective_size_drop.hpp:45-49): ESS = 1 / sum w~^2 < N / 2
    const double ess = sum_sq > 0.0 ? 1.0 / sum_sq : 0.0;
    if (ess < static_cast<double>(lead.filter_.global_size()) * 0.5) {
      if (kld) {
        uint64_t accepted = 0;
        st = kld_size(&accepted);
        if (st != BB200_OK) return rollback_group(ranks, count, st);
        for (int r = 0; r < count; ++r) ranks[r]->filter_.step_set_kld_accepted(accepted);
      }
      st = run_phases({Filter::kPhaseResample, Filter::kPhaseFinish});
      if (st == BB200_OK) st = close_batch(nullptr);
      if (st != BB200_OK) return rollback_group(ranks, count, st);
      resampled = true;
    }
  }
  out->resampled = resampled ? 1 : 0;
  out->weights_degenerate = lead.filter_.last_weights_valid() ? 0 : 1;
  for (int r = 0; r < count; ++r) {
    ranks[r]->filter_.step_abort();
    ranks[r]->commit_update(out->resampled, plan.random_state_probability);
  }
  out->updated = 1;
  return BB200_OK;
}

int Amcl::update(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out) {
  if (sharded()) {  // this process drives one shard; the peers call update() themselves
    Amcl* self = this;
    return update_group(&self, 1, control, points_xy, n_points, out);
  }
  const AmclPolicy before = policy_;
  const int st = update_device(control, points_xy, n_points, out);
  if (st != BB200_OK) policy_ = before;  // policies, control window and recovery estimator as if the call had not happened
  return st;
}

int Amcl::update_landmarks(const double control[4], const bb200_landmark_detection* detections, uint64_t n, bb200_update_result* out) {
  if (sharded()) return filter_.fail_with(BB200_ERR_STATE, "detection steps on shards run through bb200_sharded_amcl_update_landmarks; a shard joined by bb200_amcl_join_shards takes points");
  if (const int st = filter_.stage_detections(detections, n)) return st;
  return update(control, Filter::staged_detections(), 0, out);
}

bool Amcl::fused(const bb200_step_plan& plan) const {
  return plan.resample != 0 && !plan.needs_ess && !(params().min_particles < params().max_particles);
}

int Amcl::update_device(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out) {
  *out = bb200_update_result{};
  bb200_step_plan plan;
  int st = plan_update(control, &plan);
  if (st != BB200_OK || !plan.update) return st;
  if (fused(plan)) {
    // The whole step in one stream-ordered sequence with a single host synchronisation.
    st = filter_.step_begin(plan.sampling, plan.step, points_xy, n_points, plan.opts, true);
    if (st == BB200_OK) st = filter_.step_phase(Filter::kPhaseReweight);
    if (st != BB200_OK) {
      filter_.step_abort();
      return st;
    }
  } else {
    st = filter_.propagate_reweight(&plan.sampling, plan.step, points_xy, n_points);
    if (st != BB200_OK) return st;
  }
  return finish_update(plan, out);
}

int Amcl::finish_update(const bb200_step_plan& plan, bb200_update_result* out) {
  out->random_state_probability = plan.random_state_probability;
  if (fused(plan)) {
    uint64_t new_size = 0;
    const int st = filter_.finish_resample(&out->estimate, &out->weight_sum, &new_size);
    if (st != BB200_OK) return st;
    out->resampled = 1;
    out->n_particles = new_size;
  } else {
    const uint64_t n = filter_.size();
    bool do_resample = plan.resample != 0;
    double factor = 0.0, sum_sq = 0.0;
    int st = filter_.normalize(&factor, &sum_sq);
    if (st != BB200_OK) return st;
    out->weight_sum = factor;
    if (plan.needs_ess) {
      // on_effective_size_drop (on_effective_size_drop.hpp:45-49): ESS = 1 / sum w~^2 < N / 2
      const double ess = sum_sq > 0.0 ? 1.0 / sum_sq : 0.0;
      do_resample = ess < static_cast<double>(n) * 0.5;
    }
    if (do_resample) {
      uint64_t new_size = 0;
      st = filter_.resample(plan.opts, &new_size);
      if (st != BB200_OK) return st;
      out->resampled = 1;
    }
    st = filter_.estimate(&out->estimate);
    if (st != BB200_OK) return st;
    out->n_particles = filter_.size();
  }
  out->weights_degenerate = filter_.last_weights_valid() ? 0 : 1;
  commit_update(out->resampled, plan.random_state_probability);
  out->updated = 1;
  return BB200_OK;
}

int Amcl::update_begin(const double control[4], bb200_weigh_view* view) {
  error_.clear();
  if (filter_.weigh_open()) return filter_.fail_with(BB200_ERR_STATE, "a weighed step is already open (bb200_amcl_update_end closes it)");
  *view = bb200_weigh_view{};
  if (sharded() || filter_.link().world() > 1)
    return filter_.fail_with(BB200_ERR_STATE, "a shard takes weighed steps only with its filter (bb200_sharded_amcl_update_begin)");
  weighed_before_ = policy_;
  bb200_step_plan& plan = weighed_plan_;
  int st = plan_update(control, &plan);
  if (st == BB200_OK && plan.update) {
    const bool injects = plan.resample != 0 && plan.random_state_probability > 0.0;
    st = filter_.weigh_prepare(plan.opts, injects);
    if (st == BB200_OK) st = filter_.weigh_propagate(plan.sampling, plan.step, plan.opts, fused(plan));
  }
  if (st != BB200_OK) {
    policy_ = weighed_before_;  // as update(): policies, control window and recovery estimator as if the call had not happened
    filter_.step_abort();
    return st;
  }
  filter_.set_weigh_open(true);
  view->updated = plan.update;
  if (plan.update) {
    view->n = filter_.size();
    view->states = filter_.weigh_states();
    view->factors = filter_.weigh_factors();
    view->stream = filter_.stream();
  }
  return BB200_OK;
}

int Amcl::update_end(bb200_update_result* out) {
  *out = bb200_update_result{};
  // A shard's weigh_open flag belongs to its filter's step: this call leaves it open.
  if (sharded() || filter_.link().world() > 1)
    return filter_.fail_with(BB200_ERR_STATE, "a shard's weighed step is closed with its filter (bb200_sharded_amcl_update_end)");
  if (!filter_.weigh_open()) return filter_.fail_with(BB200_ERR_STATE, "no weighed step is open (bb200_amcl_update_begin)");
  filter_.set_weigh_open(false);
  if (!weighed_plan_.update) return BB200_OK;
  int st = filter_.weigh_apply();
  if (st == BB200_OK) st = finish_update(weighed_plan_, out);
  if (st != BB200_OK) {
    *out = bb200_update_result{};
    policy_ = weighed_before_;
    filter_.step_abort();
  }
  return st;
}

int Amcl::update_group_begin(Amcl* const* ranks, int count, const double control[4], bb200_weigh_view* views) {
  if (ranks == nullptr || count < 1 || count > kMaxShards) return BB200_ERR_INVALID_ARGUMENT;
  for (int r = 0; r < count; ++r)
    if (ranks[r]->filter_.weigh_open())
      return ranks[r]->filter_.fail_with(BB200_ERR_STATE, "a weighed step is already open (bb200_sharded_amcl_update_end closes it)");
  for (int r = 0; r < count; ++r) views[r] = bb200_weigh_view{};
  bb200_step_plan plan{};
  int st = plan_group(ranks, count, control, &plan);
  if (st != BB200_OK) return st;
  if (plan.update) {
    const bool resample_now = plan.resample != 0 && plan.needs_ess == 0;
    const bool injects = plan.resample != 0 && plan.random_state_probability > 0.0;
    // Every shard's checks and allocations before any shard's propagate: a refusal leaves every shard's particles as they were.
    for (int r = 0; r < count; ++r) {
      st = ranks[r]->filter_.weigh_prepare(plan.opts, injects);
      if (st != BB200_OK) return rollback_group(ranks, count, st);
    }
    for (int r = 0; r < count; ++r) {
      st = ranks[r]->filter_.weigh_propagate(plan.sampling, plan.step, plan.opts, resample_now);
      if (st != BB200_OK) return rollback_group(ranks, count, st);
    }
  }
  for (int r = 0; r < count; ++r) {
    Filter& f = ranks[r]->filter_;
    ranks[r]->weighed_plan_ = plan;
    f.set_weigh_open(true);
    views[r].updated = plan.update;
    if (plan.update) {
      views[r].n = f.size();
      views[r].states = f.weigh_states();
      views[r].factors = f.weigh_factors();
      views[r].stream = f.stream();
    }
  }
  return BB200_OK;
}

int Amcl::update_group_end(Amcl* const* ranks, int count, bb200_update_result* out) {
  *out = bb200_update_result{};
  if (ranks == nullptr || count < 1 || count > kMaxShards) return BB200_ERR_INVALID_ARGUMENT;
  for (int r = 0; r < count; ++r)
    if (!ranks[r]->filter_.weigh_open())
      return ranks[r]->filter_.fail_with(BB200_ERR_STATE, "no weighed step is open (bb200_sharded_amcl_update_begin)");
  for (int r = 0; r < count; ++r) ranks[r]->filter_.set_weigh_open(false);
  const bb200_step_plan plan = ranks[0]->weighed_plan_;
  if (!plan.update) return BB200_OK;
  for (int r = 0; r < count; ++r) {
    const int st = ranks[r]->filter_.step_phase(Filter::kPhaseApplyFactors);
    if (st != BB200_OK) return rollback_group(ranks, count, st);
  }
  // Every shard's exchanges wait for the device, with a timeout: none may start while a peer's sensor model still runs.
  for (int r = 0; r < count; ++r)
    for (int q = 0; q < count; ++q)
      if (q != r) {
        const int st = ranks[r]->filter_.wait_for_factors(ranks[q]->filter_);
        if (st != BB200_OK) return rollback_group(ranks, count, st);
      }
  const int st = finish_group(ranks, count, plan, out);
  if (st != BB200_OK) *out = bb200_update_result{};
  return st;
}

}  // namespace bb200
