// TEST INFRASTRUCTURE ONLY -- CPU parity oracle: the filter driver.
//
// Restates beluga::Amcl (algorithm/amcl_core.hpp:81-233 of /root/reference/beluga/include/beluga)
// over the scalar functions of beluga_oracle.hpp, in two RNG modes:
//   mode A  libstdc++: one std::mt19937_64 shared by propagate / bernoulli / discrete_distribution
//           in the reference's draw order (ranges::detail::get_random_engine() is a thread-local
//           std::mt19937_64; here it is seedable).  Statistical cross-check only.
//   mode B  counter: Philox4x32-10 keyed by (seed; slot, step, stream) and a fixed-point CDF.
//           This is the definition the GPU implements and the oracle of record for
//           "bit-exact resample indices" (parity unpinned in the reference, see beluga_oracle.hpp).
// `threads` > 1 parallelises propagate / reweight / normalize over particles with OpenMP, which is
// what std::execution::par covers in the reference (actions/propagate.hpp:72-77,
// actions/reweight.hpp:57-59, actions/normalize.hpp:77-82); everything else stays sequential.
#pragma once

#include <cstring>
#include <memory>
#include <string>

#include "beluga_oracle.hpp"

namespace oracle {

enum class SensorKind : int { kLikelihoodField = 0, kLikelihoodFieldProb = 1, kBeam = 2 };
enum class RngMode : int { kStd = 0, kCounter = 1 };

/// algorithm/amcl_core.hpp:34-55 plus the knobs of the drop-in backend.
struct AmclParams {
  double update_min_d = 0.25;
  double update_min_a = 0.2;
  std::size_t resample_interval = 1;
  bool selective_resampling = false;
  std::size_t min_particles = 500;
  std::size_t max_particles = 2000;
  double alpha_slow = 0.001;
  double alpha_fast = 0.1;
  double kld_epsilon = 0.05;
  double kld_z = 3.0;
  // spatial_hash<SE2d> resolutions (beluga_ros/include/beluga_ros/amcl.hpp:91-97 defaults)
  double spatial_resolution_x = 0.5;
  double spatial_resolution_y = 0.5;
  double spatial_resolution_theta = 10.0 * 3.14159265358979323846 / 180.0;
  // backend knobs
  RngMode rng_mode = RngMode::kCounter;
  ResampleScheme scheme = ResampleScheme::kMultinomial;
  std::uint64_t seed = 0;
  int threads = 1;
};

struct UpdateResult {
  bool updated{false};
  Estimate estimate{};
  std::size_t n_particles{0};
  bool resampled{false};
  double random_state_probability{0.0};
  double weight_sum{0.0};  // normalisation factor used this step
  std::uint64_t cells_visited{0};  // beam model: Bresenham cells inspected (algorithmic bytes)
};

class Amcl {
 public:
  Amcl(const AmclParams& p, const DifferentialDriveParam& motion, int motion_model = 0, const OmnidirectionalDriveParam& omni = {})
      : params_(p), motion_(motion), motion_model_(motion_model), omni_(omni), thrun_(p.alpha_slow, p.alpha_fast), engine_(p.seed) {
    update_policy_.min_distance = p.update_min_d;
    update_policy_.min_angle = p.update_min_a;
    every_n_.count = p.resample_interval;
  }

  void set_likelihood_field_model(const LikelihoodFieldParam& lp, const OccupancyGrid& grid, bool prob) {
    grid_ = grid;
    lfm_ = std::make_unique<LikelihoodFieldModel>(lp, grid_);
    sensor_ = prob ? SensorKind::kLikelihoodFieldProb : SensorKind::kLikelihoodField;
    free_ = free_cells(grid_);
  }
  void set_beam_model(const BeamModelParam& bp, const OccupancyGrid& grid) {
    grid_ = grid;
    beam_ = bp;
    sensor_ = SensorKind::kBeam;
    free_ = free_cells(grid_);
  }
  [[nodiscard]] const LikelihoodFieldModel* lfm() const { return lfm_.get(); }

  /// amcl_core.hpp:131-147 with MultivariateNormalDistribution{pose, covariance}.
  void initialize_normal(const double mean_xyt[3], const double cov[9]) {
    double transform[9];
    normal_transform(cov, transform);
    states_.resize(params_.max_particles);
    weights_.assign(params_.max_particles, 1.0);  // make_from_state: weight = 1 (particle_traits.hpp:105)
    if (params_.rng_mode == RngMode::kCounter) {
      for (std::size_t i = 0; i < states_.size(); ++i) states_[i] = normal_state_counter(mean_xyt, transform, params_.seed, i);
    } else {
      std::normal_distribution<double> n;
      for (auto& s : states_) {
        double d[3] = {n(engine_), n(engine_), n(engine_)};
        s = normal_state_from_delta(mean_xyt, transform, d);
      }
    }
    force_update_ = true;
  }

  /// beluga_ros::Amcl::initialize_from_map (beluga_ros/include/beluga_ros/amcl.hpp:192-209): max_particles samples of
  /// MultivariateUniformDistribution<SE2d, OccupancyGrid> (random/multivariate_uniform_distribution.hpp:127-161).
  void initialize_from_map() {
    if (free_.empty()) throw std::runtime_error("initialize_from_map: the map has no free cell");
    states_.resize(params_.max_particles);
    weights_.assign(params_.max_particles, 1.0);
    if (params_.rng_mode == RngMode::kCounter) {
      for (std::size_t i = 0; i < states_.size(); ++i) states_[i] = random_state_counter(grid_, free_, params_.seed, i, 0);
    } else {
      // operator()(engine): SO2d::sampleUniform(engine) first, then the free-state index (:143-145)
      std::uniform_int_distribution<std::size_t> pick(0, free_.size() - 1);
      const double pi = 3.14159265358979323846;
      std::uniform_real_distribution<double> yaw(-pi, pi);
      for (auto& s : states_) {
        const double theta = yaw(engine_);
        s = free_cell_state(grid_, free_[pick(engine_)], theta);
      }
    }
    force_update_ = true;
  }

  void set_particles(const std::vector<SE2>& states, const std::vector<double>& weights) {
    states_ = states;
    weights_ = weights;
    force_update_ = true;
  }
  void force_update() { force_update_ = true; }

  [[nodiscard]] const std::vector<SE2>& states() const { return states_; }
  [[nodiscard]] const std::vector<double>& weights() const { return weights_; }
  /// Ancestor index of each particle produced by the last resample (-1: injected random state).
  [[nodiscard]] const std::vector<std::int64_t>& last_indices() const { return last_indices_; }

  /// amcl_core.hpp:165-201
  UpdateResult update(const SE2& control_action, const Points& measurement) {
    UpdateResult out;
    if (states_.empty()) return out;
    if (!update_policy_(control_action) && !force_update_) return out;

    window_.push(control_action);
    const MotionSampling sampling = motion_model_ == 1   ? omni_drive_sampling(omni_, window_[0], window_[1])
                                    : motion_model_ == 2 ? stationary_sampling()
                                                         : to_motion_sampling(diff_drive_sampling(motion_, window_[0], window_[1]));
    ++step_;

    propagate(sampling);
    out.cells_visited = reweight(measurement);
    out.weight_sum = normalize_weights();

    // thrun_recovery_probability_estimator.hpp:69-89 on the normalised weights.
    double total_weight;
    if (params_.rng_mode == RngMode::kCounter) {
      total_weight = 1.0;  // mode B: the normalised total is 1 by construction (weights /= S)
    } else {
      total_weight = std::accumulate(weights_.begin(), weights_.end(), 0.0);
    }
    const double random_state_probability = thrun_.update(total_weight, states_.size());
    out.random_state_probability = random_state_probability;

    bool do_resample = every_n_();
    if (params_.selective_resampling) {
      // policies/policy.hpp:47-50 operator&& short-circuits: every_n always advances its counter,
      // on_effective_size_drop (stateless, on_effective_size_drop.hpp:45-49) only runs when it fired.
      do_resample = do_resample && (effective_sample_size(weights_) < static_cast<double>(weights_.size()) * 0.5);
    }
    if (do_resample) {
      if (random_state_probability > 0.0) thrun_.reset();
      resample(random_state_probability);
      out.resampled = true;
    }
    force_update_ = false;
    out.updated = true;
    out.estimate = estimate(states_, weights_);
    out.n_particles = states_.size();
    return out;
  }

 private:
  void propagate(const MotionSampling& sampling) {
    if (params_.rng_mode == RngMode::kCounter) {
      const std::int64_t n = static_cast<std::int64_t>(states_.size());
#pragma omp parallel for num_threads(params_.threads) schedule(static) if (params_.threads > 1)
      for (std::int64_t i = 0; i < n; ++i) {
        states_[static_cast<std::size_t>(i)] =
            motion_sample_counter(states_[static_cast<std::size_t>(i)], sampling, params_.seed, static_cast<std::uint64_t>(i), step_);
      }
    } else {
      motion_propagate_std(states_, sampling, motion_distribution_, engine_);
    }
  }

  std::uint64_t reweight(const Points& points) {
    const std::int64_t n = static_cast<std::int64_t>(states_.size());
    std::uint64_t visited_total = 0;
#pragma omp parallel for num_threads(params_.threads) schedule(static) reduction(+ : visited_total) if (params_.threads > 1)
    for (std::int64_t i = 0; i < n; ++i) {
      const SE2& s = states_[static_cast<std::size_t>(i)];
      double likelihood = 1.0;
      switch (sensor_) {
        case SensorKind::kLikelihoodField:
          likelihood = lfm_->weight(s, points);
          break;
        case SensorKind::kLikelihoodFieldProb:
          likelihood = lfm_->weight_prob(s, points);
          break;
        case SensorKind::kBeam: {
          std::uint64_t visited = 0;
          likelihood = beam_weight(beam_, grid_, s, points, &visited);
          visited_total += visited;
          break;
        }
      }
      weights_[static_cast<std::size_t>(i)] *= likelihood;  // actions/reweight.hpp:54-60
    }
    return visited_total;
  }

  double normalize_weights() {
    if (params_.rng_mode == RngMode::kCounter) {
      // Mode B: the normalisation factor is the fixed-point total, S = T * 2^-e (exactly
      // reproducible for any summation order / rank count).
      cdf_ = fixed_point_cdf(weights_);
      const double factor = std::ldexp(static_cast<double>(cdf_.total), -cdf_.exponent);
      if (!cdf_.valid) return factor;  // no weight can be selected: weights kept, resampling draws from the uniform CDF
      const std::int64_t n = static_cast<std::int64_t>(weights_.size());
#pragma omp parallel for num_threads(params_.threads) schedule(static) if (params_.threads > 1)
      for (std::int64_t i = 0; i < n; ++i) weights_[static_cast<std::size_t>(i)] = weights_[static_cast<std::size_t>(i)] / factor;
      return factor;
    }
    return normalize(weights_);
  }

  void resample(double random_state_probability) {
    const std::size_t max = params_.max_particles;
    std::vector<SE2> new_states;
    new_states.reserve(max);
    last_indices_.clear();
    KldCondition kld{params_.min_particles, params_.kld_epsilon, params_.kld_z, 0, {}};
    const auto hash = [this](const SE2& s) {
      return spatial_hash(s, params_.spatial_resolution_x, params_.spatial_resolution_y, params_.spatial_resolution_theta);
    };

    if (params_.rng_mode == RngMode::kCounter) {
      // cdf_ was built from the raw weights in normalize_weights(); quantised raw weights
      // and quantised normalised weights select identically (same ratios up to the grid).
      const CounterResampler rs{params_.seed, step_, params_.scheme, cdf_.total, max};
      for (std::uint64_t j = 0; new_states.size() < max; ++j) {
        SE2 s;
        std::int64_t idx = -1;
        if (random_state_probability > 0.0 && rs.inject(j, random_state_probability)) {
          s = random_state_counter(grid_, free_, params_.seed, j, step_);
        } else {
          idx = static_cast<std::int64_t>(cdf_search(cdf_.cdf, rs.position(j)));
          s = states_[static_cast<std::size_t>(idx)];
        }
        if (!kld(hash(s))) break;  // take_while: the failing element is dropped
        new_states.push_back(s);
        last_indices_.push_back(idx);
      }
    } else {
      // views/sample.hpp:128-135 | random_intersperse.hpp:93-100 | take_while_kld.hpp:134-136.
      // Draw order of the lazy pipeline: begin() draws the first sample index; each advance draws
      // one bernoulli and, when it is false, one more index.
      std::discrete_distribution<std::ptrdiff_t> distribution(weights_.begin(), weights_.end());
      std::bernoulli_distribution bernoulli(random_state_probability);
      std::uniform_int_distribution<std::size_t> cell_dist(0, free_.empty() ? 0 : free_.size() - 1);
      const double pi = 3.14159265358979323846;
      std::uniform_real_distribution<double> yaw_dist(-pi, pi);
      std::ptrdiff_t idx = distribution(engine_);
      std::optional<SE2> injected;
      while (new_states.size() < max) {
        const SE2 s = injected.value_or(states_[static_cast<std::size_t>(idx)]);
        if (!kld(hash(s))) break;
        new_states.push_back(s);
        last_indices_.push_back(injected ? -1 : idx);
        if (new_states.size() >= max) break;  // take(max) stops before advancing
        injected.reset();
        if (bernoulli(engine_)) {
          // multivariate_uniform_distribution.hpp:143-146: {SO2::sampleUniform(engine), free_states[dist(engine)]}
          // (brace-init evaluates left to right: yaw first, then the cell).
          const double yaw = yaw_dist(engine_);
          const std::size_t c = cell_dist(engine_);
          injected = free_cell_state(grid_, free_[c], yaw);
        } else {
          idx = distribution(engine_);
        }
      }
    }
    states_ = std::move(new_states);
    weights_.assign(states_.size(), 1.0);
  }

  AmclParams params_;
  DifferentialDriveParam motion_;
  int motion_model_{0};
  OmnidirectionalDriveParam omni_;
  ThrunRecoveryProbabilityEstimator thrun_;
  OnMotionPolicy update_policy_{};
  EveryNPolicy every_n_{};
  RollingWindow2 window_{};
  bool force_update_{true};
  std::uint32_t step_{0};

  SensorKind sensor_{SensorKind::kLikelihoodField};
  OccupancyGrid grid_;
  std::unique_ptr<LikelihoodFieldModel> lfm_;
  BeamModelParam beam_;
  std::vector<std::uint32_t> free_;

  std::vector<SE2> states_;
  std::vector<double> weights_;
  std::vector<std::int64_t> last_indices_;
  FixedPointCdf cdf_;

  std::mt19937_64 engine_;
  std::normal_distribution<double> motion_distribution_;
};

}  // namespace oracle
