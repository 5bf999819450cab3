// beluga_b200/amcl.hpp -- beluga::Amcl shaped driver over the C ABI.
//
// Mirrors beluga::Amcl<MotionModel, SensorModel, ...> (beluga/algorithm/amcl_core.hpp:74-233):
// same constructor argument order (motion model, sensor model, [random state generator, spatial
// hasher,] params), same public methods -- particles(), initialize(pose, covariance),
// update_map(map), update(control_action, measurement) -> std::optional<std::pair<pose, covariance>>,
// force_update() -- and the same AmclParams members and defaults (:34-55).  The particle set lives
// on the GPU; particles() copies it out on demand.  update() also takes a point cloud, as the second
// overload of beluga_ros::Amcl::update does (beluga_ros/src/amcl.cpp:67-81).
//
// What differs from the template: the random state generator is always the map's free-cell uniform
// distribution (what beluga_ros::Amcl passes, beluga_ros/include/beluga_ros/amcl.hpp:269), the
// spatial hasher is spatial_hash<SE2d> with the resolutions in AmclParams, and the execution
// policy argument is accepted and ignored (everything per-particle runs on the device).
#pragma once

#include <algorithm>
#include <array>
#include <execution>
#include <limits>
#include <map>
#include <optional>
#include <utility>
#include <variant>

#include "models.hpp"

namespace beluga_b200 {

/// beluga::AmclParams (amcl_core.hpp:34-55) plus the knobs the drop-in backend adds.
struct AmclParams {
  double update_min_d = 0.25;
  double update_min_a = 0.2;
  std::size_t resample_interval = 1UL;
  bool selective_resampling = false;
  std::size_t min_particles = 500UL;
  std::size_t max_particles = 2000UL;
  double alpha_slow = 0.001;
  double alpha_fast = 0.1;
  double kld_epsilon = 0.05;
  double kld_z = 3.0;
  // spatial_hash<SE2d>{x, y, theta} resolutions (beluga_ros/include/beluga_ros/amcl.hpp:91-97)
  double spatial_resolution_x = 0.5;
  double spatial_resolution_y = 0.5;
  double spatial_resolution_theta = 10.0 * 3.14159265358979323846 / 180.0;
  // backend
  bb200_resample_scheme resample_scheme = BB200_RESAMPLE_MULTINOMIAL;
  std::uint64_t seed = 0;  // the reference's engine is auto-seeded and cannot be set (amcl_core.hpp uses get_random_engine())
  int device = 0;
};

/// AmclParams as the C ABI's parameter block.
inline bb200_amcl_param c_amcl_param(const AmclParams& params) {
  bb200_amcl_param p{};
  p.update_min_d = params.update_min_d;
  p.update_min_a = params.update_min_a;
  p.resample_interval = params.resample_interval;
  p.selective_resampling = params.selective_resampling ? 1 : 0;
  p.min_particles = params.min_particles;
  p.max_particles = params.max_particles;
  p.alpha_slow = params.alpha_slow;
  p.alpha_fast = params.alpha_fast;
  p.kld_epsilon = params.kld_epsilon;
  p.kld_z = params.kld_z;
  p.spatial_resolution[0] = params.spatial_resolution_x;
  p.spatial_resolution[1] = params.spatial_resolution_y;
  p.spatial_resolution[2] = params.spatial_resolution_theta;
  p.resample_scheme = params.resample_scheme;
  p.seed = params.seed;
  p.device = params.device;
  return p;
}

/// The parameters of a state blob (bb200_amcl_state_params), as AmclParams.
inline AmclParams amcl_params_of_state(const std::vector<std::uint8_t>& blob, bb200_motion_param* motion = nullptr) {
  bb200_amcl_param p{};
  bb200_motion_param m{};
  const int st = bb200_amcl_state_params(blob.data(), blob.size(), &p, &m);
  if (st != BB200_OK) throw Error(st, bb200_create_error());
  if (motion != nullptr) *motion = m;
  AmclParams q;
  q.update_min_d = p.update_min_d;
  q.update_min_a = p.update_min_a;
  q.resample_interval = p.resample_interval;
  q.selective_resampling = p.selective_resampling != 0;
  q.min_particles = p.min_particles;
  q.max_particles = p.max_particles;
  q.alpha_slow = p.alpha_slow;
  q.alpha_fast = p.alpha_fast;
  q.kld_epsilon = p.kld_epsilon;
  q.kld_z = p.kld_z;
  q.spatial_resolution_x = p.spatial_resolution[0];
  q.spatial_resolution_y = p.spatial_resolution[1];
  q.spatial_resolution_theta = p.spatial_resolution[2];
  q.resample_scheme = static_cast<bb200_resample_scheme>(p.resample_scheme);
  q.seed = p.seed;
  q.device = p.device;
  return q;
}

/// Particle set copy: the two vectors of beluga::TupleVector<std::tuple<SE2d, Weight>>.
struct ParticleSet {
  std::vector<SE2d> states;
  std::vector<double> weights;
  [[nodiscard]] std::size_t size() const { return states.size(); }
  [[nodiscard]] bool empty() const { return states.empty(); }
};

/// A bearing {cos, sin} of a ray cast, taken as given (Sophus::SO2d's unit complex, not normalised).
using Bearing = std::array<double, 2>;

/// The directions of the beams a laser scan of this geometry keeps (take_evenly(max_beams), beluga_ros/laser_scan.hpp:69-80),
/// computed as bb200_scan_to_points computes them and without dropping readings by range (bb200_scan_bearings): the
/// bearings of the scan a sensor at some pose is expected to see (Amcl::cast_rays).
inline std::vector<Bearing> scan_bearings(float angle_min, float angle_increment, std::uint64_t n_ranges, std::uint64_t max_beams = 0) {
  std::uint64_t n = 0;
  int st = bb200_scan_bearings(angle_min, angle_increment, n_ranges, max_beams, nullptr, 0, &n);
  if (st != BB200_OK && st != BB200_ERR_CAPACITY) throw Error(st, "bb200_scan_bearings");
  std::vector<Bearing> out(n);
  static_assert(sizeof(Bearing) == 2 * sizeof(double), "bearings must be packed");
  st = bb200_scan_bearings(angle_min, angle_increment, n_ranges, max_beams, n > 0 ? out.front().data() : nullptr, n, &n);
  if (st != BB200_OK) throw Error(st, "bb200_scan_bearings");
  return out;
}

namespace detail {
/// The ranges of a ray cast as Ray2d::cast returns them: +inf (a miss) becomes std::nullopt.
inline std::vector<std::optional<double>> cast_results(const double* ranges, std::size_t n) {
  std::vector<std::optional<double>> out(n);
  for (std::size_t i = 0; i < n; ++i)
    if (ranges[i] != std::numeric_limits<double>::infinity()) out[i] = ranges[i];
  return out;
}
}  // namespace detail

template <class MotionModel, class SensorModel, class ExecutionPolicy = std::execution::sequenced_policy>
class Amcl {
 public:
  using state_type = typename SensorModel::state_type;
  using measurement_type = typename SensorModel::measurement_type;
  using map_type = typename SensorModel::map_type;
  using estimation_type = std::pair<state_type, Matrix3d>;

  Amcl(MotionModel motion_model, SensorModel sensor_model, const AmclParams& params = AmclParams{}, ExecutionPolicy = ExecutionPolicy{})
      : params_{params}, motion_model_{std::move(motion_model)}, sensor_model_{std::move(sensor_model)} {
    const bb200_amcl_param p = c_amcl_param(params);
    const bb200_motion_param m = motion_model_.c_motion_param();
    const int st = bb200_amcl_create_with_motion(&p, &m, &handle_);
    if (st != BB200_OK) throw Error(st, bb200_create_error());
    check(sensor_model_.attach(bb200_amcl_filter(handle_)));
  }
  ~Amcl() { bb200_amcl_destroy(handle_); }
  Amcl(const Amcl&) = delete;
  Amcl& operator=(const Amcl&) = delete;
  Amcl(Amcl&& other) noexcept
      : params_{other.params_}, motion_model_{std::move(other.motion_model_)}, sensor_model_{std::move(other.sensor_model_)}, handle_{other.handle_} {
    other.handle_ = nullptr;
  }

  /// The filter a state blob holds (bb200_amcl_create_from_state) on `device`, reading the sensor model's map: it continues
  /// exactly where the filter that wrote the blob stopped.  The motion model must be the one the blob was written with.
  static Amcl from_state(const std::vector<std::uint8_t>& blob, MotionModel motion_model, SensorModel sensor_model, int device = 0) {
    AmclParams params = amcl_params_of_state(blob);
    params.device = device;
    bb200_amcl* handle = nullptr;
    const int st = bb200_amcl_create_from_state(blob.data(), blob.size(), device, &handle);
    if (st != BB200_OK) throw Error(st, bb200_create_error());
    return Amcl(handle, params, std::move(motion_model), std::move(sensor_model));
  }
  /// This filter's state blob (bb200_amcl_export_state): parameters, policies, particles, weights, CDF and ancestors.
  [[nodiscard]] std::vector<std::uint8_t> export_state() const {
    std::uint64_t size = 0;
    check(bb200_amcl_export_state(handle_, nullptr, 0, &size));
    std::vector<std::uint8_t> blob(size);
    check(bb200_amcl_export_state(handle_, blob.data(), blob.size(), &size));
    return blob;
  }

  /// amcl_core.hpp:128 -- copies the particle set back from the device.
  [[nodiscard]] ParticleSet particles() const {
    bb200_filter* f = bb200_amcl_filter(handle_);
    std::uint64_t n = 0;
    check(bb200_filter_size(f, &n));
    ParticleSet out;
    out.states.resize(n);
    out.weights.resize(n);
    static_assert(sizeof(SE2d) == 4 * sizeof(double), "SE2d must be four packed doubles");
    if (n > 0) check(bb200_filter_get_particles(f, reinterpret_cast<double*>(out.states.data()), out.weights.data(), n));
    return out;
  }

  /// amcl_core.hpp:145-147 -- throws like MultivariateNormalDistribution on an invalid covariance.
  void initialize(const state_type& pose, const Matrix3d& covariance) {
    const double mean[3] = {pose.x(), pose.y(), pose.theta()};
    check(bb200_amcl_initialize(handle_, mean, covariance.data()));
  }
  /// amcl_core.hpp:131-137 with an explicit state list instead of a distribution.
  /// beluga_ros::Amcl::initialize_from_map() (beluga_ros/include/beluga_ros/amcl.hpp:209): max_particles samples of the
  /// map distribution -- uniform over the free cells of the sensor model's map.
  void initialize_from_map() { check(bb200_amcl_initialize_from_map(handle_)); }
  void initialize(const std::vector<state_type>& states) {
    check(bb200_amcl_initialize_states(handle_, states.empty() ? nullptr : reinterpret_cast<const double*>(states.data()), nullptr, states.size()));
  }

  /// amcl_core.hpp:150
  void update_map(const map_type& map) {
    sensor_model_.update_map(map);
    check(sensor_model_.attach(bb200_amcl_filter(handle_)));
  }

  /// amcl_core.hpp:165-201.  With a caller's device sensor model (is_weighed_token_v of its token): begin, the token's
  /// weigh on the views (not called when the policies skip the step) and end (bb200_amcl_update_begin / _end).  weigh must
  /// not throw: the step would stay open and the filter then accepts nothing but its destruction.
  auto update(const state_type& control_action, measurement_type measurement) -> std::optional<estimation_type> {
    const auto token = sensor_model_(std::move(measurement));
    bb200_update_result r{};
    if constexpr (is_weighed_token_v<std::decay_t<decltype(token)>>) {
      bb200_weigh_view view{};
      check(bb200_amcl_update_begin(handle_, control_action.data(), &view));
      if (view.updated) token.weigh(view.stream, view.states, view.n, view.factors);
      check(bb200_amcl_update_end(handle_, &r));
    } else if constexpr (is_landmark_token_v<std::decay_t<decltype(token)>>) {
      check(bb200_amcl_update_landmarks(handle_, control_action.data(), token.detections.empty() ? nullptr : token.detections.data(),
                                        token.detections.size(), &r));
    } else {
      static_assert(sizeof(std::pair<double, double>) == 2 * sizeof(double), "measurement points must be packed");
      check(bb200_amcl_update(handle_, control_action.data(), token.points.empty() ? nullptr : &token.points.front().first, token.points.size(), &r));
    }
    return estimate_of(r);
  }

  /// beluga_ros::Amcl::update(base_pose_in_odom, point_cloud) (beluga_ros/src/amcl.cpp:67-81): the cloud's points moved
  /// into the base frame, then the update above.  Throws Error(BB200_ERR_INVALID_ARGUMENT) on an unusable layout.
  auto update(const state_type& control_action, const PointCloudView& cloud) -> std::optional<estimation_type> {
    const bb200_point_cloud c = cloud.c_view();
    bb200_update_result r{};
    check(bb200_amcl_update_point_cloud(handle_, control_action.data(), &c, &r));
    return estimate_of(r);
  }
#ifdef BELUGA_B200_WITH_SOPHUS
  /// The same for any beluga::BaseSparsePointCloud-shaped cloud, e.g. beluga_ros::SparsePointCloud3f.
  template <class SparsePointCloud, std::enable_if_t<is_sparse_point_cloud_v<SparsePointCloud>, int> = 0>
  auto update(const state_type& control_action, const SparsePointCloud& cloud) -> std::optional<estimation_type> {
    const PackedPointCloud packed{cloud};
    return update(control_action, packed.view());
  }
#endif

  /// amcl_core.hpp:204
  void force_update() { bb200_amcl_force_update(handle_); }

  /// Ray2d::cast (algorithm/raycasting.hpp:79-107) on the sensor model's map for every sensor pose (map frame) and bearing,
  /// pose major: entry i * bearings.size() + j is what Ray2d{map, poses[i], max_range}.cast(bearings[j]) returns.  One
  /// kernel launch (bb200_filter_cast_rays); the particle set is not touched.
  [[nodiscard]] std::vector<std::optional<double>> cast_rays(const std::vector<state_type>& poses, const std::vector<Bearing>& bearings,
                                                             double max_range) const {
    std::vector<double> ranges(poses.size() * bearings.size());
    check(bb200_filter_cast_rays(bb200_amcl_filter(handle_), poses.empty() ? nullptr : poses.front().data(), poses.size(),
                                 bearings.empty() ? nullptr : bearings.front().data(), bearings.size(), max_range, ranges.empty() ? nullptr : ranges.data()));
    return detail::cast_results(ranges.data(), ranges.size());
  }

  [[nodiscard]] bb200_amcl* handle() const { return handle_; }

 private:
  Amcl(bb200_amcl* handle, const AmclParams& params, MotionModel motion_model, SensorModel sensor_model)
      : params_{params}, motion_model_{std::move(motion_model)}, sensor_model_{std::move(sensor_model)}, handle_{handle} {
    check(sensor_model_.attach(bb200_amcl_filter(handle_)));
  }
  void check(int status) const {
    if (status != BB200_OK) throw Error(status, bb200_amcl_last_error(handle_));
  }
  static auto estimate_of(const bb200_update_result& r) -> std::optional<estimation_type> {
    if (!r.updated) return std::nullopt;
    Matrix3d cov;
    for (int i = 0; i < 9; ++i) cov[i] = r.estimate.cov[i];
    return std::make_pair(state_type::from_data(r.estimate.mean), cov);
  }

  AmclParams params_;
  MotionModel motion_model_;
  SensorModel sensor_model_;
  bb200_amcl* handle_{nullptr};
};

template <class MotionModel, class SensorModel>
Amcl(MotionModel, SensorModel, const AmclParams&) -> Amcl<MotionModel, SensorModel>;

/// beluga::ParticleClusterizerParam (algorithm/cluster_based_estimation.hpp:259-276).
struct ParticleClusterizerParam {
  double linear_hash_resolution = 0.20;
  double angular_hash_resolution = 0.524;
  double weight_cap_percentile = 0.90;
};

/// beluga::cluster_based_estimate(states, weights, parameters) (cluster_based_estimation.hpp:415-432)
/// over the filter's device-resident particle set: what beluga_ros::Amcl::update returns
/// (beluga_ros/src/amcl.cpp:125).  Throws Error when the filter holds no particles.
template <class MotionModel, class SensorModel, class ExecutionPolicy>
[[nodiscard]] std::pair<SE2d, Matrix3d> cluster_based_estimate(
    const Amcl<MotionModel, SensorModel, ExecutionPolicy>& amcl,
    ParticleClusterizerParam parameters = {}) {
  const bb200_cluster_param p{parameters.linear_hash_resolution, parameters.angular_hash_resolution, parameters.weight_cap_percentile};
  bb200_estimate e{};
  bb200_filter* f = bb200_amcl_filter(amcl.handle());
  const int st = bb200_filter_cluster_estimate(f, &p, &e, nullptr, 0, nullptr, nullptr);
  if (st != BB200_OK) throw Error(st, bb200_last_error(f));
  Matrix3d cov;
  for (int i = 0; i < 9; ++i) cov[i] = e.cov[i];
  return std::make_pair(SE2d::from_data(e.mean), cov);
}

/// One filter over several shards (bb200_sharded_amcl), driven like Amcl: the constructor takes Amcl's arguments and the
/// CUDA ordinal of every shard (ordinals may repeat); params.max_particles is the global particle count, a multiple of the
/// shard count.  Every method marshals one C call; results equal those of one Amcl with the same parameters and seed.
template <class MotionModel, class SensorModel>
class ShardedAmcl {
 public:
  using state_type = typename SensorModel::state_type;
  using measurement_type = typename SensorModel::measurement_type;
  using map_type = typename SensorModel::map_type;
  using estimation_type = std::pair<state_type, Matrix3d>;
  /// The particle-cloud histogram: the bins in global first-occurrence order and max(1e-3, heaviest bin).
  using histogram_type = std::pair<std::vector<bb200_cluster_cell>, double>;

  ShardedAmcl(MotionModel motion_model, SensorModel sensor_model, const AmclParams& params, const std::vector<int>& devices)
      : params_{params}, motion_model_{std::move(motion_model)}, sensor_model_{std::move(sensor_model)} {
    const bb200_amcl_param p = c_amcl_param(params);
    const bb200_motion_param m = motion_model_.c_motion_param();
    const int st = bb200_sharded_amcl_create(&p, &m, static_cast<int>(devices.size()), devices.data(), &handle_);
    if (st != BB200_OK) throw Error(st, bb200_create_error());
    check(sensor_model_.attach(handle_));
  }
  ~ShardedAmcl() { bb200_sharded_amcl_destroy(handle_); }
  ShardedAmcl(const ShardedAmcl&) = delete;
  ShardedAmcl& operator=(const ShardedAmcl&) = delete;

  /// Amcl::particles in global index order.
  [[nodiscard]] ParticleSet particles() const {
    std::uint64_t n = 0;
    for (int r = 0; r < bb200_sharded_amcl_shards(handle_); ++r) {
      std::uint64_t k = 0;
      check(bb200_filter_size(bb200_amcl_filter(bb200_sharded_amcl_shard(handle_, r)), &k));
      n += k;
    }
    ParticleSet out;
    out.states.resize(n);
    out.weights.resize(n);
    if (n > 0) check(bb200_sharded_amcl_get_particles(handle_, reinterpret_cast<double*>(out.states.data()), out.weights.data(), n));
    return out;
  }

  void initialize(const state_type& pose, const Matrix3d& covariance) {
    const double mean[3] = {pose.x(), pose.y(), pose.theta()};
    check(bb200_sharded_amcl_initialize(handle_, mean, covariance.data()));
  }
  void initialize_from_map() { check(bb200_sharded_amcl_initialize_from_map(handle_)); }
  void update_map(const map_type& map) {
    sensor_model_.update_map(map);
    check(sensor_model_.attach(handle_));
  }
  void force_update() { bb200_sharded_amcl_force_update(handle_); }

  /// Amcl::update over all shards (with a landmark or bearing model, bb200_sharded_amcl_update_landmarks).  With a caller's device sensor model (is_weighed_token_v of its token; the model's
  /// attach takes the bb200_sharded_amcl*): begin, the token's weigh once per shard that holds particles, in rank order,
  /// and end (bb200_sharded_amcl_update_begin / _end).  The views of shard r live on devices[r], the device of its stream:
  /// a token that launches kernels must make that device current (cudaSetDevice) first.  weigh must not throw: the step
  /// would stay open and the filter then accepts nothing but its destruction.
  auto update(const state_type& control_action, measurement_type measurement) -> std::optional<estimation_type> {
    const auto token = sensor_model_(std::move(measurement));
    bb200_update_result r{};
    if constexpr (is_weighed_token_v<std::decay_t<decltype(token)>>) {
      std::vector<bb200_weigh_view> views(static_cast<std::size_t>(bb200_sharded_amcl_shards(handle_)));
      check(bb200_sharded_amcl_update_begin(handle_, control_action.data(), views.data()));
      for (const bb200_weigh_view& view : views)
        if (view.updated && view.n > 0) token.weigh(view.stream, view.states, view.n, view.factors);
      check(bb200_sharded_amcl_update_end(handle_, &r));
    } else if constexpr (is_landmark_token_v<std::decay_t<decltype(token)>>) {
      check(bb200_sharded_amcl_update_landmarks(handle_, control_action.data(), token.detections.empty() ? nullptr : token.detections.data(),
                                                token.detections.size(), &r));
    } else {
      check(bb200_sharded_amcl_update(handle_, control_action.data(), token.points.empty() ? nullptr : &token.points.front().first, token.points.size(), &r));
    }
    return estimate_of(r);
  }
  /// beluga_ros::Amcl::update(base_pose_in_odom, laser_scan) (bb200_sharded_amcl_update_scan).
  auto update(const state_type& control_action, const LaserScanView& scan) -> std::optional<estimation_type> {
    const bb200_laser_scan s = scan.c_view();
    bb200_update_result r{};
    check(bb200_sharded_amcl_update_scan(handle_, control_action.data(), &s, &r));
    return estimate_of(r);
  }
  /// beluga_ros::Amcl::update(base_pose_in_odom, point_cloud) (bb200_sharded_amcl_update_point_cloud).
  auto update(const state_type& control_action, const PointCloudView& cloud) -> std::optional<estimation_type> {
    const bb200_point_cloud c = cloud.c_view();
    bb200_update_result r{};
    check(bb200_sharded_amcl_update_point_cloud(handle_, control_action.data(), &c, &r));
    return estimate_of(r);
  }
#ifdef BELUGA_B200_WITH_SOPHUS
  template <class SparsePointCloud, std::enable_if_t<is_sparse_point_cloud_v<SparsePointCloud>, int> = 0>
  auto update(const state_type& control_action, const SparsePointCloud& cloud) -> std::optional<estimation_type> {
    const PackedPointCloud packed{cloud};
    return update(control_action, packed.view());
  }
#endif

  /// beluga::cluster_based_estimate over all shards (bb200_sharded_amcl_cluster_estimate).
  [[nodiscard]] estimation_type cluster_estimate(ParticleClusterizerParam parameters = {}) const {
    const bb200_cluster_param p{parameters.linear_hash_resolution, parameters.angular_hash_resolution, parameters.weight_cap_percentile};
    bb200_estimate e{};
    check(bb200_sharded_amcl_cluster_estimate(handle_, &p, &e, nullptr, nullptr));
    return estimation_of(e);
  }
  /// The particle-cloud histogram over all shards (bb200_sharded_amcl_particle_histogram).
  [[nodiscard]] histogram_type particle_histogram(double linear_resolution = 1e-3, double angular_resolution = 1e-3) const {
    std::uint64_t n = 0;
    double top = 0.0;
    check(bb200_sharded_amcl_particle_histogram(handle_, linear_resolution, angular_resolution, nullptr, 0, &n, &top));
    std::vector<bb200_cluster_cell> bins(n);
    check(bb200_sharded_amcl_particle_histogram(handle_, linear_resolution, angular_resolution, bins.data(), n, &n, &top));
    return std::make_pair(std::move(bins), top);
  }
  /// `count` states drawn by weight from the global particle set, the multinomial draws of `step`
  /// (bb200_sharded_amcl_sample_states); no particle changes.
  [[nodiscard]] std::vector<state_type> sample_states(std::size_t count, uint32_t step) const {
    std::vector<state_type> out(count);
    check(bb200_sharded_amcl_sample_states(handle_, count, step, out.empty() ? nullptr : reinterpret_cast<double*>(out.data())));
    return out;
  }
  /// Amcl::cast_rays on the shards' copies of the map (bb200_sharded_amcl_cast_rays).
  [[nodiscard]] std::vector<std::optional<double>> cast_rays(const std::vector<state_type>& poses, const std::vector<Bearing>& bearings,
                                                             double max_range) const {
    std::vector<double> ranges(poses.size() * bearings.size());
    check(bb200_sharded_amcl_cast_rays(handle_, poses.empty() ? nullptr : poses.front().data(), poses.size(),
                                       bearings.empty() ? nullptr : bearings.front().data(), bearings.size(), max_range,
                                       ranges.empty() ? nullptr : ranges.data()));
    return detail::cast_results(ranges.data(), ranges.size());
  }

  [[nodiscard]] bb200_sharded_amcl* handle() const { return handle_; }

 private:
  void check(int status) const {
    if (status != BB200_OK) throw Error(status, bb200_sharded_amcl_last_error(handle_));
  }
  static estimation_type estimation_of(const bb200_estimate& e) {
    Matrix3d cov;
    for (int i = 0; i < 9; ++i) cov[i] = e.cov[i];
    return std::make_pair(state_type::from_data(e.mean), cov);
  }
  static auto estimate_of(const bb200_update_result& r) -> std::optional<estimation_type> {
    if (!r.updated) return std::nullopt;
    return estimation_of(r.estimate);
  }

  AmclParams params_;
  MotionModel motion_model_;
  SensorModel sensor_model_;
  bb200_sharded_amcl* handle_{nullptr};
};

/// K independent filters on one GPU (bb200_amcl_batch) that read one or several maps, each for a likelihood-field model or
/// the beam model: update() steps every member with a new scan at once.  Member m behaves like an Amcl built from motions[m] and params[m]; members keep a fixed
/// particle count (min_particles == max_particles <= 32768) unless the batch is adaptive, whose members may have
/// min_particles < max_particles and resize their particle sets with KLD as a standalone Amcl does; members of a selective
/// batch may use selective_resampling, deciding on the device as a standalone Amcl does on the host.  Results are returned
/// per member, std::nullopt where the reference's update would return it or where the member had no scan this step.
class AmclBatch {
 public:
  using estimation_type = std::pair<SE2d, Matrix3d>;

  /// adaptive: BB200_BATCH_ADAPTIVE (members may have min_particles < max_particles); particles(m) then returns
  /// member_size(m) particles.  selective: BB200_BATCH_SELECTIVE (members may have selective_resampling).
  AmclBatch(const std::vector<bb200_motion_param>& motions, const std::vector<AmclParams>& params, bool adaptive = false, bool selective = false)
      : adaptive_{adaptive} {
    if (motions.size() != params.size()) throw Error(BB200_ERR_INVALID_ARGUMENT, "one motion model per member");
    std::vector<bb200_amcl_param> p;
    for (const AmclParams& q : params) p.push_back(c_amcl_param(q));
    const uint32_t flags = (adaptive ? uint32_t{BB200_BATCH_ADAPTIVE} : 0u) | (selective ? uint32_t{BB200_BATCH_SELECTIVE} : 0u);
    const int st = bb200_amcl_batch_create_with_flags(p.data(), motions.data(), static_cast<int>(p.size()), flags, &handle_);
    if (st != BB200_OK) throw Error(st, bb200_create_error());
    sizes_.reserve(params.size());
    for (const AmclParams& q : params) sizes_.push_back(q.max_particles);
  }
  ~AmclBatch() { bb200_amcl_batch_destroy(handle_); }
  AmclBatch(const AmclBatch&) = delete;
  AmclBatch& operator=(const AmclBatch&) = delete;
  /// Moves the handle (e.g. the batch from_states returns into the owner a server keeps).
  AmclBatch(AmclBatch&& other) noexcept
      : adaptive_{other.adaptive_}, handle_{std::exchange(other.handle_, nullptr)}, sizes_{std::move(other.sizes_)},
        field_cells_{std::move(other.field_cells_)} {}

  /// Slots, occupied and vacant: the length of every per-member vector a call takes.
  [[nodiscard]] std::size_t size() const { return sizes_.size(); }

  /// Adds a member (bb200_amcl_batch_add_member): it takes the lowest vacant slot or a new one after the last, and starts
  /// as a member of a freshly created batch does, with no map and no particles.  Returns its slot.  The other members
  /// keep their particles, policies and maps.
  std::size_t add_member(const bb200_motion_param& motion, const AmclParams& params) {
    const bb200_amcl_param p = c_amcl_param(params);
    int slot = -1;
    check(bb200_amcl_batch_add_member(handle_, &p, &motion, &slot));
    const std::size_t m = static_cast<std::size_t>(slot);
    if (m == sizes_.size()) sizes_.push_back(0);
    sizes_[m] = params.max_particles;
    return m;
  }
  /// Makes slot m vacant (bb200_amcl_batch_remove_member); the last occupied slot cannot be removed.
  void remove_member(std::size_t member) {
    check(bb200_amcl_batch_remove_member(handle_, index(member)));
    sizes_[member] = 0;
  }
  /// Whether slot m holds a member.
  [[nodiscard]] bool member_active(std::size_t member) const {
    int active = 0;
    check(bb200_amcl_batch_member_active(handle_, index(member), &active));
    return active != 0;
  }

  /// The batch whose members are the filters of these state blobs (bb200_amcl_batch_create_from_states), on `device`,
  /// with the batch flags as in the constructor.  It has no map: add maps and assign them with update_map.
  static AmclBatch from_states(const std::vector<std::vector<std::uint8_t>>& blobs, bool adaptive = false, bool selective = false, int device = 0) {
    std::vector<const void*> data;
    std::vector<std::uint64_t> sizes;
    std::vector<std::size_t> slots;
    for (const auto& b : blobs) {
      data.push_back(b.data());
      sizes.push_back(b.size());
      slots.push_back(amcl_params_of_state(b).max_particles);
    }
    const uint32_t flags = (adaptive ? uint32_t{BB200_BATCH_ADAPTIVE} : 0u) | (selective ? uint32_t{BB200_BATCH_SELECTIVE} : 0u);
    bb200_amcl_batch* handle = nullptr;
    const int st = bb200_amcl_batch_create_from_states(data.data(), sizes.data(), static_cast<int>(data.size()), flags, device, &handle);
    if (st != BB200_OK) throw Error(st, bb200_create_error());
    return AmclBatch(handle, std::move(slots), adaptive);
  }
  /// Member m's state blob (bb200_amcl_batch_export_member).
  [[nodiscard]] std::vector<std::uint8_t> export_member(std::size_t member) const {
    std::uint64_t size = 0;
    check(bb200_amcl_batch_export_member(handle_, index(member), nullptr, 0, &size));
    std::vector<std::uint8_t> blob(size);
    check(bb200_amcl_batch_export_member(handle_, index(member), blob.data(), blob.size(), &size));
    return blob;
  }
  /// The fleet checkpoint (bb200_amcl_batch_export_members): the state blob of every member selected by `present`
  /// (nullptr: every occupied slot), an empty vector for the others, with one kernel launch and one synchronisation.
  [[nodiscard]] std::vector<std::vector<std::uint8_t>> export_members(const std::vector<bool>* present = nullptr) const {
    const std::vector<std::uint8_t> mask = presence_mask(present);
    const std::uint8_t* m = present != nullptr ? mask.data() : nullptr;
    std::vector<std::uint64_t> sizes(size(), 0);
    check(bb200_amcl_batch_export_members(handle_, m, nullptr, nullptr, sizes.data()));
    std::vector<std::vector<std::uint8_t>> blobs(size());
    std::vector<void*> out(size(), nullptr);
    for (std::size_t k = 0; k < size(); ++k) {
      blobs[k].resize(sizes[k]);
      if (sizes[k] > 0) out[k] = blobs[k].data();
    }
    check(bb200_amcl_batch_export_members(handle_, m, out.data(), sizes.data(), sizes.data()));
    return blobs;
  }
  /// add_member with a history (bb200_amcl_batch_import_member): the blob's filter joins in the lowest vacant slot or a
  /// new one, reading map `map_id` (-1: none).  Returns its slot.
  std::size_t import_member(const std::vector<std::uint8_t>& blob, int map_id = -1) {
    const std::size_t max_particles = amcl_params_of_state(blob).max_particles;
    int slot = -1;
    check(bb200_amcl_batch_import_member(handle_, blob.data(), blob.size(), map_id, &slot));
    const std::size_t m = static_cast<std::size_t>(slot);
    if (m == sizes_.size()) sizes_.push_back(0);
    sizes_[m] = max_particles;
    return m;
  }

  /// One likelihood field for every member (prob: the LikelihoodFieldProb model).
  void set_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob = false) {
    check(bb200_amcl_batch_set_likelihood_field_map(handle_, &p, &grid, prob ? 1 : 0));
    field_cells_.clear();
    const std::size_t occupied = static_cast<std::size_t>(std::find_if(sizes_.begin(), sizes_.end(), [](std::size_t n) { return n != 0; }) - sizes_.begin());
    field_cells_[member_map(occupied)] = static_cast<std::size_t>(grid.width) * static_cast<std::size_t>(grid.height);
  }
  /// One beam-model map (BeamSensorModel) for every member; replaces the map set before, whichever model it was for.
  void set_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid) {
    check(bb200_amcl_batch_set_beam_map(handle_, &p, &grid));
    field_cells_.clear();
  }
  /// Adds a map that no member reads yet and returns its id (several floors or sites in one batch).
  int add_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob = false) {
    int id = -1;
    check(bb200_amcl_batch_add_likelihood_field_map(handle_, &p, &grid, prob ? 1 : 0, &id));
    field_cells_[id] = static_cast<std::size_t>(grid.width) * static_cast<std::size_t>(grid.height);
    return id;
  }
  int add_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid) {
    int id = -1;
    check(bb200_amcl_batch_add_beam_map(handle_, &p, &grid, &id));
    return id;
  }
  /// A landmark map (LandmarkSensorModel2d / BearingSensorModel2d on `map`) for every member, or added without assigning
  /// it; members on it step with landmark_token measurements.
  void set_landmark_map(const LandmarkModelParam& p, const LandmarkMap& map) {
    const bb200_landmark_param c = c_param(p);
    const bb200_landmark_map m = map.view();
    check(bb200_amcl_batch_set_landmark_map(handle_, &c, &m));
    field_cells_.clear();
  }
  void set_bearing_map(const BearingModelParam& p, const LandmarkMap& map) {
    const bb200_bearing_param c = c_param(p);
    const bb200_landmark_map m = map.view();
    check(bb200_amcl_batch_set_bearing_map(handle_, &c, &m));
    field_cells_.clear();
  }
  int add_landmark_map(const LandmarkModelParam& p, const LandmarkMap& map) {
    const bb200_landmark_param c = c_param(p);
    const bb200_landmark_map m = map.view();
    int id = -1;
    check(bb200_amcl_batch_add_landmark_map(handle_, &c, &m, &id));
    return id;
  }
  int add_bearing_map(const BearingModelParam& p, const LandmarkMap& map) {
    const bb200_bearing_param c = c_param(p);
    const bb200_landmark_map m = map.view();
    int id = -1;
    check(bb200_amcl_batch_add_bearing_map(handle_, &c, &m, &id));
    return id;
  }
  /// Amcl::update_map (amcl_core.hpp:150) for one member: it keeps its particles and reads map `map_id` from its next step.
  void update_map(std::size_t member, int map_id) { check(bb200_amcl_batch_update_map(handle_, index(member), map_id)); }
  /// The id of the map member m reads (-1: none).
  [[nodiscard]] int member_map(std::size_t member) const {
    int id = -1;
    check(bb200_amcl_batch_member_map(handle_, index(member), &id));
    return id;
  }
  /// Frees a map no member reads.
  void remove_map(int map_id) {
    check(bb200_amcl_batch_remove_map(handle_, map_id));
    field_cells_.erase(map_id);
  }
  /// likelihood_field() of a likelihood-field map: height x width values, row-major.
  [[nodiscard]] std::vector<float> likelihood_field(int map_id) const {
    const auto it = field_cells_.find(map_id);
    std::vector<float> out(it != field_cells_.end() ? it->second : 0);
    float unused = 0.0f;  // an unknown id still reaches the batch, which refuses it
    check(bb200_amcl_batch_get_likelihood_field(handle_, map_id, out.empty() ? &unused : out.data(), out.size()));
    return out;
  }
  void initialize(std::size_t member, const SE2d& pose, const Matrix3d& covariance) {
    const double mean[3] = {pose.x(), pose.y(), pose.theta()};
    check(bb200_amcl_batch_initialize(handle_, index(member), mean, covariance.data()));
  }
  void initialize_from_map(std::size_t member) { check(bb200_amcl_batch_initialize_from_map(handle_, index(member))); }
  void force_update(std::size_t member) { check(bb200_amcl_batch_force_update(handle_, index(member))); }

  /// controls[m] and points[m] are member m's odometry pose and scan points; present (optional) marks the members that
  /// have a scan this step.
  auto update(const std::vector<SE2d>& controls, const std::vector<std::vector<std::pair<double, double>>>& points,
              const std::vector<bool>* present = nullptr) -> std::vector<std::optional<estimation_type>> {
    const std::size_t k = size();
    if (controls.size() != k || points.size() != k || (present != nullptr && present->size() != k))
      throw Error(BB200_ERR_INVALID_ARGUMENT, "one control, one scan (and one presence flag) per member");
    static_assert(sizeof(SE2d) == 4 * sizeof(double), "SE2d must be four packed doubles");
    static_assert(sizeof(std::pair<double, double>) == 2 * sizeof(double), "measurement points must be packed");
    std::vector<const double*> pts(k);
    std::vector<std::uint64_t> counts(k);
    std::vector<std::uint8_t> mask(present != nullptr ? k : 0);
    for (std::size_t m = 0; m < k; ++m) {
      pts[m] = points[m].empty() ? nullptr : &points[m].front().first;
      counts[m] = points[m].size();
      if (present != nullptr) mask[m] = (*present)[m] ? 1 : 0;
    }
    std::vector<bb200_update_result> r(k);
    check(bb200_amcl_batch_update(handle_, controls.front().data(), pts.data(), counts.data(), present != nullptr ? mask.data() : nullptr, r.data()));
    return estimates_of(r);
  }

  /// One member's measurement in a step: base-frame points, a laser scan or a point cloud, as Amcl::update takes them, or
  /// the detections of a member on a landmark map (what LandmarkSensorModel2d / BearingSensorModel2d return).  The
  /// constructors are explicit, so that a braced list of point vectors still selects the points overload above.
  struct Measurement {
    explicit Measurement(std::vector<std::pair<double, double>> points) : value(std::move(points)) {}
    explicit Measurement(const LaserScanView& scan) : value(scan) {}
    explicit Measurement(const PointCloudView& cloud) : value(cloud) {}
    explicit Measurement(landmark_token detections) : value(std::move(detections)) {}
    std::variant<std::vector<std::pair<double, double>>, LaserScanView, PointCloudView, landmark_token> value;
  };
  /// The bb200_measurement of one member's measurement; a scan's or a cloud's C view goes to *scan or *cloud, which must
  /// outlive the call it is passed to.  Detections reach the batch through stage_detections.
  static bb200_measurement c_measurement(const Measurement& measurement, bb200_laser_scan* scan, bb200_point_cloud* cloud) {
    const auto& v = measurement.value;
    if (const auto* points = std::get_if<0>(&v))
      return bb200_measurement{BB200_MEASUREMENT_POINTS, points->empty() ? nullptr : &points->front().first, points->size(), nullptr, nullptr};
    if (const auto* s = std::get_if<LaserScanView>(&v)) {
      *scan = s->c_view();
      return bb200_measurement{BB200_MEASUREMENT_SCAN, nullptr, 0, scan, nullptr};
    }
    if (std::holds_alternative<landmark_token>(v)) return bb200_measurement{BB200_MEASUREMENT_LANDMARKS, nullptr, 0, nullptr, nullptr};
    *cloud = std::get<PointCloudView>(v).c_view();
    return bb200_measurement{BB200_MEASUREMENT_CLOUD, nullptr, 0, nullptr, cloud};
  }
  /// bb200_amcl_batch_set_detections for every selected member whose measurement is a landmark_token (none: no call).
  template <class At>
  void stage_detections(std::size_t k, At measurement_at, const std::vector<bool>* present) {
    std::vector<const bb200_landmark_detection*> dets(k, nullptr);
    std::vector<std::uint64_t> counts(k, 0);
    std::vector<std::uint8_t> mask(k, 0);
    bool any = false;
    for (std::size_t m = 0; m < k; ++m) {
      const Measurement* meas = measurement_at(m);
      const auto* token = meas != nullptr ? std::get_if<landmark_token>(&meas->value) : nullptr;
      if (token == nullptr || (present != nullptr ? !(*present)[m] : sizes_[m] == 0)) continue;
      dets[m] = token->detections.empty() ? nullptr : token->detections.data();
      counts[m] = token->detections.size();
      mask[m] = 1;
      any = true;
    }
    if (any) check(bb200_amcl_batch_set_detections(handle_, dets.data(), counts.data(), mask.data()));
  }
  /// update with member m's measurement in measurements[m], so that members with 2-D and 3-D lidars step in one call; scans
  /// and clouds are converted on the device (bb200_amcl_batch_update_measurements).  Every member's result equals its
  /// standalone Amcl::update's with the same measurement.  Throws Error(BB200_ERR_INVALID_ARGUMENT) before any member
  /// changes when some present member's scan or cloud is unusable.
  auto update(const std::vector<SE2d>& controls, const std::vector<Measurement>& measurements, const std::vector<bool>* present = nullptr)
      -> std::vector<std::optional<estimation_type>> {
    const std::size_t k = size();
    if (controls.size() != k || measurements.size() != k || (present != nullptr && present->size() != k))
      throw Error(BB200_ERR_INVALID_ARGUMENT, "one control, one measurement (and one presence flag) per member");
    static_assert(sizeof(SE2d) == 4 * sizeof(double), "SE2d must be four packed doubles");
    std::vector<bb200_laser_scan> scans(k);
    std::vector<bb200_point_cloud> clouds(k);
    std::vector<bb200_measurement> in(k);
    std::vector<std::uint8_t> mask(present != nullptr ? k : 0);
    stage_detections(k, [&](std::size_t m) { return &measurements[m]; }, present);
    for (std::size_t m = 0; m < k; ++m) {
      in[m] = c_measurement(measurements[m], &scans[m], &clouds[m]);
      if (present != nullptr) mask[m] = (*present)[m] ? 1 : 0;
    }
    std::vector<bb200_update_result> r(k);
    check(bb200_amcl_batch_update_measurements(handle_, controls.front().data(), in.data(), present != nullptr ? mask.data() : nullptr, r.data()));
    return estimates_of(r);
  }
  /// update with members weighed by the caller's own sensor model (bb200_amcl_batch_update_begin / _end): an empty
  /// measurements[m] marks a weighed member, the others pass points, a scan or a cloud.  weigh(members, views) is called
  /// once with the weighed members that update in this step and the views of every slot (views[m].states, .factors, .n,
  /// .stream), and writes each such member's factors on views[m].stream; it is not called when none of them updates.
  /// weigh must not throw: the step would stay open and the batch then accepts nothing but its destruction.
  template <class Weigh>
  auto update(const std::vector<SE2d>& controls, const std::vector<std::optional<Measurement>>& measurements, Weigh&& weigh,
              const std::vector<bool>* present = nullptr) -> std::vector<std::optional<estimation_type>> {
    const std::size_t k = size();
    if (controls.size() != k || measurements.size() != k || (present != nullptr && present->size() != k))
      throw Error(BB200_ERR_INVALID_ARGUMENT, "one control, one measurement (and one presence flag) per member");
    std::vector<bb200_laser_scan> scans(k);
    std::vector<bb200_point_cloud> clouds(k);
    std::vector<bb200_measurement> in(k);
    std::vector<std::uint8_t> mask(present != nullptr ? k : 0);
    stage_detections(k, [&](std::size_t m) { return measurements[m] ? &*measurements[m] : nullptr; }, present);
    for (std::size_t m = 0; m < k; ++m) {
      in[m] = measurements[m] ? c_measurement(*measurements[m], &scans[m], &clouds[m]) : bb200_measurement{BB200_MEASUREMENT_WEIGHTS, nullptr, 0, nullptr, nullptr};
      if (present != nullptr) mask[m] = (*present)[m] ? 1 : 0;
    }
    std::vector<bb200_weigh_view> views(k);
    check(bb200_amcl_batch_update_begin(handle_, controls.front().data(), in.data(), present != nullptr ? mask.data() : nullptr, views.data()));
    std::vector<std::size_t> weighed;
    for (std::size_t m = 0; m < k; ++m)
      if (!measurements[m] && views[m].updated) weighed.push_back(m);
    if (!weighed.empty()) weigh(static_cast<const std::vector<std::size_t>&>(weighed), static_cast<const std::vector<bb200_weigh_view>&>(views));
    std::vector<bb200_update_result> r(k);
    check(bb200_amcl_batch_update_end(handle_, nullptr, r.data(), nullptr, nullptr, nullptr));
    return estimates_of(r);
  }
  /// update with a laser scan for every member (beluga_ros::Amcl::update(base_pose_in_odom, laser_scan) per member).
  auto update(const std::vector<SE2d>& controls, const std::vector<LaserScanView>& scans, const std::vector<bool>* present = nullptr)
      -> std::vector<std::optional<estimation_type>> {
    return update(controls, std::vector<Measurement>(scans.begin(), scans.end()), present);
  }
  /// update with a point cloud for every member (beluga_ros::Amcl::update(base_pose_in_odom, point_cloud) per member).
  auto update(const std::vector<SE2d>& controls, const std::vector<PointCloudView>& clouds, const std::vector<bool>* present = nullptr)
      -> std::vector<std::optional<estimation_type>> {
    return update(controls, std::vector<Measurement>(clouds.begin(), clouds.end()), present);
  }
  /// update, then beluga::cluster_based_estimate of every member that updated, in one call
  /// (bb200_amcl_batch_update_clustered): per member what beluga_ros::Amcl::update returns, the cluster-based estimate,
  /// or std::nullopt when the member did not update.  The per-cell flood runs on the device.
  auto update_clustered(const std::vector<SE2d>& controls, const std::vector<Measurement>& measurements, const std::vector<bool>* present = nullptr,
                        ParticleClusterizerParam parameters = {}) -> std::vector<std::optional<estimation_type>> {
    const std::size_t k = size();
    if (controls.size() != k || measurements.size() != k || (present != nullptr && present->size() != k))
      throw Error(BB200_ERR_INVALID_ARGUMENT, "one control, one measurement (and one presence flag) per member");
    std::vector<bb200_laser_scan> scans(k);
    std::vector<bb200_point_cloud> clouds(k);
    std::vector<bb200_measurement> in(k);
    const std::vector<std::uint8_t> mask = presence_mask(present);
    stage_detections(k, [&](std::size_t m) { return &measurements[m]; }, present);
    for (std::size_t m = 0; m < k; ++m) in[m] = c_measurement(measurements[m], &scans[m], &clouds[m]);
    const bb200_cluster_param p{parameters.linear_hash_resolution, parameters.angular_hash_resolution, parameters.weight_cap_percentile};
    std::vector<bb200_update_result> r(k);
    std::vector<bb200_estimate> e(k);
    check(bb200_amcl_batch_update_clustered(handle_, controls.front().data(), in.data(), present != nullptr ? mask.data() : nullptr, &p, r.data(),
                                            e.data(), nullptr, nullptr));
    std::vector<std::optional<estimation_type>> out(k);
    for (std::size_t m = 0; m < k; ++m) {
      if (!r[m].updated) continue;
      Matrix3d cov;
      for (int i = 0; i < 9; ++i) cov[i] = e[m].cov[i];
      out[m] = std::make_pair(SE2d::from_data(e[m].mean), cov);
    }
    return out;
  }
  /// update_clustered with base-frame points for every member.
  auto update_clustered(const std::vector<SE2d>& controls, const std::vector<std::vector<std::pair<double, double>>>& points,
                        const std::vector<bool>* present = nullptr, ParticleClusterizerParam parameters = {})
      -> std::vector<std::optional<estimation_type>> {
    std::vector<Measurement> views;
    views.reserve(points.size());
    for (const auto& p : points) views.emplace_back(p);
    return update_clustered(controls, views, present, parameters);
  }
  /// update_clustered with a laser scan for every member.
  auto update_clustered(const std::vector<SE2d>& controls, const std::vector<LaserScanView>& scans, const std::vector<bool>* present = nullptr,
                        ParticleClusterizerParam parameters = {}) -> std::vector<std::optional<estimation_type>> {
    return update_clustered(controls, std::vector<Measurement>(scans.begin(), scans.end()), present, parameters);
  }
#ifdef BELUGA_B200_WITH_SOPHUS
  /// The same for any beluga::BaseSparsePointCloud-shaped clouds, e.g. beluga_ros::SparsePointCloud3f.
  template <class SparsePointCloud, std::enable_if_t<is_sparse_point_cloud_v<SparsePointCloud>, int> = 0>
  auto update(const std::vector<SE2d>& controls, const std::vector<SparsePointCloud>& clouds, const std::vector<bool>* present = nullptr)
      -> std::vector<std::optional<estimation_type>> {
    std::vector<PackedPointCloud> packed;
    packed.reserve(clouds.size());
    for (const auto& c : clouds) packed.emplace_back(c);
    std::vector<Measurement> views;
    views.reserve(packed.size());
    for (const auto& p : packed) views.emplace_back(p.view());
    return update(controls, views, present);
  }
#endif

  /// Member m's current particle count.
  [[nodiscard]] std::size_t member_size(std::size_t member) const {
    std::uint64_t n = 0;
    check(bb200_amcl_batch_member_size(handle_, index(member), &n));
    return static_cast<std::size_t>(n);
  }

  /// Member m's particle set, copied from the device: max_particles entries in a fixed batch, member_size(m)
  /// in an adaptive one.
  [[nodiscard]] ParticleSet particles(std::size_t member) const {
    const std::size_t n = adaptive_ ? member_size(member) : sizes_.at(member);
    ParticleSet out;
    out.states.resize(n);
    out.weights.resize(n);
    check(bb200_amcl_batch_get_particles(handle_, index(member), reinterpret_cast<double*>(out.states.data()), out.weights.data(), out.size()));
    return out;
  }

  /// beluga::cluster_based_estimate of member m's particles.
  [[nodiscard]] estimation_type cluster_based_estimate(std::size_t member, ParticleClusterizerParam parameters = {}) const {
    const bb200_cluster_param p{parameters.linear_hash_resolution, parameters.angular_hash_resolution, parameters.weight_cap_percentile};
    bb200_estimate e{};
    check(bb200_amcl_batch_cluster_estimate(handle_, index(member), &p, &e));
    Matrix3d cov;
    for (int i = 0; i < 9; ++i) cov[i] = e.cov[i];
    return std::make_pair(SE2d::from_data(e.mean), cov);
  }

  /// beluga::cluster_based_estimate of every member whose present[m] is true (present == nullptr: all of them) in one call
  /// with a fixed number of kernel launches; std::nullopt for members not selected.
  [[nodiscard]] auto cluster_based_estimates(const std::vector<bool>* present = nullptr, ParticleClusterizerParam parameters = {}) const
      -> std::vector<std::optional<estimation_type>> {
    const std::size_t k = size();
    if (present != nullptr && present->size() != k) throw Error(BB200_ERR_INVALID_ARGUMENT, "one presence flag per member");
    const bb200_cluster_param p{parameters.linear_hash_resolution, parameters.angular_hash_resolution, parameters.weight_cap_percentile};
    std::vector<std::uint8_t> mask(present != nullptr ? k : 0);
    for (std::size_t m = 0; m < mask.size(); ++m) mask[m] = (*present)[m] ? 1 : 0;
    std::vector<bb200_estimate> e(k);
    check(bb200_amcl_batch_cluster_estimates(handle_, &p, present != nullptr ? mask.data() : nullptr, e.data(), nullptr, nullptr));
    std::vector<std::optional<estimation_type>> out(k);
    for (std::size_t m = 0; m < k; ++m) {
      if ((present != nullptr && !(*present)[m]) || sizes_[m] == 0) continue;
      Matrix3d cov;
      for (int i = 0; i < 9; ++i) cov[i] = e[m].cov[i];
      out[m] = std::make_pair(SE2d::from_data(e[m].mean), cov);
    }
    return out;
  }

  /// One member's particle-cloud histogram: its bins in first-occurrence order and max(1e-3, heaviest bin).
  using histogram_type = std::pair<std::vector<bb200_cluster_cell>, double>;

  /// The particle-cloud histogram (bb200_filter_particle_histogram) of every member whose present[m] is true (present ==
  /// nullptr: all of them) in one call; std::nullopt for members not selected.  Each member's buffer holds max_particles
  /// bins (a member never has more bins than particles), so one device pass fills them all.
  [[nodiscard]] auto particle_histograms(const std::vector<bool>* present = nullptr, double linear_resolution = 1e-3,
                                         double angular_resolution = 1e-3) const -> std::vector<std::optional<histogram_type>> {
    const std::vector<std::uint8_t> mask = presence_mask(present);
    const std::size_t k = size();
    std::vector<std::vector<bb200_cluster_cell>> bins(k);
    std::vector<bb200_cluster_cell*> ptrs(k, nullptr);
    std::vector<std::uint64_t> capacity(k, 0), n_bins(k, 0);
    std::vector<double> top(k, 0.0);
    for (std::size_t m = 0; m < k; ++m) {
      if ((present != nullptr && !(*present)[m]) || sizes_[m] == 0) continue;
      bins[m].resize(sizes_[m]);
      ptrs[m] = bins[m].data();
      capacity[m] = sizes_[m];
    }
    check(bb200_amcl_batch_particle_histograms(handle_, linear_resolution, angular_resolution, present != nullptr ? mask.data() : nullptr, ptrs.data(),
                                               capacity.data(), n_bins.data(), top.data()));
    std::vector<std::optional<histogram_type>> out(k);
    for (std::size_t m = 0; m < k; ++m) {
      if (ptrs[m] == nullptr) continue;
      bins[m].resize(n_bins[m]);
      out[m] = std::make_pair(std::move(bins[m]), top[m]);
    }
    return out;
  }

  /// counts[m] states {cos, sin, x, y} drawn by weight from every member whose present[m] is true (present == nullptr: all
  /// of them), the multinomial counter-RNG draws of `step` (bb200_filter_sample_states); std::nullopt for members not
  /// selected.  No particle set changes.
  [[nodiscard]] auto sample_states(const std::vector<std::size_t>& counts, uint32_t step, const std::vector<bool>* present = nullptr) const
      -> std::vector<std::optional<std::vector<double>>> {
    const std::vector<std::uint8_t> mask = presence_mask(present);
    const std::size_t k = size();
    if (counts.size() != k) throw Error(BB200_ERR_INVALID_ARGUMENT, "one sample count per member");
    std::vector<std::vector<double>> raw(k);
    std::vector<double*> ptrs(k, nullptr);
    std::vector<std::uint64_t> n(k, 0);
    for (std::size_t m = 0; m < k; ++m) {
      n[m] = counts[m];
      raw[m].resize(4 * counts[m]);
      ptrs[m] = raw[m].empty() ? nullptr : raw[m].data();
    }
    check(bb200_amcl_batch_sample_states(handle_, n.data(), step, present != nullptr ? mask.data() : nullptr, ptrs.data()));
    std::vector<std::optional<std::vector<double>>> out(k);
    for (std::size_t m = 0; m < k; ++m)
      if ((present == nullptr || (*present)[m]) && sizes_[m] != 0) out[m] = std::move(raw[m]);
    return out;
  }

  /// Amcl::cast_rays for every member whose present[m] is true (present == nullptr: every occupied slot): poses[m] x
  /// bearings[m] rays up to max_range[m], pose major, on the member's own map or on map (*map_ids)[m] of the batch when
  /// map_ids is set and that entry is not -1; std::nullopt for members not selected.  One kernel launch whatever K is
  /// (bb200_amcl_batch_cast_rays); no member changes.
  [[nodiscard]] auto cast_rays(const std::vector<std::vector<SE2d>>& poses, const std::vector<std::vector<Bearing>>& bearings,
                               const std::vector<double>& max_range, const std::vector<bool>* present = nullptr,
                               const std::vector<int>* map_ids = nullptr) const -> std::vector<std::optional<std::vector<std::optional<double>>>> {
    const std::vector<std::uint8_t> mask = presence_mask(present);
    const std::size_t k = size();
    if (poses.size() != k || bearings.size() != k || max_range.size() != k || (map_ids != nullptr && map_ids->size() != k))
      throw Error(BB200_ERR_INVALID_ARGUMENT, "one pose list, bearing list, maximum range and map id per member");
    std::vector<std::vector<double>> raw(k);
    std::vector<const double*> p(k, nullptr), b(k, nullptr);
    std::vector<double*> r(k, nullptr);
    std::vector<std::uint64_t> np(k), nb(k);
    for (std::size_t m = 0; m < k; ++m) {
      np[m] = poses[m].size();
      nb[m] = bearings[m].size();
      p[m] = poses[m].empty() ? nullptr : poses[m].front().data();
      b[m] = bearings[m].empty() ? nullptr : bearings[m].front().data();
      raw[m].resize(poses[m].size() * bearings[m].size());
      r[m] = raw[m].empty() ? nullptr : raw[m].data();
    }
    check(bb200_amcl_batch_cast_rays(handle_, present != nullptr ? mask.data() : nullptr, map_ids != nullptr ? map_ids->data() : nullptr, p.data(),
                                     np.data(), b.data(), nb.data(), max_range.data(), r.data()));
    std::vector<std::optional<std::vector<std::optional<double>>>> out(k);
    for (std::size_t m = 0; m < k; ++m)
      if ((present == nullptr || (*present)[m]) && sizes_[m] != 0) out[m] = detail::cast_results(raw[m].data(), raw[m].size());
    return out;
  }

  [[nodiscard]] bb200_amcl_batch* handle() const { return handle_; }

 private:
  AmclBatch(bb200_amcl_batch* handle, std::vector<std::size_t> sizes, bool adaptive) : adaptive_{adaptive}, handle_{handle}, sizes_{std::move(sizes)} {}
  static std::vector<std::optional<estimation_type>> estimates_of(const std::vector<bb200_update_result>& r) {
    std::vector<std::optional<estimation_type>> out(r.size());
    for (std::size_t m = 0; m < r.size(); ++m) {
      if (!r[m].updated) continue;
      Matrix3d cov;
      for (int i = 0; i < 9; ++i) cov[i] = r[m].estimate.cov[i];
      out[m] = std::make_pair(SE2d::from_data(r[m].estimate.mean), cov);
    }
    return out;
  }
  int index(std::size_t member) const {
    if (member >= size()) throw Error(BB200_ERR_INVALID_ARGUMENT, "member index out of range");
    return static_cast<int>(member);
  }
  void check(int status) const {
    if (status != BB200_OK) throw Error(status, bb200_amcl_batch_last_error(handle_));
  }
  static bb200_landmark_param c_param(const LandmarkModelParam& p) { return bb200_landmark_param{p.sigma_range, p.sigma_bearing, p.random_prob}; }
  static bb200_bearing_param c_param(const BearingModelParam& p) {
    bb200_bearing_param c{};
    c.sigma_bearing = p.sigma_bearing;
    for (int k = 0; k < 12; ++k) c.sensor_pose_in_robot[k] = p.sensor_pose_in_robot.m[k];
    return c;
  }
  std::vector<std::uint8_t> presence_mask(const std::vector<bool>* present) const {
    if (present != nullptr && present->size() != size()) throw Error(BB200_ERR_INVALID_ARGUMENT, "one presence flag per member");
    std::vector<std::uint8_t> mask(present != nullptr ? size() : 0);
    for (std::size_t m = 0; m < mask.size(); ++m) mask[m] = (*present)[m] ? 1 : 0;
    return mask;
  }

  bool adaptive_{false};
  bb200_amcl_batch* handle_{nullptr};
  std::vector<std::size_t> sizes_;  // per slot, max_particles (0: vacant): upper bounds of every member's particle, histogram and sample counts
  std::map<int, std::size_t> field_cells_;  // cells of each likelihood-field map, by id
};

}  // namespace beluga_b200
