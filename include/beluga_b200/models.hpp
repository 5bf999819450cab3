// beluga_b200/models.hpp -- MotionModel / SensorModel shaped adaptors over the C ABI.
//
// Header-only C++17.  These types have the member types, constructor arguments and parameter
// structs of the reference models so that code written against
//   beluga::DifferentialDriveModel2d      (beluga/motion/differential_drive_model.hpp:77-174)
//   beluga::LikelihoodFieldModel<Grid>    (beluga/sensor/likelihood_field_model.hpp:41-92)
//   beluga::LikelihoodFieldProbModel<Grid>(beluga/sensor/likelihood_field_prob_model.hpp:41-92)
//   beluga::BeamSensorModel<Grid>         (beluga/sensor/beam_model.hpp:73-163)
//   beluga::LandmarkSensorModel2d<LandmarkMap>, beluga::BearingSensorModel2d<LandmarkMap>
//                                         (beluga/sensor/landmark_sensor_model.hpp, bearing_sensor_model.hpp)
// keeps compiling when the namespace is switched to beluga_b200.  The reference models return
// per-particle callables (state sampling / weighting functions); here `operator()` returns a small
// token that beluga_b200::Amcl hands to the device kernels -- the per-particle loop lives on the GPU.
//
// Sophus/Eigen are optional: define BELUGA_B200_WITH_SOPHUS before including to get converting
// constructors from/to Sophus::SE2d and Eigen::Matrix3d.
#pragma once

#include <array>
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "../beluga_b200.h"

#ifdef BELUGA_B200_WITH_SOPHUS
#include <Eigen/Core>
#include <sophus/se2.hpp>
#include <sophus/se3.hpp>
#endif

namespace beluga_b200 {

/// 2-D pose with Sophus::SE2d's memory layout {cos, sin, x, y} (Sophus::SE2d::data()).
struct SE2d {
  std::array<double, 4> v{1.0, 0.0, 0.0, 0.0};

  SE2d() = default;
  /// Sophus::SE2d{theta, translation}: the rotation is normalised through hypot like SO2::exp.
  SE2d(double theta, double x, double y) {
    const double c = std::cos(theta), s = std::sin(theta), n = std::hypot(c, s);
    v = {c / n, s / n, x, y};
  }
  static SE2d from_data(const double* d) {
    SE2d p;
    p.v = {d[0], d[1], d[2], d[3]};
    return p;
  }
#ifdef BELUGA_B200_WITH_SOPHUS
  SE2d(const Sophus::SE2d& p) : v{p.data()[0], p.data()[1], p.data()[2], p.data()[3]} {}  // NOLINT(google-explicit-constructor)
  operator Sophus::SE2d() const {                                                           // NOLINT(google-explicit-constructor)
    Sophus::SE2d out;
    std::copy(v.begin(), v.end(), out.data());
    return out;
  }
#endif
  [[nodiscard]] const double* data() const { return v.data(); }
  [[nodiscard]] double x() const { return v[2]; }
  [[nodiscard]] double y() const { return v[3]; }
  [[nodiscard]] double theta() const { return std::atan2(v[1], v[0]); }  // so2().log()
};

/// 3x3 covariance over (x, y, theta), row-major (Sophus::Matrix3d of estimation.hpp:436).
using Matrix3d = std::array<double, 9>;

/// Thrown where the reference throws (std::runtime_error / std::invalid_argument) or a CUDA call fails.
class Error : public std::runtime_error {
 public:
  Error(int status, const std::string& what) : std::runtime_error(what), status_(status) {}
  [[nodiscard]] int status() const { return status_; }

 private:
  int status_;
};

// ---- motion --------------------------------------------------------------------------------------

/// Same members and defaults as beluga::DifferentialDriveModelParam (differential_drive_model.hpp:40-68).
struct DifferentialDriveModelParam {
  double rotation_noise_from_rotation;
  double rotation_noise_from_translation;
  double translation_noise_from_translation;
  double translation_noise_from_rotation;
  double distance_threshold = 0.01;
};

class DifferentialDriveModel {
 public:
  using state_type = SE2d;
  using control_type = std::tuple<state_type, state_type>;  // (current, previous) odometry poses
  using param_type = DifferentialDriveModelParam;

  explicit DifferentialDriveModel(const param_type& params) : params_{params} {}

  /// Token of a control action: the three normal distributions of sampling_fn_2d (:141-154).
  struct sampling_token {
    bb200_diff_drive_sampling sampling;
  };

  template <class Control>
  [[nodiscard]] sampling_token operator()(const Control& action) const {
    const auto& [pose, previous_pose] = action;
    sampling_token t{};
    const bb200_diff_drive_param p = c_param();
    bb200_diff_drive_sampling_from_control(&p, state_type(pose).data(), state_type(previous_pose).data(), &t.sampling);
    return t;
  }

  [[nodiscard]] bb200_diff_drive_param c_param() const {
    return bb200_diff_drive_param{params_.rotation_noise_from_rotation, params_.rotation_noise_from_translation,
                                  params_.translation_noise_from_translation, params_.translation_noise_from_rotation,
                                  params_.distance_threshold};
  }
  [[nodiscard]] bb200_motion_param c_motion_param() const {
    return bb200_motion_param{BB200_MOTION_DIFFERENTIAL, params_.rotation_noise_from_rotation, params_.rotation_noise_from_translation,
                              params_.translation_noise_from_translation, params_.translation_noise_from_rotation, 0.0, params_.distance_threshold};
  }

 private:
  param_type params_;
};
using DifferentialDriveModel2d = DifferentialDriveModel;

/// Same members and defaults as beluga::OmnidirectionalDriveModelParam (omnidirectional_drive_model.hpp:36-68).
struct OmnidirectionalDriveModelParam {
  double rotation_noise_from_rotation;
  double rotation_noise_from_translation;
  double translation_noise_from_translation;
  double translation_noise_from_rotation;
  double strafe_noise_from_translation;
  double distance_threshold = 0.01;
};

/// beluga::OmnidirectionalDriveModel (omnidirectional_drive_model.hpp:78-158).
class OmnidirectionalDriveModel {
 public:
  using state_type = SE2d;
  using control_type = std::tuple<state_type, state_type>;
  using param_type = OmnidirectionalDriveModelParam;
  explicit OmnidirectionalDriveModel(const param_type& params) : params_{params} {}
  [[nodiscard]] bb200_motion_param c_motion_param() const {
    return bb200_motion_param{BB200_MOTION_OMNIDIRECTIONAL, params_.rotation_noise_from_rotation, params_.rotation_noise_from_translation,
                              params_.translation_noise_from_translation, params_.translation_noise_from_rotation,
                              params_.strafe_noise_from_translation, params_.distance_threshold};
  }

 private:
  param_type params_;
};

/// beluga::StationaryModel (stationary_model.hpp:39-62).
class StationaryModel {
 public:
  using state_type = SE2d;
  using control_type = std::tuple<state_type, state_type>;
  [[nodiscard]] bb200_motion_param c_motion_param() const { return bb200_motion_param{BB200_MOTION_STATIONARY, 0, 0, 0, 0, 0, 0.01}; }
};

// ---- maps ----------------------------------------------------------------------------------------

/// Flattens any type satisfying the reference's OccupancyGrid2 requirements
/// (sensor/data/occupancy_grid.hpp: width(), height(), resolution(), origin(), data(), value_traits())
/// into the trinary int8 view of the C ABI.
struct GridSnapshot {
  std::vector<std::int8_t> cells;
  std::int32_t width{0}, height{0};
  double resolution{1.0};
  SE2d origin{};

  template <class OccupancyGrid>
  explicit GridSnapshot(const OccupancyGrid& grid)
      : width(static_cast<std::int32_t>(grid.width())), height(static_cast<std::int32_t>(grid.height())), resolution(grid.resolution()), origin(grid.origin()) {
    const auto traits = grid.value_traits();
    cells.reserve(grid.size());
    for (const auto& value : grid.data()) {
      cells.push_back(traits.is_occupied(value) ? std::int8_t{100} : (traits.is_free(value) ? std::int8_t{0} : std::int8_t{-1}));
    }
  }

  /// The C-ABI view; valid while this snapshot is alive and unmodified.
  [[nodiscard]] bb200_occupancy_grid view() const {
    bb200_occupancy_grid v{};
    v.cells = cells.data();
    v.width = width;
    v.height = height;
    v.resolution = resolution;
    for (int i = 0; i < 4; ++i) v.origin[i] = origin.data()[i];
    return v;
  }
};

/// A plain occupancy grid for callers without their own grid type (ROS trinary values).
class OccupancyGrid {
 public:
  struct ValueTraits {
    [[nodiscard]] static bool is_free(std::int8_t v) { return v == 0; }
    [[nodiscard]] static bool is_unknown(std::int8_t v) { return v == -1; }
    [[nodiscard]] static bool is_occupied(std::int8_t v) { return v == 100; }
  };
  OccupancyGrid(std::vector<std::int8_t> cells, std::size_t width, double resolution, SE2d origin = SE2d{})
      : cells_(std::move(cells)), width_(width), resolution_(resolution), origin_(origin) {}
  [[nodiscard]] std::size_t width() const { return width_; }
  [[nodiscard]] std::size_t height() const { return cells_.size() / width_; }
  [[nodiscard]] std::size_t size() const { return cells_.size(); }
  [[nodiscard]] double resolution() const { return resolution_; }
  [[nodiscard]] const SE2d& origin() const { return origin_; }
  [[nodiscard]] const std::vector<std::int8_t>& data() const { return cells_; }
  [[nodiscard]] ValueTraits value_traits() const { return {}; }

 private:
  std::vector<std::int8_t> cells_;
  std::size_t width_;
  double resolution_;
  SE2d origin_;
};

// ---- sensors -------------------------------------------------------------------------------------

/// Same members and defaults as beluga::LikelihoodFieldModelBaseParam (likelihood_field_model_base.hpp:42-64).
struct LikelihoodFieldModelParam {
  double max_obstacle_distance = 100.0;
  double max_laser_distance = 2.0;
  double z_hit = 0.5;
  double z_random = 0.5;
  double sigma_hit = 0.2;
  bool model_unknown_space = false;
  bool only_obstacle_boundaries = false;
};

/// Same members and defaults as beluga::BeamModelParam (beam_model.hpp:43-58).
struct BeamModelParam {
  double z_hit{0.5};
  double z_short{0.5};
  double z_max{0.05};
  double z_rand{0.05};
  double sigma_hit{0.2};
  double lambda_short{0.1};
  double beam_max_range{60};
};

/// Measurement token: the lidar hit points in the particle frame (measurement_type of the reference).
struct measurement_token {
  std::vector<std::pair<double, double>> points;
};

/// A caller's device sensor model (the SensorModel parameter of beluga::Amcl for a sensor this library has no model for)
/// has state_type (SE2d), measurement_type and map_type, `int attach(bb200_filter*) const` (BB200_OK, or the status of the
/// bb200_filter_set_*_map call that gives the filter a map for initialize_from_map and recovery injection) and
/// `update_map(map)`, and its operator()(measurement) returns a token with
///   void weigh(void* stream, const double* states, std::uint64_t n, double* factors) const;
/// which writes factors[i] = L(state_i) for the n propagated device states {cos, sin, x, y}, enqueued on `stream` (a
/// cudaStream_t) or synchronised with it.  Amcl::update then runs bb200_amcl_update_begin, weigh and bb200_amcl_update_end.
template <class T, class = void>
struct is_weighed_token : std::false_type {};
template <class T>
struct is_weighed_token<T, std::void_t<decltype(std::declval<const T&>().weigh(std::declval<void*>(), std::declval<const double*>(),
                                                                                std::declval<std::uint64_t>(), std::declval<double*>()))>>
    : std::true_type {};
template <class T>
constexpr bool is_weighed_token_v = is_weighed_token<T>::value;

// ---- point clouds --------------------------------------------------------------------------------

/// A sensor_msgs/PointCloud2 buffer as beluga_ros::SparsePointCloud3f reads it
/// (beluga_ros/include/beluga_ros/sparse_point_cloud.hpp:102-125): point i is the three scalars x, y, z at
/// data + i * point_step + x_offset.  `origin` is the cloud's frame in the base frame as a 3x4 row-major [R | t]
/// (nullptr: the identity).  A view: the buffers must outlive it.
struct PointCloudView {
  const void* data = nullptr;
  std::uint64_t size = 0;  // width * height
  std::uint32_t point_step = 0;
  std::uint32_t x_offset = 0;
  bb200_point_datatype datatype = BB200_POINT_FLOAT32;
  const double* origin = nullptr;

  [[nodiscard]] bb200_point_cloud c_view() const { return bb200_point_cloud{data, size, point_step, x_offset, datatype, origin}; }
};

/// A sensor_msgs/LaserScan as beluga_ros::LaserScan reads it (beluga_ros/include/beluga_ros/laser_scan.hpp:69-80): the ranges,
/// angle_min and angle_increment of the message, the range limits already combined with the node's, the max_beams of
/// take_evenly (0: every reading) and the laser's frame in the base frame as a 3x4 row-major [R | t] (nullptr: the
/// identity).  A view: the buffers must outlive it.
struct LaserScanView {
  const float* ranges = nullptr;
  std::uint64_t size = 0;
  float angle_min = 0.0f;
  float angle_increment = 0.0f;
  double min_range = 0.0;
  double max_range = HUGE_VAL;
  std::uint64_t max_beams = 0;
  const double* origin = nullptr;

  [[nodiscard]] bb200_laser_scan c_view() const {
    return bb200_laser_scan{ranges, size, angle_min, angle_increment, min_range, max_range, max_beams, origin};
  }
};

/// The base-frame (x, y) of every point, in order (beluga_ros/src/amcl.cpp:67-78); host only, needs no GPU.
/// Throws Error(BB200_ERR_INVALID_ARGUMENT) where SparsePointCloud3 throws std::invalid_argument on the layout.
[[nodiscard]] inline std::vector<std::pair<double, double>> point_cloud_points(const PointCloudView& cloud) {
  static_assert(sizeof(std::pair<double, double>) == 2 * sizeof(double), "measurement points must be packed");
  std::vector<std::pair<double, double>> out(cloud.size);
  const bb200_point_cloud c = cloud.c_view();
  std::uint64_t n = 0;
  const int st = bb200_point_cloud_to_points(&c, out.empty() ? nullptr : &out.front().first, out.size(), &n);
  if (st != BB200_OK) throw Error(st, "point cloud: datatype must be FLOAT32 or FLOAT64 and x, y, z must fit in point_step");
  return out;
}

#ifdef BELUGA_B200_WITH_SOPHUS
namespace detail {
template <class T, class = void>
struct is_sparse_point_cloud : std::false_type {};
/// Shaped like beluga::BaseSparsePointCloud (beluga/sensor/data/sparse_point_cloud.hpp): points() is a range of 3-vectors
/// with x(), y(), z(), and origin() is the Sophus::SE3d of the cloud's frame in the filter's base frame.
template <class T>
struct is_sparse_point_cloud<T, std::void_t<decltype((*std::declval<const T&>().points().begin()).z()),
                                            decltype(std::declval<const T&>().origin().matrix3x4())>>
    : std::is_convertible<decltype(std::declval<const T&>().origin()), Sophus::SE3d> {};
}  // namespace detail
template <class T>
inline constexpr bool is_sparse_point_cloud_v = detail::is_sparse_point_cloud<T>::value;

/// A BaseSparsePointCloud-shaped cloud packed into float32 x, y, z records plus its origin: the C-ABI view of it.
/// Coordinates are narrowed to float, which is what beluga_ros's SparsePointCloud3f alias hands to Amcl::update.
struct PackedPointCloud {
  std::vector<float> xyz;
  std::array<double, 12> origin{};

  template <class SparsePointCloud, std::enable_if_t<is_sparse_point_cloud_v<SparsePointCloud>, int> = 0>
  explicit PackedPointCloud(const SparsePointCloud& cloud) {
    for (const auto& p : cloud.points()) {
      xyz.push_back(static_cast<float>(p.x()));
      xyz.push_back(static_cast<float>(p.y()));
      xyz.push_back(static_cast<float>(p.z()));
    }
    const auto m = cloud.origin().matrix3x4();
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c) origin[static_cast<std::size_t>(4 * r + c)] = m(r, c);
  }
  [[nodiscard]] PointCloudView view() const {
    return PointCloudView{xyz.data(), xyz.size() / 3, 3 * sizeof(float), 0, BB200_POINT_FLOAT32, origin.data()};
  }
};
#endif

namespace detail {

template <class OccupancyGridT, bool kProb>
class LikelihoodFieldModelImpl {
 public:
  using state_type = SE2d;
  using weight_type = double;
  using measurement_type = std::vector<std::pair<double, double>>;
  using map_type = OccupancyGridT;
  using param_type = LikelihoodFieldModelParam;

  explicit LikelihoodFieldModelImpl(const param_type& params, const map_type& grid) : params_{params}, grid_{grid} {}
  void update_map(const map_type& grid) {
    grid_ = GridSnapshot{grid};
    ++map_version_;
  }
  [[nodiscard]] measurement_token operator()(measurement_type&& points) const { return measurement_token{std::move(points)}; }

  // -- used by beluga_b200::Amcl --
  [[nodiscard]] int attach(bb200_filter* f) const {
    const bb200_likelihood_field_param p{params_.max_obstacle_distance, params_.max_laser_distance, params_.z_hit,      params_.z_random,
                                         params_.sigma_hit,             params_.model_unknown_space ? 1 : 0, params_.only_obstacle_boundaries ? 1 : 0};
    const bb200_occupancy_grid g = grid_.view();
    return bb200_filter_set_likelihood_field_map(f, &p, &g, kProb ? 1 : 0);
  }
  // -- used by beluga_b200::ShardedAmcl --
  [[nodiscard]] int attach(bb200_sharded_amcl* g) const {
    const bb200_likelihood_field_param p{params_.max_obstacle_distance, params_.max_laser_distance, params_.z_hit,      params_.z_random,
                                         params_.sigma_hit,             params_.model_unknown_space ? 1 : 0, params_.only_obstacle_boundaries ? 1 : 0};
    const bb200_occupancy_grid g_view = grid_.view();
    return bb200_sharded_amcl_set_likelihood_field_map(g, &p, &g_view, kProb ? 1 : 0);
  }
  [[nodiscard]] unsigned map_version() const { return map_version_; }

 private:
  param_type params_;
  GridSnapshot grid_;
  unsigned map_version_{0};
};

}  // namespace detail

template <class OccupancyGridT = OccupancyGrid>
using LikelihoodFieldModel = detail::LikelihoodFieldModelImpl<OccupancyGridT, false>;
template <class OccupancyGridT = OccupancyGrid>
using LikelihoodFieldProbModel = detail::LikelihoodFieldModelImpl<OccupancyGridT, true>;

template <class OccupancyGridT = OccupancyGrid>
class BeamSensorModel {
 public:
  using state_type = SE2d;
  using weight_type = double;
  using measurement_type = std::vector<std::pair<double, double>>;
  using map_type = OccupancyGridT;
  using param_type = BeamModelParam;

  explicit BeamSensorModel(const param_type& params, const map_type& grid) : params_{params}, grid_{grid} {}
  void update_map(const map_type& grid) {
    grid_ = GridSnapshot{grid};
    ++map_version_;
  }
  [[nodiscard]] measurement_token operator()(measurement_type&& points) const { return measurement_token{std::move(points)}; }

  [[nodiscard]] int attach(bb200_filter* f) const {
    const bb200_beam_param p{params_.z_hit, params_.z_short, params_.z_max, params_.z_rand, params_.sigma_hit, params_.lambda_short, params_.beam_max_range};
    const bb200_occupancy_grid g = grid_.view();
    return bb200_filter_set_beam_map(f, &p, &g);
  }
  [[nodiscard]] int attach(bb200_sharded_amcl* g) const {
    const bb200_beam_param p{params_.z_hit, params_.z_short, params_.z_max, params_.z_rand, params_.sigma_hit, params_.lambda_short, params_.beam_max_range};
    const bb200_occupancy_grid g_view = grid_.view();
    return bb200_sharded_amcl_set_beam_map(g, &p, &g_view);
  }
  [[nodiscard]] unsigned map_version() const { return map_version_; }

 private:
  param_type params_;
  GridSnapshot grid_;
  unsigned map_version_{0};
};


// ---- landmark and bearing models ----------------------------------------------------------------------------------------

/// A position in 3-D: beluga's LandmarkPosition3 / LandmarkBearing3 (types/landmark_detection_types.hpp:33-34).
using LandmarkPosition3 = std::array<double, 3>;

/// types/landmark_detection_types.hpp:39-42: a detection's position in the robot frame and its category.
struct LandmarkPositionDetection {
  LandmarkPosition3 detection_position_in_robot{};
  std::uint32_t category{0};
};

/// types/landmark_detection_types.hpp:45-48: a detection's bearing vector in the sensor frame and its category.
struct LandmarkBearingDetection {
  LandmarkPosition3 detection_bearing_in_sensor{};
  std::uint32_t category{0};
};

/// The axis-aligned bounds of a LandmarkMap (LandmarkMapBoundaries, types/landmark_detection_types.hpp:36).
struct LandmarkMapBoundaries {
  LandmarkPosition3 min{}, max{};
};

/// beluga::LandmarkMap (sensor/data/landmark_map.hpp:40-166): the landmarks, in the world frame, with explicit bounds
/// or, without them, the landmarks' own (:61-71, computed by the library).  The library keeps a copy on the device.
class LandmarkMap {
 public:
  using landmarks_set_position_data = std::vector<LandmarkPositionDetection>;
  explicit LandmarkMap(const LandmarkMapBoundaries& boundaries, landmarks_set_position_data landmarks)
      : landmarks_(std::move(landmarks)), boundaries_(boundaries), explicit_bounds_(true) {}
  explicit LandmarkMap(landmarks_set_position_data landmarks) : landmarks_(std::move(landmarks)) {}

  /// The C view of this map; valid while the map lives and is not modified.
  [[nodiscard]] bb200_landmark_map view() const {
    c_.resize(landmarks_.size());
    for (std::size_t k = 0; k < landmarks_.size(); ++k) {
      const auto& p = landmarks_[k].detection_position_in_robot;
      c_[k] = bb200_landmark{p[0], p[1], p[2], landmarks_[k].category};
    }
    return bb200_landmark_map{c_.empty() ? nullptr : c_.data(), c_.size(), explicit_bounds_ ? boundaries_.min.data() : nullptr,
                              explicit_bounds_ ? boundaries_.max.data() : nullptr};
  }

 private:
  landmarks_set_position_data landmarks_;
  LandmarkMapBoundaries boundaries_{};
  bool explicit_bounds_{false};
  mutable std::vector<bb200_landmark> c_;
};

/// A pose in 3-D as the C ABI takes it: a row-major 3x4 [R | t].  With BELUGA_B200_WITH_SOPHUS it converts from
/// Sophus::SE3d (SE3d::matrix3x4()).
struct SE3d {
  std::array<double, 12> m{1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0};
  SE3d() = default;
  explicit SE3d(const std::array<double, 12>& matrix3x4) : m(matrix3x4) {}
#ifdef BELUGA_B200_WITH_SOPHUS
  SE3d(const Sophus::SE3d& p) {  // NOLINT(google-explicit-constructor)
    const auto r = p.matrix3x4();
    for (int row = 0; row < 3; ++row)
      for (int col = 0; col < 4; ++col) m[4 * row + col] = r(row, col);
  }
#endif
};

/// Same members and defaults as beluga::LandmarkModelParam (sensor/landmark_sensor_model.hpp:44-48).
struct LandmarkModelParam {
  double sigma_range{1.0};
  double sigma_bearing{1.0};
  double random_prob{1e-4};
};

/// Same members and defaults as beluga::BearingModelParam (sensor/bearing_sensor_model.hpp:42-45).
struct BearingModelParam {
  double sigma_bearing{1.0};
  SE3d sensor_pose_in_robot{};
};

/// Measurement token of the landmark and bearing models: the detections as the C ABI takes them.
struct landmark_token {
  std::vector<bb200_landmark_detection> detections;
};

template <class T, class = void>
struct is_landmark_token : std::false_type {};
template <class T>
struct is_landmark_token<T, std::void_t<decltype(std::declval<const T&>().detections)>> : std::true_type {};
template <class T>
constexpr bool is_landmark_token_v = is_landmark_token<T>::value;

/// beluga::LandmarkSensorModel2d<LandmarkMap> (sensor/landmark_sensor_model.hpp:63-172): range and bearing to the nearest
/// landmark of each detection's category.
template <class LandmarkMapT = LandmarkMap>
class LandmarkSensorModel2d {
 public:
  using state_type = SE2d;
  using weight_type = double;
  using measurement_type = std::vector<LandmarkPositionDetection>;
  using map_type = LandmarkMapT;
  using param_type = LandmarkModelParam;

  explicit LandmarkSensorModel2d(const param_type& params, map_type map) : params_{params}, map_{std::move(map)} {}
  void update_map(const map_type& map) { map_ = map; }
  [[nodiscard]] landmark_token operator()(measurement_type&& detections) const {
    landmark_token t;
    for (const auto& d : detections) {
      const auto& p = d.detection_position_in_robot;
      t.detections.push_back(bb200_landmark_detection{p[0], p[1], p[2], d.category});
    }
    return t;
  }
  [[nodiscard]] int attach(bb200_filter* f) const {
    const bb200_landmark_param p{params_.sigma_range, params_.sigma_bearing, params_.random_prob};
    const bb200_landmark_map m = map_.view();
    return bb200_filter_set_landmark_map(f, &p, &m);
  }
  [[nodiscard]] int attach(bb200_sharded_amcl* g) const {
    const bb200_landmark_param p{params_.sigma_range, params_.sigma_bearing, params_.random_prob};
    const bb200_landmark_map m = map_.view();
    return bb200_sharded_amcl_set_landmark_map(g, &p, &m);
  }

 private:
  param_type params_;
  map_type map_;
};

/// beluga::BearingSensorModel2d<LandmarkMap> (sensor/bearing_sensor_model.hpp:59-156): bearing alone, from a sensor at
/// params.sensor_pose_in_robot, to the best-aligned landmark of each detection's category.
template <class LandmarkMapT = LandmarkMap>
class BearingSensorModel2d {
 public:
  using state_type = SE2d;
  using weight_type = double;
  using measurement_type = std::vector<LandmarkBearingDetection>;
  using map_type = LandmarkMapT;
  using param_type = BearingModelParam;

  explicit BearingSensorModel2d(const param_type& params, map_type map) : params_{params}, map_{std::move(map)} {}
  void update_map(const map_type& map) { map_ = map; }
  [[nodiscard]] landmark_token operator()(measurement_type&& detections) const {
    landmark_token t;
    for (const auto& d : detections) {
      const auto& b = d.detection_bearing_in_sensor;
      t.detections.push_back(bb200_landmark_detection{b[0], b[1], b[2], d.category});
    }
    return t;
  }
  [[nodiscard]] int attach(bb200_filter* f) const {
    const bb200_bearing_param p = c_param();
    const bb200_landmark_map m = map_.view();
    return bb200_filter_set_bearing_map(f, &p, &m);
  }
  [[nodiscard]] int attach(bb200_sharded_amcl* g) const {
    const bb200_bearing_param p = c_param();
    const bb200_landmark_map m = map_.view();
    return bb200_sharded_amcl_set_bearing_map(g, &p, &m);
  }

 private:
  [[nodiscard]] bb200_bearing_param c_param() const {
    bb200_bearing_param p{};
    p.sigma_bearing = params_.sigma_bearing;
    for (int k = 0; k < 12; ++k) p.sensor_pose_in_robot[k] = params_.sensor_pose_in_robot.m[k];
    return p;
  }

  param_type params_;
  map_type map_;
};

}  // namespace beluga_b200
