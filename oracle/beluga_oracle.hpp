// TEST INFRASTRUCTURE ONLY -- CPU parity oracle for the MCL update hot path.
//
// This is a dependency-free, scalar C++17 restatement of the reference algorithm
// (Ekumen-OS/beluga @ 947326fe, /root/reference), one function per hot-path row of
// SURVEY.md section 8(a).  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may build, link or execute it.  The product
// (beluga_b200/) never includes anything from this directory.
//
// The reference itself cannot be compiled here (Eigen 3.4.0, Sophus 1.22.10,
// range-v3 0.12.0, oneTBB are absent and there is no network), so there is no
// oracle/_ref.  PINNING: every deterministic function below is checked against the
// reference's own known-answer tests (tests/test_oracle_golden.py cites each
// test file:line).  "Parity unpinned" -- NOT pinned by anything in the reference:
//   (1) resample indices for a seed, (2) diff-drive samples for a seed,
//   (3) systematic resampling (absent from the reference), (4) per-step pose
//   mean/covariance along a trajectory.  For those the oracle of record is the
//   counter-RNG mode ("mode B") defined in this file; the libstdc++ mode ("mode A")
//   follows the reference's <random> arithmetic literally and is compared with
//   mode B statistically, using the reference tests' own tolerances.
//
// All paths below are relative to /root/reference/beluga/include/beluga/.
#pragma once

#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <numeric>
#include <optional>
#include <queue>
#include <random>
#include <stdexcept>
#include <unordered_set>
#include <utility>
#include <vector>

#include "se2.hpp"

namespace oracle {

// ---------------------------------------------------------------------------------------------
// Grids (sensor/data/*.hpp)
// ---------------------------------------------------------------------------------------------

/// Occupancy grid with the ROS trinary value traits
/// (beluga_ros/include/beluga_ros/occupancy_grid.hpp:48-64; test fixture
/// test/beluga/include/beluga/test/static_occupancy_grid.hpp:39-50).
struct OccupancyGrid {
  static constexpr std::int8_t kFree = 0;
  static constexpr std::int8_t kUnknown = -1;
  static constexpr std::int8_t kOccupied = 100;

  int width{0};
  int height{0};
  double resolution{1.0};
  SE2 origin{};
  std::vector<std::int8_t> data;  // row-major, index = yi*width + xi (linear_grid.hpp:73-75)

  [[nodiscard]] std::size_t size() const { return data.size(); }
  [[nodiscard]] static bool is_free(std::int8_t v) { return v == kFree; }
  [[nodiscard]] static bool is_unknown(std::int8_t v) { return v == kUnknown; }
  [[nodiscard]] static bool is_occupied(std::int8_t v) { return v == kOccupied; }

  /// dense_grid.hpp:92-96
  [[nodiscard]] bool contains(int xi, int yi) const { return xi >= 0 && yi >= 0 && xi < width && yi < height; }
  /// linear_grid.hpp:73-75
  [[nodiscard]] std::size_t index_at(int xi, int yi) const {
    return static_cast<std::size_t>(yi) * static_cast<std::size_t>(width) + static_cast<std::size_t>(xi);
  }
  /// occupancy_grid.hpp:101-107 (+ linear_grid.hpp:102-104: index >= size -> nullopt -> not free)
  [[nodiscard]] bool free_at(std::size_t index) const { return index < data.size() && is_free(data[index]); }
  [[nodiscard]] bool free_at(int xi, int yi) const { return free_at(index_at(xi, yi)); }
};

/// regular_grid.hpp:75-78: floor(p * (1/resolution)) cast to int.  The cast is undefined for NaN and outside
/// [-2^31, 2^31); x86-64 gives INT_MIN there, stated here explicitly.  INT_MIN lies outside every grid.
inline int cell_coord_near(double p, double resolution) {
  const double inv_resolution = 1. / resolution;
  const double floored = std::floor(p * inv_resolution);
  return floored >= -0x1p31 && floored < 0x1p31 ? static_cast<int>(floored) : std::numeric_limits<int>::min();
}

/// The largest span, in cells along either axis, for which Ray2d's int Bresenham arithmetic (bresenham.hpp:84-160)
/// cannot overflow: error + dyspan <= 4 * span < 2^31.
constexpr int kMaxRaySpan = (1 << 29) - 1;

/// regular_grid.hpp:87-89: (cell + 0.5) * resolution.
inline double cell_centroid(int cell, double resolution) { return (static_cast<double>(cell) + 0.5) * resolution; }

/// linear_grid.hpp:113-130: right, down(+width), left, up, in that order.
inline void neighborhood4(std::size_t index, std::size_t width, std::size_t height, std::vector<std::size_t>& out) {
  out.clear();
  const std::size_t xi = index % width;
  const std::size_t yi = index / width;
  if (xi < (width - 1)) out.push_back(index + 1);
  if (yi < (height - 1)) out.push_back(index + width);
  if (xi > 0) out.push_back(index - 1);
  if (yi > 0) out.push_back(index - width);
}

/// occupancy_grid.hpp:184-201
inline std::vector<bool> obstacle_edge_mask(const OccupancyGrid& g) {
  std::vector<bool> mask(g.size(), false);
  std::vector<std::size_t> nb;
  for (std::size_t i = 0; i < g.size(); ++i) {
    if (!OccupancyGrid::is_occupied(g.data[i])) continue;
    neighborhood4(i, static_cast<std::size_t>(g.width), static_cast<std::size_t>(g.height), nb);
    bool any_free = false;
    for (const auto n : nb) any_free = any_free || OccupancyGrid::is_free(g.data[n]);
    mask[i] = any_free;
  }
  return mask;
}

/// ValueGrid2<float> (sensor/data/value_grid.hpp:36-69).
struct ValueGrid {
  std::vector<float> data;
  int width{0};
  int height{0};
  double resolution{1.0};

  /// dense_grid.hpp:127-129 -> regular_grid.hpp:75-78 -> dense_grid.hpp:105-107.
  [[nodiscard]] std::optional<float> data_near(double x, double y) const {
    const int xi = cell_coord_near(x, resolution);
    const int yi = cell_coord_near(y, resolution);
    if (!(xi >= 0 && yi >= 0 && xi < width && yi < height)) return std::nullopt;
    return data[static_cast<std::size_t>(yi) * static_cast<std::size_t>(width) + static_cast<std::size_t>(xi)];
  }
};

// ---------------------------------------------------------------------------------------------
// a15: likelihood field construction
// ---------------------------------------------------------------------------------------------

/// algorithm/distance_map.hpp:55-98 -- priority-queue brushfire.  The result depends on the
/// heap pop order among equal keys, so this restatement uses the very same
/// std::priority_queue<IndexPair, vector, compare-on-distance_map> as the reference.
template <class DistanceFunction>
std::vector<float> nearest_obstacle_distance_map(
    const std::vector<bool>& obstacle_mask,
    DistanceFunction&& distance_function,
    std::size_t width,
    std::size_t height,
    float max_distance_value) {
  struct IndexPair {
    std::size_t nearest_obstacle_index;
    std::size_t index;
  };
  std::vector<float> distance_map(obstacle_mask.size(), max_distance_value);
  std::vector<bool> visited(obstacle_mask.size(), false);
  auto compare = [&distance_map](const IndexPair& first, const IndexPair& second) {
    return distance_map[first.index] > distance_map[second.index];
  };
  std::priority_queue<IndexPair, std::vector<IndexPair>, decltype(compare)> queue{compare};
  for (std::size_t index = 0; index < obstacle_mask.size(); ++index) {
    if (obstacle_mask[index]) {
      visited[index] = true;
      distance_map[index] = 0;
      queue.push(IndexPair{index, index});
    }
  }
  std::vector<std::size_t> nb;
  while (!queue.empty()) {
    const auto parent = queue.top();
    queue.pop();
    neighborhood4(parent.index, width, height, nb);
    for (const std::size_t index : nb) {
      if (!visited[index]) {
        visited[index] = true;
        const float distance = distance_function(parent.nearest_obstacle_index, index);
        if (distance < max_distance_value) {
          distance_map[index] = distance;
          queue.push(IndexPair{parent.nearest_obstacle_index, index});
        }
      }
    }
  }
  return distance_map;
}

/// sensor/likelihood_field_model_base.hpp:42-64
struct LikelihoodFieldParam {
  double max_obstacle_distance = 100.0;
  double max_laser_distance = 2.0;
  double z_hit = 0.5;
  double z_random = 0.5;
  double sigma_hit = 0.2;
  bool model_unknown_space = false;
  bool only_obstacle_boundaries = false;
};

/// sensor/likelihood_field_model_base.hpp:130-185
inline ValueGrid make_likelihood_field(const LikelihoodFieldParam& params, const OccupancyGrid& grid) {
  const std::size_t width = static_cast<std::size_t>(grid.width);
  const std::size_t height = static_cast<std::size_t>(grid.height);
  // :131-133 squared distance between cell centroids, computed in double, stored as float.
  const auto squared_distance = [&grid, width](std::size_t first, std::size_t second) {
    const double ax = cell_centroid(static_cast<int>(first % width), grid.resolution);
    const double ay = cell_centroid(static_cast<int>(first / width), grid.resolution);
    const double bx = cell_centroid(static_cast<int>(second % width), grid.resolution);
    const double by = cell_centroid(static_cast<int>(second / width), grid.resolution);
    const double dx = ax - bx;
    const double dy = ay - by;
    return static_cast<float>(dx * dx + dy * dy);
  };
  const double two_squared_sigma = 2 * params.sigma_hit * params.sigma_hit;
  const double pi = 3.14159265358979323846;  // Sophus::Constants<double>::pi()
  const double amplitude = params.z_hit / (params.sigma_hit * std::sqrt(2 * pi));
  const double offset = params.z_random / params.max_laser_distance;
  const auto to_likelihood = [amplitude, two_squared_sigma, offset](double sq) {
    return amplitude * std::exp(-sq / two_squared_sigma) + offset;
  };
  const float squared_max_distance = static_cast<float>(params.max_obstacle_distance * params.max_obstacle_distance);

  std::vector<bool> obstacle(grid.size());
  for (std::size_t i = 0; i < grid.size(); ++i) obstacle[i] = OccupancyGrid::is_occupied(grid.data[i]);
  const std::vector<bool> edge = obstacle_edge_mask(grid);

  std::vector<float> distance_map = nearest_obstacle_distance_map(
      params.only_obstacle_boundaries ? edge : obstacle, squared_distance, width, height, squared_max_distance);

  if (params.model_unknown_space) {  // :158-177
    const double inverse_max_distance = 1 / params.max_laser_distance;
    const double squared_background_distance = -two_squared_sigma * std::log((inverse_max_distance - offset) / amplitude);
    const float mask_value = std::min(squared_max_distance, static_cast<float>(squared_background_distance));
    for (std::size_t i = 0; i < grid.size(); ++i) {
      const bool is_unknown = OccupancyGrid::is_unknown(grid.data[i]);
      const bool effective =
          params.only_obstacle_boundaries ? (is_unknown || (obstacle[i] && !edge[i])) : is_unknown;
      if (effective) distance_map[i] = mask_value;  // actions/overlay.hpp:46-62
    }
  }

  ValueGrid field;
  field.width = grid.width;
  field.height = grid.height;
  field.resolution = grid.resolution;
  field.data.resize(distance_map.size());
  // :179-182 ranges::actions::transform in place on a vector<float>: double result stored as float.
  for (std::size_t i = 0; i < distance_map.size(); ++i) {
    field.data[i] = static_cast<float>(to_likelihood(static_cast<double>(distance_map[i])));
  }
  return field;
}

// ---------------------------------------------------------------------------------------------
// a3 / a3': likelihood field sensor models
// ---------------------------------------------------------------------------------------------

using Points = std::vector<std::pair<double, double>>;

/// libstdc++ std::transform_reduce(first, last, init, plus, f) for random-access iterators:
/// /usr/include/c++/13/numeric:439-462 groups by four -- init += ((f0+f1)+(f2+f3)) -- then a
/// scalar tail.  The reference inherits this order; so does the CUDA kernel.
template <class F>
double transform_reduce_plus(std::size_t n, double init, F&& f) {
  std::size_t i = 0;
  while (n - i >= 4) {
    const double v1 = f(i) + f(i + 1);
    const double v2 = f(i + 2) + f(i + 3);
    const double v3 = v1 + v2;
    init = init + v3;
    i += 4;
  }
  for (; i < n; ++i) init = init + f(i);
  return init;
}

struct LikelihoodFieldModel {
  LikelihoodFieldParam params;
  ValueGrid field;
  SE2 world_to_field;  // grid.origin().inverse() (likelihood_field_model_base.hpp:99)

  LikelihoodFieldModel(const LikelihoodFieldParam& p, const OccupancyGrid& grid)
      : params(p), field(make_likelihood_field(p, grid)), world_to_field(grid.origin.inverse()) {}

  [[nodiscard]] double pz_at(const SE2& transform, double px, double py) const {
    const float unknown_space_occupancy_prob = static_cast<float>(1. / params.max_laser_distance);
    const double x = px * transform.r.c - py * transform.r.s + transform.x;
    const double y = px * transform.r.s + py * transform.r.c + transform.y;
    return static_cast<double>(field.data_near(x, y).value_or(unknown_space_occupancy_prob));
  }

  /// sensor/likelihood_field_model.hpp:69-90: 1.0 + sum pz^3.
  [[nodiscard]] double weight(const SE2& state, const Points& points) const {
    const SE2 transform = world_to_field * state;
    return transform_reduce_plus(points.size(), 1.0, [&](std::size_t i) {
      const double pz = pz_at(transform, points[i].first, points[i].second);
      return pz * pz * pz;
    });
  }

  /// sensor/likelihood_field_prob_model.hpp:69-90: exp(sum log pz).
  [[nodiscard]] double weight_prob(const SE2& state, const Points& points) const {
    const SE2 transform = world_to_field * state;
    return std::exp(transform_reduce_plus(points.size(), 0.0, [&](std::size_t i) {
      return std::log(pz_at(transform, points[i].first, points[i].second));
    }));
  }
};

// ---------------------------------------------------------------------------------------------
// a4: beam model, raycasting, Bresenham
// ---------------------------------------------------------------------------------------------

/// algorithm/raycasting/bresenham.hpp:84-160.  Iterates the cells of a line from p0 to p1
/// (both inclusive).  `modified` selects the supercover variant (:141-157).
struct BresenhamLine {
  int x_, y_, xspan_, yspan_, dxspan_, dyspan_, xstep_, ystep_, step_{0}, prev_error_, error_;
  std::size_t checks_{0};
  bool modified_{false};
  bool reversed_{false};
  int cx, cy;  // current point

  BresenhamLine(int x0, int y0, int x1, int y1, bool modified) : x_(x0), y_(y0), cx(x0), cy(y0) {
    xspan_ = x1 - x0;
    xstep_ = 1;
    if (xspan_ < 0) {
      xspan_ = -xspan_;
      xstep_ = -xstep_;
    }
    yspan_ = y1 - y0;
    ystep_ = 1;
    if (yspan_ < 0) {
      yspan_ = -yspan_;
      ystep_ = -ystep_;
    }
    if (xspan_ < yspan_) {
      std::swap(x_, y_);
      std::swap(xspan_, yspan_);
      std::swap(xstep_, ystep_);
      reversed_ = true;
    }
    dxspan_ = 2 * xspan_;
    dyspan_ = 2 * yspan_;
    error_ = prev_error_ = xspan_;
    modified_ = modified;
  }

  [[nodiscard]] bool done() const { return step_ > xspan_; }  // sentinel, :179

  void step_to(int x, int y) {
    if (reversed_) std::swap(x, y);
    cx = x;
    cy = y;
  }

  void next() {  // operator++, :122-160
    if (checks_ == 0) {
      if (++step_ > xspan_) return;
      x_ += xstep_;
      error_ += dyspan_;
      ++checks_;
      if (error_ > dxspan_) {
        y_ += ystep_;
        error_ -= dxspan_;
        if (modified_) {
          ++checks_;
          ++checks_;
        }
      }
    }
    if (checks_ > 1) {
      if (checks_ > 2) {
        --checks_;
        if (error_ + prev_error_ <= dxspan_) {
          step_to(x_, y_ - ystep_);
          return;
        }
      }
      --checks_;
      if (error_ + prev_error_ >= dxspan_) {
        step_to(x_ - xstep_, y_);
        return;
      }
    }
    --checks_;
    step_to(x_, y_);
    prev_error_ = error_;
  }
};

/// algorithm/raycasting.hpp:44-115
struct Ray2d {
  const OccupancyGrid& grid;
  SE2 source_pose_in_local_frame;
  int source_x, source_y;
  double max_range;
  bool modified{false};

  Ray2d(const OccupancyGrid& g, const SE2& source_pose, double range, bool modified_variant = false)
      : grid(g),
        source_pose_in_local_frame(g.origin.inverse() * source_pose),
        source_x(cell_coord_near(source_pose_in_local_frame.x, g.resolution)),
        source_y(cell_coord_near(source_pose_in_local_frame.y, g.resolution)),
        max_range(range),
        modified(modified_variant) {}

  /// :79-88 far end cell for a bearing, for a source cell inside the grid.  Returns false when the far end is not
  /// finite: the ray is then a miss.  Where the span from the source reaches kMaxRaySpan + 1 cells, the reference's
  /// int arithmetic overflows; the far end is then pulled back, per axis, to kMaxRaySpan cells from the source.
  /// Below that the far end is the reference's cell.
  [[nodiscard]] bool far_end_cell(const SO2& bearing, int& fx, int& fy) const {
    const SO2& r1 = source_pose_in_local_frame.r;
    const Vec2 t2{bearing.c * max_range, bearing.s * max_range};
    const Vec2 rt = r1 * t2;
    const double ex = rt.x + source_pose_in_local_frame.x;
    const double ey = rt.y + source_pose_in_local_frame.y;
    if (!std::isfinite(ex) || !std::isfinite(ey)) return false;
    const double inv_resolution = 1. / grid.resolution;
    const auto span = [](double e, int source) {  // exact: both terms are integers far below 2^53, or the clamp applies
      const double s = std::floor(e) - static_cast<double>(source);
      return static_cast<int>(std::min(std::max(s, -static_cast<double>(kMaxRaySpan)), static_cast<double>(kMaxRaySpan)));
    };
    fx = source_x + span(ex * inv_resolution, source_x);
    fy = source_y + span(ey * inv_resolution, source_y);
    return true;
  }

  /// :97-107.  `visited` (optional) counts the cells inspected (for the algorithmic-bytes figure).
  [[nodiscard]] std::optional<double> cast(const SO2& bearing, std::uint64_t* visited = nullptr) const {
    if (!grid.contains(source_x, source_y)) return std::nullopt;  // the first cell of the line fails cell_is_valid
    int fx = 0, fy = 0;
    if (!far_end_cell(bearing, fx, fy)) return std::nullopt;
    for (BresenhamLine line(source_x, source_y, fx, fy, modified); !line.done(); line.next()) {
      if (!grid.contains(line.cx, line.cy)) break;  // take_while(cell_is_valid), :86-87
      if (visited != nullptr) ++*visited;
      if (!grid.free_at(line.cx, line.cy)) {
        const double sx = cell_centroid(source_x, grid.resolution);
        const double sy = cell_centroid(source_y, grid.resolution);
        const double cxp = cell_centroid(line.cx, grid.resolution);
        const double cyp = cell_centroid(line.cy, grid.resolution);
        const double dx = cxp - sx;
        const double dy = cyp - sy;
        const double distance = std::sqrt(dx * dx + dy * dy);  // Eigen norm()
        return std::min(distance, max_range);
      }
    }
    return std::nullopt;
  }
};

/// sensor/beam_model.hpp:43-58
struct BeamModelParam {
  double z_hit{0.5};
  double z_short{0.5};
  double z_max{0.05};
  double z_rand{0.05};
  double sigma_hit{0.2};
  double lambda_short{0.1};
  double beam_max_range{60};
};

/// sensor/beam_model.hpp:104-150
inline double beam_weight(
    const BeamModelParam& params,
    const OccupancyGrid& grid,
    const SE2& state,
    const Points& points,
    std::uint64_t* visited = nullptr) {
  const Ray2d beam{grid, state, params.beam_max_range};
  const double n = 1. / (std::sqrt(2. * M_PI) * params.sigma_hit);
  return transform_reduce_plus(points.size(), 0.0, [&](std::size_t i) {
    const double px = points[i].first;
    const double py = points[i].second;
    const double z = std::sqrt(px * px + py * py);
    const SO2 beam_bearing = SO2::raw(px / z, py / z);
    const double z_mean = beam.cast(beam_bearing, visited).value_or(params.beam_max_range);
    const double eta_hit = 2. / (std::erf((params.beam_max_range - z_mean) / (std::sqrt(2.) * params.sigma_hit)) -
                                 std::erf(-z_mean / (std::sqrt(2.) * params.sigma_hit)));
    const double d = (z - z_mean) / params.sigma_hit;
    double pz = params.z_hit * eta_hit * n * std::exp(-(d * d) / 2.);
    if (z < z_mean) {
      const double eta_short = 1. / (1. - std::exp(-params.lambda_short * z_mean));
      pz += params.z_short * params.lambda_short * eta_short * std::exp(-params.lambda_short * z);
    }
    if (z < params.beam_max_range) {
      pz += params.z_rand / params.beam_max_range;
    } else {
      pz += params.z_max;
    }
    return pz * pz * pz;
  });
}

// ---------------------------------------------------------------------------------------------
// a2: differential drive motion model
// ---------------------------------------------------------------------------------------------

/// motion/differential_drive_model.hpp:40-68
struct DifferentialDriveParam {
  double rotation_noise_from_rotation{0.0};        // alpha1
  double rotation_noise_from_translation{0.0};     // alpha2
  double translation_noise_from_translation{0.0};  // alpha3
  double translation_noise_from_rotation{0.0};     // alpha4
  double distance_threshold{0.01};
};

/// The six scalars of the three std::normal_distribution param_types (:141-154).
struct DiffDriveSampling {
  double rot1_mean, rot1_std;
  double trans_mean, trans_std;
  double rot2_mean, rot2_std;
};

/// motion/differential_drive_model.hpp:167-173
inline double rotation_variance(const SO2& rotation) {
  static const SO2 kFlippingRotation{3.14159265358979323846};  // Sophus::Constants<double>::pi()
  const SO2 flipped_rotation = rotation * kFlippingRotation;
  const double delta = std::min(std::abs(rotation.log()), std::abs(flipped_rotation.log()));
  return delta * delta;
}

/// motion/differential_drive_model.hpp:129-154 (host part of sampling_fn_2d).
inline DiffDriveSampling diff_drive_sampling(const DifferentialDriveParam& params, const SE2& pose, const SE2& previous_pose) {
  const double tx = pose.x - previous_pose.x;
  const double ty = pose.y - previous_pose.y;
  const double distance = std::sqrt(tx * tx + ty * ty);  // Eigen norm()
  const double distance_variance = distance * distance;
  const SO2& previous_orientation = previous_pose.r;
  const SO2& current_orientation = pose.r;
  const SO2 heading_rotation{std::atan2(ty, tx)};
  const SO2 first_rotation =
      distance > params.distance_threshold ? heading_rotation * previous_orientation.inverse() : SO2{};
  const SO2 second_rotation = current_orientation * previous_orientation.inverse() * first_rotation.inverse();
  DiffDriveSampling out{};
  out.rot1_mean = first_rotation.log();
  out.rot1_std = std::sqrt(
      params.rotation_noise_from_rotation * rotation_variance(first_rotation) +
      params.rotation_noise_from_translation * distance_variance);
  out.trans_mean = distance;
  out.trans_std = std::sqrt(
      params.translation_noise_from_translation * distance_variance +
      params.translation_noise_from_rotation * (rotation_variance(first_rotation) + rotation_variance(second_rotation)));
  out.rot2_mean = second_rotation.log();
  out.rot2_std = std::sqrt(
      params.rotation_noise_from_rotation * rotation_variance(second_rotation) +
      params.rotation_noise_from_translation * distance_variance);
  return out;
}

/// motion/differential_drive_model.hpp:156-163 given the three sampled scalars.
inline SE2 diff_drive_apply(const SE2& state, double rot1, double trans, double rot2) {
  const SO2 first_rotation{rot1};
  const SO2 second_rotation{rot2};
  return state * SE2{first_rotation, 0.0, 0.0} * SE2{second_rotation, trans, 0.0};
}

/// Generic form of what a motion model derives from a control action: three normal distributions
/// and (omnidirectional only) the deterministic first rotation.  model: 0 differential,
/// 1 omnidirectional, 2 stationary.
struct MotionSampling {
  int model{0};
  double mean[3]{0, 0, 0};
  double stddev[3]{0, 0, 0};
  SO2 first_rotation{};
};

/// motion/omnidirectional_drive_model.hpp:36-68
struct OmnidirectionalDriveParam {
  double rotation_noise_from_rotation{0.0};
  double rotation_noise_from_translation{0.0};
  double translation_noise_from_translation{0.0};
  double translation_noise_from_rotation{0.0};
  double strafe_noise_from_translation{0.0};
  double distance_threshold{0.01};
};

inline MotionSampling to_motion_sampling(const DiffDriveSampling& d) {
  MotionSampling m;
  m.model = 0;
  m.mean[0] = d.rot1_mean, m.stddev[0] = d.rot1_std;
  m.mean[1] = d.trans_mean, m.stddev[1] = d.trans_std;
  m.mean[2] = d.rot2_mean, m.stddev[2] = d.rot2_std;
  return m;
}

/// motion/omnidirectional_drive_model.hpp:101-129 (host part).
inline MotionSampling omni_drive_sampling(const OmnidirectionalDriveParam& params, const SE2& pose, const SE2& previous_pose) {
  const double tx = pose.x - previous_pose.x;
  const double ty = pose.y - previous_pose.y;
  const double distance = std::sqrt(tx * tx + ty * ty);
  const double distance_variance = distance * distance;
  const SO2& previous_orientation = previous_pose.r;
  const SO2& current_orientation = pose.r;
  const SO2 rotation = current_orientation * previous_orientation.inverse();
  const SO2 heading_rotation{std::atan2(ty, tx)};
  const SO2 first_rotation = distance > params.distance_threshold ? heading_rotation * previous_orientation.inverse() : SO2{};
  MotionSampling m;
  m.model = 1;
  m.mean[0] = rotation.log();
  m.stddev[0] = std::sqrt(params.rotation_noise_from_rotation * rotation_variance(rotation) + params.rotation_noise_from_translation * distance_variance);
  m.mean[1] = distance;
  m.stddev[1] = std::sqrt(params.translation_noise_from_translation * distance_variance + params.translation_noise_from_rotation * rotation_variance(rotation));
  m.mean[2] = 0.0;
  m.stddev[2] = std::sqrt(params.strafe_noise_from_translation * distance_variance + params.translation_noise_from_rotation * rotation_variance(rotation));
  m.first_rotation = first_rotation;
  return m;
}

/// motion/stationary_model.hpp:52-60: three draws from N(0, 0.02).
inline MotionSampling stationary_sampling() {
  MotionSampling m;
  m.model = 2;
  for (int k = 0; k < 3; ++k) m.stddev[k] = 0.02;
  return m;
}

/// The per-particle composition given the three sampled scalars (in draw order):
/// differential_drive_model.hpp:158-162, omnidirectional_drive_model.hpp:138-144, stationary_model.hpp:56-58.
inline SE2 motion_apply(const MotionSampling& m, const SE2& state, double d0, double d1, double d2) {
  if (m.model == 1) {
    const SO2 second_rotation = SO2{d0} * m.first_rotation.inverse();
    return state * SE2{m.first_rotation, 0.0, 0.0} * SE2{second_rotation, d1, -d2};
  }
  if (m.model == 2) return state * SE2{SO2{d0}, d1, d2};
  return diff_drive_apply(state, d0, d1, d2);
}

// ---------------------------------------------------------------------------------------------
// Counter-mode RNG ("mode B"): Philox4x32-10 (Salmon et al., SC'11; Random123 constants).
// The GPU kernels use the same counters, so draws are reproducible per (seed, step, slot).
// ---------------------------------------------------------------------------------------------

struct Philox4 {
  std::uint32_t v[4];
};

inline Philox4 philox4x32_10(std::uint32_t c0, std::uint32_t c1, std::uint32_t c2, std::uint32_t c3, std::uint32_t k0, std::uint32_t k1) {
  constexpr std::uint32_t kM0 = 0xD2511F53u, kM1 = 0xCD9E8D57u, kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
  for (int round = 0; round < 10; ++round) {
    const std::uint64_t p0 = static_cast<std::uint64_t>(kM0) * c0;
    const std::uint64_t p1 = static_cast<std::uint64_t>(kM1) * c2;
    const std::uint32_t n0 = static_cast<std::uint32_t>(p1 >> 32) ^ c1 ^ k0;
    const std::uint32_t n1 = static_cast<std::uint32_t>(p1);
    const std::uint32_t n2 = static_cast<std::uint32_t>(p0 >> 32) ^ c3 ^ k1;
    const std::uint32_t n3 = static_cast<std::uint32_t>(p0);
    c0 = n0;
    c1 = n1;
    c2 = n2;
    c3 = n3;
    k0 += kW0;
    k1 += kW1;
  }
  return Philox4{{c0, c1, c2, c3}};
}

/// Stream identifiers (4th counter word).
enum Stream : std::uint32_t {
  kStreamInit0 = 0,      // initial normal sample, first Box-Muller pair
  kStreamInit1 = 1,      // initial normal sample, second pair
  kStreamMotion0 = 2,    // propagate: (rot1, trans)
  kStreamMotion1 = 3,    // propagate: (rot2, unused)
  kStreamResample = 4,   // per output slot: .a = Bernoulli(recovery), .b = multinomial position
  kStreamSystematic = 5, // per step (slot 0): .a = systematic offset
  kStreamRandomState = 6 // per injected slot: .a = free cell, .b = yaw
};

struct Draw {
  std::uint64_t a, b;
};

inline Draw counter_draw(std::uint64_t seed, std::uint64_t index, std::uint32_t step, std::uint32_t stream) {
  const Philox4 r = philox4x32_10(
      static_cast<std::uint32_t>(index), static_cast<std::uint32_t>(index >> 32), step, stream,
      static_cast<std::uint32_t>(seed), static_cast<std::uint32_t>(seed >> 32));
  return Draw{(static_cast<std::uint64_t>(r.v[1]) << 32) | r.v[0], (static_cast<std::uint64_t>(r.v[3]) << 32) | r.v[2]};
}

/// 53-bit uniform in the open interval (0, 1).
inline double uniform01(std::uint64_t bits) { return (static_cast<double>(bits >> 11) + 0.5) * 0x1.0p-53; }

inline std::uint64_t mulhi64(std::uint64_t a, std::uint64_t b) {
  return static_cast<std::uint64_t>((static_cast<unsigned __int128>(a) * b) >> 64);
}

/// Box-Muller pair from one draw.
inline void box_muller(const Draw& d, double& z0, double& z1) {
  const double radius = std::sqrt(-2.0 * std::log(uniform01(d.a)));
  const double angle = 6.283185307179586476925 * uniform01(d.b);
  z0 = radius * std::cos(angle);
  z1 = radius * std::sin(angle);
}

/// Mode-B propagate of one particle (global index `index`).
inline SE2 diff_drive_sample_counter(const SE2& state, const DiffDriveSampling& p, std::uint64_t seed, std::uint64_t index, std::uint32_t step) {
  double z0, z1, z2, unused;
  box_muller(counter_draw(seed, index, step, kStreamMotion0), z0, z1);
  box_muller(counter_draw(seed, index, step, kStreamMotion1), z2, unused);
  // libstdc++ normal_distribution: ret * stddev + mean (bits/random.tcc:1843).
  const double rot1 = z0 * p.rot1_std + p.rot1_mean;
  const double trans = z1 * p.trans_std + p.trans_mean;
  const double rot2 = z2 * p.rot2_std + p.rot2_mean;
  return diff_drive_apply(state, rot1, trans, rot2);
}

/// Mode-B propagate for any motion model.
inline SE2 motion_sample_counter(const SE2& state, const MotionSampling& m, std::uint64_t seed, std::uint64_t index, std::uint32_t step) {
  double z0, z1, z2, unused;
  box_muller(counter_draw(seed, index, step, kStreamMotion0), z0, z1);
  box_muller(counter_draw(seed, index, step, kStreamMotion1), z2, unused);
  return motion_apply(m, state, z0 * m.stddev[0] + m.mean[0], z1 * m.stddev[1] + m.mean[1], z2 * m.stddev[2] + m.mean[2]);
}

/// Mode-A propagate for any motion model: one shared std::normal_distribution like the reference's
/// `static thread_local auto distribution` in each model's lambda.
template <class URNG>
void motion_propagate_std(std::vector<SE2>& states, const MotionSampling& m, std::normal_distribution<double>& distribution, URNG& gen) {
  using Param = std::normal_distribution<double>::param_type;
  const Param p0{m.mean[0], m.stddev[0]}, p1{m.mean[1], m.stddev[1]}, p2{m.mean[2], m.stddev[2]};
  for (auto& s : states) {
    const double d0 = distribution(gen, p0);
    const double d1 = distribution(gen, p1);
    const double d2 = distribution(gen, p2);
    s = motion_apply(m, s, d0, d1, d2);
  }
}

/// Mode-A propagate: actions/propagate.hpp:57-79 with the thread-local normal_distribution of
/// differential_drive_model.hpp:157 (one distribution object shared by all particles, so the
/// polar method's cached second value carries over from one particle to the next).
template <class URNG>
void diff_drive_propagate_std(std::vector<SE2>& states, const DiffDriveSampling& p, std::normal_distribution<double>& distribution, URNG& gen) {
  using Param = std::normal_distribution<double>::param_type;
  const Param first{p.rot1_mean, p.rot1_std}, trans{p.trans_mean, p.trans_std}, second{p.rot2_mean, p.rot2_std};
  for (auto& s : states) {
    const double r1 = distribution(gen, first);
    const double t = distribution(gen, trans);
    const double r2 = distribution(gen, second);
    s = diff_drive_apply(s, r1, t, r2);
  }
}

// ---------------------------------------------------------------------------------------------
// a7 / a8 / a9: normalize, recovery probability, ESS, policies
// ---------------------------------------------------------------------------------------------

/// actions/normalize.hpp:54-85
inline double normalize(std::vector<double>& weights) {
  const double factor = std::accumulate(weights.begin(), weights.end(), 0.0);
  if (std::abs(factor - 1.0) < std::numeric_limits<double>::epsilon()) return factor;
  for (auto& w : weights) w = w / factor;
  return factor;
}

/// algorithm/effective_sample_size.hpp:46-59
inline double effective_sample_size(const std::vector<double>& weights) {
  const double total_weight = std::accumulate(weights.begin(), weights.end(), 0.0);
  if (total_weight == 0.0) return 0.0;
  double acc = 0.0;
  for (const double w : weights) {
    const double nw = w / total_weight;
    acc = acc + nw * nw;
  }
  return 1.0 / acc;
}

/// algorithm/exponential_filter.hpp:35-44
struct ExponentialFilter {
  double output{0.};
  double alpha{0.};
  void reset() { output = 0.; }
  double operator()(double input) {
    output += (output == 0.) ? input : alpha * (input - output);
    return output;
  }
};

/// algorithm/thrun_recovery_probability_estimator.hpp:40-94
struct ThrunRecoveryProbabilityEstimator {
  ExponentialFilter slow, fast;
  ThrunRecoveryProbabilityEstimator(double alpha_slow, double alpha_fast) {
    slow.alpha = alpha_slow;
    fast.alpha = alpha_fast;
  }
  void reset() {
    slow.reset();
    fast.reset();
  }
  /// :69-89 given the total weight and the particle count.
  double update(double total_weight, std::size_t size) {
    if (size == 0) {
      reset();
      return 0.0;
    }
    const double average_weight = total_weight / static_cast<double>(size);
    const double fast_average = fast(average_weight);
    const double slow_average = slow(average_weight);
    if (std::abs(slow_average) < std::numeric_limits<double>::epsilon()) return 0.0;
    return std::clamp(1.0 - fast_average / slow_average, 0.0, 1.0);
  }
};

/// policies/on_motion.hpp:63-67,121-133
struct OnMotionPolicy {
  double min_distance, min_angle;
  std::optional<SE2> latest_pose;
  bool operator()(const SE2& pose) {
    if (!latest_pose) {
      latest_pose = pose;
      return true;
    }
    const SE2 delta = latest_pose->inverse() * pose;
    const bool moved = std::sqrt(delta.x * delta.x + delta.y * delta.y) > min_distance || std::abs(delta.r.log()) > min_angle;
    if (moved) latest_pose = pose;
    return moved;
  }
};

/// policies/every_n.hpp:47-50
struct EveryNPolicy {
  std::size_t count{1};
  std::size_t current{0};
  bool operator()() {
    current = (current + 1) % count;
    return current == 0;
  }
};

/// containers/circular_array.hpp:461-480,353-361: RollingWindow<SE2d,2> -- push_front,
/// index clamped to size-1 (extrapolate on read).
struct RollingWindow2 {
  SE2 data[2];
  std::size_t size{0};
  void push(const SE2& v) {
    data[1] = data[0];
    data[0] = v;
    size = std::min<std::size_t>(size + 1, 2);
  }
  [[nodiscard]] const SE2& operator[](std::size_t i) const { return data[std::min(i, size - 1)]; }
};

// ---------------------------------------------------------------------------------------------
// a12: spatial hash + KLD
// ---------------------------------------------------------------------------------------------

/// algorithm/spatial_hash.hpp:45-75 with N=21 bits per axis on 64-bit size_t (:93).
inline std::uint64_t floor_and_fibo_hash(double value, unsigned shift) {
  constexpr std::uint64_t kFib = 11400714819323198485LLU;
  // The reference casts std::floor(value) to int64; for NaN and values outside [-2^63, 2^63) the cast is undefined and
  // x86-64 gives INT64_MIN.  That result is stated here, so that the oracle gives it on every host.
  const double floored = std::floor(value);
  const std::int64_t signed_value = floored >= -0x1p63 && floored < 0x1p63 ? static_cast<std::int64_t>(floored)
                                                                            : std::numeric_limits<std::int64_t>::min();
  const auto unsigned_value = static_cast<std::uint64_t>(signed_value);
  const std::uint64_t h = kFib * unsigned_value;
  if (shift != 0) return (h << shift) | (h >> (64 - shift));
  return h;
}

/// algorithm/spatial_hash.hpp:88-94,190-193
inline std::uint64_t spatial_hash(const SE2& state, double rx, double ry, double rtheta) {
  return floor_and_fibo_hash(state.x / rx, 0) ^ floor_and_fibo_hash(state.y / ry, 21) ^
         floor_and_fibo_hash(state.r.log() / rtheta, 42);
}

/// views/take_while_kld.hpp:73-80
inline std::size_t kld_target_size(std::size_t k, double epsilon, double z) {
  const double two_epsilon = 2 * epsilon;
  if (k <= 2U) return std::numeric_limits<std::size_t>::max();
  const double common = 2. / static_cast<double>(9 * (k - 1));
  const double base = 1. - common + std::sqrt(common) * z;
  const double result = (static_cast<double>(k - 1) / two_epsilon) * base * base * base;
  return static_cast<std::size_t>(std::ceil(result));
}

/// views/take_while_kld.hpp:72-88: stateful predicate.
struct KldCondition {
  std::size_t min;
  double epsilon, z;
  unsigned long long count{0};
  std::unordered_set<std::size_t> buckets;
  bool operator()(std::size_t hash) {
    count++;
    buckets.insert(hash);
    return count <= min || count <= kld_target_size(buckets.size(), epsilon, z);
  }
};

/// take_while_kld over a finite hash sequence (:134-136: take_while(cond) | take(max)):
/// number of elements kept.
inline std::size_t kld_take_count(const std::vector<std::uint64_t>& hashes, std::size_t min, std::size_t max, double epsilon, double z) {
  KldCondition cond{min, epsilon, z, 0, {}};
  std::size_t kept = 0;
  for (const auto h : hashes) {
    if (kept >= max) break;
    if (!cond(h)) break;
    ++kept;
  }
  return kept;
}

// ---------------------------------------------------------------------------------------------
// a14: estimate
// ---------------------------------------------------------------------------------------------

struct Estimate {
  SE2 mean;
  double cov[9];  // row-major 3x3
};

/// algorithm/estimation.hpp:436-475 (mean_fn :42-73, covariance_fn :230-272).
inline Estimate estimate(const std::vector<SE2>& states, const std::vector<double>& weights) {
  const double sum = std::accumulate(weights.begin(), weights.end(), 0.0);
  double m[4] = {0, 0, 0, 0};  // cos, sin, x, y (Sophus data() order)
  for (std::size_t i = 0; i < states.size(); ++i) {
    const double w = weights[i] / sum;
    m[0] += w * states[i].r.c;
    m[1] += w * states[i].r.s;
    m[2] += w * states[i].x;
    m[3] += w * states[i].y;
  }
  Estimate out{};
  for (double& c : out.cov) c = 0.0;
  double acc[4] = {0, 0, 0, 0};
  double squared_weight_sum = 0.0;
  for (std::size_t i = 0; i < states.size(); ++i) {
    const double w = weights[i] / sum;
    const double cx = states[i].x - m[2];
    const double cy = states[i].y - m[3];
    acc[0] += w * cx * cx;
    acc[1] += w * cx * cy;
    acc[2] += w * cy * cx;
    acc[3] += w * cy * cy;
    squared_weight_sum += w * w;
  }
  const double corr = 1.0 - squared_weight_sum;
  out.cov[0] = acc[0] / corr;
  out.cov[1] = acc[1] / corr;
  out.cov[3] = acc[2] / corr;
  out.cov[4] = acc[3] / corr;
  const double norm = std::sqrt(m[0] * m[0] + m[1] * m[1]);
  out.mean.x = m[2];
  out.mean.y = m[3];
  if (norm < std::numeric_limits<double>::epsilon()) {
    out.cov[8] = std::numeric_limits<double>::infinity();
    out.mean.r = SO2{0.0};
  } else {
    out.cov[8] = -2.0 * std::log(norm);
    out.mean.r = SO2::raw(m[0], m[1]);
    out.mean.r.normalize();
  }
  return out;
}

// ---------------------------------------------------------------------------------------------
// a16: initial distributions
// ---------------------------------------------------------------------------------------------

/// Symmetric 3x3 eigen-decomposition by cyclic Jacobi; eigenvalues sorted increasing like
/// Eigen::SelfAdjointEigenSolver (random/multivariate_normal_distribution.hpp:117-125).
/// Eigenvector signs are convention-free in the reference (seeded parity is unpinned).
inline void symmetric_eigen3(const double a_in[9], double eval[3], double evec[9]) {
  double a[3][3], v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) a[i][j] = a_in[3 * i + j];
  for (int sweep = 0; sweep < 64; ++sweep) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    if (off == 0.0) break;
    for (int p = 0; p < 2; ++p) {
      for (int q = p + 1; q < 3; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::abs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0);
        const double s = t * c;
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - s * vkq;
          v[k][q] = s * vkp + c * vkq;
        }
      }
    }
  }
  int order[3] = {0, 1, 2};
  std::sort(order, order + 3, [&](int i, int j) { return a[i][i] < a[j][j]; });
  for (int j = 0; j < 3; ++j) {
    eval[j] = a[order[j]][order[j]];
    for (int i = 0; i < 3; ++i) evec[3 * i + j] = v[i][order[j]];
  }
}

/// random/multivariate_normal_distribution.hpp:109-126: transform = V * sqrt(Lambda).
inline void normal_transform(const double cov[9], double transform[9]) {
  // Eigen isApprox(transpose): ||C - C^T||_F^2 <= prec^2 * min(||C||_F^2, ||C^T||_F^2), prec = 1e-12.
  double diff2 = 0.0, norm2 = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double d = cov[3 * i + j] - cov[3 * j + i];
      diff2 += d * d;
      norm2 += cov[3 * i + j] * cov[3 * i + j];
    }
  if (!(diff2 <= 1e-24 * norm2)) throw std::runtime_error("Invalid covariance matrix, it is not symmetric.");
  double eval[3], evec[9];
  symmetric_eigen3(cov, eval, evec);
  for (double e : eval)
    if (e < 0.0) throw std::runtime_error("Invalid covariance matrix, it has negative eigenvalues.");
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) transform[3 * i + j] = evec[3 * i + j] * std::sqrt(eval[j]);
}

/// random/multivariate_normal_distribution.hpp:96-103 + multivariate_distribution_traits.hpp:102-113:
/// vector (x, y, theta) = mean + T * delta ; SE2(SO2::exp(theta), (x, y)).
inline SE2 normal_state_from_delta(const double mean_xyt[3], const double transform[9], const double delta[3]) {
  double v[3];
  for (int i = 0; i < 3; ++i) {
    v[i] = mean_xyt[i] + (transform[3 * i + 0] * delta[0] + transform[3 * i + 1] * delta[1] + transform[3 * i + 2] * delta[2]);
  }
  return SE2{SO2{v[2]}, v[0], v[1]};
}

/// Mode-B initial sample of particle `index`.
inline SE2 normal_state_counter(const double mean_xyt[3], const double transform[9], std::uint64_t seed, std::uint64_t index) {
  double d[3], unused;
  box_muller(counter_draw(seed, index, 0, kStreamInit0), d[0], d[1]);
  box_muller(counter_draw(seed, index, 0, kStreamInit1), d[2], unused);
  return normal_state_from_delta(mean_xyt, transform, d);
}

/// Free-cell centroids in the global frame (random/multivariate_uniform_distribution.hpp:158-160,
/// occupancy_grid.hpp:150-156,166-172).
inline std::vector<std::uint32_t> free_cells(const OccupancyGrid& g) {
  std::vector<std::uint32_t> out;
  for (std::size_t i = 0; i < g.size(); ++i)
    if (OccupancyGrid::is_free(g.data[i])) out.push_back(static_cast<std::uint32_t>(i));
  return out;
}

inline SE2 free_cell_state(const OccupancyGrid& g, std::uint32_t cell, double yaw) {
  const double lx = cell_centroid(static_cast<int>(cell % static_cast<std::uint32_t>(g.width)), g.resolution);
  const double ly = cell_centroid(static_cast<int>(cell / static_cast<std::uint32_t>(g.width)), g.resolution);
  const Vec2 p = g.origin * Vec2{lx, ly};
  return SE2{SO2{yaw}, p.x, p.y};
}

/// Mode-B random state for output slot `slot` (recovery injection).
inline SE2 random_state_counter(const OccupancyGrid& g, const std::vector<std::uint32_t>& free, std::uint64_t seed, std::uint64_t slot, std::uint32_t step) {
  const Draw d = counter_draw(seed, slot, step, kStreamRandomState);
  const std::uint32_t cell = free[mulhi64(d.a, free.size())];
  // std::uniform_real_distribution(-pi, pi): u * (b - a) + a  (Sophus SO2::sampleUniform)
  const double pi = 3.14159265358979323846;
  const double yaw = uniform01(d.b) * (pi - (-pi)) + (-pi);
  return free_cell_state(g, cell, yaw);
}

// ---------------------------------------------------------------------------------------------
// a10: resampling
// ---------------------------------------------------------------------------------------------

/// Mode-A: std::discrete_distribution exactly as views/sample.hpp:128-135 builds it.
/// (The CDF arithmetic is libstdc++'s: bits/random.tcc:2657-2677.)

/// Mode-B fixed-point CDF.  Weights are scaled by a power of two so that the largest weight
/// lands in [2^(P-1), 2^P) and truncated to integers; P = min(52, 62 - ceil(log2(N))) keeps the
/// total below 2^62.  Integer addition is associative, so any scan order -- sequential here,
/// decoupled look-back on the GPU, any number of ranks -- yields the identical CDF.
inline int ceil_log2(std::uint64_t n) {
  int b = 0;
  while ((std::uint64_t{1} << b) < n) ++b;
  return b;
}

struct FixedPointCdf {
  int exponent{0};                 // q = floor(w * 2^exponent)
  std::vector<std::uint64_t> cdf;  // inclusive
  std::uint64_t total{0};
  bool valid{true};  // false: no weight can be selected and `cdf` is the uniform fallback
};

/// The one rule for which weights can be selected: 0 < w <= DBL_MAX.  Zero, negative, NaN and +-inf weights never are.
inline bool weight_selectable(double w) { return w > 0.0 && w <= std::numeric_limits<double>::max(); }

/// What every particle quantises to when no weight can be selected: a uniform CDF.
constexpr std::uint64_t kUniformFallbackWeight = std::uint64_t{1} << 20;

/// wmax = 0 (no weight can be selected) counts as 2^0: the exponent is then P.
inline int fixed_point_exponent(double wmax, std::uint64_t n_total) {
  const int p = std::min(52, 62 - ceil_log2(n_total));
  int ex = 0;
  if (weight_selectable(wmax)) (void)std::frexp(wmax, &ex);  // wmax = m * 2^ex, m in [0.5, 1)
  return p - ex;
}

inline std::uint64_t quantize_weight(double w, int exponent) {
  if (!weight_selectable(w)) return 0;  // zero, negative, NaN or infinite weights never get selected
  return static_cast<std::uint64_t>(std::ldexp(w, exponent));
}

/// With no weight that can be selected, every particle gets kUniformFallbackWeight and `valid` is false (the reference
/// would divide by zero in normalize.hpp:82).
inline FixedPointCdf fixed_point_cdf(const std::vector<double>& weights, std::uint64_t n_total = 0) {
  FixedPointCdf out;
  double wmax = 0.0;
  for (const double w : weights)
    if (weight_selectable(w) && w > wmax) wmax = w;
  out.valid = wmax > 0.0;
  out.exponent = fixed_point_exponent(wmax, n_total == 0 ? weights.size() : n_total);
  out.cdf.resize(weights.size());
  std::uint64_t acc = 0;
  for (std::size_t i = 0; i < weights.size(); ++i) {
    acc += out.valid ? quantize_weight(weights[i], out.exponent) : kUniformFallbackWeight;
    out.cdf[i] = acc;
  }
  out.total = acc;
  return out;
}

/// Smallest i with cdf[i] > t.
inline std::size_t cdf_search(const std::vector<std::uint64_t>& cdf, std::uint64_t t) {
  return static_cast<std::size_t>(std::upper_bound(cdf.begin(), cdf.end(), t) - cdf.begin());
}

enum class ResampleScheme : int { kMultinomial = 0, kSystematic = 1 };

/// Mode-B position of output slot j in [0, total).
struct CounterResampler {
  std::uint64_t seed;
  std::uint32_t step;
  ResampleScheme scheme;
  std::uint64_t total;
  std::uint64_t m;  // number of output slots the systematic comb is laid over
  std::uint64_t stride{0}, offset{0};

  CounterResampler(std::uint64_t seed_, std::uint32_t step_, ResampleScheme scheme_, std::uint64_t total_, std::uint64_t m_)
      : seed(seed_), step(step_), scheme(scheme_), total(total_), m(m_) {
    if (scheme == ResampleScheme::kSystematic) {
      stride = total / m;
      offset = mulhi64(counter_draw(seed, 0, step, kStreamSystematic).a, stride);
    }
  }
  [[nodiscard]] std::uint64_t position(std::uint64_t j) const {
    if (scheme == ResampleScheme::kSystematic) return offset + j * stride;
    return mulhi64(counter_draw(seed, j, step, kStreamResample).b, total);
  }
  /// Bernoulli(p) for slot j (views/random_intersperse.hpp:93-100 in counter form).  The coin is tossed on every
  /// ADVANCE of the view, so the first element always comes from the input range
  /// (test_random_intersperse.cpp: GuaranteedIntersperseFirstElement).
  [[nodiscard]] bool inject(std::uint64_t j, double p) const {
    return j > 0 && uniform01(counter_draw(seed, j, step, kStreamResample).a) < p;
  }
};

}  // namespace oracle
