// beluga_b200::ShardedAmcl<DifferentialDriveModel, LandmarkSensorModel2d<LandmarkMap>> and the bearing model (include/
// beluga_b200/amcl.hpp, models.hpp).  Without a device the constructor throws Error(BB200_ERR_NO_DEVICE); with one, a filter
// of shards on device 0 follows a beluga_b200::Amcl with the same parameters and seed bit for bit, from a Gaussian and from
// the map's box, and the same models attach again through update_map.  With -DBELUGA_B200_WITH_SOPHUS the camera pose is a
// Sophus::SE3d.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {

using beluga_b200::LandmarkMap;
using beluga_b200::LandmarkMapBoundaries;
using beluga_b200::SE2d;

LandmarkMap make_map(double scale) {
  std::vector<beluga_b200::LandmarkPositionDetection> lms;
  for (int k = 0; k < 12; ++k)
    lms.push_back({{std::cos(0.5 * k) * scale, std::sin(0.5 * k) * scale, 0.5 * (k % 3)}, static_cast<std::uint32_t>(k % 4)});
  return LandmarkMap{LandmarkMapBoundaries{{-8.0, -8.0, 0.0}, {8.0, 8.0, 2.0}}, lms};
}

beluga_b200::AmclParams params() {
  beluga_b200::AmclParams p;
  p.update_min_d = 0.0;
  p.update_min_a = 0.0;
  p.min_particles = 2400;
  p.max_particles = 2400;
  p.resample_scheme = BB200_RESAMPLE_SYSTEMATIC;
  p.seed = 3;
  return p;
}

bool same_bytes(const void* a, const void* b, std::size_t n) { return std::memcmp(a, b, n) == 0; }

template <class A, class S>
bool same_particles(const A& single, const S& sharded) {
  const auto p = single.particles(), q = sharded.particles();
  return p.size() == q.size() && same_bytes(p.states.data(), q.states.data(), p.size() * sizeof(SE2d)) &&
         same_bytes(p.weights.data(), q.weights.data(), p.size() * sizeof(double));
}

/// Five steps of both filters with the detections of `detect(step)`, then the moved map and two more: 0 when every step
/// equals, otherwise the failing step + 1.
template <class Model, class Detect>
int follow(const Model& model, const LandmarkMap& moved, const std::vector<int>& devices, bool from_map, Detect detect) {
  const beluga_b200::DifferentialDriveModel motion{beluga_b200::DifferentialDriveModelParam{0.1, 0.05, 0.1, 0.05}};
  beluga_b200::ShardedAmcl sharded(motion, model, params(), devices);
  beluga_b200::Amcl single(motion, model, params());
  if (from_map) {
    sharded.initialize_from_map();
    single.initialize_from_map();
  } else {
    const beluga_b200::Matrix3d cov{0.3, 0, 0, 0, 0.3, 0, 0, 0, 0.1};
    sharded.initialize(SE2d{0.0, 0.0, 0.0}, cov);
    single.initialize(SE2d{0.0, 0.0, 0.0}, cov);
  }
  if (!same_particles(single, sharded)) return 100;
  for (int step = 0; step < 7; ++step) {
    if (step == 5) {
      sharded.update_map(moved);
      single.update_map(moved);
    }
    const SE2d odom{0.05 * step, 0.2 * step, 0.0};
    const auto a = single.update(odom, detect(step));
    const auto b = sharded.update(odom, detect(step));
    if (!a || !b || !same_particles(single, sharded)) return step + 1;
  }
  return 0;
}

}  // namespace

int main() {
  using Landmark = beluga_b200::LandmarkSensorModel2d<LandmarkMap>;
  using Bearing = beluga_b200::BearingSensorModel2d<LandmarkMap>;
  beluga_b200::BearingModelParam bp;
  bp.sigma_bearing = 0.3;
  bp.sensor_pose_in_robot = beluga_b200::SE3d{{0.0, 0.0, 1.0, 0.2, -1.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.5}};  // a camera along x
#ifdef BELUGA_B200_WITH_SOPHUS
  bp.sensor_pose_in_robot = Sophus::SE3d{};
#endif
  auto positions = [](int step) {
    return std::vector<beluga_b200::LandmarkPositionDetection>{{{6.0 - 0.2 * step, 0.0, 0.0}, 0},
                                                               {{std::cos(0.5) * 6.0 - 0.2 * step, std::sin(0.5) * 6.0, 0.5}, 1},
                                                               {{1.0, 1.0, 0.0}, 9}};  // a category the map lacks
  };
  auto bearings = [](int step) {
    return std::vector<beluga_b200::LandmarkBearingDetection>{{{0.0, 0.1 * step, 1.0}, 0}, {{0.5, 0.0, 1.0}, 2}};
  };
  try {
    const Landmark landmark{{0.5, 0.3, 1e-3}, make_map(6.0)};
    const Bearing bearing{bp, make_map(6.0)};
    const LandmarkMap moved = make_map(5.0);
    const std::vector<std::vector<int>> layouts{{0, 0}, {0, 0, 0, 0}};
    for (const auto& devices : layouts)
      for (const bool from_map : {false, true}) {
        if (const int st = follow(landmark, moved, devices, from_map, positions)) {
          std::printf("landmark model, %zu shards, from_map %d: step %d differs from the single filter\n", devices.size(), from_map, st);
          return 1;
        }
        if (const int st = follow(bearing, moved, devices, from_map, bearings)) {
          std::printf("bearing model, %zu shards, from_map %d: step %d differs from the single filter\n", devices.size(), from_map, st);
          return 2;
        }
      }
  } catch (const beluga_b200::Error& e) {
    if (e.status() == BB200_ERR_NO_DEVICE) {
      std::printf("SHARDED_LANDMARK_ADAPTOR_NO_DEVICE\n");
      return 0;
    }
    std::printf("error %d: %s\n", e.status(), e.what());
    return 3;
  }
  std::printf("SHARDED_LANDMARK_ADAPTOR_OK\n");
  return 0;
}
