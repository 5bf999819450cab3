// beluga_b200::Amcl<DifferentialDriveModel, LandmarkSensorModel2d<LandmarkMap>> and the bearing model (include/beluga_b200/
// models.hpp).  Without a device the Amcl constructor throws Error(BB200_ERR_NO_DEVICE); with one, each step equals a twin
// driven through the C ABI (bb200_filter_set_landmark_map / _set_bearing_map, bb200_amcl_update_landmarks) and the
// estimate follows the robot.  With -DBELUGA_B200_WITH_SOPHUS the camera pose is a Sophus::SE3d.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <vector>

namespace {

using beluga_b200::LandmarkMap;
using beluga_b200::LandmarkMapBoundaries;

LandmarkMap make_map() {
  std::vector<beluga_b200::LandmarkPositionDetection> lms;
  for (int k = 0; k < 12; ++k) lms.push_back({{std::cos(0.5 * k) * 6.0, std::sin(0.5 * k) * 6.0, 0.5 * (k % 3)}, static_cast<std::uint32_t>(k % 4)});
  return LandmarkMap{LandmarkMapBoundaries{{-8.0, -8.0, 0.0}, {8.0, 8.0, 2.0}}, lms};
}

beluga_b200::AmclParams params() {
  beluga_b200::AmclParams p;
  p.update_min_d = 0.0;
  p.update_min_a = 0.0;
  p.min_particles = 2000;
  p.max_particles = 2000;
  p.seed = 3;
  return p;
}

bool same(const bb200_update_result& r, const std::optional<std::pair<beluga_b200::SE2d, std::array<double, 9>>>& e) {
  if (!e) return r.updated == 0;
  for (int k = 0; k < 4; ++k)
    if (r.estimate.mean[k] != e->first.v[k]) return false;
  return true;
}

}  // namespace

int main() {
  using Landmark = beluga_b200::LandmarkSensorModel2d<LandmarkMap>;
  using Bearing = beluga_b200::BearingSensorModel2d<LandmarkMap>;
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  beluga_b200::BearingModelParam bp;
  bp.sigma_bearing = 0.3;
#ifdef BELUGA_B200_WITH_SOPHUS
  bp.sensor_pose_in_robot = Sophus::SE3d{};
#endif
  try {
    beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, Landmark> amcl{beluga_b200::DifferentialDriveModel{motion}, Landmark{{0.5, 0.3, 1e-3}, make_map()},
                                                                          params()};
    beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, Bearing> bearing{beluga_b200::DifferentialDriveModel{motion}, Bearing{bp, make_map()}, params()};
    // The twin through the C ABI.
    const bb200_amcl_param cp = beluga_b200::c_amcl_param(params());
    const bb200_motion_param mp = beluga_b200::DifferentialDriveModel{motion}.c_motion_param();
    bb200_amcl* twin = nullptr;
    if (bb200_amcl_create_with_motion(&cp, &mp, &twin) != BB200_OK) return 1;
    const LandmarkMap map = make_map();
    const bb200_landmark_map m = map.view();
    const bb200_landmark_param lp{0.5, 0.3, 1e-3};
    if (bb200_filter_set_landmark_map(bb200_amcl_filter(twin), &lp, &m) != BB200_OK) return 2;
    const std::array<double, 9> cov{0.3, 0, 0, 0, 0.3, 0, 0, 0, 0.1};
    amcl.initialize(beluga_b200::SE2d{0.0, 0.0, 0.0}, cov);
    bearing.initialize(beluga_b200::SE2d{0.0, 0.0, 0.0}, cov);
    const double mean[3] = {0.0, 0.0, 0.0};  // {x, y, theta}
    if (bb200_amcl_initialize(twin, mean, cov.data()) != BB200_OK) return 3;
    for (int step = 0; step < 5; ++step) {
      const beluga_b200::SE2d odom{0.0, 0.2 * step, 0.0};
      std::vector<beluga_b200::LandmarkPositionDetection> dets{{{6.0 - 0.2 * step, 0.0, 0.0}, 0}, {{std::cos(0.5) * 6.0 - 0.2 * step, std::sin(0.5) * 6.0, 0.5}, 1}};
      std::vector<bb200_landmark_detection> cdets;
      for (const auto& d : dets) cdets.push_back({d.detection_position_in_robot[0], d.detection_position_in_robot[1], d.detection_position_in_robot[2], d.category});
      const auto e = amcl.update(odom, dets);
      bb200_update_result r{};
      if (bb200_amcl_update_landmarks(twin, odom.data(), cdets.data(), cdets.size(), &r) != BB200_OK) return 4;
      if (!e || !same(r, e)) {
        std::printf("step %d differs from the C ABI twin\n", step);
        return 5;
      }
      std::vector<beluga_b200::LandmarkBearingDetection> bdets{{{0.0, 0.0, 1.0}, 0}};
      if (!bearing.update(odom, bdets)) return 6;
    }
    bb200_amcl_destroy(twin);
  } catch (const beluga_b200::Error& e) {
    if (e.status() == BB200_ERR_NO_DEVICE) {
      std::printf("LANDMARK_ADAPTOR_NO_DEVICE\n");
      return 0;
    }
    std::printf("error %d: %s\n", e.status(), e.what());
    return 7;
  }
  std::printf("LANDMARK_ADAPTOR_OK\n");
  return 0;
}
