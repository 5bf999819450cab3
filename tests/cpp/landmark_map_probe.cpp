// Host-only probe of prepare_landmark_map (csrc/reweight_landmark.cu), the argument checks behind
// bb200_filter_set_landmark_map / _set_bearing_map: it runs on the host before anything reaches a device, so it is
// checked here without one (tests/test_landmark_cpu.py).  Prints one status per case, then the box of a valid map.
#include <cmath>
#include <cstdio>
#include <limits>
#include <string>

#include "device_map.hpp"

using namespace bb200;

int main() {
  const bb200_landmark lms[2] = {{1.0, -2.0, 0.5, 0}, {-3.0, 4.0, 0.0, 1}};
  const bb200_landmark_map map{lms, 2, nullptr, nullptr};
  const double lo[3] = {-1.0, -1.0, 0.0}, hi[3] = {1.0, 1.0, 0.0};
  const double nan = std::numeric_limits<double>::quiet_NaN();
  const bb200_landmark_param landmark[] = {{1.0, 1.0, 0.1}, {0.0, 1.0, 0.1}, {1.0, -1.0, 0.1}, {nan, 1.0, 0.1}, {1.0, INFINITY, 0.1},
                                           {1.0, 1.0, -0.1}, {1.0, 1.0, 1.5}, {1.0, 1.0, nan}};
  MapTables t;
  std::string error;
  for (const auto& p : landmark) std::printf("landmark %d\n", prepare_landmark_map(&p, nullptr, map, &t, &error));
  bb200_bearing_param b{1.0, {1, 0, 0, 0.2, 0, 1, 0, 0, 0, 0, 1, 0.5}};
  std::printf("bearing %d\n", prepare_landmark_map(nullptr, &b, map, &t, &error));
  bb200_bearing_param bad = b;
  bad.sensor_pose_in_robot[10] = 1.0 + 1e-6;  // not orthonormal
  std::printf("bearing %d\n", prepare_landmark_map(nullptr, &bad, map, &t, &error));
  bad = b;
  bad.sensor_pose_in_robot[10] = -1.0;  // a reflection
  std::printf("bearing %d\n", prepare_landmark_map(nullptr, &bad, map, &t, &error));
  bad = b;
  bad.sigma_bearing = 0.0;
  std::printf("bearing %d\n", prepare_landmark_map(nullptr, &bad, map, &t, &error));
  const bb200_landmark_map null_landmarks{nullptr, 2, nullptr, nullptr};
  std::printf("map %d\n", prepare_landmark_map(&landmark[0], nullptr, null_landmarks, &t, &error));
  const bb200_landmark_map half_bounds{lms, 2, lo, nullptr};
  std::printf("map %d\n", prepare_landmark_map(&landmark[0], nullptr, half_bounds, &t, &error));
  const bb200_landmark_map bounded{lms, 2, lo, hi};
  std::printf("map %d\n", prepare_landmark_map(&landmark[0], nullptr, bounded, &t, &error));
  std::printf("box %g %g %g %g %d\n", t.box[0], t.box[1], t.box[2], t.box[3], t.box_valid ? 1 : 0);
  prepare_landmark_map(&landmark[0], nullptr, map, &t, &error);
  std::printf("box %g %g %g %g %d\n", t.box[0], t.box[1], t.box[2], t.box[3], t.box_valid ? 1 : 0);
  const bb200_landmark_map empty{nullptr, 0, nullptr, nullptr};
  prepare_landmark_map(&landmark[0], nullptr, empty, &t, &error);
  std::printf("box - - - - %d\n", t.box_valid ? 1 : 0);
  return 0;
}
