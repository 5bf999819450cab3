// beluga_b200::AmclBatch with landmark maps (set_landmark_map / add_bearing_map) and landmark_token measurements.  Without
// a device the constructor throws Error(BB200_ERR_NO_DEVICE); with one, a landmark member and a bearing member take a few
// steps through update and update_clustered next to beluga_b200::Amcl<..., LandmarkSensorModel2d> and
// <..., BearingSensorModel2d> twins, and every member's estimate and particles equal its twin's byte for byte.  With
// -DBELUGA_B200_WITH_SOPHUS the camera pose is a Sophus::SE3d.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <optional>
#include <vector>

namespace {

using beluga_b200::LandmarkMap;

LandmarkMap make_map() {
  std::vector<beluga_b200::LandmarkPositionDetection> lms;
  for (int k = 0; k < 12; ++k) lms.push_back({{std::cos(0.5 * k) * 6.0, std::sin(0.5 * k) * 6.0, 0.5 * (k % 3)}, static_cast<std::uint32_t>(k % 4)});
  return LandmarkMap{beluga_b200::LandmarkMapBoundaries{{-8.0, -8.0, 0.0}, {8.0, 8.0, 2.0}}, lms};
}

}  // namespace

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::SE2d;
  using Model = beluga_b200::DifferentialDriveModel;
  using Landmark = beluga_b200::LandmarkSensorModel2d<LandmarkMap>;
  using Bearing = beluga_b200::BearingSensorModel2d<LandmarkMap>;
  std::vector<beluga_b200::AmclParams> params(2);
  for (std::size_t m = 0; m < params.size(); ++m) {
    params[m].update_min_d = params[m].update_min_a = 0.0;
    params[m].min_particles = params[m].max_particles = 1500 + 500 * m;
    params[m].seed = 40 + m;
  }
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  const std::vector<bb200_motion_param> motions(2, Model(motion).c_motion_param());
  const beluga_b200::LandmarkModelParam lp{0.5, 0.3, 1e-3};
  beluga_b200::BearingModelParam bp;
  bp.sigma_bearing = 0.3;
#ifdef BELUGA_B200_WITH_SOPHUS
  bp.sensor_pose_in_robot = Sophus::SE3d{};
#endif
  try {
    AmclBatch batch(motions, params);
    batch.set_landmark_map(lp, make_map());
    batch.update_map(1, batch.add_bearing_map(bp, make_map()));
    const Landmark landmark_model{lp, make_map()};
    const Bearing bearing_model{bp, make_map()};
    beluga_b200::Amcl<Model, Landmark> a{Model(motion), Landmark{lp, make_map()}, params[0]};
    beluga_b200::Amcl<Model, Bearing> b{Model(motion), Bearing{bp, make_map()}, params[1]};
    const beluga_b200::Matrix3d cov = {0.3, 0, 0, 0, 0.3, 0, 0, 0, 0.1};
    const SE2d start(0.0, 0.0, 0.0);
    for (std::size_t m = 0; m < batch.size(); ++m) batch.initialize(m, start, cov);
    a.initialize(start, cov);
    b.initialize(start, cov);
    auto same = [](const std::optional<AmclBatch::estimation_type>& x, const std::optional<AmclBatch::estimation_type>& y) {
      if (!x || !y) return !x && !y;
      return std::memcmp(x->first.data(), y->first.data(), 4 * sizeof(double)) == 0 && std::memcmp(x->second.data(), y->second.data(), 9 * sizeof(double)) == 0;
    };
    auto same_particles = [](const beluga_b200::ParticleSet& x, const beluga_b200::ParticleSet& y) {
      return x.size() == y.size() && std::memcmp(x.states.data(), y.states.data(), x.size() * sizeof(SE2d)) == 0 &&
             std::memcmp(x.weights.data(), y.weights.data(), x.size() * sizeof(double)) == 0;
    };
    for (int step = 0; step < 4; ++step) {
      const SE2d odom(0.0, 0.2 * step, 0.0);
      std::vector<beluga_b200::LandmarkPositionDetection> dets{{{6.0 - 0.2 * step, 0.0, 0.0}, 0}, {{std::cos(0.5) * 6.0 - 0.2 * step, std::sin(0.5) * 6.0, 0.5}, 1}};
      std::vector<beluga_b200::LandmarkBearingDetection> bdets{{{0.0, 0.0, 1.0}, 0}, {{0.3, 0.1, 1.0}, 1}};
      std::vector<AmclBatch::Measurement> in;
      in.emplace_back(landmark_model(std::vector<beluga_b200::LandmarkPositionDetection>(dets)));
      in.emplace_back(bearing_model(std::vector<beluga_b200::LandmarkBearingDetection>(bdets)));
      const auto out = step % 2 == 0 ? batch.update({odom, odom}, in) : batch.update_clustered({odom, odom}, in);
      const auto ea = a.update(odom, dets);
      const auto eb = b.update(odom, bdets);
      if (step % 2 == 0 && (!same(out[0], ea) || !same(out[1], eb))) return 1;
      if (!out[0] || !out[1]) return 2;
      if (!same_particles(batch.particles(0), a.particles()) || !same_particles(batch.particles(1), b.particles())) return 3;
    }
    std::printf("BATCH_LANDMARK_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 4;
    }
    std::printf("BATCH_LANDMARK_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
