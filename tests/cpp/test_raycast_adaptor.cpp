// Amcl::cast_rays, AmclBatch::cast_rays and beluga_b200::scan_bearings through the C ABI.  Without a device the Amcl
// constructor throws Error(BB200_ERR_NO_DEVICE); with one, the reference's Ray2d known answers (test_raycasting.cpp:31-131)
// come back through a beam-model Amcl, a likelihood-field Amcl and a batch, as Ray2d::cast returns them (std::nullopt for
// a miss).
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <optional>
#include <vector>

namespace {

constexpr double kPi = 3.14159265358979323846;

struct Case {
  beluga_b200::SE2d pose;
  double max_range;
  double bearing;
  std::optional<double> expected;
};

beluga_b200::Bearing bearing_of(double theta) { return {std::cos(theta), std::sin(theta)}; }

}  // namespace

int main() {
  using beluga_b200::SE2d;
  std::vector<int8_t> cells(25, 0);
  cells[2 * 5 + 2] = 100;
  const beluga_b200::OccupancyGrid map(cells, 5, 0.5);
  const std::vector<Case> cases = {{SE2d(0.0, 0.5, 0.0), 5.0, 0.0, std::nullopt},          {SE2d(0.0, 0.0, 1.0), 5.0, 0.0, 1.0},
                                   {SE2d(0.0, 0.0, 1.0), 5.0, kPi / 2, std::nullopt},      {SE2d(0.0, 1.0, 1.0), 5.0, kPi / 2, 0.0},
                                   {SE2d(kPi / 2, 0.0, 0.0), 1.0, 0.0, std::nullopt},      {SE2d(0.0, 1.0, 0.0), 5.0, kPi / 2, 1.0},
                                   {SE2d(0.0, 0.0, 0.0), 5.0, kPi / 4, std::sqrt(2.0)}};
  // scan_bearings: take_evenly's directions of a 360-reading scan, 60 kept
  const std::vector<beluga_b200::Bearing> scan = beluga_b200::scan_bearings(static_cast<float>(-kPi), static_cast<float>(2 * kPi / 360), 360, 60);
  if (scan.size() != 60 || std::abs(scan[0][0] + 1.0) > 1e-6) return 1;
  try {
    beluga_b200::AmclParams params;
    params.min_particles = params.max_particles = 100;
    const beluga_b200::DifferentialDriveModel motion{beluga_b200::DifferentialDriveModelParam{}};
    beluga_b200::Amcl beam(motion, beluga_b200::BeamSensorModel<>{beluga_b200::BeamModelParam{}, map}, params);
    beluga_b200::Amcl field(motion, beluga_b200::LikelihoodFieldModel<>{beluga_b200::LikelihoodFieldModelParam{}, map}, params);
    beluga_b200::AmclBatch batch({motion.c_motion_param()}, {params});
    const beluga_b200::GridSnapshot snapshot{map};
    const bb200_beam_param c_beam{0.5, 0.5, 0.05, 0.05, 0.2, 0.1, 60.0};
    batch.set_beam_map(c_beam, snapshot.view());
    for (const Case& c : cases) {
      const std::vector<SE2d> poses{c.pose};
      const std::vector<beluga_b200::Bearing> bearings{bearing_of(c.bearing)};
      const auto a = beam.cast_rays(poses, bearings, c.max_range);
      const auto b = field.cast_rays(poses, bearings, c.max_range);
      const auto k = batch.cast_rays({poses}, {bearings}, {c.max_range});
      if (a.size() != 1 || b.size() != 1 || !k[0] || k[0]->size() != 1) return 2;
      if (a[0] != c.expected || b[0] != c.expected || (*k[0])[0] != c.expected) {
        std::printf("pose (%g, %g) bearing %g: got %g / %g / %g\n", c.pose.x(), c.pose.y(), c.bearing, a[0].value_or(-1), b[0].value_or(-1),
                    (*k[0])[0].value_or(-1));
        return 3;
      }
    }
    // every pose against every bearing, pose major
    std::vector<SE2d> poses;
    std::vector<beluga_b200::Bearing> bearings;
    for (const Case& c : cases) {
      poses.push_back(c.pose);
      bearings.push_back(bearing_of(c.bearing));
    }
    const auto all = beam.cast_rays(poses, bearings, 5.0);
    if (all.size() != poses.size() * bearings.size()) return 4;
    for (std::size_t i = 0; i < poses.size(); ++i) {
      const auto one = beam.cast_rays({poses[i]}, bearings, 5.0);
      for (std::size_t j = 0; j < bearings.size(); ++j)
        if (all[i * bearings.size() + j] != one[j]) return 5;
    }
    std::printf("RAYCAST_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 7;
    }
    std::printf("RAYCAST_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
