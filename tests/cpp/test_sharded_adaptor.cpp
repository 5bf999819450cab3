// beluga_b200::ShardedAmcl through the C ABI.  Without a device the constructor throws Error(BB200_ERR_NO_DEVICE); with one,
// a filter of two shards on device 0 follows an Amcl with the same parameters bit for bit through updates with points, a
// laser scan and a point cloud, and its histogram, pose samples and ray casts equal the Amcl's filter calls.
#include <beluga_b200/amcl.hpp>

#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <optional>
#include <vector>

namespace {

constexpr double kPi = 3.14159265358979323846;

bool same_bytes(const void* a, const void* b, std::size_t n) { return std::memcmp(a, b, n) == 0; }

template <class A, class S>
bool same_particles(const A& single, const S& sharded) {
  const auto p = single.particles(), q = sharded.particles();
  return p.size() == q.size() && same_bytes(p.states.data(), q.states.data(), p.size() * sizeof(beluga_b200::SE2d)) &&
         same_bytes(p.weights.data(), q.weights.data(), p.size() * sizeof(double));
}

}  // namespace

int main() {
  using beluga_b200::SE2d;
  // a 40 x 40 room of 0.1 m cells with walls on its border and one pillar
  const std::size_t w = 40;
  std::vector<int8_t> cells(w * w, 0);
  for (std::size_t i = 0; i < w; ++i) cells[i] = cells[(w - 1) * w + i] = cells[i * w] = cells[i * w + w - 1] = 100;
  cells[20 * w + 20] = 100;
  const beluga_b200::OccupancyGrid map(cells, w, 0.1);
  beluga_b200::AmclParams params;
  params.min_particles = params.max_particles = 2000;
  params.resample_scheme = BB200_RESAMPLE_MULTINOMIAL;
  params.seed = 7;
  const beluga_b200::DifferentialDriveModel motion{beluga_b200::DifferentialDriveModelParam{}};
  const beluga_b200::LikelihoodFieldModel<> sensor{beluga_b200::LikelihoodFieldModelParam{}, map};
  try {
    beluga_b200::ShardedAmcl sharded(motion, sensor, params, {0, 0});
    beluga_b200::Amcl single(motion, sensor, params);
    beluga_b200::Matrix3d cov{};
    cov[0] = cov[4] = 0.05;
    cov[8] = 0.1;
    sharded.initialize(SE2d(0.0, 2.0, 2.0), cov);
    single.initialize(SE2d(0.0, 2.0, 2.0), cov);
    if (!same_particles(single, sharded)) return 1;

    // points, then a laser scan, then a point cloud
    std::vector<std::pair<double, double>> points;
    for (int k = 0; k < 36; ++k) points.emplace_back(1.5 * std::cos(k * kPi / 18), 1.5 * std::sin(k * kPi / 18));
    const auto a = single.update(SE2d(0.0, 0.3, 0.0), points);
    const auto b = sharded.update(SE2d(0.0, 0.3, 0.0), points);
    if (!a || !b || !same_particles(single, sharded)) return 2;

    std::vector<float> ranges(90, 1.5F);
    ranges[3] = NAN;
    const beluga_b200::LaserScanView scan{ranges.data(), ranges.size(), static_cast<float>(-kPi), static_cast<float>(2 * kPi / 90), 0.1, 3.0, 30, nullptr};
    const bb200_laser_scan c_scan = scan.c_view();
    bb200_update_result r{};
    if (bb200_amcl_update_scan(single.handle(), SE2d(0.0, 0.6, 0.0).data(), &c_scan, &r) != BB200_OK) return 3;
    if (!sharded.update(SE2d(0.0, 0.6, 0.0), scan) || !same_particles(single, sharded)) return 4;

    std::vector<float> xyz;
    for (int k = 0; k < 50; ++k) {
      xyz.push_back(static_cast<float>(1.2 * std::cos(k * kPi / 25)));
      xyz.push_back(static_cast<float>(1.2 * std::sin(k * kPi / 25)));
      xyz.push_back(0.2F);
    }
    const beluga_b200::PointCloudView cloud{xyz.data(), 50, 3 * sizeof(float), 0, BB200_POINT_FLOAT32, nullptr};
    if (!single.update(SE2d(0.0, 0.9, 0.0), cloud) || !sharded.update(SE2d(0.0, 0.9, 0.0), cloud) || !same_particles(single, sharded)) return 5;

    // an unusable cloud is refused with the standalone call's status and changes nothing
    const beluga_b200::PointCloudView bad{xyz.data(), 50, 4, 0, BB200_POINT_FLOAT32, nullptr};
    const auto before = sharded.particles();
    try {
      (void)sharded.update(SE2d(0.0, 1.2, 0.0), bad);
      return 6;
    } catch (const beluga_b200::Error& e) {
      if (e.status() != BB200_ERR_INVALID_ARGUMENT) return 7;
    }
    if (!same_bytes(before.states.data(), sharded.particles().states.data(), before.size() * sizeof(SE2d))) return 8;

    // histogram, samples and rays against the standalone filter's calls
    bb200_filter* f = bb200_amcl_filter(single.handle());
    const auto histogram = sharded.particle_histogram(0.05, 0.1);
    std::uint64_t n_bins = 0;
    double top = 0.0;
    if (bb200_filter_particle_histogram(f, 0.05, 0.1, nullptr, 0, &n_bins, &top) != BB200_OK) return 9;
    std::vector<bb200_cluster_cell> bins(n_bins);
    if (bb200_filter_particle_histogram(f, 0.05, 0.1, bins.data(), n_bins, &n_bins, &top) != BB200_OK) return 10;
    if (histogram.first.size() != n_bins || histogram.second != top) return 11;
    for (std::size_t k = 0; k < n_bins; ++k)
      if (histogram.first[k].hash != bins[k].hash || histogram.first[k].count != bins[k].count || histogram.first[k].first_index != bins[k].first_index)
        return 12;

    const auto samples = sharded.sample_states(777, 0xFFFFFFF0u);
    std::vector<double> expected(4 * 777);
    if (bb200_filter_sample_states(f, 777, 0xFFFFFFF0u, expected.data()) != BB200_OK) return 13;
    if (samples.size() != 777 || !same_bytes(samples.data(), expected.data(), expected.size() * sizeof(double))) return 14;

    const std::vector<SE2d> poses{SE2d(0.0, 2.0, 2.0), SE2d(kPi / 3, 1.0, 3.0), SE2d(0.0, -5.0, 1.0)};
    const std::vector<beluga_b200::Bearing> bearings = beluga_b200::scan_bearings(static_cast<float>(-kPi), static_cast<float>(2 * kPi / 64), 64);
    if (sharded.cast_rays(poses, bearings, 3.0) != single.cast_rays(poses, bearings, 3.0)) return 15;

    const auto cs = sharded.cluster_estimate();
    if (!std::isfinite(cs.first.x()) || !same_particles(single, sharded)) return 16;
    std::printf("SHARDED_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 20;
    }
    std::printf("SHARDED_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
