// AmclBatch::update with laser scans, point clouds and points through the C ABI.  Without a device the constructor throws
// Error(BB200_ERR_NO_DEVICE); with one, three members (a scan, a cloud, points) step twice in one call per step, and each
// member's estimate equals, bit for bit, that of a second batch stepped with the points the host conversions return.  The
// all-scans and all-clouds overloads and the refusal of an unusable cloud are exercised too.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {

std::vector<std::pair<double, double>> scan_points(const beluga_b200::LaserScanView& scan) {
  const bb200_laser_scan c = scan.c_view();
  std::vector<std::pair<double, double>> out(scan.size + 1);
  std::uint64_t n = 0;
  if (bb200_scan_to_points(&c, &out.front().first, out.size(), &n) != BB200_OK) throw beluga_b200::Error(BB200_ERR_STATE, "scan_to_points");
  out.resize(n);
  return out;
}

bool same(const std::optional<beluga_b200::AmclBatch::estimation_type>& a, const std::optional<beluga_b200::AmclBatch::estimation_type>& b) {
  if (a.has_value() != b.has_value()) return false;
  if (!a) return true;
  return std::memcmp(a->first.data(), b->first.data(), 4 * sizeof(double)) == 0 && std::memcmp(&a->second, &b->second, sizeof(a->second)) == 0;
}

}  // namespace

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  std::vector<AmclParams> params(3);
  for (std::size_t m = 0; m < params.size(); ++m) {
    params[m].min_particles = params[m].max_particles = 500 + 700 * m;
    params[m].seed = 40 + m;
  }
  const bb200_motion_param diff = beluga_b200::DifferentialDriveModel(beluga_b200::DifferentialDriveModelParam{0.1, 0.05, 0.1, 0.05}).c_motion_param();
  const std::vector<bb200_motion_param> motions(3, diff);
  try {
    AmclBatch batch(motions, params);
    AmclBatch twin(motions, params);
    std::vector<int8_t> cells(100 * 100, 0);  // a 100 x 100 free map with a wall on every side, 5 cm cells
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const bb200_occupancy_grid grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}};
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    for (AmclBatch* b : {&batch, &twin}) {
      b->set_likelihood_field_map(bb200_likelihood_field_param{2.0, 100.0, 0.5, 0.5, 0.2, 0, 0}, grid);
      for (std::size_t m = 0; m < b->size(); ++m) b->initialize(m, truth, cov);
    }
    std::vector<float> ranges(360);  // the walls seen from the centre of the map, one reading per degree
    for (std::size_t k = 0; k < ranges.size(); ++k) {
      const double a = static_cast<double>(k) * 3.14159265358979323846 / 180.0;
      ranges[k] = static_cast<float>(2.45 / std::max(std::fabs(std::cos(a)), std::fabs(std::sin(a))));
    }
    ranges[7] = NAN;
    const double laser[12] = {1, 0, 0, 0.05, 0, 1, 0, -0.02, 0, 0, 1, 0.3};
    const beluga_b200::LaserScanView scan{ranges.data(), ranges.size(), -3.14159265f, 0.0174532925f, 0.1, 3.0, 120, laser};
    std::vector<float> xyz;  // a cloud: every second reading of the scan at three heights
    for (std::size_t k = 0; k < ranges.size(); k += 2)
      for (float z : {-0.1f, 0.2f, 0.5f}) {
        const double a = static_cast<double>(k) * 3.14159265358979323846 / 180.0;
        xyz.insert(xyz.end(), {static_cast<float>(ranges[k] * std::cos(a)), static_cast<float>(ranges[k] * std::sin(a)), z});
      }
    const double lidar[12] = {0.99955, -0.0299955, 0, 0.1, 0.0299955, 0.99955, 0, 0, 0, 0, 1, 0.8};
    const beluga_b200::PointCloudView cloud{xyz.data(), xyz.size() / 3, 3 * sizeof(float), 0, BB200_POINT_FLOAT32, lidar};
    const auto points = scan_points(scan);
    const auto scan_xy = scan_points(scan), cloud_xy = beluga_b200::point_cloud_points(cloud);
    for (int step = 0; step < 2; ++step) {
      for (std::size_t m = 0; m < batch.size(); ++m) batch.force_update(m), twin.force_update(m);
      const std::vector<AmclBatch::Measurement> mixed{AmclBatch::Measurement(scan), AmclBatch::Measurement(cloud), AmclBatch::Measurement(points)};
      const auto got = batch.update({truth, truth, truth}, mixed);
      const auto want = twin.update({truth, truth, truth}, {scan_xy, cloud_xy, points});
      for (std::size_t m = 0; m < 3; ++m)
        if (!got[m] || !same(got[m], want[m])) return 1 + static_cast<int>(m);
    }
    for (std::size_t m = 0; m < batch.size(); ++m) batch.force_update(m), twin.force_update(m);
    const std::vector<bool> present = {true, false, true};
    if (!same(batch.update({truth, truth, truth}, std::vector<beluga_b200::LaserScanView>(3, scan), &present)[2],
              twin.update({truth, truth, truth}, {scan_xy, scan_xy, scan_xy}, &present)[2]))
      return 5;
    for (std::size_t m = 0; m < batch.size(); ++m) batch.force_update(m), twin.force_update(m);
    if (!same(batch.update({truth, truth, truth}, std::vector<beluga_b200::PointCloudView>(3, cloud))[1],
              twin.update({truth, truth, truth}, {cloud_xy, cloud_xy, cloud_xy})[1]))
      return 6;
    beluga_b200::PointCloudView bad = cloud;
    bad.x_offset = 4;  // 4 + 12 > 12
    try {
      (void)batch.update({truth, truth, truth}, std::vector<beluga_b200::PointCloudView>{cloud, bad, cloud});
      return 7;
    } catch (const beluga_b200::Error& e) {
      if (e.status() != BB200_ERR_INVALID_ARGUMENT) return 8;
    }
    std::printf("BATCH_MEASUREMENTS_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 9;
    }
    std::printf("BATCH_MEASUREMENTS_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
