// beluga_b200::AmclBatch through the C ABI.  Without a device the constructor throws Error(BB200_ERR_NO_DEVICE); with one,
// two members on a small open map take a few steps and each member's estimate stays near its ground truth.
#include <beluga_b200/amcl.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  std::vector<AmclParams> params(2);
  for (std::size_t m = 0; m < params.size(); ++m) {
    params[m].min_particles = params[m].max_particles = 1000 + 500 * m;
    params[m].seed = m;
    params[m].resample_scheme = m == 0 ? BB200_RESAMPLE_SYSTEMATIC : BB200_RESAMPLE_MULTINOMIAL;
  }
  const std::vector<bb200_motion_param> motions = {
      beluga_b200::DifferentialDriveModel(beluga_b200::DifferentialDriveModelParam{0.1, 0.05, 0.1, 0.05}).c_motion_param(),
      beluga_b200::StationaryModel{}.c_motion_param()};
  try {
    AmclBatch batch(motions, params);
    // a 100 x 100 free map with a wall on every side, 5 cm cells
    std::vector<int8_t> cells(100 * 100, 0);
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const bb200_occupancy_grid grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}};
    batch.set_likelihood_field_map(bb200_likelihood_field_param{2.0, 100.0, 0.5, 0.5, 0.2, 0, 0}, grid);
    const beluga_b200::Matrix3d cov = {0.01, 0, 0, 0, 0.01, 0, 0, 0, 0.01};
    const SE2d truth(0.0, 2.5, 2.5);
    for (std::size_t m = 0; m < batch.size(); ++m) batch.initialize(m, truth, cov);
    std::vector<std::pair<double, double>> scan;  // the walls seen from the centre of the map
    for (int k = 0; k < 72; ++k) {
      const double a = k * 3.14159265358979323846 / 36.0, c = std::cos(a), s = std::sin(a);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    for (int step = 0; step < 3; ++step) {
      const std::vector<bool> present = {true, step != 1};
      for (std::size_t m = 0; m < batch.size(); ++m) batch.force_update(m);  // the robots stand still: no update otherwise
      const auto out = batch.update({truth, truth}, {scan, scan}, &present);
      for (std::size_t m = 0; m < out.size(); ++m) {
        if (!present[m]) {
          if (out[m]) return 1;
          continue;
        }
        if (!out[m] || std::hypot(out[m]->first.x() - 2.5, out[m]->first.y() - 2.5) > 0.3) return 2;
      }
    }
    if (batch.particles(1).size() != 1500) return 3;
    (void)batch.cluster_based_estimate(0);
    std::printf("BATCH_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 4;
    }
    std::printf("BATCH_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
