// beluga_b200::AmclBatch::cluster_based_estimates through the C ABI.  Without a device the constructor throws
// Error(BB200_ERR_NO_DEVICE); with one, three members take two steps, and the batched estimates equal the per-member
// cluster_based_estimate(m) byte for byte, with std::nullopt for the member left out.
#include <beluga_b200/amcl.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  std::vector<AmclParams> params(3);
  for (std::size_t m = 0; m < params.size(); ++m) {
    params[m].min_particles = params[m].max_particles = 700 + 900 * m;
    params[m].seed = 10 + m;
    params[m].resample_scheme = m % 2 == 0 ? BB200_RESAMPLE_SYSTEMATIC : BB200_RESAMPLE_MULTINOMIAL;
  }
  params[2].resample_interval = 2;  // non-unit weights after the first step
  const bb200_motion_param diff = beluga_b200::DifferentialDriveModel(beluga_b200::DifferentialDriveModelParam{0.1, 0.05, 0.1, 0.05}).c_motion_param();
  const std::vector<bb200_motion_param> motions = {diff, beluga_b200::StationaryModel{}.c_motion_param(), diff};
  try {
    AmclBatch batch(motions, params);
    // a 100 x 100 free map with a wall on every side, 5 cm cells
    std::vector<int8_t> cells(100 * 100, 0);
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const bb200_occupancy_grid grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}};
    batch.set_likelihood_field_map(bb200_likelihood_field_param{2.0, 100.0, 0.5, 0.5, 0.2, 0, 0}, grid);
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    for (std::size_t m = 0; m < batch.size(); ++m) batch.initialize(m, truth, cov);
    std::vector<std::pair<double, double>> scan;  // the walls seen from the centre of the map
    for (int k = 0; k < 72; ++k) {
      const double a = k * 3.14159265358979323846 / 36.0, c = std::cos(a), s = std::sin(a);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    auto same = [](const AmclBatch::estimation_type& a, const AmclBatch::estimation_type& b) {
      return std::memcmp(a.first.data(), b.first.data(), 4 * sizeof(double)) == 0 && std::memcmp(a.second.data(), b.second.data(), 9 * sizeof(double)) == 0;
    };
    for (int step = 0; step < 2; ++step) {
      for (std::size_t m = 0; m < batch.size(); ++m) batch.force_update(m);  // the robots stand still: no update otherwise
      (void)batch.update({truth, truth, truth}, {scan, scan, scan});
      const auto all = batch.cluster_based_estimates();
      for (std::size_t m = 0; m < all.size(); ++m)
        if (!all[m] || !same(*all[m], batch.cluster_based_estimate(m))) return 1;
      const std::vector<bool> present = {true, false, true};
      const auto some = batch.cluster_based_estimates(&present);
      if (some.size() != 3 || some[1] || !some[0] || !some[2] || !same(*some[0], *all[0]) || !same(*some[2], *all[2])) return 2;
    }
    std::printf("BATCH_CLUSTER_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 4;
    }
    std::printf("BATCH_CLUSTER_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
