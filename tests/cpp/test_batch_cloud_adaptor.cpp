// beluga_b200::particle_cloud_markers / sample_poses over an AmclBatch through the C ABI.  Without a device the constructor
// throws Error(BB200_ERR_NO_DEVICE); with one, three members take two steps, and each selected member's markers and poses
// equal those of the batch's per-member histogram and draw, with std::nullopt for the member left out.
#include <beluga_b200/particle_cloud.hpp>

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
    params[m].seed = 20 + m;
    params[m].resample_scheme = m % 2 == 0 ? BB200_RESAMPLE_SYSTEMATIC : BB200_RESAMPLE_MULTINOMIAL;
  }
  params[2].resample_interval = 2;  // a normalising step: member 2 draws from the step's CDF
  const bb200_motion_param diff = beluga_b200::DifferentialDriveModel(beluga_b200::DifferentialDriveModelParam{0.1, 0.05, 0.1, 0.05}).c_motion_param();
  const std::vector<bb200_motion_param> motions = {diff, beluga_b200::StationaryModel{}.c_motion_param(), diff};
  try {
    AmclBatch batch(motions, params);
    std::vector<int8_t> cells(100 * 100, 0);  // a 100 x 100 free map with a wall on every side, 5 cm cells
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
    const std::vector<bool> present = {true, false, true};
    for (uint32_t step = 0; step < 2; ++step) {
      for (std::size_t m = 0; m < batch.size(); ++m) batch.force_update(m);
      (void)batch.update({truth, truth, truth}, {scan, scan, scan});
      const auto markers = beluga_b200::particle_cloud_markers(batch, &present);
      const auto histograms = batch.particle_histograms(&present);
      const auto poses = beluga_b200::sample_poses(batch, 50, step, &present);
      const auto raw = batch.sample_states({50, 50, 50}, 0xFFFFFFFFu - step, &present);
      if (markers.size() != 3 || markers[1] || poses[1] || histograms[1] || raw[1]) return 1;
      for (std::size_t m : {std::size_t{0}, std::size_t{2}}) {
        if (!markers[m] || !histograms[m] || !poses[m] || !raw[m]) return 2;
        const std::vector<bb200_cluster_cell>& bins = histograms[m]->first;
        if (bins.empty() || markers[m]->bodies.size() != 2 * bins.size() || markers[m]->heads.size() != 3 * bins.size()) return 3;
        if (histograms[m]->second < 1e-3) return 4;
        const std::vector<double>& r = *raw[m];
        for (std::size_t i = 0; i < 50; ++i) {
          const beluga_b200::Pose2d& p = (*poses[m])[i];
          if (p.x != r[4 * i + 2] || p.y != r[4 * i + 3] || p.cos_yaw != r[4 * i] || p.sin_yaw != r[4 * i + 1]) return 5;
        }
      }
    }
    std::printf("BATCH_CLOUD_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 4;
    }
    std::printf("BATCH_CLOUD_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
