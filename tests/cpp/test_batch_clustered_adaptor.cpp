// AmclBatch::update_clustered through the C ABI: one call steps every member and returns its cluster-based estimate, what
// beluga_ros::Amcl::update returns.  Without a device the constructor throws Error(BB200_ERR_NO_DEVICE); with one, a fixed,
// a KLD and a selective member step next to standalone beluga_b200::Amcl twins: each clustered estimate equals
// cluster_based_estimate of its twin after the twin's update, bit for bit, and so do the particle states and weights.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  std::vector<AmclParams> params(3);
  params[0].min_particles = params[0].max_particles = 2000;
    params[0].resample_scheme = BB200_RESAMPLE_SYSTEMATIC;
  params[0].seed = 21;
  params[1].min_particles = 300;
  params[1].max_particles = 5000;
    params[1].seed = 22;
  params[2].min_particles = params[2].max_particles = 1000;
  params[2].selective_resampling = true;
  params[2].seed = 23;
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  const std::vector<bb200_motion_param> motions(3, beluga_b200::DifferentialDriveModel(motion).c_motion_param());
  try {
    AmclBatch batch(motions, params, true, true);
    std::vector<int8_t> cells(100 * 100, 0);  // a 100 x 100 free map with a wall on every side, 5 cm cells
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const bb200_occupancy_grid grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}};
    const beluga_b200::LikelihoodFieldModelParam lfm{2.0, 100.0, 0.5, 0.5, 0.2, false};
    batch.set_likelihood_field_map(bb200_likelihood_field_param{2.0, 100.0, 0.5, 0.5, 0.2, 0, 0}, grid);
    const beluga_b200::OccupancyGrid map(cells, 100, 0.05);
    using Twin = beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, beluga_b200::LikelihoodFieldModel<>>;
    std::vector<Twin> twins;
    twins.reserve(3);
    for (std::size_t m = 0; m < 3; ++m)
      twins.emplace_back(beluga_b200::DifferentialDriveModel{motion}, beluga_b200::LikelihoodFieldModel<>{lfm, map}, params[m]);
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    for (std::size_t m = 0; m < 3; ++m) {
      batch.initialize(m, truth, cov);
      twins[m].initialize(truth, cov);
    }
    std::vector<std::pair<double, double>> scan;  // the walls seen from the centre of the map
    for (int k = 0; k < 72; ++k) {
      const double a = k * 3.14159265358979323846 / 36.0, c = std::cos(a), s = std::sin(a);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    for (int step = 0; step < 6; ++step) {
      for (std::size_t m = 0; m < 3; ++m) batch.force_update(m), twins[m].force_update();  // the robots stand still
      const std::vector<AmclBatch::Measurement> meas(3, AmclBatch::Measurement(scan));
      const auto got = batch.update_clustered({truth, truth, truth}, meas);
      for (std::size_t m = 0; m < 3; ++m) {
        if (!got[m] || !twins[m].update(truth, scan)) return 1;
        const auto want = beluga_b200::cluster_based_estimate(twins[m]);
        if (std::memcmp(got[m]->first.data(), want.first.data(), 4 * sizeof(double)) != 0 ||
            std::memcmp(&got[m]->second, &want.second, sizeof(want.second)) != 0)
          return 2;
        const beluga_b200::ParticleSet a = batch.particles(m), b = twins[m].particles();
        if (a.size() != b.size() || batch.member_size(m) != b.size()) return 3;
        for (std::size_t i = 0; i < a.size(); ++i)
          if (std::memcmp(a.states[i].data(), b.states[i].data(), 4 * sizeof(double)) != 0 || std::memcmp(&a.weights[i], &b.weights[i], sizeof(double)) != 0)
            return 4;
      }
    }
    std::printf("BATCH_CLUSTERED_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 6;
    }
    std::printf("BATCH_CLUSTERED_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
