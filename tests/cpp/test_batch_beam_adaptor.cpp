// beluga_b200::AmclBatch::set_beam_map through the C ABI.  Without a device the constructor throws
// Error(BB200_ERR_NO_DEVICE); with one, three members on a beam-model map take a few steps next to three
// beluga_b200::Amcl<..., BeamSensorModel> twins built from the same parameters, and every member's estimate and
// particles equal its twin's byte for byte.
#include <beluga_b200/amcl.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <optional>
#include <vector>

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  using Model = beluga_b200::DifferentialDriveModel;
  using Sensor = beluga_b200::BeamSensorModel<>;
  std::vector<AmclParams> params(3);
  for (std::size_t m = 0; m < params.size(); ++m) {
    params[m].min_particles = params[m].max_particles = 700 + 900 * m;
    params[m].seed = 20 + m;
    params[m].resample_scheme = m % 2 == 0 ? BB200_RESAMPLE_SYSTEMATIC : BB200_RESAMPLE_MULTINOMIAL;
  }
  params[2].resample_interval = 2;  // non-unit weights after the first step
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  const std::vector<bb200_motion_param> motions(3, Model(motion).c_motion_param());
  try {
    AmclBatch batch(motions, params);
    // a 100 x 100 free map with a wall on every side, 5 cm cells
    std::vector<int8_t> cells(100 * 100, 0);
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const beluga_b200::BeamModelParam beam{};
    const bb200_beam_param c_beam{beam.z_hit, beam.z_short, beam.z_max, beam.z_rand, beam.sigma_hit, beam.lambda_short, beam.beam_max_range};
    batch.set_beam_map(c_beam, bb200_occupancy_grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}});
    const beluga_b200::OccupancyGrid map(cells, 100, 0.05);
    std::vector<beluga_b200::Amcl<Model, Sensor>> twins;
    for (std::size_t m = 0; m < params.size(); ++m) twins.emplace_back(Model(motion), Sensor(beam, map), params[m]);
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    for (std::size_t m = 0; m < batch.size(); ++m) {
      batch.initialize(m, truth, cov);
      twins[m].initialize(truth, cov);
    }
    std::vector<std::pair<double, double>> scan;  // the walls seen from the centre of the map
    for (int k = 0; k < 72; ++k) {
      const double a = k * 3.14159265358979323846 / 36.0, c = std::cos(a), s = std::sin(a);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    auto same = [](const std::optional<AmclBatch::estimation_type>& a, const std::optional<AmclBatch::estimation_type>& b) {
      if (!a || !b) return !a && !b;
      return std::memcmp(a->first.data(), b->first.data(), 4 * sizeof(double)) == 0 && std::memcmp(a->second.data(), b->second.data(), 9 * sizeof(double)) == 0;
    };
    for (int step = 0; step < 3; ++step) {
      for (std::size_t m = 0; m < batch.size(); ++m) {  // the robots stand still: no update otherwise
        batch.force_update(m);
        twins[m].force_update();
      }
      const auto out = batch.update({truth, truth, truth}, {scan, scan, scan});
      for (std::size_t m = 0; m < out.size(); ++m) {
        const auto exp = twins[m].update(truth, scan);
        if (!out[m] || !same(out[m], exp)) return 1;
        const beluga_b200::ParticleSet a = batch.particles(m), b = twins[m].particles();
        if (a.size() != b.size() || std::memcmp(a.states.data(), b.states.data(), a.size() * sizeof(SE2d)) != 0 ||
            std::memcmp(a.weights.data(), b.weights.data(), a.size() * sizeof(double)) != 0)
          return 2;
        if (std::hypot(out[m]->first.x() - 2.5, out[m]->first.y() - 2.5) > 0.3) return 3;
      }
    }
    std::printf("BATCH_BEAM_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 4;
    }
    std::printf("BATCH_BEAM_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
