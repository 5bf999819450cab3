// beluga_b200::AmclBatch with two maps through the C ABI.  Without a device the constructor throws
// Error(BB200_ERR_NO_DEVICE); with one, three members on two likelihood-field maps (room A, and room B: room A with a
// wider free area) take a few steps next to three beluga_b200::Amcl<..., LikelihoodFieldModel> twins, member 0 moves
// from A to B with update_map while its twin calls Amcl::update_map, and every member's estimate and particles equal its
// twin's byte for byte.
#include <beluga_b200/amcl.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <optional>
#include <vector>

namespace {

/// A free width x 100 map with a wall on every side, 5 cm cells.
std::vector<int8_t> room(int width) {
  std::vector<int8_t> cells(static_cast<std::size_t>(width) * 100, 0);
  for (int i = 0; i < width; ++i) cells[i] = cells[99 * width + i] = 100;
  for (int j = 0; j < 100; ++j) cells[j * width] = cells[j * width + width - 1] = 100;
  return cells;
}

}  // namespace

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  using Model = beluga_b200::DifferentialDriveModel;
  using Sensor = beluga_b200::LikelihoodFieldModel<>;
  std::vector<AmclParams> params(3);
  for (std::size_t m = 0; m < params.size(); ++m) {
    params[m].min_particles = params[m].max_particles = 800 + 600 * m;
    params[m].seed = 60 + m;
    params[m].resample_scheme = m % 2 == 0 ? BB200_RESAMPLE_SYSTEMATIC : BB200_RESAMPLE_MULTINOMIAL;
  }
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  const std::vector<bb200_motion_param> motions(3, Model(motion).c_motion_param());
  try {
    AmclBatch batch(motions, params);
    const std::vector<int8_t> cells_a = room(100), cells_b = room(140);
    const beluga_b200::LikelihoodFieldModelParam lfm{2.0, 100.0, 0.5, 0.5, 0.2, false, false};
    const bb200_likelihood_field_param c_lfm{lfm.max_obstacle_distance, lfm.max_laser_distance, lfm.z_hit, lfm.z_random, lfm.sigma_hit, 0, 0};
    const int a = batch.add_likelihood_field_map(c_lfm, bb200_occupancy_grid{cells_a.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}});
    const int b = batch.add_likelihood_field_map(c_lfm, bb200_occupancy_grid{cells_b.data(), 140, 100, 0.05, {1.0, 0.0, 0.0, 0.0}});
    if (a != 0 || b != 1) return 5;
    if (batch.likelihood_field(b).size() != 140u * 100u) return 6;
    const beluga_b200::OccupancyGrid map_a(cells_a, 100, 0.05), map_b(cells_b, 140, 0.05);
    const int start[3] = {a, a, b};
    std::vector<beluga_b200::Amcl<Model, Sensor>> twins;
    for (std::size_t m = 0; m < params.size(); ++m) {
      batch.update_map(m, start[m]);
      twins.emplace_back(Model(motion), Sensor(lfm, start[m] == a ? map_a : map_b), params[m]);
    }
    if (batch.member_map(2) != b) return 7;
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    for (std::size_t m = 0; m < batch.size(); ++m) {
      batch.initialize(m, truth, cov);
      twins[m].initialize(truth, cov);
    }
    std::vector<std::pair<double, double>> scan;  // the walls seen from (2.5, 2.5) in room A
    for (int k = 0; k < 72; ++k) {
      const double t = k * 3.14159265358979323846 / 36.0, c = std::cos(t), s = std::sin(t);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    auto same = [](const std::optional<AmclBatch::estimation_type>& x, const std::optional<AmclBatch::estimation_type>& y) {
      if (!x || !y) return !x && !y;
      return std::memcmp(x->first.data(), y->first.data(), 4 * sizeof(double)) == 0 && std::memcmp(x->second.data(), y->second.data(), 9 * sizeof(double)) == 0;
    };
    for (int step = 0; step < 4; ++step) {
      if (step == 2) {
        batch.update_map(0, b);
        twins[0].update_map(map_b);
      }
      for (std::size_t m = 0; m < batch.size(); ++m) {  // the robots stand still: no update otherwise
        batch.force_update(m);
        twins[m].force_update();
      }
      const auto out = batch.update({truth, truth, truth}, {scan, scan, scan});
      for (std::size_t m = 0; m < out.size(); ++m) {
        const auto exp = twins[m].update(truth, scan);
        if (!out[m] || !same(out[m], exp)) return 1;
        const beluga_b200::ParticleSet x = batch.particles(m), y = twins[m].particles();
        if (x.size() != y.size() || std::memcmp(x.states.data(), y.states.data(), x.size() * sizeof(SE2d)) != 0 ||
            std::memcmp(x.weights.data(), y.weights.data(), x.size() * sizeof(double)) != 0)
          return 2;
      }
    }
    try {
      batch.remove_map(b);  // members 0 and 2 read it
      return 3;
    } catch (const beluga_b200::Error& e) {
      if (e.status() != BB200_ERR_STATE) return 3;
    }
    std::printf("BATCH_MAPS_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 4;
    }
    std::printf("BATCH_MAPS_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
