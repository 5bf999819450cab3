// AmclBatch::add_member / remove_member / member_active through the C ABI.  Without a device the constructor throws
// Error(BB200_ERR_NO_DEVICE); with one, two members step next to standalone beluga_b200::Amcl twins, a third joins (with its
// own twin, created when it joins), the first leaves, and after every step each occupied member's estimate, particle states
// and weights equal its twin's bit for bit.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  std::vector<AmclParams> params(3);
  for (std::size_t m = 0; m < 3; ++m) {
    params[m].min_particles = params[m].max_particles = 1000 + 500 * m;
    params[m].seed = 31 + m;
  }
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  const bb200_motion_param c_motion = beluga_b200::DifferentialDriveModel(motion).c_motion_param();
  try {
    AmclBatch batch({c_motion, c_motion}, {params[0], params[1]});
    std::vector<int8_t> cells(100 * 100, 0);  // a 100 x 100 free map with a wall on every side, 5 cm cells
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const bb200_occupancy_grid grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}};
    const beluga_b200::LikelihoodFieldModelParam lfm{2.0, 100.0, 0.5, 0.5, 0.2, false};
    const bb200_likelihood_field_param c_lfm{2.0, 100.0, 0.5, 0.5, 0.2, 0, 0};
    batch.set_likelihood_field_map(c_lfm, grid);
    const beluga_b200::OccupancyGrid map(cells, 100, 0.05);
    using Twin = beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, beluga_b200::LikelihoodFieldModel<>>;
    std::vector<std::unique_ptr<Twin>> twins(3);
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    auto join = [&](std::size_t m) {
      twins[m] = std::make_unique<Twin>(beluga_b200::DifferentialDriveModel{motion}, beluga_b200::LikelihoodFieldModel<>{lfm, map}, params[m]);
      batch.initialize(m, truth, cov);
      twins[m]->initialize(truth, cov);
    };
    join(0);
    join(1);
    std::vector<std::pair<double, double>> scan;  // the walls seen from the centre of the map
    for (int k = 0; k < 72; ++k) {
      const double a = k * 3.14159265358979323846 / 36.0, c = std::cos(a), s = std::sin(a);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    for (int step = 0; step < 6; ++step) {
      if (step == 2) {  // a third robot joins: a new slot after the last
        if (batch.add_member(c_motion, params[2]) != 2 || batch.size() != 3 || !batch.member_active(2)) return 1;
        if (batch.member_map(2) != -1) return 1;
        batch.update_map(2, batch.member_map(1));
        join(2);
      }
      if (step == 4) {  // the first one leaves; its slot stays, vacant
        batch.remove_member(0);
        twins[0].reset();
        if (batch.size() != 3 || batch.member_active(0)) return 1;
        try {
          (void)batch.particles(0);
          return 1;
        } catch (const beluga_b200::Error& e) {
          if (e.status() != BB200_ERR_INVALID_ARGUMENT) return 1;
        }
      }
      const std::size_t k = batch.size();
      for (std::size_t m = 0; m < k; ++m)
        if (twins[m]) batch.force_update(m), twins[m]->force_update();  // the robots stand still
      const auto got = batch.update(std::vector<SE2d>(k, truth), std::vector<std::vector<std::pair<double, double>>>(k, scan));
      for (std::size_t m = 0; m < k; ++m) {
        if (!twins[m]) {
          if (got[m]) return 2;
          continue;
        }
        const auto want = twins[m]->update(truth, scan);
        if (!got[m] || !want) return 3;
        if (std::memcmp(got[m]->first.data(), want->first.data(), 4 * sizeof(double)) != 0 ||
            std::memcmp(&got[m]->second, &want->second, sizeof(want->second)) != 0)
          return 4;
        const beluga_b200::ParticleSet a = batch.particles(m), b = twins[m]->particles();
        if (a.size() != b.size()) return 5;
        for (std::size_t i = 0; i < a.size(); ++i)
          if (std::memcmp(a.states[i].data(), b.states[i].data(), 4 * sizeof(double)) != 0 || std::memcmp(&a.weights[i], &b.weights[i], sizeof(double)) != 0)
            return 6;
      }
    }
    std::printf("BATCH_MEMBERS_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 7;
    }
    std::printf("BATCH_MEMBERS_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
