// AmclBatch::export_member / import_member / from_states and Amcl::export_state / from_state through the C ABI.  Without a
// device the batch constructor throws Error(BB200_ERR_NO_DEVICE); with one, two members step next to standalone
// beluga_b200::Amcl twins, member 1 moves out of the batch into a standalone Amcl, steps there, moves back into the batch
// (a vacant slot after it left), and the whole batch is checkpointed and restored with from_states; after every step each
// copy's estimate, particle states and weights equal its twin's bit for bit.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <optional>
#include <vector>

namespace {

bool same(const beluga_b200::ParticleSet& a, const beluga_b200::ParticleSet& b) {
  if (a.size() != b.size()) return false;
  for (std::size_t i = 0; i < a.size(); ++i)
    if (std::memcmp(a.states[i].data(), b.states[i].data(), 4 * sizeof(double)) != 0 || std::memcmp(&a.weights[i], &b.weights[i], sizeof(double)) != 0)
      return false;
  return true;
}

template <class Estimate>
bool same(const std::optional<Estimate>& a, const std::optional<Estimate>& b) {
  return a && b && std::memcmp(a->first.data(), b->first.data(), 4 * sizeof(double)) == 0 && std::memcmp(&a->second, &b->second, sizeof(b->second)) == 0;
}

}  // namespace

int main() {
  using beluga_b200::AmclBatch;
  using beluga_b200::AmclParams;
  using beluga_b200::SE2d;
  std::vector<AmclParams> params(2);
  for (std::size_t m = 0; m < 2; ++m) {
    params[m].min_particles = params[m].max_particles = 1000 + 500 * m;
    params[m].seed = 61 + m;
  }
  const beluga_b200::DifferentialDriveModelParam motion{0.1, 0.05, 0.1, 0.05};
  const bb200_motion_param c_motion = beluga_b200::DifferentialDriveModel(motion).c_motion_param();
  try {
    std::unique_ptr<AmclBatch> batch = std::make_unique<AmclBatch>(std::vector<bb200_motion_param>{c_motion, c_motion}, params);
    std::vector<int8_t> cells(100 * 100, 0);  // a 100 x 100 free map with a wall on every side, 5 cm cells
    for (int i = 0; i < 100; ++i) cells[i] = cells[99 * 100 + i] = cells[i * 100] = cells[i * 100 + 99] = 100;
    const bb200_occupancy_grid grid{cells.data(), 100, 100, 0.05, {1.0, 0.0, 0.0, 0.0}};
    const beluga_b200::LikelihoodFieldModelParam lfm{2.0, 100.0, 0.5, 0.5, 0.2, false};
    const bb200_likelihood_field_param c_lfm{2.0, 100.0, 0.5, 0.5, 0.2, 0, 0};
    batch->set_likelihood_field_map(c_lfm, grid);
    const beluga_b200::OccupancyGrid map(cells, 100, 0.05);
    using Solo = beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, beluga_b200::LikelihoodFieldModel<>>;
    auto make = [&](std::size_t m) {
      return std::make_unique<Solo>(beluga_b200::DifferentialDriveModel{motion}, beluga_b200::LikelihoodFieldModel<>{lfm, map}, params[m]);
    };
    std::vector<std::unique_ptr<Solo>> twins;
    twins.push_back(make(0));
    twins.push_back(make(1));
    const beluga_b200::Matrix3d cov = {0.04, 0, 0, 0, 0.04, 0, 0, 0, 0.04};
    const SE2d truth(0.0, 2.5, 2.5);
    for (std::size_t m = 0; m < 2; ++m) {
      batch->initialize(m, truth, cov);
      twins[m]->initialize(truth, cov);
    }
    std::vector<std::pair<double, double>> scan;  // the walls seen from the centre of the map
    for (int k = 0; k < 72; ++k) {
      const double a = k * 3.14159265358979323846 / 36.0, c = std::cos(a), s = std::sin(a);
      const double r = 2.45 / std::max(std::fabs(c), std::fabs(s));
      scan.emplace_back(r * c, r * s);
    }
    std::unique_ptr<Solo> solo;  // member 1 while it is out of the batch
    std::size_t slot1 = 1;
    for (int step = 0; step < 8; ++step) {
      if (step == 2) {  // member 1 leaves the batch for a standalone filter
        const std::vector<std::uint8_t> blob = batch->export_member(1);
        if (blob != twins[1]->export_state()) return 10;
        batch->remove_member(1);
        solo = std::make_unique<Solo>(Solo::from_state(blob, beluga_b200::DifferentialDriveModel{motion}, beluga_b200::LikelihoodFieldModel<>{lfm, map}));
      }
      if (step == 4) {  // ... and comes back
        slot1 = batch->import_member(solo->export_state(), batch->member_map(0));
        if (slot1 != 1) return 11;
        solo.reset();
      }
      if (step == 6) {  // the fleet checkpoint, restored into a new batch
        const std::vector<std::vector<std::uint8_t>> blobs = batch->export_members();
        auto restored = std::make_unique<AmclBatch>(AmclBatch::from_states(blobs));
        restored->set_likelihood_field_map(c_lfm, grid);
        batch = std::move(restored);
      }
      for (auto& t : twins) t->force_update();  // the robots stand still
      for (std::size_t m = 0; m < batch->size(); ++m)
        if (batch->member_active(m)) batch->force_update(m);
      if (solo) solo->force_update();
      const std::size_t k = batch->size();
      const auto got = batch->update(std::vector<SE2d>(k, truth), std::vector<std::vector<std::pair<double, double>>>(k, scan));
      for (std::size_t m = 0; m < 2; ++m) {
        const auto want = twins[m]->update(truth, scan);
        const bool in_batch = m == 0 || !solo;
        const auto have = in_batch ? got[m == 0 ? 0 : slot1] : solo->update(truth, scan);
        if (!same(have, want)) return 3;
        if (!same(in_batch ? batch->particles(m == 0 ? 0 : slot1) : solo->particles(), twins[m]->particles())) return 4;
      }
    }
    std::printf("BATCH_STATE_ADAPTOR_OK\n");
  } catch (const beluga_b200::Error& e) {
    if (e.status() != BB200_ERR_NO_DEVICE) {
      std::printf("unexpected error %d: %s\n", e.status(), e.what());
      return 7;
    }
    std::printf("BATCH_STATE_ADAPTOR_NO_DEVICE\n");
  }
  return 0;
}
