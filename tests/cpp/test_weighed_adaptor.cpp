// Amcl with a caller's device sensor model (include/beluga_b200/amcl.hpp, models.hpp: is_weighed_token_v).  The model is a
// Gaussian position fix whose kernel (position_fix.cu) runs on the stream the step hands out.  Without a device the Amcl
// constructor throws Error(BB200_ERR_NO_DEVICE); with one, every step equals a twin driven through the C ABI
// (bb200_amcl_update_begin, the same kernel, bb200_amcl_update_end), a step the policies skip returns std::nullopt, and the
// estimate settles on the fix.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <optional>
#include <utility>
#include <vector>

void launch_position_fix(void* stream, const double* states, std::uint64_t n, double fx, double fy, double sigma, double* factors);

namespace {

struct PositionFix {
  double x, y, sigma;
};

struct PositionFixToken {
  PositionFix fix;
  void weigh(void* stream, const double* states, std::uint64_t n, double* factors) const {
    launch_position_fix(stream, states, n, fix.x, fix.y, fix.sigma, factors);
  }
};

/// A sensor model without a map: measurement_type is the fix, the token weighs on the device.
class PositionFixModel {
 public:
  using state_type = beluga_b200::SE2d;
  using measurement_type = PositionFix;
  using map_type = beluga_b200::OccupancyGrid;
  [[nodiscard]] PositionFixToken operator()(measurement_type&& fix) const { return PositionFixToken{fix}; }
  [[nodiscard]] int attach(bb200_filter*) const { return BB200_OK; }
  void update_map(const map_type&) {}
};

static_assert(beluga_b200::is_weighed_token_v<PositionFixToken>, "the token weighs on the device");
static_assert(!beluga_b200::is_weighed_token_v<beluga_b200::measurement_token>, "stock tokens carry points");

/// AmclBatch's weighed overload, compiled here (the batch form runs in tests/test_gpu_weighed_update.py).
[[maybe_unused]] std::size_t batch_step(beluga_b200::AmclBatch& batch, const PositionFix& fix) {
  using Measurement = beluga_b200::AmclBatch::Measurement;
  std::vector<std::optional<Measurement>> in(batch.size());
  in[0] = Measurement{std::vector<std::pair<double, double>>{{1.0, 0.0}}};
  const auto estimates = batch.update(std::vector<beluga_b200::SE2d>(batch.size()), in,
                                      [&](const std::vector<std::size_t>& members, const std::vector<bb200_weigh_view>& views) {
                                        for (const std::size_t m : members)
                                          launch_position_fix(views[m].stream, views[m].states, views[m].n, fix.x, fix.y, fix.sigma, views[m].factors);
                                      });
  return estimates.size();
}

int fail(const char* what) {
  std::printf("WEIGHED_ADAPTOR_FAIL %s\n", what);
  return 1;
}

}  // namespace

int main() {
  using beluga_b200::SE2d;
  beluga_b200::AmclParams params;
  params.min_particles = params.max_particles = 4096;
  params.resample_interval = 1;
  params.update_min_d = 0.1;
  params.seed = 5;
  const beluga_b200::DifferentialDriveModelParam motion{0.05, 0.05, 0.05, 0.05};
  std::optional<beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, PositionFixModel>> amcl;
  try {
    amcl.emplace(beluga_b200::DifferentialDriveModel{motion}, PositionFixModel{}, params);
  } catch (const beluga_b200::Error& e) {
    if (e.status() == BB200_ERR_NO_DEVICE) {
      std::printf("WEIGHED_ADAPTOR_NO_DEVICE\n");
      return 0;
    }
    throw;
  }
  // the twin: the same parameters through the C ABI
  const bb200_amcl_param p = beluga_b200::c_amcl_param(params);
  const bb200_motion_param m = beluga_b200::DifferentialDriveModel{motion}.c_motion_param();
  bb200_amcl* twin = nullptr;
  if (bb200_amcl_create_with_motion(&p, &m, &twin) != BB200_OK) return fail("twin create");

  beluga_b200::Matrix3d cov{};
  cov[0] = cov[4] = 1.0;
  cov[8] = 0.1;
  amcl->initialize(SE2d{0.0, 0.0, 0.0}, cov);
  const double mean[3] = {0.0, 0.0, 0.0};
  if (bb200_amcl_initialize(twin, mean, cov.data()) != BB200_OK) return fail("twin initialize");

  const PositionFix fix{1.5, -0.5, 0.3};
  int rc = 0;
  for (int k = 0; k < 6; ++k) {
    // step 3 repeats step 2's pose: the policies skip it
    const double x = 0.25 * (k == 3 ? 2 : k);
    const SE2d control{x, 0.0, 0.0};
    const auto est = amcl->update(control, PositionFix{fix});
    bb200_weigh_view view{};
    if (bb200_amcl_update_begin(twin, control.data(), &view) != BB200_OK) return fail("twin begin");
    if (view.updated) launch_position_fix(view.stream, view.states, view.n, fix.x, fix.y, fix.sigma, view.factors);
    bb200_update_result r{};
    if (bb200_amcl_update_end(twin, &r) != BB200_OK) return fail("twin end");
    if (est.has_value() != (r.updated != 0)) return fail("updated flags differ");
    if (k == 3 && est.has_value()) return fail("the repeated pose was not skipped");
    if (!est) continue;
    for (int j = 0; j < 4; ++j)
      if (est->first.data()[j] != r.estimate.mean[j]) rc = fail("estimate differs from the C ABI twin");
  }
  const auto particles = amcl->particles();
  double mx = 0.0, my = 0.0;
  for (const SE2d& s : particles.states) mx += s.x(), my += s.y();
  mx /= static_cast<double>(particles.states.size());
  my /= static_cast<double>(particles.states.size());
  bb200_amcl_destroy(twin);
  if (std::fabs(mx - (fix.x)) > 0.5 || std::fabs(my - fix.y) > 0.5) return fail("the cloud did not settle on the fix");
  if (rc == 0) std::printf("WEIGHED_ADAPTOR_OK mean=(%.3f, %.3f)\n", mx, my);
  return rc;
}
