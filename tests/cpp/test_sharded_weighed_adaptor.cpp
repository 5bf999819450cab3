// ShardedAmcl with a caller's device sensor model (include/beluga_b200/amcl.hpp: ShardedAmcl::update with a token that
// weighs on the device).  The model is the Gaussian position fix of position_fix.cu.  Without a device the ShardedAmcl
// constructor throws Error(BB200_ERR_NO_DEVICE); with one, every step of a 2-shard filter equals a twin driven through the
// C ABI (bb200_sharded_amcl_update_begin, the kernel once per shard, bb200_sharded_amcl_update_end) and a standalone Amcl
// weighed by the same token, a step the policies skip returns std::nullopt, and the particles of the sharded filter are
// the standalone filter's.
#include <beluga_b200/amcl.hpp>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <optional>
#include <vector>

void launch_position_fix(void* stream, const double* states, std::uint64_t n, double fx, double fy, double sigma, double* factors);

namespace {

struct PositionFix {
  double x, y, sigma;
};

struct PositionFixToken {
  PositionFix fix;
  // Every shard of these filters lives on device 0, the current device: a token for shards on several devices would make
  // each view's device current before it launches.
  void weigh(void* stream, const double* states, std::uint64_t n, double* factors) const {
    launch_position_fix(stream, states, n, fix.x, fix.y, fix.sigma, factors);
  }
};

/// A sensor model without a map, for a standalone and for a sharded filter.
class PositionFixModel {
 public:
  using state_type = beluga_b200::SE2d;
  using measurement_type = PositionFix;
  using map_type = beluga_b200::OccupancyGrid;
  [[nodiscard]] PositionFixToken operator()(measurement_type&& fix) const { return PositionFixToken{fix}; }
  [[nodiscard]] int attach(bb200_filter*) const { return BB200_OK; }
  [[nodiscard]] int attach(bb200_sharded_amcl*) const { return BB200_OK; }
  void update_map(const map_type&) {}
};

int fail(const char* what) {
  std::printf("SHARDED_WEIGHED_ADAPTOR_FAIL %s\n", what);
  return 1;
}

}  // namespace

int main() {
  using beluga_b200::SE2d;
  beluga_b200::AmclParams params;
  params.min_particles = params.max_particles = 8192;
  params.resample_interval = 1;
  params.update_min_d = 0.1;
  params.seed = 5;
  const beluga_b200::DifferentialDriveModelParam motion{0.05, 0.05, 0.05, 0.05};
  const std::vector<int> devices{0, 0};
  std::optional<beluga_b200::ShardedAmcl<beluga_b200::DifferentialDriveModel, PositionFixModel>> sharded;
  try {
    sharded.emplace(beluga_b200::DifferentialDriveModel{motion}, PositionFixModel{}, params, devices);
  } catch (const beluga_b200::Error& e) {
    if (e.status() == BB200_ERR_NO_DEVICE) {
      std::printf("SHARDED_WEIGHED_ADAPTOR_NO_DEVICE\n");
      return 0;
    }
    throw;
  }
  beluga_b200::Amcl<beluga_b200::DifferentialDriveModel, PositionFixModel> single{beluga_b200::DifferentialDriveModel{motion}, PositionFixModel{}, params};
  // the twin: the same parameters through the C ABI
  const bb200_amcl_param p = beluga_b200::c_amcl_param(params);
  const bb200_motion_param m = beluga_b200::DifferentialDriveModel{motion}.c_motion_param();
  bb200_sharded_amcl* twin = nullptr;
  if (bb200_sharded_amcl_create(&p, &m, 2, devices.data(), &twin) != BB200_OK) return fail("twin create");

  beluga_b200::Matrix3d cov{};
  cov[0] = cov[4] = 1.0;
  cov[8] = 0.1;
  sharded->initialize(SE2d{0.0, 0.0, 0.0}, cov);
  single.initialize(SE2d{0.0, 0.0, 0.0}, cov);
  const double mean[3] = {0.0, 0.0, 0.0};
  if (bb200_sharded_amcl_initialize(twin, mean, cov.data()) != BB200_OK) return fail("twin initialize");

  const PositionFix fix{1.5, -0.5, 0.3};
  int rc = 0;
  for (int k = 0; k < 6; ++k) {
    // step 3 repeats step 2's pose: the policies skip it
    const double x = 0.25 * (k == 3 ? 2 : k);
    const SE2d control{x, 0.0, 0.0};
    const auto est = sharded->update(control, PositionFix{fix});
    const auto est_single = single.update(control, PositionFix{fix});
    bb200_weigh_view views[2]{};
    if (bb200_sharded_amcl_update_begin(twin, control.data(), views) != BB200_OK) return fail("twin begin");
    for (const bb200_weigh_view& v : views)
      if (v.updated && v.n > 0) launch_position_fix(v.stream, v.states, v.n, fix.x, fix.y, fix.sigma, v.factors);
    bb200_update_result r{};
    if (bb200_sharded_amcl_update_end(twin, &r) != BB200_OK) return fail("twin end");
    if (est.has_value() != (r.updated != 0) || est.has_value() != est_single.has_value()) return fail("updated flags differ");
    if (k == 3 && est.has_value()) return fail("the repeated pose was not skipped");
    if (!est) continue;
    for (int j = 0; j < 4; ++j) {
      if (est->first.data()[j] != r.estimate.mean[j]) rc = fail("estimate differs from the C ABI twin");
      if (std::fabs(est->first.data()[j] - est_single->first.data()[j]) > 1e-12) rc = fail("estimate differs from the standalone filter");
    }
  }
  const auto a = sharded->particles();
  const auto b = single.particles();
  bb200_sharded_amcl_destroy(twin);
  if (a.size() != b.size() || std::memcmp(a.states.data(), b.states.data(), a.size() * sizeof(SE2d)) != 0)
    return fail("particles differ from the standalone filter");
  double mx = 0.0, my = 0.0;
  for (const SE2d& s : a.states) mx += s.x(), my += s.y();
  mx /= static_cast<double>(a.size());
  my /= static_cast<double>(a.size());
  if (std::fabs(mx - fix.x) > 0.5 || std::fabs(my - fix.y) > 0.5) return fail("the cloud did not settle on the fix");
  if (rc == 0) std::printf("SHARDED_WEIGHED_ADAPTOR_OK mean=(%.3f, %.3f)\n", mx, my);
  return rc;
}
