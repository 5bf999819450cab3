// Host-only probe: prints what csrc/kernels.cuh's schedule_from_moments and bordered_index compute, so that the CPU model
// tests (tests/test_schedule_model.py, tests/test_fixed_point_lookup_model.py) are checked against the code the kernels
// are built from, not only against their own restatement.  Compiled with nvcc, runs without a GPU (no CUDA call).
#include <cstdio>

#include "kernels.cuh"

int main() {
  using namespace bb200;
  struct Case {
    double cbar, sbar, mx, my, vx, vy, n, mean_range, min_bin;
  };
  const Case cases[] = {
      {0.45, 0.87, 30.0, 40.0, 0.25, 0.30, 1e6, 21.0, 0.025},
      {0.45, 0.87, 30.0, 40.0, 0.25, 0.30, 1.25e7, 21.0, 0.025},
      {1.0, 0.0, 3.0, 4.0, 0.0, 0.0, 1e4, 10.0, 0.025},
      {0.0, 0.0, 0.0, 0.0, 1.0, 1.0, 1e4, 10.0, 0.025},
      {-0.2, 0.1, -5.0, 7.5, 4.0, 0.01, 32769.0, 3.0, 0.05},      // just above the scheduling threshold; heading spread clamped
      {0.486, -0.648, 12.5, -3.0, 0.04, 2.25, 2.5e5, 8.0, 0.05},  // 3 sigma of the heading just inside the +-2 rad clamp
  };
  for (const Case& c : cases) {
    Schedule g{};
    schedule_from_moments(g, c.cbar, c.sbar, c.mx, c.my, c.vx, c.vy, c.n, c.mean_range, c.min_bin);
    std::printf("grid %u %u %u %u %.17g %.17g %.17g %.9g %.9g %.9g\n", g.nt, g.nx, g.ny, g.n_bins, g.c0, g.s0, g.half_u,
                static_cast<double>(g.kt), static_cast<double>(g.kx), static_cast<double>(g.ky));
  }
  for (int kx = 0; kx < 4; ++kx)
    for (uint32_t py = 0; py < 9; ++py)
      for (uint32_t px = 0; px < (4u << kx); ++px) std::printf("index %d %u %u %u\n", kx, px, py, bordered_index(px, py, kx));
  std::printf("max_bins %u\n", kScheduleMaxBins);
  // se2_math.cuh: the counter RNG (Philox4x32-10 keyed by seed, counter = index | step | stream) and the spatial hash
  const uint32_t kat[3][6] = {{0u, 0u, 0u, 0u, 0u, 0u},
                              {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu},
                              {0x243f6a88u, 0x85a308d3u, 0x13198a2eu, 0x03707344u, 0xa4093822u, 0x299f31d0u}};
  for (const auto& k : kat) {
    const Draw d = counter_draw((static_cast<uint64_t>(k[5]) << 32) | k[4], (static_cast<uint64_t>(k[1]) << 32) | k[0], k[2], k[3]);
    std::printf("philox %08x %08x %08x %08x\n", static_cast<uint32_t>(d.a), static_cast<uint32_t>(d.a >> 32), static_cast<uint32_t>(d.b),
                static_cast<uint32_t>(d.b >> 32));
  }
  for (uint64_t i = 0; i < 64; ++i) {
    const Draw d = counter_draw(0x9e3779b97f4a7c15ull, i * 0x100000001ull + 7, 3, kStreamRandomState);
    double z0, z1;
    box_muller(d, z0, z1);
    const Pose2 st = pose_from_xytheta(40.0 * uniform01(d.a) - 20.0, 40.0 * uniform01(d.b) - 20.0, 3.0 * z0);
    std::printf("hash %.17g %.17g %.17g %.17g %llu %llu %.17g %.17g %llu\n", st.c, st.s, st.x, st.y,
                static_cast<unsigned long long>(spatial_hash(st, 0.5, 0.5, 0.17453292519943295)),
                static_cast<unsigned long long>(spatial_hash(st, 0.05, 0.1, 0.01)), z0, z1,
                static_cast<unsigned long long>(mulhi64(d.a, d.b)));
  }
  return 0;
}
