// Host-only probe: prints what csrc/kernels.cuh's schedule_from_moments and bordered_index compute, so that the CPU model
// tests (tests/test_schedule_model.py, tests/test_fixed_point_lookup_model.py) are checked against the code the kernels
// are built from, not only against their own restatement.  Compiled with nvcc, runs without a GPU (no CUDA call).
#include <cstdio>
#include <cstring>

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
  // the spatial hash where floor() leaves the int64 range (tests/test_integer_edges_cpu.py): values as bit patterns
  const uint64_t edges[] = {
      0x0000000000000000ull, 0x8000000000000000ull,  // +-0
      0x0000000000000001ull, 0x8000000000000001ull, 0x000fffffffffffffull, 0x800fffffffffffffull,  // subnormals
      0x3ff0000000000000ull, 0x3fefffffffffffffull, 0x3ff0000000000001ull,  // 1 and one ulp either side
      0xbff0000000000000ull, 0xbfefffffffffffffull, 0xbff0000000000001ull,  // -1 and one ulp either side
      0x4059000000000000ull, 0x4058ffffffffffffull, 0x4059000000000001ull,  // 100 and one ulp either side
      0xbfe0000000000000ull, 0xbf847ae147ae147bull, 0x8000000000000010ull,  // -0.5, -0.01, a negative subnormal
      0x4340000000000000ull, 0xc340000000000000ull, 0x4340000000000001ull,  // +-2^53, 2^53 + 2
      0x43dfffffffffffffull, 0xc3dfffffffffffffull,  // +-(2^63 - 1024)
      0x43e0000000000000ull, 0xc3e0000000000000ull,  // +-2^63
      0x43e0000000000001ull, 0xc3e0000000000001ull,  // one ulp beyond +-2^63
      0x7e37e43c8800759cull, 0xfe37e43c8800759cull,  // +-1e300
      0x7fefffffffffffffull, 0xffefffffffffffffull,  // +-DBL_MAX
      0x7ff0000000000000ull, 0xfff0000000000000ull,  // +-inf
      0x7ff8000000000000ull, 0xfff8000000000000ull, 0x7ff0000000000001ull,  // NaNs
  };
  for (const uint64_t bits : edges) {
    double v;
    std::memcpy(&v, &bits, sizeof v);
    std::printf("floor %016llx %lld %llu %llu\n", static_cast<unsigned long long>(bits), static_cast<long long>(floor_to_int64(v)),
                static_cast<unsigned long long>(floor_and_fibo_hash(v, 0)), static_cast<unsigned long long>(floor_and_fibo_hash(v, 21)));
    // the value as x, as y, and as the heading's cosine and sine (the bucket of atan2(s, c)), at resolutions that keep
    // the quotient exact (1, 0.5) or push it past the int64 range (rtheta = 5e-324)
    const Pose2 poses[] = {{1.0, 0.0, v, 0.25}, {1.0, 0.0, 0.25, v}, {v, 0.0, 0.25, 0.25}, {-1.0, v, 0.25, 0.25}, {1.0, v, 0.25, 0.25}};
    for (const Pose2& st : poses)
      std::printf("pose %016llx %.17g %.17g %.17g %.17g %llu %llu %llu\n", static_cast<unsigned long long>(bits), st.c, st.s, st.x, st.y,
                  static_cast<unsigned long long>(spatial_hash(st, 1.0, 1.0, 0.1)),
                  static_cast<unsigned long long>(spatial_hash(st, 0.5, 0.5, 0.17453292519943295)),
                  static_cast<unsigned long long>(spatial_hash(st, 0.5, 0.5, 5e-324)));
  }
  return 0;
}
