// The point-cloud input of the C++ adaptors: beluga_b200::PointCloudView, point_cloud_points and
// Amcl::update(control, cloud), the counterpart of beluga_ros::Amcl::update(pose, SparsePointCloud3f)
// (beluga_ros/src/amcl.cpp:67-81).  Built by tests/test_cpp_point_cloud.py with g++ against libbeluga_b200.so, with and
// without the Sophus stub headers.  Without arguments only the host-side conversion runs; `--gpu` adds the filter updates.
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "beluga_b200/amcl.hpp"

namespace {

int g_failures = 0;
#define ASSERT_TRUE(cond)                                                               \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      std::fprintf(stderr, "%s:%d: assertion failed: %s\n", __FILE__, __LINE__, #cond); \
      ++g_failures;                                                                     \
      return;                                                                           \
    }                                                                                   \
  } while (0)

/// Velodyne-style records (x, y, z, intensity: FLOAT32, ring: UINT16, time: FLOAT32; 22 bytes, no padding).
std::vector<unsigned char> velodyne_records(const std::vector<std::array<float, 3>>& points) {
  constexpr std::size_t kStep = 22;
  std::vector<unsigned char> out(points.size() * kStep, 0);
  for (std::size_t i = 0; i < points.size(); ++i) {
    std::memcpy(out.data() + i * kStep, points[i].data(), 3 * sizeof(float));
    const float intensity = 1.1F, time = 0.1F;
    const std::uint16_t ring = 1;
    std::memcpy(out.data() + i * kStep + 12, &intensity, 4);
    std::memcpy(out.data() + i * kStep + 16, &ring, 2);
    std::memcpy(out.data() + i * kStep + 18, &time, 4);
  }
  return out;
}

std::vector<std::array<float, 3>> ring_of_points(std::size_t n, float radius) {
  std::vector<std::array<float, 3>> pts;
  for (std::size_t i = 0; i < n; ++i) {
    const double a = 2.0 * 3.14159265358979323846 * static_cast<double>(i) / static_cast<double>(n);
    pts.push_back({static_cast<float>(radius * std::cos(a)), static_cast<float>(radius * std::sin(a)), static_cast<float>(0.1 * static_cast<double>(i % 4))});
  }
  return pts;
}

// yaw 90 degrees, lifted by 0.5 m, shifted by (0.3, -0.2)
const std::array<double, 12> kOrigin = {0.0, -1.0, 0.0, 0.3, 1.0, 0.0, 0.0, -0.2, 0.0, 0.0, 1.0, 0.5};

void PointsFollowTheOrigin() {
  const auto pts = ring_of_points(8, 2.0F);
  const auto bytes = velodyne_records(pts);
  const beluga_b200::PointCloudView view{bytes.data(), pts.size(), 22, 0, BB200_POINT_FLOAT32, kOrigin.data()};
  const auto xy = beluga_b200::point_cloud_points(view);
  ASSERT_TRUE(xy.size() == pts.size());
  for (std::size_t i = 0; i < pts.size(); ++i) {
    const double x = pts[i][0], y = pts[i][1], z = pts[i][2];
    ASSERT_TRUE(xy[i].first == ((0.0 * x + -1.0 * y) + 0.0 * z) + 0.3);
    ASSERT_TRUE(xy[i].second == ((1.0 * x + 0.0 * y) + 0.0 * z) + -0.2);
  }
  const beluga_b200::PointCloudView plain{bytes.data(), pts.size(), 22, 0, BB200_POINT_FLOAT32, nullptr};
  const auto same = beluga_b200::point_cloud_points(plain);
  for (std::size_t i = 0; i < pts.size(); ++i) ASSERT_TRUE(same[i].first == pts[i][0] && same[i].second == pts[i][1]);
}

void BadLayoutThrows() {
  const auto bytes = velodyne_records(ring_of_points(2, 1.0F));
  for (const beluga_b200::PointCloudView& bad : {beluga_b200::PointCloudView{bytes.data(), 2, 22, 12, BB200_POINT_FLOAT32, nullptr},
                                                  beluga_b200::PointCloudView{bytes.data(), 2, 22, 0, static_cast<bb200_point_datatype>(5), nullptr},
                                                  beluga_b200::PointCloudView{nullptr, 2, 22, 0, BB200_POINT_FLOAT32, nullptr}}) {
    bool thrown = false;
    try {
      (void)beluga_b200::point_cloud_points(bad);
    } catch (const beluga_b200::Error& e) {
      thrown = e.status() == BB200_ERR_INVALID_ARGUMENT;
    }
    ASSERT_TRUE(thrown);
  }
}

#ifdef BELUGA_B200_WITH_SOPHUS
/// Shaped like beluga_ros::SparsePointCloud3f: points() as 3-vectors, origin() as Sophus::SE3d.
struct Vec3f {
  float v[3];
  float x() const { return v[0]; }
  float y() const { return v[1]; }
  float z() const { return v[2]; }
};
struct StubSparseCloud {
  std::vector<Vec3f> pts;
  Sophus::SE3d frame;
  const std::vector<Vec3f>& points() const { return pts; }
  const Sophus::SE3d& origin() const { return frame; }
};

StubSparseCloud stub_cloud(const std::vector<std::array<float, 3>>& pts) {
  StubSparseCloud c;
  for (const auto& p : pts) c.pts.push_back(Vec3f{{p[0], p[1], p[2]}});
  Sophus::Matrix3x4d m{};
  for (int k = 0; k < 12; ++k) m.m[k] = kOrigin[static_cast<std::size_t>(k)];
  c.frame = Sophus::SE3d{m};
  return c;
}

static_assert(beluga_b200::is_sparse_point_cloud_v<StubSparseCloud>, "a BaseSparsePointCloud-shaped type is recognised");
static_assert(!beluga_b200::is_sparse_point_cloud_v<std::vector<std::pair<double, double>>>, "a measurement vector is not a cloud");

void SparseCloudPacksLikeTheView() {
  const auto pts = ring_of_points(16, 3.0F);
  const beluga_b200::PackedPointCloud packed{stub_cloud(pts)};
  const auto bytes = velodyne_records(pts);
  const auto a = beluga_b200::point_cloud_points(packed.view());
  const auto b = beluga_b200::point_cloud_points(beluga_b200::PointCloudView{bytes.data(), pts.size(), 22, 0, BB200_POINT_FLOAT32, kOrigin.data()});
  ASSERT_TRUE(a == b);
}
#endif

// ---- on the GPU --------------------------------------------------------------------------------

using Grid = beluga_b200::OccupancyGrid;

Grid walled_grid() {  // 40 x 40 cells of 0.1 m with a wall all around
  std::vector<std::int8_t> cells(40 * 40, 0);
  for (int i = 0; i < 40; ++i) {
    cells[static_cast<std::size_t>(i)] = cells[static_cast<std::size_t>(39 * 40 + i)] = 100;
    cells[static_cast<std::size_t>(i * 40)] = cells[static_cast<std::size_t>(i * 40 + 39)] = 100;
  }
  return Grid{cells, 40, 0.1};
}

auto make_amcl() {
  beluga_b200::AmclParams params;
  params.min_particles = params.max_particles = 4096;
  params.seed = 9;
  return beluga_b200::Amcl{beluga_b200::DifferentialDriveModel{beluga_b200::DifferentialDriveModelParam{0.1, 0.05, 0.1, 0.05}},
                           beluga_b200::LikelihoodFieldModel<Grid>{beluga_b200::LikelihoodFieldModelParam{}, walled_grid()}, params};
}

void UpdateWithCloudEqualsUpdateWithPoints() {
  auto a = make_amcl();
  auto b = make_amcl();
  const beluga_b200::Matrix3d cov{0.01, 0, 0, 0, 0.01, 0, 0, 0, 0.01};
  a.initialize(beluga_b200::SE2d{0.0, 2.0, 2.0}, cov);
  b.initialize(beluga_b200::SE2d{0.0, 2.0, 2.0}, cov);
  const auto pts = ring_of_points(3000, 1.5F);
  const auto bytes = velodyne_records(pts);
  const beluga_b200::PointCloudView view{bytes.data(), pts.size(), 22, 0, BB200_POINT_FLOAT32, kOrigin.data()};
  const auto ea = a.update(beluga_b200::SE2d{}, view);
  const auto eb = b.update(beluga_b200::SE2d{}, beluga_b200::point_cloud_points(view));
  ASSERT_TRUE(ea.has_value() && eb.has_value());
  ASSERT_TRUE(ea->first.v == eb->first.v && ea->second == eb->second);
  ASSERT_TRUE(a.particles().states.size() == b.particles().states.size());
  const auto pa = a.particles(), pb = b.particles();
  for (std::size_t i = 0; i < pa.states.size(); ++i) ASSERT_TRUE(pa.states[i].v == pb.states[i].v && pa.weights[i] == pb.weights[i]);
#ifdef BELUGA_B200_WITH_SOPHUS
  auto c = make_amcl();
  c.initialize(beluga_b200::SE2d{0.0, 2.0, 2.0}, cov);
  const auto ec = c.update(beluga_b200::SE2d{}, stub_cloud(pts));
  ASSERT_TRUE(ec.has_value() && ec->first.v == ea->first.v && ec->second == ea->second);
#endif
  bool thrown = false;
  try {
    a.force_update();
    (void)a.update(beluga_b200::SE2d{}, beluga_b200::PointCloudView{bytes.data(), pts.size(), 10, 0, BB200_POINT_FLOAT32, nullptr});
  } catch (const beluga_b200::Error& e) {
    thrown = e.status() == BB200_ERR_INVALID_ARGUMENT;
  }
  ASSERT_TRUE(thrown);
}

}  // namespace

int main(int argc, char** argv) {
  PointsFollowTheOrigin();
  BadLayoutThrows();
#ifdef BELUGA_B200_WITH_SOPHUS
  SparseCloudPacksLikeTheView();
#endif
  if (argc > 1 && std::string(argv[1]) == "--gpu") UpdateWithCloudEqualsUpdateWithPoints();
  if (g_failures == 0) std::printf("CPP_POINT_CLOUD_OK\n");
  return g_failures == 0 ? 0 : 1;
}
