// Host-only probe of csrc/reweight_landmark.cuh, the per-particle body of the landmark reweight kernel
// (tests/test_landmark_oracle_cpu.py).  Built with g++ -ffp-contract=off; needs no GPU and no CUDA header.
//
// Reads cases from the file named by argv[1], each a run of doubles:
//   model (3 landmark, 4 bearing), n_states, n_detections, n_landmarks, sigma_range, sigma_bearing, random_prob,
//   sensor_pose_in_robot[12], then n_states x {c, s, x, y}, n_detections x {x, y, z, category},
//   n_landmarks x {x, y, z, category} in map order,
// and writes landmark_likelihood of every state, case after case, as doubles to argv[2].  The map is stably sorted by
// category and the detections are prepared here as the library prepares them.
#include <algorithm>
#include <cstdio>
#include <numeric>
#include <vector>

#include "reweight_landmark.cuh"

using namespace bb200;

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  FILE* out = std::fopen(argv[2], "wb");
  if (in == nullptr || out == nullptr) return 2;
  double head[19];
  while (std::fread(head, sizeof(double), 19, in) == 19) {
    const int model = static_cast<int>(head[0]);
    const size_t n = static_cast<size_t>(head[1]), nd = static_cast<size_t>(head[2]), nl = static_cast<size_t>(head[3]);
    std::vector<double> st(4 * n), det(4 * nd), lm(4 * nl);
    if (std::fread(st.data(), sizeof(double), st.size(), in) != st.size() || std::fread(det.data(), sizeof(double), det.size(), in) != det.size() ||
        std::fread(lm.data(), sizeof(double), lm.size(), in) != lm.size())
      return 3;
    LandmarkParams p;
    p.model = model;
    p.range_den = 2. * head[4] * head[4];
    p.bearing_den = 2. * head[5] * head[5];
    p.random_prob = head[6];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) p.sensor_r[3 * r + c] = head[7 + 4 * r + c];
      p.sensor_t[r] = head[7 + 4 * r + 3];
    }
    std::vector<size_t> order(nl);
    std::iota(order.begin(), order.end(), size_t{0});
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return lm[4 * a + 3] < lm[4 * b + 3]; });
    std::vector<LandmarkPoint> points;
    for (size_t k : order) points.push_back(LandmarkPoint{lm[4 * k], lm[4 * k + 1], lm[4 * k + 2], 0.0});
    std::vector<LandmarkDetection> d(nd);
    for (size_t k = 0; k < nd; ++k) {
      const Vec3 v{det[4 * k], det[4 * k + 1], det[4 * k + 2]};
      const Vec3 u = lm_normalized(v);
      d[k] = LandmarkDetection{{v.x, v.y, v.z}, {u.x, u.y, u.z}, std::sqrt(lm_dot(v, v)), 0, 0};
      for (size_t j = 0; j < nl; ++j) {
        if (lm[4 * order[j] + 3] != det[4 * k + 3]) continue;
        if (d[k].end == 0) d[k].begin = static_cast<uint32_t>(j);
        d[k].end = static_cast<uint32_t>(j + 1);
      }
    }
    std::vector<double> w(n);
    for (size_t i = 0; i < n; ++i) {
      const Pose2 s{st[4 * i], st[4 * i + 1], st[4 * i + 2], st[4 * i + 3]};
      w[i] = model == BB200_SENSOR_BEARING ? landmark_likelihood<BB200_SENSOR_BEARING>(s, d.data(), static_cast<uint32_t>(nd), points.data(), p)
                                           : landmark_likelihood<BB200_SENSOR_LANDMARK>(s, d.data(), static_cast<uint32_t>(nd), points.data(), p);
    }
    std::fwrite(w.data(), sizeof(double), n, out);
  }
  std::fclose(in);
  std::fclose(out);
  return 0;
}
