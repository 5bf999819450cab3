// Landmark and bearing sensor models of one filter: the host preparation of a landmark map and of a step's detections,
// and the reweight kernel.
#include "reweight_landmark.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>

#include "device_map.hpp"
#include "reweight_landmark_block.cuh"

namespace bb200 {

namespace {

template <int kModel>
__global__ void __launch_bounds__(kLandmarkThreads)
    reweight_landmark_kernel(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, LandmarkParams params,
                             const LandmarkPoint* __restrict__ landmarks, const LandmarkDetection* __restrict__ detections, uint32_t n_detections,
                             Scalars* __restrict__ scalars) {
  reweight_landmark_block<kModel>(states, weights, n, params, landmarks, detections, n_detections, scalars, blockIdx.x);
}

bool positive_finite(double v) { return std::isfinite(v) && v > 0.0; }

/// R R^T = I and det R = 1, each within 1e-9.
bool is_rotation(const double m[12]) {
  for (int k = 0; k < 12; ++k)
    if (!std::isfinite(m[k])) return false;
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) {
      const double d = m[4 * a] * m[4 * b] + m[4 * a + 1] * m[4 * b + 1] + m[4 * a + 2] * m[4 * b + 2];
      if (std::fabs(d - (a == b ? 1.0 : 0.0)) > 1e-9) return false;
    }
  }
  const double det = m[0] * (m[5] * m[10] - m[6] * m[9]) - m[1] * (m[4] * m[10] - m[6] * m[8]) + m[2] * (m[4] * m[9] - m[5] * m[8]);
  return std::fabs(det - 1.0) <= 1e-9;
}

}  // namespace

void launch_reweight_landmark(const Pose2* states, double* weights, uint64_t n, const LandmarkParams& params, const LandmarkPoint* landmarks,
                              const LandmarkDetection* detections, uint32_t n_detections, Scalars* scalars, cudaStream_t stream) {
  if (n == 0) return;
  const unsigned blocks = static_cast<unsigned>((n + kLandmarkThreads - 1) / kLandmarkThreads);
  if (params.model == BB200_SENSOR_BEARING) {
    reweight_landmark_kernel<BB200_SENSOR_BEARING><<<blocks, kLandmarkThreads, 0, stream>>>(states, weights, n, params, landmarks, detections,
                                                                                             n_detections, scalars);
  } else {
    reweight_landmark_kernel<BB200_SENSOR_LANDMARK><<<blocks, kLandmarkThreads, 0, stream>>>(states, weights, n, params, landmarks, detections,
                                                                                              n_detections, scalars);
  }
}

int prepare_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map, MapTables* out,
                         std::string* error) {
  if (map.n > 0 && map.landmarks == nullptr) return reject(BB200_ERR_INVALID_ARGUMENT, "landmarks is null", error);
  if (map.n >= 0xffffffffull) return reject(BB200_ERR_INVALID_ARGUMENT, "too many landmarks", error);
  if ((map.bounds_min3 == nullptr) != (map.bounds_max3 == nullptr))
    return reject(BB200_ERR_INVALID_ARGUMENT, "bounds_min3 and bounds_max3 are both given or both null", error);
  LandmarkParams p;
  if (lp != nullptr) {
    if (!positive_finite(lp->sigma_range) || !positive_finite(lp->sigma_bearing))
      return reject(BB200_ERR_INVALID_ARGUMENT, "sigma_range and sigma_bearing must be positive and finite", error);
    if (!(lp->random_prob >= 0.0 && lp->random_prob <= 1.0)) return reject(BB200_ERR_INVALID_ARGUMENT, "random_prob must lie in [0, 1]", error);
    p.model = BB200_SENSOR_LANDMARK;
    p.range_den = 2. * lp->sigma_range * lp->sigma_range;  // landmark_sensor_model.hpp:147
    p.bearing_den = 2. * lp->sigma_bearing * lp->sigma_bearing;
    p.random_prob = lp->random_prob;
  } else {
    if (!positive_finite(bp->sigma_bearing)) return reject(BB200_ERR_INVALID_ARGUMENT, "sigma_bearing must be positive and finite", error);
    if (!is_rotation(bp->sensor_pose_in_robot))
      return reject(BB200_ERR_INVALID_ARGUMENT, "sensor_pose_in_robot must be a finite [R | t] with R a rotation (within 1e-9)", error);
    p.model = BB200_SENSOR_BEARING;
    p.bearing_den = 2. * bp->sigma_bearing * bp->sigma_bearing;  // bearing_sensor_model.hpp:134
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) p.sensor_r[3 * r + c] = bp->sensor_pose_in_robot[4 * r + c];
      p.sensor_t[r] = bp->sensor_pose_in_robot[4 * r + 3];
    }
  }
  *out = MapTables{};
  out->sensor = p.model;
  out->landmark = p;
  // Stable sort by category: each category is one contiguous slice in the map's own order, so the first minimum of a
  // slice is the first minimum of the reference's filtered view (landmark_map.hpp:84-92).
  std::vector<uint64_t> order(map.n);
  std::iota(order.begin(), order.end(), uint64_t{0});
  std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return map.landmarks[a].category < map.landmarks[b].category; });
  out->landmark_points.reserve(map.n);
  for (uint64_t k = 0; k < map.n; ++k) {
    const bb200_landmark& l = map.landmarks[order[k]];
    out->landmark_points.push_back(LandmarkPoint{l.x, l.y, l.z, 0.0});
    if (out->landmark_slices.empty() || out->landmark_slices.back().category != l.category)
      out->landmark_slices.push_back(LandmarkSlice{l.category, static_cast<uint32_t>(k), static_cast<uint32_t>(k)});
    out->landmark_slices.back().end = static_cast<uint32_t>(k + 1);
  }
  out->n_landmarks = static_cast<uint32_t>(map.n);
  // The box of MultivariateUniformDistribution<SE2d, AlignedBox2d>: the explicit bounds, or cwiseMin / cwiseMax over
  // the landmarks from the first one (landmark_map.hpp:61-71); an empty map without bounds has an empty box.
  if (map.bounds_min3 != nullptr) {
    out->box[0] = map.bounds_min3[0], out->box[1] = map.bounds_max3[0], out->box[2] = map.bounds_min3[1], out->box[3] = map.bounds_max3[1];
  } else if (map.n > 0) {
    out->box[0] = out->box[1] = map.landmarks[0].x;
    out->box[2] = out->box[3] = map.landmarks[0].y;
    for (uint64_t k = 1; k < map.n; ++k) {
      const bb200_landmark& l = map.landmarks[k];
      out->box[0] = l.x < out->box[0] ? l.x : out->box[0];
      out->box[1] = out->box[1] < l.x ? l.x : out->box[1];
      out->box[2] = l.y < out->box[2] ? l.y : out->box[2];
      out->box[3] = out->box[3] < l.y ? l.y : out->box[3];
    }
  }
  const double* b = out->box;
  out->box_valid = (map.bounds_min3 != nullptr || map.n > 0) && std::isfinite(b[0]) && std::isfinite(b[1]) && std::isfinite(b[2]) &&
                   std::isfinite(b[3]) && b[0] <= b[1] && b[2] <= b[3];
  return BB200_OK;
}

void prepare_detections(const std::vector<LandmarkSlice>& slices, const bb200_landmark_detection* in, uint64_t n, std::vector<LandmarkDetection>* out) {
  out->resize(n);
  for (uint64_t k = 0; k < n; ++k) {
    LandmarkDetection& d = (*out)[k];
    const Vec3 p{in[k].x, in[k].y, in[k].z};
    const Vec3 u = lm_normalized(p);
    d.p[0] = p.x, d.p[1] = p.y, d.p[2] = p.z;
    d.u[0] = u.x, d.u[1] = u.y, d.u[2] = u.z;
    d.range = std::sqrt(lm_dot(p, p));  // landmark_sensor_model.hpp:116
    const auto it = std::lower_bound(slices.begin(), slices.end(), in[k].category,
                                     [](const LandmarkSlice& s, uint32_t c) { return s.category < c; });
    const bool found = it != slices.end() && it->category == in[k].category;
    d.begin = found ? it->begin : 0;
    d.end = found ? it->end : 0;
  }
}

}  // namespace bb200
