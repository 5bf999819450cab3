// The landmark and bearing sensor models of one particle (host + device): LandmarkSensorModel2d
// (sensor/landmark_sensor_model.hpp:96-156) and BearingSensorModel2d (sensor/bearing_sensor_model.hpp:92-140) over a
// beluga::LandmarkMap (sensor/data/landmark_map.hpp:40-166).  The reweight kernel (reweight_landmark.cu) and the host
// probe (tests/cpp/landmark_probe.cpp) run these same functions.
//
// Evaluation order, fixed here because Sophus SO3/SE3 and Eigen are not part of the reference checkout (DESIGN.md §1):
//   - the rotation about z is the particle's stored unit complex (c, s), not SO3d::rotZ(so2().log());
//   - R * p is ((R00 p0 + R01 p1) + R02 p2) row by row, with the zero entries of the z rotation left out;
//     a pose applied to a point is R * p + t, its inverse R^T * (p - t);
//   - dot products and squared norms add left to right; norm() is sqrt(squaredNorm());
//   - normalized() is v / sqrt(squaredNorm) when squaredNorm > 0 and v unchanged otherwise (Eigen's rule);
//   - no contraction anywhere (the library is built with -fmad=false, the probe with -ffp-contract=off).
// The landmark a detection is matched to depends only on correctly rounded +, -, *, / and sqrt, so it is the oracle's bit
// for bit; the factor goes through exp and atan2, which may differ from glibc by a few ulps on the device.
#pragma once

#include <cmath>
#include <cstdint>

#include "../../include/beluga_b200.h"
#include "se2_math.cuh"

namespace bb200 {

/// One landmark of the device map: its position in the world frame (the category is implied by its slice).
struct __attribute__((aligned(32))) LandmarkPoint {
  double x, y, z, pad;
};

/// The particle-independent part of one detection, prepared on the host (prepare_detections).
struct __attribute__((aligned(16))) LandmarkDetection {
  double p[3];     // landmark model: the position in the robot frame; bearing model: the bearing in the sensor frame, as given
  double u[3];     // p.normalized()
  double range;    // landmark model: p.norm()
  uint32_t begin;  // the detection's candidates: landmarks [begin, end) of the category-sorted map
  uint32_t end;
};

/// Model constants.  The denominators are the reference's (2. * sigma * sigma), evaluated once on the host.
struct LandmarkParams {
  int model{0};  // BB200_SENSOR_LANDMARK or BB200_SENSOR_BEARING
  double range_den{1.0}, bearing_den{1.0};
  double random_prob{0.0};
  double sensor_r[9]{1, 0, 0, 0, 1, 0, 0, 0, 1};  // bearing model: sensor_pose_in_robot, row-major R ...
  double sensor_t[3]{0, 0, 0};                   // ... and t
};

struct Vec3 {
  double x, y, z;
};

BB_HD double lm_dot(const Vec3& a, const Vec3& b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
BB_HD Vec3 lm_normalized(const Vec3& v) {
  const double n = lm_dot(v, v);
  if (n > 0.0) {
    const double r = sqrt(n);
    return Vec3{v.x / r, v.y / r, v.z / r};
  }
  return v;
}
BB_HD double lm_cross_norm(const Vec3& a, const Vec3& b) {
  const Vec3 c{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
  return sqrt(lm_dot(c, c));
}
/// atan2(|a x b|, a . b): the aperture angle of both models (landmark_sensor_model.hpp:137-139, bearing_sensor_model.hpp:125-129).
BB_HD double lm_aperture(const Vec3& a, const Vec3& b) { return atan2(lm_cross_norm(a, b), lm_dot(a, b)); }
BB_HD double lm_gauss(double e, double den) { return exp(-e * e / den); }

/// The frame a particle reads its candidates in.  Landmark model: the robot pose (R = Rz(c, s), t = (x, y, 0)).  Bearing
/// model: the sensor pose in the world, robot_pose * sensor_pose_in_robot (bearing_sensor_model.hpp:107).
struct LandmarkFrame {
  double r[9];
  double t[3];
};

BB_HD LandmarkFrame landmark_frame(const Pose2& st, const LandmarkParams& p) {
  LandmarkFrame f;
  if (p.model == BB200_SENSOR_BEARING) {
    const double* R = p.sensor_r;
    for (int j = 0; j < 3; ++j) {
      f.r[j] = st.c * R[j] - st.s * R[3 + j];
      f.r[3 + j] = st.s * R[j] + st.c * R[3 + j];
      f.r[6 + j] = R[6 + j];
    }
    f.t[0] = (st.c * p.sensor_t[0] - st.s * p.sensor_t[1]) + st.x;
    f.t[1] = (st.s * p.sensor_t[0] + st.c * p.sensor_t[1]) + st.y;
    f.t[2] = p.sensor_t[2];
  } else {
    f.r[0] = st.c, f.r[1] = -st.s, f.r[2] = 0.0;
    f.r[3] = st.s, f.r[4] = st.c, f.r[5] = 0.0;
    f.r[6] = 0.0, f.r[7] = 0.0, f.r[8] = 1.0;
    f.t[0] = st.x, f.t[1] = st.y, f.t[2] = 0.0;
  }
  return f;
}

/// frame^-1 * l = R^T * (l - t).
BB_HD Vec3 lm_to_frame(const LandmarkFrame& f, double lx, double ly, double lz) {
  const double dx = lx - f.t[0], dy = ly - f.t[1], dz = lz - f.t[2];
  return Vec3{(f.r[0] * dx + f.r[3] * dy) + f.r[6] * dz, (f.r[1] * dx + f.r[4] * dy) + f.r[7] * dz, (f.r[2] * dx + f.r[5] * dy) + f.r[8] * dz};
}

/// The landmark model's query point: the detection in the world frame, robot_pose * p (landmark_sensor_model.hpp:120).
BB_HD Vec3 lm_query(const LandmarkFrame& f, const LandmarkDetection& d) {
  return Vec3{(f.r[0] * d.p[0] + f.r[1] * d.p[1]) + f.t[0], (f.r[3] * d.p[0] + f.r[4] * d.p[1]) + f.t[1], d.p[2] + f.t[2]};
}

/// The search key of one candidate.  Landmark model: the squared distance to the query point (landmark_map.hpp:98-101).
/// Bearing model: the dot product of the candidate's bearing in the sensor frame with the detection as given (:145-152).
template <int kModel>
BB_HD double landmark_key(const LandmarkFrame& f, const LandmarkDetection& d, const Vec3& query, const LandmarkPoint& l) {
  if (kModel == BB200_SENSOR_BEARING) {
    const Vec3 b = lm_normalized(lm_to_frame(f, l.x, l.y, l.z));
    return lm_dot(b, Vec3{d.p[0], d.p[1], d.p[2]});
  }
  const Vec3 e{l.x - query.x, l.y - query.y, l.z - query.z};
  return lm_dot(e, e);
}

/// std::min_element's step with the reference's comparators: the candidate replaces the current minimum only when it is
/// strictly better (distance a < b, bearing dot_a > dot_b); a NaN comparison keeps the current one.
template <int kModel>
BB_HD bool landmark_better(double candidate, double best) {
  return kModel == BB200_SENSOR_BEARING ? candidate > best : candidate < best;
}

/// The factor of one detection given its matched landmark (`found` false: no landmark of the category).
template <int kModel>
BB_HD double landmark_factor(const LandmarkFrame& f, const LandmarkDetection& d, bool found, const LandmarkPoint& l, const LandmarkParams& p) {
  const Vec3 u{d.u[0], d.u[1], d.u[2]};
  if (kModel == BB200_SENSOR_BEARING) {
    if (!found) return 0.0;  // bearing_sensor_model.hpp:115-117
    const Vec3 b = lm_normalized(lm_to_frame(f, l.x, l.y, l.z));
    return lm_gauss(lm_aperture(u, b), p.bearing_den);  // :120-134
  }
  if (!found) return p.random_prob;  // landmark_sensor_model.hpp:126-128
  const Vec3 q = lm_to_frame(f, l.x, l.y, l.z);  // :133
  const double range = sqrt(lm_dot(q, q));
  const Vec3 b = lm_normalized(q);
  const double bearing_error = lm_aperture(b, u);
  const double range_error = d.range - range;
  return lm_gauss(range_error, p.range_den) * lm_gauss(bearing_error, p.bearing_den) + p.random_prob;  // :146-152
}

/// std::transform_reduce(first, last, 1.0, std::multiplies{}, f) as libstdc++ 13 evaluates it (<numeric>:439-462):
/// init *= ((f0 * f1) * (f2 * f3)) per group of four, then a scalar tail.
struct ProductByFours {
  double init{1.0};
  double f[3];
  int k{0};
  BB_HD void push(double v) {
    if (k < 3) {
      f[k++] = v;
    } else {
      init = init * ((f[0] * f[1]) * (f[2] * v));
      k = 0;
    }
  }
  BB_HD double finish() const {
    double r = init;
    for (int i = 0; i < k; ++i) r = r * f[i];
    return r;
  }
};

/// The whole per-particle likelihood over `n` detections and the category-sorted landmarks: the body the kernel runs with
/// its candidates staged through shared memory.
template <int kModel>
BB_HD double landmark_likelihood(const Pose2& st, const LandmarkDetection* det, uint32_t n, const LandmarkPoint* landmarks, const LandmarkParams& p) {
  const LandmarkFrame f = landmark_frame(st, p);
  ProductByFours prod;
  for (uint32_t k = 0; k < n; ++k) {
    const LandmarkDetection& d = det[k];
    const Vec3 query = kModel == BB200_SENSOR_BEARING ? Vec3{0.0, 0.0, 0.0} : lm_query(f, d);
    uint32_t best = d.begin;
    double best_key = 0.0;
    for (uint32_t j = d.begin; j < d.end; ++j) {
      const double key = landmark_key<kModel>(f, d, query, landmarks[j]);
      if (j == d.begin || landmark_better<kModel>(key, best_key)) best = j, best_key = key;
    }
    const bool found = d.end > d.begin;
    prod.push(landmark_factor<kModel>(f, d, found, found ? landmarks[best] : LandmarkPoint{0, 0, 0, 0}, p));
  }
  return prod.finish();
}

}  // namespace bb200
