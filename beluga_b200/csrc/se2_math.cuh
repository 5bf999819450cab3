// SE(2) arithmetic and the counter RNG of the CUDA MCL backend (host + device).
//
// Particle states are Sophus::SE2d values in the reference; every operation the hot path applies
// to them is reproduced here with the same order of floating-point operations, because pose
// parity is judged to 1e-5 on the mean/covariance and the likelihood-field lookup depends on the
// exact cell each beam end point lands in.  Reference call sites (relative to
// /root/reference/beluga/include/beluga): motion/differential_drive_model.hpp:136-139,158-162,
// sensor/likelihood_field_model.hpp:70-74, algorithm/raycasting.hpp:69,81-85,
// algorithm/spatial_hash.hpp:190-193, policies/on_motion.hpp:63-67.
//
// Sophus 1.22.10 conventions followed (Sophus itself is not part of the reference checkout):
// SO2 is a unit complex {cos, sin}; the (real, imag) constructor and exp() normalise through
// hypot; the group product renormalises with 2/(1+|z|^2) when |z|^2 != 1 and then goes through
// that constructor; inverse() conjugates (through the constructor); log() is atan2(sin, cos).
//
// This translation unit is compiled with -fmad=false / -ffp-contract=off: the reference targets
// baseline x86-64, where a*b+c rounds twice.
#pragma once

#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define BB_HD __host__ __device__ __forceinline__
#else
#define BB_HD inline
#endif

namespace bb200 {

struct Rot2 {
  double c, s;
};

/// A particle state / pose in Sophus::SE2d::data() order.
struct __attribute__((aligned(32))) Pose2 {
  double c, s, x, y;
};

BB_HD Rot2 rot_make(double re, double im) {
  const double len = hypot(re, im);
  return Rot2{re / len, im / len};
}
BB_HD Rot2 rot_exp(double theta) { return rot_make(cos(theta), sin(theta)); }
BB_HD Rot2 rot_inverse(const Rot2& r) { return rot_make(r.c, -r.s); }
BB_HD double rot_log(const Rot2& r) { return atan2(r.s, r.c); }
BB_HD Rot2 rot_mul(const Rot2& a, const Rot2& b) {
  double re = a.c * b.c - a.s * b.s;
  double im = a.c * b.s + a.s * b.c;
  const double sq = re * re + im * im;
  if (sq != 1.0) {
    const double scale = 2.0 / (1.0 + sq);
    re = re * scale;
    im = im * scale;
  }
  return rot_make(re, im);
}

BB_HD Pose2 pose_mul(const Pose2& a, const Pose2& b) {
  const Rot2 r = rot_mul(Rot2{a.c, a.s}, Rot2{b.c, b.s});
  const double rx = a.c * b.x - a.s * b.y;
  const double ry = a.s * b.x + a.c * b.y;
  return Pose2{r.c, r.s, a.x + rx, a.y + ry};
}
BB_HD Pose2 pose_inverse(const Pose2& a) {
  const Rot2 inv = rot_inverse(Rot2{a.c, a.s});
  const double nx = a.x * -1.0, ny = a.y * -1.0;
  return Pose2{inv.c, inv.s, inv.c * nx - inv.s * ny, inv.s * nx + inv.c * ny};
}
BB_HD Pose2 pose_from_xytheta(double x, double y, double theta) {
  const Rot2 r = rot_exp(theta);
  return Pose2{r.c, r.s, x, y};
}

/// state * SE2{SO2{rot1}, (0,0)} * SE2{SO2{rot2}, (trans, 0)} -- differential_drive_model.hpp:158-162.
BB_HD Pose2 diff_drive_apply(const Pose2& st, double rot1, double trans, double rot2) {
  const Rot2 r1 = rot_exp(rot1);
  const Rot2 r2 = rot_exp(rot2);
  const Pose2 a = pose_mul(st, Pose2{r1.c, r1.s, 0.0, 0.0});
  return pose_mul(a, Pose2{r2.c, r2.s, trans, 0.0});
}

/// The per-particle composition of the three motion models given their three sampled scalars.
///   0 differential   (differential_drive_model.hpp:158-162)
///   1 omnidirectional (omnidirectional_drive_model.hpp:138-144): second = SO2(d0) * first^-1,
///     translation = (d1, -d2), state * SE2(first, 0) * SE2(second, translation)
///   2 stationary     (stationary_model.hpp:56-58): state * SE2(SO2(d0), (d1, d2))
BB_HD Pose2 motion_apply(int model, const Pose2& st, double d0, double d1, double d2, const Rot2& first) {
  if (model == 1) {
    const Rot2 second = rot_mul(rot_exp(d0), rot_inverse(first));
    const Pose2 a = pose_mul(st, Pose2{first.c, first.s, 0.0, 0.0});
    return pose_mul(a, Pose2{second.c, second.s, d1, -d2});
  }
  if (model == 2) {
    const Rot2 r = rot_exp(d0);
    return pose_mul(st, Pose2{r.c, r.s, d1, d2});
  }
  return diff_drive_apply(st, d0, d1, d2);
}

#if defined(__CUDACC__)
// ---- device-only variants for the propagate kernel ------------------------------------------------
// Same quantities as rot_make / rot_exp / rot_mul / pose_mul / box_muller above with fewer FP64 instructions:
// sqrt(c^2 + s^2) instead of hypot (the arguments are within an ulp of the unit circle: no overflow guard needed),
// one reciprocal and two multiplications instead of two divisions, sincos / sincospi instead of separate calls, and
// no normalisation that the next product repeats.
// Each substitution moves a result by at most an ulp or two -- the size of the CUDA-vs-glibc libm difference the
// states carry anyway (tests bound them at 1e-12, the north star at 1e-5); nothing downstream is bit-compared
// against these values except through the likelihood-field CELL they select.
__device__ __forceinline__ Rot2 rot_make_fast(double re, double im) {
  const double inv = 1.0 / sqrt(re * re + im * im);
  return Rot2{re * inv, im * inv};
}
__device__ __forceinline__ Rot2 rot_exp_fast(double theta) {
  // sincos returns a unit vector to within an ulp; the products below renormalise anyway
  double sn, cs;
  sincos(theta, &sn, &cs);
  return Rot2{cs, sn};
}
__device__ __forceinline__ Rot2 rot_mul_fast(const Rot2& a, const Rot2& b) {
  // Sophus scales the product by 2 / (1 + |z|^2) before normalising it; a positive scale cancels in the normalisation
  const double re = a.c * b.c - a.s * b.s;
  const double im = a.c * b.s + a.s * b.c;
  return rot_make_fast(re, im);
}
__device__ __forceinline__ Pose2 pose_mul_fast(const Pose2& a, const Pose2& b) {
  const Rot2 r = rot_mul_fast(Rot2{a.c, a.s}, Rot2{b.c, b.s});
  const double rx = a.c * b.x - a.s * b.y;
  const double ry = a.s * b.x + a.c * b.y;
  return Pose2{r.c, r.s, a.x + rx, a.y + ry};
}
__device__ __forceinline__ Pose2 motion_apply_fast(int model, const Pose2& st, double d0, double d1, double d2, const Rot2& first) {
  if (model == 1) {
    const Rot2 e = rot_exp_fast(d0);
    const Rot2 second = rot_mul_fast(e, rot_make_fast(first.c, -first.s));
    const Pose2 a = pose_mul_fast(st, Pose2{first.c, first.s, 0.0, 0.0});
    return pose_mul_fast(a, Pose2{second.c, second.s, d1, -d2});
  }
  if (model == 2) {
    const Rot2 r = rot_exp_fast(d0);
    return pose_mul_fast(st, Pose2{r.c, r.s, d1, d2});
  }
  const Rot2 r1 = rot_exp_fast(d0);
  const Rot2 r2 = rot_exp_fast(d2);
  const Pose2 a = pose_mul_fast(st, Pose2{r1.c, r1.s, 0.0, 0.0});
  return pose_mul_fast(a, Pose2{r2.c, r2.s, d1, 0.0});
}
#endif

// ---- counter RNG -------------------------------------------------------------------------------
// Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11).
// Counter = (index lo, index hi, step, stream); key = seed.  A draw yields two 64-bit words.

enum Stream : uint32_t {
  kStreamInit0 = 0,
  kStreamInit1 = 1,
  kStreamMotion0 = 2,
  kStreamMotion1 = 3,
  kStreamResample = 4,
  kStreamSystematic = 5,
  kStreamRandomState = 6
};

struct Draw {
  uint64_t a, b;
};

BB_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return static_cast<uint32_t>((static_cast<uint64_t>(a) * b) >> 32);
#endif
}

BB_HD Draw counter_draw(uint64_t seed, uint64_t index, uint32_t step, uint32_t stream) {
  uint32_t c0 = static_cast<uint32_t>(index), c1 = static_cast<uint32_t>(index >> 32), c2 = step, c3 = stream;
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
#pragma unroll
  for (int round = 0; round < 10; ++round) {
    const uint32_t hi0 = mulhi32(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = mulhi32(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Draw{(static_cast<uint64_t>(c1) << 32) | c0, (static_cast<uint64_t>(c3) << 32) | c2};
}

/// 53-bit uniform in the open interval (0, 1).
BB_HD double uniform01(uint64_t bits) { return (static_cast<double>(bits >> 11) + 0.5) * 0x1.0p-53; }

BB_HD uint64_t mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return static_cast<uint64_t>((static_cast<unsigned __int128>(a) * b) >> 64);
#endif
}

BB_HD void box_muller(const Draw& d, double& z0, double& z1) {
  const double radius = sqrt(-2.0 * log(uniform01(d.a)));
  const double angle = 6.283185307179586476925 * uniform01(d.b);
  z0 = radius * cos(angle);
  z1 = radius * sin(angle);
}

#if defined(__CUDACC__)
/// box_muller with the angle's range reduction done exactly (sincospi of 2u instead of sin/cos of the rounded 2 pi u).
__device__ __forceinline__ void box_muller_fast(const Draw& d, double& z0, double& z1) {
  const double radius = sqrt(-2.0 * log(uniform01(d.a)));
  double sn, cs;
  sincospi(2.0 * uniform01(d.b), &sn, &cs);
  z0 = radius * cs;
  z1 = radius * sn;
}
/// Only the first normal of the pair.
__device__ __forceinline__ double box_muller_first(const Draw& d) {
  return sqrt(-2.0 * log(uniform01(d.a))) * cospi(2.0 * uniform01(d.b));
}
#endif

// ---- spatial hash (algorithm/spatial_hash.hpp:45-94,190-193) ------------------------------------
/// floor(v) as an int64, or INT64_MIN when floor(v) is NaN or outside [-2^63, 2^63).  The reference's
/// static_cast<int64_t>(std::floor(v)) is undefined out there; on x86-64 (cvttsd2si) it yields INT64_MIN, which this
/// states explicitly, so that host and device agree (the device conversion saturates and turns NaN into 0).
BB_HD int64_t floor_to_int64(double v) {
  const double f = floor(v);
  return f >= -0x1p63 && f < 0x1p63 ? static_cast<int64_t>(f) : INT64_MIN;
}
BB_HD uint64_t floor_and_fibo_hash(double value, unsigned shift) {
  const int64_t signed_value = floor_to_int64(value);
  const uint64_t h = 11400714819323198485ull * static_cast<uint64_t>(signed_value);
  return shift != 0 ? ((h << shift) | (h >> (64 - shift))) : h;
}
BB_HD uint64_t spatial_hash(const Pose2& st, double rx, double ry, double rtheta) {
  return floor_and_fibo_hash(st.x / rx, 0) ^ floor_and_fibo_hash(st.y / ry, 21) ^
         floor_and_fibo_hash(atan2(st.s, st.c) / rtheta, 42);
}

}  // namespace bb200
