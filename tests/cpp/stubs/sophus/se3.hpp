// Minimal stand-in for <sophus/se3.hpp> (Sophus is not in this image): the one member the point-cloud adaptor reads --
// SE3d::matrix3x4(), the [R | t] block indexed as m(row, col) (Sophus 1.22.10 se3.hpp returns an Eigen 3x4 matrix).
#pragma once
namespace Sophus {
struct Matrix3x4d {
  double m[12];
  double operator()(int r, int c) const { return m[4 * r + c]; }
};
class SE3d {
 public:
  SE3d() = default;
  explicit SE3d(const Matrix3x4d& m) : m_(m) {}  // stub only: real Sophus builds an SE3d from a rotation and a translation
  Matrix3x4d matrix3x4() const { return m_; }

 private:
  Matrix3x4d m_{{1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0}};
};
}  // namespace Sophus
