// The host half of turning a sensor message into base-frame points, shared by the single filter's conversion
// (bb200_scan_to_points, bb200_point_cloud_to_points) and the batch, which converts on the device from what these return.
// One definition for both keeps the two bit-identical: the beam directions come from glibc's cos / sin on both paths (the
// device's differ by an ulp now and then, enough to move an end point across a cell edge).
#pragma once

#include <cmath>
#include <cstdint>
#include <cstring>

#include "../../include/beluga_b200.h"

namespace bb200 {

/// take_evenly(max_beams) over a scan's readings (views/take_evenly.hpp:47-57): how many are kept.
inline uint64_t scan_beam_count(const bb200_laser_scan& scan) {
  const uint64_t size = scan.n_ranges;
  const uint64_t count = scan.max_beams == 0 ? size : scan.max_beams;
  return size == 0 ? 0 : (count > size ? size : count);
}

/// The pos-th kept reading of a scan (pos < scan_beam_count): its index and direction (cos theta, sin theta).
struct ScanBeam {
  uint64_t index;
  double c, s;
};
inline ScanBeam scan_beam(const bb200_laser_scan& scan, uint64_t pos) {
  const uint64_t size = scan.n_ranges;
  const uint64_t count = scan.max_beams == 0 ? size : scan.max_beams;
  uint64_t i = pos;
  if (count <= size && pos != 0) {  // take_evenly's compute_offset (views/take_evenly.hpp:118-145); count >= 2 here
    const uint64_t a = pos * (size - 1), b = count - 1;
    i = a / b + ((a % b == 0) ? 0 : 1);
  }
  // beluga_ros/laser_scan.hpp:73-74: float arithmetic, then widened.
  const double theta = static_cast<double>(scan.angle_min + static_cast<float>(static_cast<int>(i)) * scan.angle_increment);
  return ScanBeam{i, std::cos(theta), std::sin(theta)};  // laser_scan.hpp:66-69
}

/// Whether a reading survives the range filter (beluga_ros/laser_scan.hpp:80-84).
inline bool scan_range_kept(double range, const bb200_laser_scan& scan) {
  return !(std::isnan(range) || !(range >= scan.min_range) || !(range <= scan.max_range));
}

/// One coordinate of a packed point cloud record.  The record has no alignment guarantee (PointCloud2 packs its fields),
/// hence the copy.  float64 values are narrowed to float: SparsePointCloud3f casts them (sparse_point_cloud.hpp:106-116).
template <class Scalar>
float cloud_scalar(const unsigned char* p) {
  Scalar v;
  std::memcpy(&v, p, sizeof(Scalar));
  return static_cast<float>(v);
}

/// The checks bb200_point_cloud_to_points makes before it reads a cloud (the std::invalid_argument cases of the reference).
inline bool cloud_valid(const bb200_point_cloud& c) {
  const bool f32 = c.datatype == BB200_POINT_FLOAT32;
  if (!f32 && c.datatype != BB200_POINT_FLOAT64) return false;
  const uint64_t scalar = f32 ? sizeof(float) : sizeof(double);
  return static_cast<uint64_t>(c.x_offset) + 3 * scalar <= c.point_step && (c.data != nullptr || c.n_points == 0);
}

/// Point i of a valid cloud as the three floats it holds.
template <class Scalar>
void cloud_point(const bb200_point_cloud& c, uint64_t i, float xyz[3]) {
  const unsigned char* p = static_cast<const unsigned char*>(c.data) + c.x_offset + i * c.point_step;
  xyz[0] = cloud_scalar<Scalar>(p);
  xyz[1] = cloud_scalar<Scalar>(p + sizeof(Scalar));
  xyz[2] = cloud_scalar<Scalar>(p + 2 * sizeof(Scalar));
}

}  // namespace bb200
