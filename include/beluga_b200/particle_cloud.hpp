// Output side of the CUDA backend with the shapes of beluga_ros/include/beluga_ros/particle_cloud.hpp and
// likelihood_field.hpp, minus the ROS message types (plain vectors a node copies into its messages):
//
//   beluga_ros::assign_particle_cloud(particles, size, PoseArray)          -> beluga_b200::sample_poses(amcl, size, draw)
//   beluga_ros::assign_particle_cloud(particles, lin, ang, MarkerArray)    -> beluga_b200::particle_cloud_markers(amcl, lin, ang)
//   beluga_ros::assign_likelihood_field(field, origin, OccupancyGrid)      -> beluga_b200::likelihood_field_cells(amcl)
//
// The histogram behind the markers runs on the device (bb200_filter_particle_histogram): a publish of a million
// particles moves a few thousand bins, not 40 MB of states.  The AmclBatch overloads publish every selected member of a
// batch with one histogram call and one sample call (bb200_amcl_batch_particle_histograms / _sample_states).
#pragma once

#include <cstdint>
#include <optional>
#include <vector>

#include "../beluga_b200.h"
#include "amcl.hpp"

namespace beluga_b200 {

namespace detail_io {
inline void check_filter(bb200_filter* f, int status) {
  if (status != BB200_OK) throw Error(status, bb200_last_error(f));
}
}  // namespace detail_io

struct Pose2d {
  double x, y, cos_yaw, sin_yaw;
};

/// Arrow markers of the pose distribution: the two markers assign_particle_cloud fills (particle_cloud.hpp:233-294).
struct ParticleCloudMarkers {
  std::vector<bb200_marker_vertex> bodies;  // LINE_LIST, ns "bodies", id 0: 2 vertices per bin
  std::vector<bb200_marker_vertex> heads;   // TRIANGLE_LIST, ns "heads", id 1: 3 vertices per bin
  double body_scale_x{0.0};                 // arrow_bodies.scale.x
};

template <class AmclT>
ParticleCloudMarkers particle_cloud_markers(AmclT& amcl, double linear_resolution = 1e-3, double angular_resolution = 1e-3) {
  bb200_filter* f = bb200_amcl_filter(amcl.handle());
  uint64_t n = 0;
  double top = 0.0;
  detail_io::check_filter(f, bb200_filter_particle_histogram(f, linear_resolution, angular_resolution, nullptr, 0, &n, &top));
  std::vector<bb200_cluster_cell> bins(static_cast<size_t>(n));
  detail_io::check_filter(f, bb200_filter_particle_histogram(f, linear_resolution, angular_resolution, bins.data(), n, &n, &top));
  ParticleCloudMarkers out;
  out.bodies.resize(2 * bins.size());
  out.heads.resize(3 * bins.size());
  detail_io::check_filter(f, bb200_particle_cloud_markers(bins.data(), bins.size(), out.bodies.data(), out.heads.data(), &out.body_scale_x));
  return out;
}

/// `size` poses drawn by weight; `draw` numbers the publish (the counter RNG uses step 0xFFFFFFFF - draw).
template <class AmclT>
std::vector<Pose2d> sample_poses(AmclT& amcl, std::size_t size, uint32_t draw = 0) {
  std::vector<double> raw(4 * size);
  bb200_filter* f = bb200_amcl_filter(amcl.handle());
  detail_io::check_filter(f, bb200_filter_sample_states(f, size, 0xFFFFFFFFu - draw, raw.data()));
  std::vector<Pose2d> out(size);
  for (std::size_t i = 0; i < size; ++i) out[i] = Pose2d{raw[4 * i + 2], raw[4 * i + 3], raw[4 * i], raw[4 * i + 1]};
  return out;
}

/// The markers of every member of a batch whose present[m] is true (present == nullptr: all of them), from one batched
/// histogram call; std::nullopt for members not selected.
inline std::vector<std::optional<ParticleCloudMarkers>> particle_cloud_markers(AmclBatch& batch, const std::vector<bool>* present = nullptr,
                                                                                double linear_resolution = 1e-3, double angular_resolution = 1e-3) {
  const auto histograms = batch.particle_histograms(present, linear_resolution, angular_resolution);
  std::vector<std::optional<ParticleCloudMarkers>> out(histograms.size());
  for (std::size_t m = 0; m < histograms.size(); ++m) {
    if (!histograms[m]) continue;
    const std::vector<bb200_cluster_cell>& bins = histograms[m]->first;
    ParticleCloudMarkers markers;
    markers.bodies.resize(2 * bins.size());
    markers.heads.resize(3 * bins.size());
    const int st = bb200_particle_cloud_markers(bins.data(), bins.size(), markers.bodies.data(), markers.heads.data(), &markers.body_scale_x);
    if (st != BB200_OK) throw Error(st, "bb200_particle_cloud_markers");
    out[m] = std::move(markers);
  }
  return out;
}

/// `size` poses drawn by weight from every member of a batch whose present[m] is true (present == nullptr: all of them),
/// with the step convention of sample_poses above; std::nullopt for members not selected.
inline std::vector<std::optional<std::vector<Pose2d>>> sample_poses(AmclBatch& batch, std::size_t size, uint32_t draw = 0,
                                                                     const std::vector<bool>* present = nullptr) {
  const auto raw = batch.sample_states(std::vector<std::size_t>(batch.size(), size), 0xFFFFFFFFu - draw, present);
  std::vector<std::optional<std::vector<Pose2d>>> out(raw.size());
  for (std::size_t m = 0; m < raw.size(); ++m) {
    if (!raw[m]) continue;
    const std::vector<double>& r = *raw[m];
    std::vector<Pose2d> poses(size);
    for (std::size_t i = 0; i < size; ++i) poses[i] = Pose2d{r[4 * i + 2], r[4 * i + 3], r[4 * i], r[4 * i + 1]};
    out[m] = std::move(poses);
  }
  return out;
}

/// nav_msgs/OccupancyGrid cells of the likelihood field, [0, 100] (likelihood_field.hpp:44-79).
template <class AmclT>
std::vector<int8_t> likelihood_field_cells(AmclT& amcl, std::size_t width, std::size_t height) {
  std::vector<float> field(width * height);
  bb200_filter* f = bb200_amcl_filter(amcl.handle());
  detail_io::check_filter(f, bb200_filter_get_likelihood_field(f, field.data(), field.size()));
  std::vector<int8_t> cells(field.size());
  detail_io::check_filter(f, bb200_likelihood_field_to_occupancy(field.data(), field.size(), cells.data()));
  return cells;
}

}  // namespace beluga_b200
