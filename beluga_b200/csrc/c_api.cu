// extern "C" surface of libbeluga_b200.so (declared in include/beluga_b200.h).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/beluga_b200.h"
#include "amcl.hpp"
#include "batch.hpp"
#include "cluster_host.hpp"
#include "filter.hpp"
#include "measurement_host.hpp"
#include "sharded_amcl.hpp"
#include "state_blob.hpp"

using bb200::Amcl;
using bb200::Batch;
using bb200::Filter;
using bb200::ShardedAmcl;

struct bb200_filter {
  Filter impl;
  explicit bb200_filter(const bb200_filter_config& c) : impl(c) {}
};

struct bb200_amcl {
  Amcl impl;
  bb200_amcl(const bb200_amcl_param& p, const bb200_motion_param& m) : impl(p, m) {}
};

struct bb200_amcl_batch {
  Batch impl;
  bb200_amcl_batch(const bb200_amcl_param* p, const bb200_motion_param* m, int n, uint32_t flags) : impl(p, m, n, flags) {}
};

struct bb200_sharded_amcl {
  ShardedAmcl impl;
  bb200_sharded_amcl(const bb200_amcl_param& p, const bb200_motion_param& m, int n, const int* devices) : impl(p, m, n, devices) {}
};

namespace {
thread_local std::string g_create_error;

// bb200_filter and bb200_amcl are layout-compatible with their only member, so the Amcl-owned Filter and the
// ShardedAmcl-owned shards can be viewed through the same handle types without a second allocation.
static_assert(sizeof(bb200_filter) == sizeof(Filter), "bb200_filter must wrap Filter exactly");
static_assert(sizeof(bb200_amcl) == sizeof(Amcl), "bb200_amcl must wrap Amcl exactly");

// Nothing throws across the C boundary: the host side allocates (std::vector, std::string, unordered_map), so every
// entry point runs its body under this guard and turns an exception into a status + last_error message.
template <class Context, class Body>
int guarded(Context& context, Body&& body) noexcept {
  try {
    return body();
  } catch (const std::bad_alloc&) {
    try {
      context.record_error("out of host memory");
    } catch (...) {
    }
    return BB200_ERR_CAPACITY;
  } catch (const std::exception& e) {
    try {
      context.record_error(std::string("internal error: ") + e.what());
    } catch (...) {
    }
    return BB200_ERR_STATE;
  } catch (...) {
    try {
      context.record_error("internal error: unknown exception");
    } catch (...) {
    }
    return BB200_ERR_STATE;
  }
}
struct CreateErrorContext {
  void record_error(const std::string& m) { g_create_error = m; }
};
template <class Body>
int guarded_create(Body&& body) noexcept {
  CreateErrorContext c;
  return guarded(c, body);
}

/// SparsePointCloud3f::points() | transform(origin * p, keep (x, y))  (beluga_ros/src/amcl.cpp:73-78)
template <class Scalar>
void cloud_to_points(const bb200_point_cloud& c, double* points_xy) {
  const double* m = c.origin;
  for (uint64_t i = 0; i < c.n_points; ++i) {
    float xyz[3];
    bb200::cloud_point<Scalar>(c, i, xyz);
    const double x = xyz[0], y = xyz[1], z = xyz[2];
    double px = x, py = y;
    if (m != nullptr) {
      px = ((m[0] * x + m[1] * y) + m[2] * z) + m[3];
      py = ((m[4] * x + m[5] * y) + m[6] * z) + m[7];
    }
    points_xy[2 * i] = px;
    points_xy[2 * i + 1] = py;
  }
}

const char* const kCloudRefused = "point cloud: datatype must be 7 (FLOAT32) or 8 (FLOAT64), x, y and z must fit in point_step, data must be set";
/// update(points_xy, n_points) on the base-frame points of a laser scan (bb200_scan_to_points): the standalone and the
/// sharded filter convert alike.
template <class Update>
int with_scan_points(const bb200_laser_scan& scan, Update&& update) {
  std::vector<double> points(2 * (scan.n_ranges + 1), 0.0);
  uint64_t n = 0;
  const int st = bb200_scan_to_points(&scan, points.data(), scan.n_ranges + 1, &n);
  return st != BB200_OK ? st : update(points.data(), n);
}
/// ... and on those of a point cloud (bb200_point_cloud_to_points); a refused cloud is reported to `context`.
template <class Context, class Update>
int with_cloud_points(Context& context, const bb200_point_cloud& cloud, Update&& update) {
  std::vector<double> points(2 * cloud.n_points, 0.0);
  uint64_t n = 0;
  const int st = bb200_point_cloud_to_points(&cloud, points.data(), cloud.n_points, &n);
  if (st != BB200_OK) {
    context.record_error(kCloudRefused);
    return st;
  }
  return update(points.data(), n);
}

int create_batch(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags, bb200_amcl_batch** out) {
  if (out == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *out = nullptr;
  {
    const int st = Batch::validate(params, motions, n_members, flags, &g_create_error);  // before any device is touched
    if (st != BB200_OK) return st;
  }
  return guarded_create([&] {
    auto b = std::make_unique<bb200_amcl_batch>(params, motions, n_members, flags);
    if (!b->impl.ok()) {
      g_create_error = b->impl.last_error();
      return b->impl.create_status();
    }
    *out = b.release();
    return static_cast<int>(BB200_OK);
  });
}
}  // namespace

extern "C" {

int bb200_abi_version(void) { return BB200_ABI_VERSION; }

int bb200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return n;
}

const char* bb200_create_error(void) { return g_create_error.c_str(); }

int bb200_filter_create(const bb200_filter_config* config, bb200_filter** out) {
  if (config == nullptr || out == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *out = nullptr;
  return guarded_create([&] {
    bb200_filter* f = new bb200_filter(*config);
    if (!f->impl.ok()) {
      g_create_error = f->impl.last_error();
      const int st = f->impl.create_status();
      delete f;
      return st;
    }
    *out = f;
    return static_cast<int>(BB200_OK);
  });
}

void bb200_filter_destroy(bb200_filter* f) { delete f; }
const char* bb200_last_error(const bb200_filter* f) { return f != nullptr ? f->impl.last_error() : "null filter"; }

#define BB_REQUIRE(cond)                              \
  do {                                                \
    if (!(cond)) return BB200_ERR_INVALID_ARGUMENT;   \
  } while (0)
// While a weighed step is open (bb200_amcl_update_begin .. _end) a filter refuses every call but the step's end and destroy;
// a sharded filter and a batch likewise between their update_begin and _end.
#define BB_REFUSE_OPEN(filter)                                                                              \
  do {                                                                                                      \
    if ((filter).weigh_open()) {                                                                            \
      (filter).record_error("a weighed step is open: only bb200_amcl_update_end and destroy are accepted"); \
      return BB200_ERR_STATE;                                                                               \
    }                                                                                                       \
  } while (0)
#define BB_REFUSE_OPEN_STEP(handle, message)                   \
  do {                                                         \
    if ((handle) != nullptr && (handle)->impl.step_open()) {   \
      (handle)->impl.record_error(message);                    \
      return BB200_ERR_STATE;                                  \
    }                                                          \
  } while (0)
namespace {
const char* const kShardedStepOpen = "a weighed step is open: only bb200_sharded_amcl_update_end and destroy are accepted";
const char* const kBatchStepOpen = "a weighed step is open: only bb200_amcl_batch_update_end and destroy are accepted";
}  // namespace

int bb200_filter_set_likelihood_field_map(bb200_filter* f, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid, int prob) {
  BB_REQUIRE(f && p && grid);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.set_likelihood_field_map(*p, *grid, prob != 0); });
}
int bb200_filter_set_beam_map(bb200_filter* f, const bb200_beam_param* p, const bb200_occupancy_grid* grid) {
  BB_REQUIRE(f && p && grid);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.set_beam_map(*p, *grid); });
}
int bb200_filter_set_landmark_map(bb200_filter* f, const bb200_landmark_param* p, const bb200_landmark_map* map) {
  BB_REQUIRE(f && p && map);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.set_landmark_map(p, nullptr, *map); });
}
int bb200_filter_set_bearing_map(bb200_filter* f, const bb200_bearing_param* p, const bb200_landmark_map* map) {
  BB_REQUIRE(f && p && map);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.set_landmark_map(nullptr, p, *map); });
}
int bb200_filter_reweight_landmarks(bb200_filter* f, const bb200_landmark_detection* detections, uint64_t n) {
  BB_REQUIRE(f && (detections || n == 0));
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] {
    const int st = f->impl.stage_detections(detections, n);
    return st != BB200_OK ? st : f->impl.propagate_reweight(nullptr, 0, Filter::staged_detections(), 0);
  });
}
int bb200_filter_get_likelihood_field(const bb200_filter* f, float* out, uint64_t capacity) {
  BB_REQUIRE(f && out);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.get_likelihood_field(out, capacity); });
}
int bb200_filter_set_particles(bb200_filter* f, const double* states, const double* weights, uint64_t n) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.set_particles(states, weights, n); });
}
int bb200_filter_size(const bb200_filter* f, uint64_t* n) {
  BB_REQUIRE(f && n);
  BB_REFUSE_OPEN(f->impl);
  *n = f->impl.size();
  return BB200_OK;
}
int bb200_filter_get_particles(bb200_filter* f, double* states, double* weights, uint64_t capacity) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.get_particles(states, weights, capacity); });
}
int bb200_filter_initialize_normal(bb200_filter* f, const double mean_xytheta[3], const double cov[9], uint64_t n) {
  BB_REQUIRE(f && mean_xytheta && cov);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.initialize_normal(mean_xytheta, cov, n); });
}
int bb200_filter_initialize_uniform(bb200_filter* f, uint64_t n) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.initialize_uniform(n); });
}
int bb200_filter_propagate(bb200_filter* f, const bb200_motion_sampling* s, uint32_t step) {
  BB_REQUIRE(f && s);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.propagate_reweight(s, step, nullptr, 0); });
}
int bb200_filter_reweight(bb200_filter* f, const double* points_xy, uint64_t n_points) {
  BB_REQUIRE(f && (points_xy || n_points == 0));
  BB_REFUSE_OPEN(f->impl);
  static const double kNoPoints[2] = {0.0, 0.0};
  return guarded(f->impl, [&] { return f->impl.propagate_reweight(nullptr, 0, points_xy != nullptr ? points_xy : kNoPoints, n_points); });
}
int bb200_filter_propagate_reweight(bb200_filter* f, const bb200_motion_sampling* s, uint32_t step, const double* points_xy, uint64_t n_points) {
  BB_REQUIRE(f && s && (points_xy || n_points == 0));
  BB_REFUSE_OPEN(f->impl);
  static const double kNoPoints[2] = {0.0, 0.0};
  return guarded(f->impl, [&] { return f->impl.propagate_reweight(s, step, points_xy != nullptr ? points_xy : kNoPoints, n_points); });
}
int bb200_filter_max_weight(bb200_filter* f, double* wmax) {
  BB_REQUIRE(f && wmax);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.max_weight(wmax); });
}
int bb200_filter_build_cdf(bb200_filter* f, double global_wmax, uint64_t* local_total, int* exponent) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.build_cdf(global_wmax, local_total, exponent); });
}
int bb200_filter_normalize_by(bb200_filter* f, uint64_t global_total, double* local_sum_sq) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.normalize_by(global_total, local_sum_sq); });
}
int bb200_filter_normalize(bb200_filter* f, double* factor, double* sum_sq) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.normalize(factor, sum_sq); });
}
int bb200_filter_resample(bb200_filter* f, const bb200_resample_opts* o, uint64_t* new_size) {
  BB_REQUIRE(f && o);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.resample(*o, new_size); });
}
int bb200_filter_resample_range(bb200_filter* f, const bb200_resample_opts* o, uint64_t global_total, uint64_t cdf_offset, uint64_t slot_begin,
                                uint64_t slot_end) {
  BB_REQUIRE(f && o);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.resample_range(*o, global_total, cdf_offset, slot_begin, slot_end); });
}
int bb200_filter_adopt(bb200_filter* f, uint64_t n, int from_staging) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.adopt(n, from_staging); });
}
int bb200_systematic_comb(uint64_t seed, uint32_t step, uint64_t global_total, uint64_t total_slots, uint64_t* stride, uint64_t* offset) {
  BB_REQUIRE(stride && offset && total_slots > 0);
  *stride = global_total / total_slots;
  *offset = bb200::mulhi64(bb200::counter_draw(seed, 0, step, bb200::kStreamSystematic).a, *stride);
  return BB200_OK;
}
int bb200_estimate_from_moments(const double moments[9], const double pivot_xy[2], bb200_estimate* out) {
  BB_REQUIRE(moments && pivot_xy && out);
  // Pure host arithmetic (estimation.hpp:436-475 from raw moments); needs no device.
  bb200::estimate_from_moments(moments, pivot_xy, out);
  return BB200_OK;
}
int bb200_filter_set_stream(bb200_filter* f, void* cuda_stream) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.set_stream(cuda_stream); });
}
int bb200_filter_enqueue_propagate_reweight(bb200_filter* f, const bb200_motion_sampling* s, uint32_t step, const double* points_xy, uint64_t n_points) {
  BB_REQUIRE(f && s && points_xy);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.enqueue_propagate_reweight(s, step, points_xy, n_points); });
}
int bb200_filter_enqueue_build_cdf(bb200_filter* f) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.enqueue_build_cdf(-1.0); });
}
int bb200_filter_enqueue_resample_range(bb200_filter* f, const bb200_resample_opts* o, uint64_t global_total, uint64_t cdf_offset, uint64_t slot_begin,
                                        uint64_t slot_end) {
  BB_REQUIRE(f && o);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.enqueue_resample_range(*o, global_total, cdf_offset, slot_begin, slot_end); });
}
int bb200_filter_enqueue_adopt(bb200_filter* f, uint64_t n) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.enqueue_adopt(n); });
}
int bb200_filter_enqueue_moments(bb200_filter* f, const double pivot_xy[2]) {
  BB_REQUIRE(f && pivot_xy);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.enqueue_moments(pivot_xy); });
}
int bb200_filter_ancestors(bb200_filter* f, int64_t* out, uint64_t capacity) {
  BB_REQUIRE(f && out);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.ancestors(out, capacity); });
}
int bb200_filter_cdf(bb200_filter* f, uint64_t* out, uint64_t capacity) {
  BB_REQUIRE(f && out);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.cdf(out, capacity); });
}
int bb200_filter_estimate(bb200_filter* f, bb200_estimate* out) {
  BB_REQUIRE(f && out);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.estimate(out); });
}
void bb200_cluster_param_default(bb200_cluster_param* p) {
  if (p == nullptr) return;
  p->linear_hash_resolution = 0.20;
  p->angular_hash_resolution = 0.524;
  p->weight_cap_percentile = 0.90;
}
int bb200_filter_cluster_estimate(bb200_filter* f, const bb200_cluster_param* p, bb200_estimate* out, uint32_t* cluster_ids, uint64_t ids_capacity,
                                  uint32_t* n_cells, uint32_t* n_clusters) {
  BB_REQUIRE(f && p);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.cluster_estimate(*p, out, cluster_ids, ids_capacity, n_cells, n_clusters); });
}
int bb200_cluster_select_host(const bb200_cluster_cell* cells, uint64_t n_cells, uint64_t n_particles, const bb200_cluster_param* p,
                              uint32_t* cluster_of_cell, uint32_t* n_clusters, int* found, uint32_t* best, double moments_out[9]) {
  if ((cells == nullptr && n_cells > 0) || p == nullptr || !(p->linear_hash_resolution > 0.0) || !(p->angular_hash_resolution > 0.0) ||
      !(p->weight_cap_percentile >= 0.0) || !(p->weight_cap_percentile < 1.0))
    return BB200_ERR_INVALID_ARGUMENT;
  static_assert(sizeof(bb200_cluster_cell) == sizeof(bb200::HostCell), "public and internal cell records must agree");
  return guarded_create([&] {
    const bb200::ClusterSelection sel = bb200::select_cluster(reinterpret_cast<const bb200::HostCell*>(cells), n_cells, n_particles,
                                                              p->linear_hash_resolution, p->angular_hash_resolution, p->weight_cap_percentile);
    if (cluster_of_cell != nullptr)
      for (uint64_t k = 0; k < n_cells; ++k) cluster_of_cell[k] = sel.cluster_of_cell[k];
    if (n_clusters != nullptr) *n_clusters = sel.clusters;
    if (found != nullptr) *found = sel.found ? 1 : 0;
    if (best != nullptr) *best = sel.best;
    if (moments_out != nullptr)
      for (int j = 0; j < 9; ++j) moments_out[j] = sel.moments[j];
    return static_cast<int>(BB200_OK);
  });
}
int bb200_filter_particle_histogram(bb200_filter* f, double linear_resolution, double angular_resolution, bb200_cluster_cell* bins, uint64_t capacity,
                                    uint64_t* n_bins, double* max_bin_weight) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.particle_histogram(linear_resolution, angular_resolution, bins, capacity, n_bins, max_bin_weight); });
}
int bb200_filter_sample_states(bb200_filter* f, uint64_t count, uint32_t step, double* states_out) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.sample_states(count, step, states_out); });
}
int bb200_filter_cast_rays(bb200_filter* f, const double* poses, uint64_t n_poses, const double* bearings_cs, uint64_t n_bearings, double max_range,
                           double* ranges) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.cast_rays(poses, n_poses, bearings_cs, n_bearings, max_range, ranges); });
}

namespace {
// detail::alphaHueToRGBA (beluga_ros/particle_cloud.hpp:56-70): single-precision HSV -> RGB for V = S = 1.
void alpha_hue_to_rgba(float hue, float alpha, float rgba[4]) {
  const float kr = std::fmod(5.0F + hue / 60.0F, 6.0F);
  const float kg = std::fmod(3.0F + hue / 60.0F, 6.0F);
  const float kb = std::fmod(1.0F + hue / 60.0F, 6.0F);
  rgba[0] = 1.0F - 1.0F * std::max(0.0F, std::min({kr, 4.0F - kr, 1.0F}));
  rgba[1] = 1.0F - 1.0F * std::max(0.0F, std::min({kg, 4.0F - kg, 1.0F}));
  rgba[2] = 1.0F - 1.0F * std::max(0.0F, std::min({kb, 4.0F - kb, 1.0F}));
  rgba[3] = alpha;
}
}  // namespace

int bb200_particle_cloud_markers(const bb200_cluster_cell* bins, uint64_t n_bins, bb200_marker_vertex* bodies, bb200_marker_vertex* heads,
                                 double* body_scale_x) {
  BB_REQUIRE((bins || n_bins == 0) && (bodies || n_bins == 0) && (heads || n_bins == 0) && body_scale_x);
  // beluga_ros/particle_cloud.hpp:212-294: arrows as a line list (bodies) and a triangle list (heads), sizes and
  // colours scaled by the bin weight relative to the heaviest bin.
  const double kArrowBodyLength = 0.5, kArrowHeadLength = 0.1, kArrowHeadWidth = kArrowHeadLength / 5.0;
  const double kArrowLength = kArrowBodyLength + kArrowHeadLength;
  double max_bin_weight = 1e-3;
  for (uint64_t k = 0; k < n_bins; ++k) max_bin_weight = bins[k].weight > max_bin_weight ? bins[k].weight : max_bin_weight;
  double min_scale_factor = 1.0;
  for (uint64_t k = 0; k < n_bins; ++k) {
    const double* st = bins[k].representative;  // {cos, sin, x, y}
    const double scale_factor = std::max(bins[k].weight / max_bin_weight, 1e-1);
    if (scale_factor < min_scale_factor) min_scale_factor = scale_factor;
    float rgba[4];
    alpha_hue_to_rgba(static_cast<float>((1.0 - scale_factor) * 270.0), static_cast<float>(0.25 + 0.75 * scale_factor), rgba);
    auto put = [&](bb200_marker_vertex& v, double lx, double ly) {  // state * (scale_factor * local point)
      const double px = scale_factor * lx, py = scale_factor * ly;
      v.x = (st[0] * px - st[1] * py) + st[2];
      v.y = (st[1] * px + st[0] * py) + st[3];
      v.z = 0.0;
      v.r = rgba[0], v.g = rgba[1], v.b = rgba[2], v.a = rgba[3];
    };
    put(bodies[2 * k], 0.0, 0.0);
    put(bodies[2 * k + 1], kArrowBodyLength, 0.0);
    put(heads[3 * k], kArrowBodyLength, kArrowHeadWidth / 2.0);
    put(heads[3 * k + 1], kArrowBodyLength, -(kArrowHeadWidth / 2.0));
    put(heads[3 * k + 2], kArrowLength, 0.0);
  }
  *body_scale_x = static_cast<double>(min_scale_factor * kArrowHeadWidth) * 0.8;
  return BB200_OK;
}

int bb200_likelihood_field_to_occupancy(const float* field, uint64_t n, int8_t* out) {
  BB_REQUIRE((field && out) || n == 0);
  if (n == 0) return BB200_OK;
  // beluga_ros/likelihood_field.hpp:44-79
  float min_val = field[0], max_val = field[0];
  for (uint64_t i = 1; i < n; ++i) {
    if (field[i] < min_val) min_val = field[i];
    if (max_val < field[i]) max_val = field[i];
  }
  const float range = max_val - min_val;
  if (range <= std::numeric_limits<float>::epsilon()) {
    for (uint64_t i = 0; i < n; ++i) out[i] = 0;
    return BB200_OK;
  }
  for (uint64_t i = 0; i < n; ++i) {
    const float normalized = (field[i] - min_val) / range;
    out[i] = static_cast<int8_t>(normalized * 100.0f);
  }
  return BB200_OK;
}

int bb200_filter_moments(bb200_filter* f, const double pivot_xy[2], double out[9]) {
  BB_REQUIRE(f && pivot_xy && out);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.moments(pivot_xy, out); });
}
int bb200_filter_set_timing(bb200_filter* f, int enabled) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  f->impl.set_timing(enabled != 0);
  return BB200_OK;
}
int bb200_filter_clear_timings(bb200_filter* f) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  f->impl.clear_timings();
  return BB200_OK;
}
int bb200_filter_last_timings(const bb200_filter* f, const char** names, float* ms, int capacity) {
  if (f == nullptr) return 0;
  return guarded(f->impl, [&] { return f->impl.last_timings(names, ms, capacity); });
}
uint64_t bb200_filter_launch_count(const bb200_filter* f) { return f != nullptr ? f->impl.launch_count() : 0; }
int bb200_filter_synchronize(bb200_filter* f) {
  BB_REQUIRE(f);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.synchronize(); });
}
int bb200_filter_device_pointer(bb200_filter* f, int which, void** ptr, uint64_t* bytes) {
  BB_REQUIRE(f && ptr && bytes);
  BB_REFUSE_OPEN(f->impl);
  return guarded(f->impl, [&] { return f->impl.device_pointer(which, ptr, bytes); });
}

// ---- amcl ---------------------------------------------------------------------------------------

int bb200_amcl_create_with_motion(const bb200_amcl_param* p, const bb200_motion_param* motion, bb200_amcl** out) {
  if (p == nullptr || motion == nullptr || out == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *out = nullptr;
  if (const int st = Amcl::validate(*p, *motion, &g_create_error)) return st;
  return guarded_create([&] {
    bb200_amcl* a = new bb200_amcl(*p, *motion);
    if (!a->impl.ok()) {
      g_create_error = a->impl.last_error();
      const int st = a->impl.create_status();
      delete a;
      return st;
    }
    *out = a;
    return static_cast<int>(BB200_OK);
  });
}
int bb200_amcl_create(const bb200_amcl_param* p, const bb200_diff_drive_param* motion, bb200_amcl** out) {
  if (motion == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  const bb200_motion_param m{BB200_MOTION_DIFFERENTIAL, motion->rotation_noise_from_rotation, motion->rotation_noise_from_translation,
                             motion->translation_noise_from_translation, motion->translation_noise_from_rotation, 0.0, motion->distance_threshold};
  return bb200_amcl_create_with_motion(p, &m, out);
}
void bb200_amcl_destroy(bb200_amcl* a) { delete a; }
const char* bb200_amcl_last_error(const bb200_amcl* a) { return a != nullptr ? a->impl.last_error() : "null amcl"; }
bb200_filter* bb200_amcl_filter(bb200_amcl* a) { return a != nullptr ? reinterpret_cast<bb200_filter*>(&a->impl.filter()) : nullptr; }
int bb200_amcl_initialize(bb200_amcl* a, const double mean_xytheta[3], const double cov[9]) {
  BB_REQUIRE(a && mean_xytheta && cov);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.initialize(mean_xytheta, cov); });
}
int bb200_amcl_initialize_from_map(bb200_amcl* a) {
  BB_REQUIRE(a);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.initialize_from_map(); });
}
int bb200_amcl_initialize_states(bb200_amcl* a, const double* states, const double* weights, uint64_t n) {
  BB_REQUIRE(a);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.initialize_states(states, weights, n); });
}
void bb200_amcl_force_update(bb200_amcl* a) {
  if (a != nullptr && !a->impl.filter().weigh_open()) a->impl.force_update();
}
int bb200_amcl_update(bb200_amcl* a, const double control_pose[4], const double* points_xy, uint64_t n_points, bb200_update_result* out) {
  BB_REQUIRE(a && control_pose && out && (points_xy || n_points == 0));
  BB_REFUSE_OPEN(a->impl.filter());
  static const double kNoPoints[2] = {0.0, 0.0};
  return guarded(a->impl, [&] { return a->impl.update(control_pose, points_xy != nullptr ? points_xy : kNoPoints, n_points, out); });
}
int bb200_amcl_update_landmarks(bb200_amcl* a, const double control_pose[4], const bb200_landmark_detection* detections, uint64_t n,
                                bb200_update_result* out) {
  BB_REQUIRE(a && control_pose && out && (detections || n == 0));
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.update_landmarks(control_pose, detections, n, out); });
}
int bb200_amcl_update_begin(bb200_amcl* a, const double control_pose[4], bb200_weigh_view* view) {
  BB_REQUIRE(a && control_pose && view);
  return guarded(a->impl, [&] { return a->impl.update_begin(control_pose, view); });
}
int bb200_amcl_update_end(bb200_amcl* a, bb200_update_result* out) {
  BB_REQUIRE(a && out);
  return guarded(a->impl, [&] { return a->impl.update_end(out); });
}
int bb200_take_evenly_indices(uint64_t size, uint64_t count, uint64_t* indices, uint64_t capacity, uint64_t* n_indices) {
  BB_REQUIRE(indices && n_indices);
  // take_evenly_view::size() and compute_offset() (views/take_evenly.hpp:47-57,118-145)
  uint64_t kept = size == 0 ? 0 : (count > size ? size : count);
  if (kept > capacity) return BB200_ERR_CAPACITY;
  for (uint64_t pos = 0; pos < kept; ++pos) {
    uint64_t idx;
    if (count > size) {
      idx = pos;
    } else if (pos == 0) {
      idx = 0;
    } else {  // count >= 2 here: pos < kept <= count
      const uint64_t a = pos * (size - 1), b = count - 1;
      idx = a / b + ((a % b == 0) ? 0 : 1);
    }
    indices[pos] = idx;
  }
  *n_indices = kept;
  return BB200_OK;
}

int bb200_scan_to_points(const bb200_laser_scan* scan, double* points_xy, uint64_t capacity, uint64_t* n_points) {
  BB_REQUIRE(scan && points_xy && n_points && (scan->ranges || scan->n_ranges == 0));
  const uint64_t kept = bb200::scan_beam_count(*scan);
  uint64_t n = 0;
  for (uint64_t pos = 0; pos < kept; ++pos) {
    const bb200::ScanBeam beam = bb200::scan_beam(*scan, pos);
    const double range = static_cast<double>(scan->ranges[beam.index]);
    if (!bb200::scan_range_kept(range, *scan)) continue;
    const double x = range * beam.c, y = range * beam.s;
    double px = x, py = y;
    if (scan->laser_origin != nullptr) {  // origin * (x, y, 0), keep (x, y)  (beluga_ros/src/amcl.cpp:59-61)
      const double* m = scan->laser_origin;
      px = m[0] * x + m[1] * y + m[3];
      py = m[4] * x + m[5] * y + m[7];
    }
    if (n >= capacity) return BB200_ERR_CAPACITY;
    points_xy[2 * n] = px;
    points_xy[2 * n + 1] = py;
    ++n;
  }
  *n_points = n;
  return BB200_OK;
}

int bb200_amcl_update_scan(bb200_amcl* a, const double control_pose[4], const bb200_laser_scan* scan, bb200_update_result* out) {
  BB_REQUIRE(a && control_pose && scan && out);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] {
    return with_scan_points(*scan, [&](const double* points, uint64_t n) { return bb200_amcl_update(a, control_pose, points, n, out); });
  });
}

int bb200_scan_bearings(float angle_min, float angle_increment, uint64_t n_ranges, uint64_t max_beams, double* bearings_cs, uint64_t capacity,
                        uint64_t* n) {
  BB_REQUIRE(n && (bearings_cs || capacity == 0));
  bb200_laser_scan scan{};
  scan.n_ranges = n_ranges;
  scan.angle_min = angle_min;
  scan.angle_increment = angle_increment;
  scan.max_beams = max_beams;
  const uint64_t kept = bb200::scan_beam_count(scan);
  *n = kept;
  if (kept > capacity) return BB200_ERR_CAPACITY;
  for (uint64_t pos = 0; pos < kept; ++pos) {
    const bb200::ScanBeam beam = bb200::scan_beam(scan, pos);
    bearings_cs[2 * pos] = beam.c;
    bearings_cs[2 * pos + 1] = beam.s;
  }
  return BB200_OK;
}

int bb200_point_cloud_to_points(const bb200_point_cloud* cloud, double* points_xy, uint64_t capacity, uint64_t* n_points) {
  BB_REQUIRE(cloud && n_points && (points_xy || capacity == 0));
  BB_REQUIRE(bb200::cloud_valid(*cloud));
  if (cloud->n_points > capacity) return BB200_ERR_CAPACITY;
  if (cloud->datatype == BB200_POINT_FLOAT32) {
    cloud_to_points<float>(*cloud, points_xy);
  } else {
    cloud_to_points<double>(*cloud, points_xy);
  }
  *n_points = cloud->n_points;
  return BB200_OK;
}

int bb200_amcl_update_point_cloud(bb200_amcl* a, const double control_pose[4], const bb200_point_cloud* cloud, bb200_update_result* out) {
  BB_REQUIRE(a && control_pose && cloud && out);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] {
    return with_cloud_points(a->impl, *cloud, [&](const double* points, uint64_t n) { return bb200_amcl_update(a, control_pose, points, n, out); });
  });
}

// ---- sharded filters ---------------------------------------------------------------------------------

int bb200_amcl_export_shard(bb200_amcl* a, void* out256) {
  BB_REQUIRE(a && out256);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.filter().link().export_handles(out256); });
}
int bb200_amcl_join_shards(bb200_amcl* a, int world, int rank, const void* handles) {
  BB_REQUIRE(a && handles);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.filter().link().join_ipc(world, rank, handles); });
}
int bb200_amcl_leave_shards(bb200_amcl* a) {
  BB_REQUIRE(a);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] {
    bb200::Filter& f = a->impl.filter();
    return f.link().leave(f.stream());
  });
}

int bb200_sharded_amcl_create(const bb200_amcl_param* p, const bb200_motion_param* motion, int n_shards, const int* devices, bb200_sharded_amcl** out) {
  if (p == nullptr || motion == nullptr || out == nullptr || devices == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *out = nullptr;
  if (const int st = ShardedAmcl::validate(*p, *motion, n_shards, &g_create_error)) return st;  // before any device is touched
  return guarded_create([&] {
    auto g = std::make_unique<bb200_sharded_amcl>(*p, *motion, n_shards, devices);
    if (!g->impl.ok()) {
      g_create_error = g->impl.last_error();
      return g->impl.create_status();
    }
    *out = g.release();
    return static_cast<int>(BB200_OK);
  });
}
void bb200_sharded_amcl_destroy(bb200_sharded_amcl* g) { delete g; }
const char* bb200_sharded_amcl_last_error(const bb200_sharded_amcl* g) { return g != nullptr ? g->impl.last_error() : "null sharded amcl"; }
int bb200_sharded_amcl_shards(const bb200_sharded_amcl* g) { return g != nullptr ? g->impl.shards() : 0; }
bb200_amcl* bb200_sharded_amcl_shard(bb200_sharded_amcl* g, int rank) {
  return g != nullptr ? reinterpret_cast<bb200_amcl*>(g->impl.shard(rank)) : nullptr;
}

int bb200_sharded_amcl_set_likelihood_field_map(bb200_sharded_amcl* g, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid, int prob) {
  BB_REQUIRE(g && p && grid);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] {
    return g->impl.set_map([&](bb200::MapTables* t, std::string* e) { return bb200::prepare_likelihood_field_map(*p, *grid, prob != 0, t, e); });
  });
}
int bb200_sharded_amcl_set_beam_map(bb200_sharded_amcl* g, const bb200_beam_param* p, const bb200_occupancy_grid* grid) {
  BB_REQUIRE(g && p && grid);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.set_map([&](bb200::MapTables* t, std::string* e) { return bb200::prepare_beam_map(*p, *grid, t, e); }); });
}
int bb200_sharded_amcl_set_landmark_map(bb200_sharded_amcl* g, const bb200_landmark_param* p, const bb200_landmark_map* map) {
  BB_REQUIRE(g && p && map);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.set_landmark_map(p, nullptr, *map); });
}
int bb200_sharded_amcl_set_bearing_map(bb200_sharded_amcl* g, const bb200_bearing_param* p, const bb200_landmark_map* map) {
  BB_REQUIRE(g && p && map);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.set_landmark_map(nullptr, p, *map); });
}
int bb200_sharded_amcl_initialize(bb200_sharded_amcl* g, const double mean_xytheta[3], const double cov[9]) {
  BB_REQUIRE(mean_xytheta && cov);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  BB_REQUIRE(g);
  return guarded(g->impl, [&] { return g->impl.initialize(mean_xytheta, cov); });
}
int bb200_sharded_amcl_initialize_from_map(bb200_sharded_amcl* g) {
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  BB_REQUIRE(g);
  return guarded(g->impl, [&] { return g->impl.initialize_from_map(); });
}
void bb200_sharded_amcl_force_update(bb200_sharded_amcl* g) {
  if (g != nullptr && !g->impl.step_open()) g->impl.force_update();
}
int bb200_sharded_amcl_update(bb200_sharded_amcl* g, const double control_pose[4], const double* points_xy, uint64_t n_points, bb200_update_result* out) {
  BB_REQUIRE(g && control_pose && out && (points_xy || n_points == 0));
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  static const double kNoPoints[2] = {0.0, 0.0};
  return guarded(g->impl, [&] { return g->impl.update(control_pose, points_xy != nullptr ? points_xy : kNoPoints, n_points, out); });
}
int bb200_sharded_amcl_update_landmarks(bb200_sharded_amcl* g, const double control_pose[4], const bb200_landmark_detection* detections, uint64_t n,
                                        bb200_update_result* out) {
  BB_REQUIRE(g && control_pose && out && (detections || n == 0));
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.update_landmarks(control_pose, detections, n, out); });
}
int bb200_sharded_amcl_update_begin(bb200_sharded_amcl* g, const double control_pose[4], bb200_weigh_view* views) {
  BB_REQUIRE(g && control_pose && views);
  return guarded(g->impl, [&] { return g->impl.update_begin(control_pose, views); });
}
int bb200_sharded_amcl_update_end(bb200_sharded_amcl* g, bb200_update_result* out) {
  BB_REQUIRE(g && out);
  return guarded(g->impl, [&] { return g->impl.update_end(out); });
}
int bb200_cluster_merge_host(const bb200_cluster_cell* const* shard_cells, const uint64_t* shard_counts, const uint64_t* shard_first_index, int shards,
                             bb200_cluster_cell* merged, uint64_t capacity, uint64_t* n_merged) {
  BB_REQUIRE(shard_cells && shard_counts && n_merged && shards >= 1);
  return guarded_create([&] { return bb200::merge_cells(shard_cells, shard_counts, shard_first_index, shards, merged, capacity, n_merged); });
}

int bb200_sharded_amcl_cluster_estimate(bb200_sharded_amcl* g, const bb200_cluster_param* p, bb200_estimate* out, uint32_t* n_cells,
                                        uint32_t* n_clusters) {
  BB_REQUIRE(g && p && out);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.cluster_estimate(*p, out, n_cells, n_clusters); });
}

int bb200_sharded_amcl_get_particles(bb200_sharded_amcl* g, double* states, double* weights, uint64_t capacity) {
  BB_REQUIRE(g);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.get_particles(states, weights, capacity); });
}

int bb200_sharded_amcl_update_scan(bb200_sharded_amcl* g, const double control_pose[4], const bb200_laser_scan* scan, bb200_update_result* out) {
  BB_REQUIRE(g && control_pose && scan && out);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  g->impl.record_error("");  // a refused measurement leaves no earlier message behind
  return guarded(g->impl, [&] {
    return with_scan_points(*scan, [&](const double* points, uint64_t n) { return bb200_sharded_amcl_update(g, control_pose, points, n, out); });
  });
}

int bb200_sharded_amcl_update_point_cloud(bb200_sharded_amcl* g, const double control_pose[4], const bb200_point_cloud* cloud,
                                          bb200_update_result* out) {
  BB_REQUIRE(g && control_pose && cloud && out);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  g->impl.record_error("");  // a refused measurement leaves no earlier message behind
  return guarded(g->impl, [&] {
    return with_cloud_points(g->impl, *cloud, [&](const double* points, uint64_t n) { return bb200_sharded_amcl_update(g, control_pose, points, n, out); });
  });
}

int bb200_sharded_amcl_particle_histogram(bb200_sharded_amcl* g, double linear_resolution, double angular_resolution, bb200_cluster_cell* bins,
                                          uint64_t capacity, uint64_t* n_bins, double* max_bin_weight) {
  BB_REQUIRE(g);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.particle_histogram(linear_resolution, angular_resolution, bins, capacity, n_bins, max_bin_weight); });
}

int bb200_sharded_amcl_sample_states(bb200_sharded_amcl* g, uint64_t count, uint32_t step, double* states_out) {
  BB_REQUIRE(g);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.sample_states(count, step, states_out); });
}

int bb200_sharded_amcl_cast_rays(bb200_sharded_amcl* g, const double* poses, uint64_t n_poses, const double* bearings_cs, uint64_t n_bearings,
                                 double max_range, double* ranges) {
  BB_REQUIRE(g);
  BB_REFUSE_OPEN_STEP(g, kShardedStepOpen);
  return guarded(g->impl, [&] { return g->impl.cast_rays(poses, n_poses, bearings_cs, n_bearings, max_range, ranges); });
}

// ---- batches ------------------------------------------------------------------------------------------

int bb200_amcl_batch_create(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, bb200_amcl_batch** out) {
  return create_batch(params, motions, n_members, 0, out);
}
int bb200_amcl_batch_create_adaptive(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, bb200_amcl_batch** out) {
  return create_batch(params, motions, n_members, BB200_BATCH_ADAPTIVE, out);
}
int bb200_amcl_batch_create_with_flags(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags,
                                       bb200_amcl_batch** out) {
  return create_batch(params, motions, n_members, flags, out);
}
int bb200_amcl_batch_member_size(const bb200_amcl_batch* b, int member, uint64_t* n) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && n);
  return guarded(b->impl, [&] { return b->impl.member_size(member, n); });
}
void bb200_amcl_batch_destroy(bb200_amcl_batch* b) { delete b; }
const char* bb200_amcl_batch_last_error(const bb200_amcl_batch* b) { return b != nullptr ? b->impl.last_error() : "null batch"; }
int bb200_amcl_batch_members(const bb200_amcl_batch* b) { return b != nullptr ? b->impl.members() : 0; }
int bb200_amcl_batch_set_likelihood_field_map(bb200_amcl_batch* b, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid,
                                              int prob) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && grid);
  return guarded(b->impl, [&] { return b->impl.set_likelihood_field_map(*p, *grid, prob != 0); });
}
int bb200_amcl_batch_set_beam_map(bb200_amcl_batch* b, const bb200_beam_param* p, const bb200_occupancy_grid* grid) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && grid);
  return guarded(b->impl, [&] { return b->impl.set_beam_map(*p, *grid); });
}
int bb200_amcl_batch_add_likelihood_field_map(bb200_amcl_batch* b, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid,
                                              int prob, int* map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && grid && map_id);
  return guarded(b->impl, [&] { return b->impl.add_likelihood_field_map(*p, *grid, prob != 0, map_id); });
}
int bb200_amcl_batch_add_beam_map(bb200_amcl_batch* b, const bb200_beam_param* p, const bb200_occupancy_grid* grid, int* map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && grid && map_id);
  return guarded(b->impl, [&] { return b->impl.add_beam_map(*p, *grid, map_id); });
}
int bb200_amcl_batch_set_landmark_map(bb200_amcl_batch* b, const bb200_landmark_param* p, const bb200_landmark_map* map) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && map);
  return guarded(b->impl, [&] { return b->impl.set_landmark_map(p, nullptr, *map); });
}
int bb200_amcl_batch_set_bearing_map(bb200_amcl_batch* b, const bb200_bearing_param* p, const bb200_landmark_map* map) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && map);
  return guarded(b->impl, [&] { return b->impl.set_landmark_map(nullptr, p, *map); });
}
int bb200_amcl_batch_add_landmark_map(bb200_amcl_batch* b, const bb200_landmark_param* p, const bb200_landmark_map* map, int* map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && map && map_id);
  return guarded(b->impl, [&] { return b->impl.add_landmark_map(p, nullptr, *map, map_id); });
}
int bb200_amcl_batch_add_bearing_map(bb200_amcl_batch* b, const bb200_bearing_param* p, const bb200_landmark_map* map, int* map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && map && map_id);
  return guarded(b->impl, [&] { return b->impl.add_landmark_map(nullptr, p, *map, map_id); });
}
int bb200_amcl_batch_set_detections(bb200_amcl_batch* b, const bb200_landmark_detection* const* detections, const uint64_t* n, const uint8_t* present) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && n);
  return guarded(b->impl, [&] { return b->impl.set_detections(detections, n, present); });
}
int bb200_amcl_batch_update_map(bb200_amcl_batch* b, int member, int map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.update_map(member, map_id); });
}
int bb200_amcl_batch_member_map(const bb200_amcl_batch* b, int member, int* map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && map_id);
  return guarded(b->impl, [&] { return b->impl.member_map(member, map_id); });
}
int bb200_amcl_batch_remove_map(bb200_amcl_batch* b, int map_id) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.remove_map(map_id); });
}
int bb200_amcl_batch_get_likelihood_field(const bb200_amcl_batch* b, int map_id, float* out, uint64_t capacity) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && out);
  return guarded(b->impl, [&] { return b->impl.get_likelihood_field(map_id, out, capacity); });
}
int bb200_amcl_batch_initialize(bb200_amcl_batch* b, int member, const double mean_xytheta[3], const double cov[9]) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && mean_xytheta && cov);
  return guarded(b->impl, [&] { return b->impl.initialize(member, mean_xytheta, cov); });
}
int bb200_amcl_batch_initialize_from_map(bb200_amcl_batch* b, int member) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.initialize_from_map(member); });
}
int bb200_amcl_batch_initialize_states(bb200_amcl_batch* b, int member, const double* states, const double* weights, uint64_t n) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.initialize_states(member, states, weights, n); });
}
int bb200_amcl_batch_force_update(bb200_amcl_batch* b, int member) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return b->impl.force_update(member);
}
int bb200_amcl_batch_get_particles(bb200_amcl_batch* b, int member, double* states, double* weights, uint64_t capacity) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.get_particles(member, states, weights, capacity); });
}
int bb200_amcl_batch_ancestors(bb200_amcl_batch* b, int member, int64_t* out, uint64_t capacity) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && (out || capacity == 0));
  return guarded(b->impl, [&] { return b->impl.ancestors(member, out, capacity); });
}
int bb200_amcl_batch_cluster_estimate(bb200_amcl_batch* b, int member, const bb200_cluster_param* p, bb200_estimate* out) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && out);
  return guarded(b->impl, [&] { return b->impl.cluster_estimate(member, *p, out); });
}
int bb200_amcl_batch_cluster_estimates(bb200_amcl_batch* b, const bb200_cluster_param* p, const uint8_t* present, bb200_estimate* out,
                                       uint32_t* n_cells, uint32_t* n_clusters) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && p && out);
  return guarded(b->impl, [&] { return b->impl.cluster_estimates(*p, present, out, n_cells, n_clusters); });
}
int bb200_amcl_batch_particle_histograms(bb200_amcl_batch* b, double linear_resolution, double angular_resolution, const uint8_t* present,
                                         bb200_cluster_cell* const* bins, const uint64_t* capacity, uint64_t* n_bins, double* max_bin_weight) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.particle_histograms(linear_resolution, angular_resolution, present, bins, capacity, n_bins, max_bin_weight); });
}
int bb200_amcl_batch_sample_states(bb200_amcl_batch* b, const uint64_t* counts, uint32_t step, const uint8_t* present, double* const* states_out) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && counts && states_out);
  return guarded(b->impl, [&] { return b->impl.sample_states(counts, step, present, states_out); });
}
int bb200_amcl_batch_update(bb200_amcl_batch* b, const double* control_poses, const double* const* points_xy, const uint64_t* n_points,
                            const uint8_t* present, bb200_update_result* out) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && control_poses && points_xy && n_points && out);
  return guarded(b->impl, [&] { return b->impl.update(control_poses, points_xy, n_points, present, out); });
}
int bb200_amcl_batch_update_measurements(bb200_amcl_batch* b, const double* control_poses, const bb200_measurement* measurements,
                                         const uint8_t* present, bb200_update_result* out) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && control_poses && measurements && out);
  return guarded(b->impl, [&] { return b->impl.update_measurements(control_poses, measurements, present, out); });
}
int bb200_amcl_batch_update_clustered(bb200_amcl_batch* b, const double* control_poses, const bb200_measurement* measurements,
                                      const uint8_t* present, const bb200_cluster_param* p, bb200_update_result* out, bb200_estimate* clustered,
                                      uint32_t* n_cells, uint32_t* n_clusters) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && control_poses && measurements && p && out && clustered);
  return guarded(b->impl, [&] { return b->impl.update_clustered(control_poses, measurements, present, *p, out, clustered, n_cells, n_clusters); });
}
int bb200_amcl_batch_update_begin(bb200_amcl_batch* b, const double* control_poses, const bb200_measurement* measurements, const uint8_t* present,
                                  bb200_weigh_view* views) {
  BB_REQUIRE(b && control_poses && measurements && views);
  return guarded(b->impl, [&] { return b->impl.update_begin(control_poses, measurements, present, views); });
}
int bb200_amcl_batch_update_end(bb200_amcl_batch* b, const bb200_cluster_param* cluster, bb200_update_result* out, bb200_estimate* clustered,
                                uint32_t* n_cells, uint32_t* n_clusters) {
  BB_REQUIRE(b && out && (cluster == nullptr || clustered != nullptr));
  return guarded(b->impl, [&] { return b->impl.update_end(cluster, out, clustered, n_cells, n_clusters); });
}
int bb200_amcl_batch_cast_rays(bb200_amcl_batch* b, const uint8_t* present, const int* map_ids, const double* const* poses, const uint64_t* n_poses,
                               const double* const* bearings_cs, const uint64_t* n_bearings, const double* max_range, double* const* ranges) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && poses && n_poses && bearings_cs && n_bearings && max_range && ranges);
  return guarded(b->impl, [&] { return b->impl.cast_rays(present, map_ids, poses, n_poses, bearings_cs, n_bearings, max_range, ranges); });
}
uint64_t bb200_amcl_batch_launch_count(const bb200_amcl_batch* b) { return b != nullptr ? b->impl.launch_count() : 0; }
int bb200_amcl_batch_add_member(bb200_amcl_batch* b, const bb200_amcl_param* params, const bb200_motion_param* motion, int* member) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && params && motion && member);
  return guarded(b->impl, [&] { return b->impl.add_member(*params, *motion, member); });
}
int bb200_amcl_batch_remove_member(bb200_amcl_batch* b, int member) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b);
  return guarded(b->impl, [&] { return b->impl.remove_member(member); });
}
int bb200_amcl_batch_member_active(const bb200_amcl_batch* b, int member, int* active) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && active);
  return guarded(b->impl, [&] { return b->impl.member_active(member, active); });
}

int bb200_amcl_batch_export_members(bb200_amcl_batch* b, const uint8_t* present, void* const* out, const uint64_t* capacity, uint64_t* size) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && size);
  return guarded(b->impl, [&] { return b->impl.export_members(present, out, capacity, size); });
}
int bb200_amcl_batch_export_member(bb200_amcl_batch* b, int member, void* out, uint64_t capacity, uint64_t* size) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && size);
  return guarded(b->impl, [&] { return b->impl.export_member(member, out, capacity, size); });
}
int bb200_amcl_batch_import_member(bb200_amcl_batch* b, const void* blob, uint64_t size, int map_id, int* member) {
  BB_REFUSE_OPEN_STEP(b, kBatchStepOpen);
  BB_REQUIRE(b && blob && member);
  return guarded(b->impl, [&] { return b->impl.import_member(blob, size, map_id, member); });
}
int bb200_amcl_batch_create_from_states(const void* const* blobs, const uint64_t* sizes, int n_members, uint32_t flags, int device,
                                        bb200_amcl_batch** out) {
  if (blobs == nullptr || sizes == nullptr || out == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *out = nullptr;
  if (n_members < 1) {
    g_create_error = "a batch needs at least one member";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  return guarded_create([&] {
    std::vector<bb200::FilterState> states(static_cast<size_t>(n_members));
    std::vector<bb200_amcl_param> params(states.size());
    std::vector<bb200_motion_param> motions(states.size());
    for (size_t k = 0; k < states.size(); ++k) {
      std::string message;
      if (const int st = bb200::read_state_blob(blobs[k], sizes[k], &states[k], &message)) {
        g_create_error = "member " + std::to_string(k) + ": " + message;
        return st;
      }
      states[k].params.device = device;  // the receiver's device
      params[k] = states[k].params;
      motions[k] = states[k].motion;
    }
    bb200_amcl_batch* b = nullptr;
    if (const int st = create_batch(params.data(), motions.data(), n_members, flags, &b)) return st;
    if (const int st = b->impl.restore_members(states)) {
      g_create_error = b->impl.last_error();
      delete b;
      return st;
    }
    *out = b;
    return static_cast<int>(BB200_OK);
  });
}

int bb200_amcl_state_params(const void* blob, uint64_t size, bb200_amcl_param* params, bb200_motion_param* motion) {
  if (params == nullptr || motion == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  return guarded_create([&] {
    bb200::FilterState s;
    if (const int st = bb200::read_state_blob(blob, size, &s, &g_create_error)) return st;
    *params = s.params;
    *motion = s.motion;
    return static_cast<int>(BB200_OK);
  });
}
int bb200_amcl_export_state(bb200_amcl* a, void* out, uint64_t capacity, uint64_t* size) {
  BB_REQUIRE(a && size);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.export_state(out, capacity, size); });
}
int bb200_amcl_create_from_state(const void* blob, uint64_t size, int device, bb200_amcl** out) {
  if (out == nullptr) {
    g_create_error = "null argument";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *out = nullptr;
  bb200::FilterState s;
  int st = guarded_create([&] { return bb200::read_state_blob(blob, size, &s, &g_create_error); });
  if (st != BB200_OK) return st;
  s.params.device = device;  // the receiver's device
  bb200_amcl* a = nullptr;
  st = bb200_amcl_create_with_motion(&s.params, &s.motion, &a);
  if (st != BB200_OK) return st;
  st = guarded(a->impl, [&] { return a->impl.restore_state(s); });
  if (st != BB200_OK) {
    g_create_error = a->impl.last_error();
    bb200_amcl_destroy(a);
    return st;
  }
  *out = a;
  return BB200_OK;
}

int bb200_amcl_plan_update(bb200_amcl* a, const double control_pose[4], bb200_step_plan* plan) {
  BB_REQUIRE(a && control_pose && plan);
  BB_REFUSE_OPEN(a->impl.filter());
  return guarded(a->impl, [&] { return a->impl.plan_update(control_pose, plan); });
}
void bb200_amcl_commit_update(bb200_amcl* a, int resampled, double random_state_probability) {
  if (a != nullptr && !a->impl.filter().weigh_open()) a->impl.commit_update(resampled, random_state_probability);
}
int bb200_motion_sampling_from_control(const bb200_motion_param* p, const double pose[4], const double previous_pose[4], bb200_motion_sampling* out) {
  BB_REQUIRE(p && pose && previous_pose && out);
  *out = bb200::motion_sampling(*p, bb200::Pose2{pose[0], pose[1], pose[2], pose[3]},
                                bb200::Pose2{previous_pose[0], previous_pose[1], previous_pose[2], previous_pose[3]});
  return BB200_OK;
}
int bb200_diff_drive_sampling_from_control(const bb200_diff_drive_param* p, const double pose[4], const double previous_pose[4], bb200_diff_drive_sampling* out) {
  BB_REQUIRE(p && pose && previous_pose && out);
  *out = bb200::diff_drive_sampling(*p, bb200::Pose2{pose[0], pose[1], pose[2], pose[3]},
                                    bb200::Pose2{previous_pose[0], previous_pose[1], previous_pose[2], previous_pose[3]});
  return BB200_OK;
}

}  // extern "C"
