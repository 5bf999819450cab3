// TEST INFRASTRUCTURE ONLY -- flat C entry points over the CPU parity oracle so that the
// pytest suite (ctypes) and bench.py's cpu_baseline / --impl reference legs can drive it.
// Never linked into, loaded by or called from the product library.
#include <cstdint>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "amcl_oracle.hpp"
#include "cluster_oracle.hpp"

using namespace oracle;

namespace {

SE2 se2_from_data(const double* d) { return SE2{SO2::raw(d[0], d[1]), d[2], d[3]}; }

OccupancyGrid make_grid(const std::int8_t* cells, int width, int height, double resolution, const double* origin) {
  OccupancyGrid g;
  g.width = width;
  g.height = height;
  g.resolution = resolution;
  g.origin = se2_from_data(origin);
  g.data.assign(cells, cells + static_cast<std::size_t>(width) * static_cast<std::size_t>(height));
  return g;
}

Points make_points(const double* xy, std::size_t n) {
  Points p(n);
  for (std::size_t i = 0; i < n; ++i) p[i] = {xy[2 * i], xy[2 * i + 1]};
  return p;
}

thread_local std::string g_error;

}  // namespace

extern "C" {

// Mirrors oracle::LikelihoodFieldParam / BeamModelParam / DifferentialDriveParam / AmclParams as POD.
struct orc_lfm_param {
  double max_obstacle_distance, max_laser_distance, z_hit, z_random, sigma_hit;
  int model_unknown_space, only_obstacle_boundaries;
};
struct orc_beam_param {
  double z_hit, z_short, z_max, z_rand, sigma_hit, lambda_short, beam_max_range;
};
struct orc_motion_param {
  double alpha1, alpha2, alpha3, alpha4, distance_threshold;
};
struct orc_amcl_param {
  double update_min_d, update_min_a;
  std::uint64_t resample_interval;
  int selective_resampling;
  std::uint64_t min_particles, max_particles;
  double alpha_slow, alpha_fast, kld_epsilon, kld_z;
  double spatial_resolution_x, spatial_resolution_y, spatial_resolution_theta;
  int rng_mode;  // 0 libstdc++ (mode A), 1 counter (mode B)
  int scheme;    // 0 multinomial, 1 systematic
  std::uint64_t seed;
  int threads;
};
struct orc_update_result {
  int updated, resampled;
  std::uint64_t n_particles;
  double mean[4];  // cos, sin, x, y
  double cov[9];
  double random_state_probability, weight_sum;
  std::uint64_t cells_visited;
};

const char* orc_last_error() { return g_error.c_str(); }

static LikelihoodFieldParam to_lfm(const orc_lfm_param* p) {
  LikelihoodFieldParam o;
  o.max_obstacle_distance = p->max_obstacle_distance;
  o.max_laser_distance = p->max_laser_distance;
  o.z_hit = p->z_hit;
  o.z_random = p->z_random;
  o.sigma_hit = p->sigma_hit;
  o.model_unknown_space = p->model_unknown_space != 0;
  o.only_obstacle_boundaries = p->only_obstacle_boundaries != 0;
  return o;
}
static BeamModelParam to_beam(const orc_beam_param* p) {
  return BeamModelParam{p->z_hit, p->z_short, p->z_max, p->z_rand, p->sigma_hit, p->lambda_short, p->beam_max_range};
}
static DifferentialDriveParam to_motion(const orc_motion_param* p) {
  return DifferentialDriveParam{p->alpha1, p->alpha2, p->alpha3, p->alpha4, p->distance_threshold};
}

// ---- stateless functions ---------------------------------------------------------------------

void orc_philox4x32_10(const std::uint32_t ctr[4], const std::uint32_t key[2], std::uint32_t out[4]) {
  const Philox4 r = philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1]);
  std::memcpy(out, r.v, sizeof(r.v));
}

void orc_se2_compose(const double* a, const double* b, double* out) {
  const SE2 r = se2_from_data(a) * se2_from_data(b);
  out[0] = r.r.c, out[1] = r.r.s, out[2] = r.x, out[3] = r.y;
}
void orc_se2_inverse(const double* a, double* out) {
  const SE2 r = se2_from_data(a).inverse();
  out[0] = r.r.c, out[1] = r.r.s, out[2] = r.x, out[3] = r.y;
}
void orc_se2_from_xytheta(double x, double y, double theta, double* out) {
  const SE2 r{theta, x, y};
  out[0] = r.r.c, out[1] = r.r.s, out[2] = r.x, out[3] = r.y;
}

void orc_distance_map(const std::uint8_t* obstacle, int width, int height, float max_distance, int squared_euclidean, float* out) {
  // test/beluga/algorithm/test_distance_map.cpp uses integer Manhattan-free "distance" lambdas;
  // squared_euclidean=0 -> |dx|+|dy| (manhattan), 1 -> dx^2+dy^2 on unit cells.
  std::vector<bool> mask(static_cast<std::size_t>(width) * height);
  for (std::size_t i = 0; i < mask.size(); ++i) mask[i] = obstacle[i] != 0;
  const auto w = static_cast<std::size_t>(width);
  auto dist = [w, squared_euclidean](std::size_t a, std::size_t b) {
    const double dx = static_cast<double>(a % w) - static_cast<double>(b % w);
    const double dy = static_cast<double>(a / w) - static_cast<double>(b / w);
    return squared_euclidean ? static_cast<float>(dx * dx + dy * dy) : static_cast<float>(std::abs(dx) + std::abs(dy));
  };
  const auto m = nearest_obstacle_distance_map(mask, dist, w, static_cast<std::size_t>(height), max_distance);
  std::memcpy(out, m.data(), m.size() * sizeof(float));
}

int orc_likelihood_field(const orc_lfm_param* p, const std::int8_t* cells, int width, int height, double resolution, const double* origin, float* out) {
  try {
    const ValueGrid f = make_likelihood_field(to_lfm(p), make_grid(cells, width, height, resolution, origin));
    std::memcpy(out, f.data.data(), f.data.size() * sizeof(float));
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

/// weights[i] = L(states[i]) for n states (cos,sin,x,y each); kind: 0 LFM, 1 LFM-prob, 2 beam.
int orc_sensor_weights(
    int kind, const void* param, const std::int8_t* cells, int width, int height, double resolution, const double* origin,
    const double* points_xy, std::uint64_t n_points, const double* states, std::uint64_t n, double* weights, std::uint64_t* cells_visited) {
  try {
    const OccupancyGrid grid = make_grid(cells, width, height, resolution, origin);
    const Points points = make_points(points_xy, n_points);
    std::uint64_t visited = 0;
    if (kind == 2) {
      const BeamModelParam bp = to_beam(static_cast<const orc_beam_param*>(param));
      // particles are independent (the reference runs them under std::execution::par): threaded to keep the big parity cases short
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : visited)
      for (std::int64_t i = 0; i < static_cast<std::int64_t>(n); ++i) {
        std::uint64_t v = 0;
        weights[i] = beam_weight(bp, grid, se2_from_data(states + 4 * i), points, &v);
        visited += v;
      }
    } else {
      const LikelihoodFieldModel model{to_lfm(static_cast<const orc_lfm_param*>(param)), grid};
#pragma omp parallel for schedule(static)
      for (std::int64_t i = 0; i < static_cast<std::int64_t>(n); ++i) {
        const SE2 s = se2_from_data(states + 4 * i);
        weights[i] = kind == 0 ? model.weight(s, points) : model.weight_prob(s, points);
      }
    }
    if (cells_visited != nullptr) *cells_visited = visited;
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

/// Bresenham trace p0 -> p1 (inclusive); returns the number of cells written (<= capacity).
std::uint64_t orc_bresenham(int x0, int y0, int x1, int y1, int modified, int* out_xy, std::uint64_t capacity) {
  std::uint64_t n = 0;
  for (BresenhamLine line(x0, y0, x1, y1, modified != 0); !line.done(); line.next()) {
    if (n < capacity) {
      out_xy[2 * n] = line.cx;
      out_xy[2 * n + 1] = line.cy;
    }
    ++n;
  }
  return n;
}

/// Ray2d::cast for a bearing angle; returns 1 and *distance when something is hit, 0 otherwise.
int orc_raycast(const std::int8_t* cells, int width, int height, double resolution, const double* origin, const double* pose, double max_range, double bearing, double* distance) {
  const OccupancyGrid grid = make_grid(cells, width, height, resolution, origin);
  const Ray2d ray{grid, se2_from_data(pose), max_range};
  const auto r = ray.cast(SO2{bearing});
  if (r.has_value()) {
    *distance = *r;
    return 1;
  }
  return 0;
}

void orc_diff_drive_sampling(const orc_motion_param* p, const double* pose, const double* previous_pose, double* out6) {
  const DiffDriveSampling s = diff_drive_sampling(to_motion(p), se2_from_data(pose), se2_from_data(previous_pose));
  out6[0] = s.rot1_mean, out6[1] = s.rot1_std, out6[2] = s.trans_mean, out6[3] = s.trans_std, out6[4] = s.rot2_mean, out6[5] = s.rot2_std;
}

/// Mode-A / mode-B propagate of n states in place.  mode 0: std::mt19937_64(seed) shared engine.
void orc_diff_drive_propagate(const double* sampling6, int mode, std::uint64_t seed, std::uint32_t step, std::uint64_t first_index, double* states, std::uint64_t n) {
  const DiffDriveSampling s{sampling6[0], sampling6[1], sampling6[2], sampling6[3], sampling6[4], sampling6[5]};
  if (mode == 0) {
    std::vector<SE2> v(n);
    for (std::uint64_t i = 0; i < n; ++i) v[i] = se2_from_data(states + 4 * i);
    std::mt19937_64 gen(seed);
    std::normal_distribution<double> dist;
    diff_drive_propagate_std(v, s, dist, gen);
    for (std::uint64_t i = 0; i < n; ++i) states[4 * i] = v[i].r.c, states[4 * i + 1] = v[i].r.s, states[4 * i + 2] = v[i].x, states[4 * i + 3] = v[i].y;
  } else {
    for (std::uint64_t i = 0; i < n; ++i) {
      const SE2 r = diff_drive_sample_counter(se2_from_data(states + 4 * i), s, seed, first_index + i, step);
      states[4 * i] = r.r.c, states[4 * i + 1] = r.r.s, states[4 * i + 2] = r.x, states[4 * i + 3] = r.y;
    }
  }
}

struct orc_omni_param {
  double alpha1, alpha2, alpha3, alpha4, alpha5, distance_threshold;
};

/// Sampling parameters of any motion model: out10 = {mean[3], stddev[3], first_rotation cos, sin, model, 0}.
void orc_motion_sampling(int model, const orc_omni_param* p, const double* pose, const double* previous_pose, double* out10) {
  MotionSampling m;
  if (model == 1) {
    m = omni_drive_sampling(OmnidirectionalDriveParam{p->alpha1, p->alpha2, p->alpha3, p->alpha4, p->alpha5, p->distance_threshold}, se2_from_data(pose),
                            se2_from_data(previous_pose));
  } else if (model == 2) {
    m = stationary_sampling();
  } else {
    m = to_motion_sampling(diff_drive_sampling(DifferentialDriveParam{p->alpha1, p->alpha2, p->alpha3, p->alpha4, p->distance_threshold},
                                               se2_from_data(pose), se2_from_data(previous_pose)));
  }
  for (int k = 0; k < 3; ++k) out10[k] = m.mean[k], out10[3 + k] = m.stddev[k];
  out10[6] = m.first_rotation.c, out10[7] = m.first_rotation.s, out10[8] = m.model, out10[9] = 0.0;
}

/// Propagate n states with a generic sampling block (layout of orc_motion_sampling); mode 0 std, 1 counter.
void orc_motion_propagate(const double* sampling10, int mode, std::uint64_t seed, std::uint32_t step, std::uint64_t first_index, double* states, std::uint64_t n) {
  MotionSampling m;
  for (int k = 0; k < 3; ++k) m.mean[k] = sampling10[k], m.stddev[k] = sampling10[3 + k];
  m.first_rotation = SO2::raw(sampling10[6], sampling10[7]);
  m.model = static_cast<int>(sampling10[8]);
  std::vector<SE2> v(n);
  for (std::uint64_t i = 0; i < n; ++i) v[i] = se2_from_data(states + 4 * i);
  if (mode == 0) {
    std::mt19937_64 gen(seed);
    std::normal_distribution<double> dist;
    motion_propagate_std(v, m, dist, gen);
  } else {
    for (std::uint64_t i = 0; i < n; ++i) v[i] = motion_sample_counter(v[i], m, seed, first_index + i, step);
  }
  for (std::uint64_t i = 0; i < n; ++i) states[4 * i] = v[i].r.c, states[4 * i + 1] = v[i].r.s, states[4 * i + 2] = v[i].x, states[4 * i + 3] = v[i].y;
}

double orc_normalize(double* weights, std::uint64_t n) {
  std::vector<double> w(weights, weights + n);
  const double f = normalize(w);
  std::memcpy(weights, w.data(), n * sizeof(double));
  return f;
}

double orc_effective_sample_size(const double* weights, std::uint64_t n) { return effective_sample_size(std::vector<double>(weights, weights + n)); }

/// Feeds `count` (total_weight, size) samples through a fresh estimator; writes each probability.
void orc_thrun(double alpha_slow, double alpha_fast, const double* total_weights, const std::uint64_t* sizes, std::uint64_t count, double* out) {
  ThrunRecoveryProbabilityEstimator e{alpha_slow, alpha_fast};
  for (std::uint64_t i = 0; i < count; ++i) out[i] = e.update(total_weights[i], sizes[i]);
}

std::uint64_t orc_spatial_hash(const double* state, double rx, double ry, double rtheta) { return spatial_hash(se2_from_data(state), rx, ry, rtheta); }

std::uint64_t orc_kld_target_size(std::uint64_t k, double epsilon, double z) { return kld_target_size(k, epsilon, z); }

std::uint64_t orc_kld_take_count(const std::uint64_t* hashes, std::uint64_t n, std::uint64_t min, std::uint64_t max, double epsilon, double z) {
  return kld_take_count(std::vector<std::uint64_t>(hashes, hashes + n), min, max, epsilon, z);
}

void orc_estimate(const double* states, const double* weights, std::uint64_t n, double* mean4, double* cov9) {
  std::vector<SE2> s(n);
  for (std::uint64_t i = 0; i < n; ++i) s[i] = se2_from_data(states + 4 * i);
  const Estimate e = estimate(s, std::vector<double>(weights, weights + n));
  mean4[0] = e.mean.r.c, mean4[1] = e.mean.r.s, mean4[2] = e.mean.x, mean4[3] = e.mean.y;
  std::memcpy(cov9, e.cov, sizeof(e.cov));
}

/// Mode-B coin of views::random_intersperse for output slots 0..m-1 (CounterResampler::inject).
void orc_inject_flags(std::uint64_t seed, std::uint32_t step, double probability, std::uint64_t m, std::uint8_t* out) {
  const CounterResampler rs{seed, step, ResampleScheme::kMultinomial, 1ull << 40, m};
  for (std::uint64_t j = 0; j < m; ++j) out[j] = rs.inject(j, probability) ? 1 : 0;
}

/// ExponentialFilter (algorithm/exponential_filter.hpp:35-44): out[i] = filter(values[i]); reset() before sample reset_before (or never: -1).
void orc_exponential_filter(double alpha, const double* values, std::uint64_t n, std::int64_t reset_before, double* out) {
  ExponentialFilter f;
  f.alpha = alpha;
  for (std::uint64_t i = 0; i < n; ++i) {
    if (static_cast<std::int64_t>(i) == reset_before) f.reset();
    out[i] = f(values[i]);
  }
}

// ---- cluster-based estimate (cluster_oracle.hpp) ----------------------------------------------

double orc_percentile_threshold(const double* values, std::uint64_t n, double percentile) {
  return calculate_percentile_threshold(std::vector<double>(values, values + n), percentile);
}

static std::vector<SE2> states_from_data(const double* states, std::uint64_t n) {
  std::vector<SE2> s(n);
  for (std::uint64_t i = 0; i < n; ++i) s[i] = se2_from_data(states + 4 * i);
  return s;
}

void orc_cluster_ids(const double* states, const double* weights, std::uint64_t n, double linear, double angular, double percentile,
                     std::uint64_t* ids_out) {
  const auto ids = ParticleClusterizer{ParticleClusterizerParam{linear, angular, percentile}}(states_from_data(states, n),
                                                                                              std::vector<double>(weights, weights + n));
  for (std::uint64_t i = 0; i < n; ++i) ids_out[i] = ids[i];
}

/// assign_clusters on a hand-made map (one cell per entry, inserted with emplace in the given order,
/// as test_cluster_based_estimation.cpp:171-176 does); n_neighbors = 4 (the test's own neighbour
/// function, :178-189) or 6 (ParticleClusterizer::neighbors).
void orc_assign_clusters(const double* states, const double* cell_weights, std::uint64_t n, double linear, double angular, int n_neighbors,
                         std::uint64_t* ids_out) {
  const ParticleClusterizer c{ParticleClusterizerParam{linear, angular, 0.9}};
  const auto s = states_from_data(states, n);
  ClusterMap map;
  for (std::uint64_t i = 0; i < n; ++i) map.emplace(c.hash(s[i]), ClusterCell{s[i], cell_weights[i], 0, std::nullopt});
  assign_clusters(map, [&](const SE2& pose) {
    auto all = c.neighbors(pose);
    all.resize(static_cast<std::size_t>(n_neighbors));
    return all;
  });
  for (std::uint64_t i = 0; i < n; ++i) ids_out[i] = map[c.hash(s[i])].cluster_id.value();
}

std::uint64_t orc_estimate_clusters(const double* states, const double* weights, const std::uint64_t* clusters, std::uint64_t n,
                                    std::uint64_t max_out, double* weight_out, double* mean4_out, double* cov9_out, std::uint64_t* id_out) {
  const auto per = estimate_clusters(states_from_data(states, n), std::vector<double>(weights, weights + n),
                                     std::vector<std::size_t>(clusters, clusters + n));
  for (std::size_t k = 0; k < per.size() && k < max_out; ++k) {
    weight_out[k] = per[k].weight;
    const Estimate& e = per[k].estimate;
    mean4_out[4 * k + 0] = e.mean.r.c, mean4_out[4 * k + 1] = e.mean.r.s, mean4_out[4 * k + 2] = e.mean.x, mean4_out[4 * k + 3] = e.mean.y;
    std::memcpy(cov9_out + 9 * k, e.cov, sizeof(e.cov));
    id_out[k] = per[k].cluster;
  }
  return per.size();
}

void orc_cluster_based_estimate(const double* states, const double* weights, std::uint64_t n, double linear, double angular, double percentile,
                                double* mean4, double* cov9) {
  const Estimate e = cluster_based_estimate(states_from_data(states, n), std::vector<double>(weights, weights + n),
                                            ParticleClusterizerParam{linear, angular, percentile});
  mean4[0] = e.mean.r.c, mean4[1] = e.mean.r.s, mean4[2] = e.mean.x, mean4[3] = e.mean.y;
  std::memcpy(cov9, e.cov, sizeof(e.cov));
}

int orc_normal_transform(const double* cov9, double* transform9) {
  try {
    normal_transform(cov9, transform9);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

/// Mode-B resampling of a weight vector: indices[j] for j < m (no injection, no KLD).
int orc_resample_indices(const double* weights, std::uint64_t n, std::uint64_t n_total, int scheme, std::uint64_t seed, std::uint32_t step, std::uint64_t m, std::int64_t* indices, std::uint64_t* cdf_out, int* exponent_out, int* valid_out) {
  try {
    const FixedPointCdf cdf = fixed_point_cdf(std::vector<double>(weights, weights + n), n_total);
    const CounterResampler rs{seed, step, static_cast<ResampleScheme>(scheme), cdf.total, m};
    for (std::uint64_t j = 0; j < m; ++j) indices[j] = static_cast<std::int64_t>(cdf_search(cdf.cdf, rs.position(j)));
    if (cdf_out != nullptr) std::memcpy(cdf_out, cdf.cdf.data(), n * sizeof(std::uint64_t));
    if (exponent_out != nullptr) *exponent_out = cdf.exponent;
    if (valid_out != nullptr) *valid_out = cdf.valid ? 1 : 0;
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

/// Mode-A resampling: std::discrete_distribution over `weights` with std::mt19937_64(seed).
void orc_resample_indices_std(const double* weights, std::uint64_t n, std::uint64_t seed, std::uint64_t m, std::int64_t* indices) {
  std::discrete_distribution<std::ptrdiff_t> d(weights, weights + n);
  std::mt19937_64 gen(seed);
  for (std::uint64_t j = 0; j < m; ++j) indices[j] = d(gen);
}

// ---- the filter ------------------------------------------------------------------------------

struct orc_amcl {
  Amcl impl;
};

orc_amcl* orc_amcl_create_motion(const orc_amcl_param* p, int motion_model, const orc_omni_param* m);

orc_amcl* orc_amcl_create(const orc_amcl_param* p, const orc_motion_param* m) {
  const orc_omni_param o{m->alpha1, m->alpha2, m->alpha3, m->alpha4, 0.0, m->distance_threshold};
  return orc_amcl_create_motion(p, 0, &o);
}

orc_amcl* orc_amcl_create_motion(const orc_amcl_param* p, int motion_model, const orc_omni_param* m) {
  AmclParams a;
  a.update_min_d = p->update_min_d;
  a.update_min_a = p->update_min_a;
  a.resample_interval = p->resample_interval;
  a.selective_resampling = p->selective_resampling != 0;
  a.min_particles = p->min_particles;
  a.max_particles = p->max_particles;
  a.alpha_slow = p->alpha_slow;
  a.alpha_fast = p->alpha_fast;
  a.kld_epsilon = p->kld_epsilon;
  a.kld_z = p->kld_z;
  a.spatial_resolution_x = p->spatial_resolution_x;
  a.spatial_resolution_y = p->spatial_resolution_y;
  a.spatial_resolution_theta = p->spatial_resolution_theta;
  a.rng_mode = static_cast<RngMode>(p->rng_mode);
  a.scheme = static_cast<ResampleScheme>(p->scheme);
  a.seed = p->seed;
  a.threads = p->threads;
  return new (std::nothrow) orc_amcl{Amcl{a, DifferentialDriveParam{m->alpha1, m->alpha2, m->alpha3, m->alpha4, m->distance_threshold}, motion_model,
                                          OmnidirectionalDriveParam{m->alpha1, m->alpha2, m->alpha3, m->alpha4, m->alpha5, m->distance_threshold}}};
}
void orc_amcl_destroy(orc_amcl* a) { delete a; }

int orc_amcl_set_map(orc_amcl* a, int kind, const void* param, const std::int8_t* cells, int width, int height, double resolution, const double* origin) {
  try {
    const OccupancyGrid grid = make_grid(cells, width, height, resolution, origin);
    if (kind == 2) {
      a->impl.set_beam_model(to_beam(static_cast<const orc_beam_param*>(param)), grid);
    } else {
      a->impl.set_likelihood_field_model(to_lfm(static_cast<const orc_lfm_param*>(param)), grid, kind == 1);
    }
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

int orc_amcl_get_likelihood_field(const orc_amcl* a, float* out) {
  if (a->impl.lfm() == nullptr) return -1;
  const auto& d = a->impl.lfm()->field.data;
  std::memcpy(out, d.data(), d.size() * sizeof(float));
  return 0;
}

int orc_amcl_initialize_normal(orc_amcl* a, const double* mean_xyt, const double* cov9) {
  try {
    a->impl.initialize_normal(mean_xyt, cov9);
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

int orc_amcl_initialize_from_map(orc_amcl* a) {
  try {
    a->impl.initialize_from_map();
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

void orc_amcl_set_particles(orc_amcl* a, const double* states, const double* weights, std::uint64_t n) {
  std::vector<SE2> s(n);
  for (std::uint64_t i = 0; i < n; ++i) s[i] = se2_from_data(states + 4 * i);
  a->impl.set_particles(s, std::vector<double>(weights, weights + n));
}

std::uint64_t orc_amcl_size(const orc_amcl* a) { return a->impl.states().size(); }

void orc_amcl_get_particles(const orc_amcl* a, double* states, double* weights) {
  const auto& s = a->impl.states();
  for (std::size_t i = 0; i < s.size(); ++i) states[4 * i] = s[i].r.c, states[4 * i + 1] = s[i].r.s, states[4 * i + 2] = s[i].x, states[4 * i + 3] = s[i].y;
  std::memcpy(weights, a->impl.weights().data(), s.size() * sizeof(double));
}

std::uint64_t orc_amcl_last_indices(const orc_amcl* a, std::int64_t* out, std::uint64_t capacity) {
  const auto& idx = a->impl.last_indices();
  const std::uint64_t n = std::min<std::uint64_t>(capacity, idx.size());
  if (out != nullptr) std::memcpy(out, idx.data(), n * sizeof(std::int64_t));
  return idx.size();
}

void orc_amcl_force_update(orc_amcl* a) { a->impl.force_update(); }

int orc_amcl_update(orc_amcl* a, const double* control_pose, const double* points_xy, std::uint64_t n_points, orc_update_result* out) {
  try {
    const UpdateResult r = a->impl.update(se2_from_data(control_pose), make_points(points_xy, n_points));
    out->updated = r.updated ? 1 : 0;
    out->resampled = r.resampled ? 1 : 0;
    out->n_particles = r.n_particles;
    out->mean[0] = r.estimate.mean.r.c, out->mean[1] = r.estimate.mean.r.s, out->mean[2] = r.estimate.mean.x, out->mean[3] = r.estimate.mean.y;
    std::memcpy(out->cov, r.estimate.cov, sizeof(r.estimate.cov));
    out->random_state_probability = r.random_state_probability;
    out->weight_sum = r.weight_sum;
    out->cells_visited = r.cells_visited;
    return 0;
  } catch (const std::exception& e) {
    g_error = e.what();
    return -1;
  }
}

}  // extern "C"
