#include "sharded_amcl.hpp"

#include <algorithm>

#include "cluster_host.hpp"

namespace bb200 {

namespace {

/// Shard r's parameters: the filter's, on devices[r], holding the r-th of n_shards equal particle ranges.
bb200_amcl_param shard_param(const bb200_amcl_param& p, int n_shards, int r, int device) {
  const uint64_t shard = p.max_particles / static_cast<uint64_t>(n_shards);
  bb200_amcl_param q = p;
  q.device = device;
  q.shard_capacity = shard;
  q.shard_first_index = static_cast<uint64_t>(r) * shard;
  return q;
}

}  // namespace

int ShardedAmcl::validate(const bb200_amcl_param& p, const bb200_motion_param& motion, int n_shards, std::string* error) {
  if (n_shards < 1 || n_shards > kMaxShards || p.max_particles == 0 || p.max_particles % static_cast<uint64_t>(n_shards) != 0) {
    if (error != nullptr) *error = "a filter splits into 1..8 equal shards: max_particles must be a multiple of n_shards";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  for (int r = 0; r < n_shards; ++r)
    if (const int st = Amcl::validate(shard_param(p, n_shards, r, p.device), motion, error)) return st;
  return BB200_OK;
}

ShardedAmcl::ShardedAmcl(const bb200_amcl_param& p, const bb200_motion_param& motion, int n_shards, const int* devices) {
  create_status_ = validate(p, motion, n_shards, &error_);
  if (create_status_ != BB200_OK) return;
  std::vector<ShardLink*> links;
  for (int r = 0; r < n_shards; ++r) {
    auto a = std::make_unique<Amcl>(shard_param(p, n_shards, r, devices[r]), motion);
    if (!a->ok()) {
      error_ = a->last_error();
      create_status_ = a->create_status();
      return;
    }
    links.push_back(&a->filter().link());
    ranks_.push_back(a.get());
    shards_.push_back(std::move(a));
  }
  create_status_ = ShardLink::join_local(links.data(), n_shards);
  if (create_status_ != BB200_OK) {
    error_ = "joining the shards failed (peer access between the devices?)";
    for (Amcl* a : ranks_)
      if (a->filter().last_error()[0] != '\0') error_ = a->filter().last_error();
    return;
  }
  created_ = true;
}

const char* ShardedAmcl::last_error() const {
  if (!error_.empty()) return error_.c_str();
  for (const Amcl* a : ranks_)
    if (a->last_error()[0] != '\0') return a->last_error();
  return "";
}

int ShardedAmcl::set_map(const std::function<int(MapTables*, std::string*)>& prepare) {
  error_.clear();
  MapTables tables;
  std::string message;
  int st = prepare(&tables, &message);
  if (st != BB200_OK) return ranks_[0]->filter().fail_with(st, message);
  for (auto a = ranks_.begin(); st == BB200_OK && a != ranks_.end(); ++a) st = (*a)->filter().set_map(tables);
  return st;
}

int ShardedAmcl::set_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map) {
  return set_map([&](MapTables* t, std::string* e) { return prepare_landmark_map(lp, bp, map, t, e); });
}

int ShardedAmcl::initialize(const double mean[3], const double cov[9]) {
  error_.clear();
  for (Amcl* a : ranks_)
    if (const int st = a->initialize(mean, cov)) return st;
  return BB200_OK;
}

int ShardedAmcl::initialize_from_map() {
  error_.clear();
  for (Amcl* a : ranks_)
    if (const int st = a->initialize_from_map()) return st;
  return BB200_OK;
}

void ShardedAmcl::force_update() {
  for (Amcl* a : ranks_) a->force_update();
}

int ShardedAmcl::update(const double control[4], const double* points_xy, uint64_t n_points, bb200_update_result* out) {
  error_.clear();
  return Amcl::update_group(ranks_.data(), shards(), control, points_xy, n_points, out);
}

int ShardedAmcl::update_landmarks(const double control[4], const bb200_landmark_detection* detections, uint64_t n, bb200_update_result* out) {
  error_.clear();
  *out = bb200_update_result{};
  if (detections == nullptr && n > 0) {
    error_ = "detections is null";
    return static_cast<int>(BB200_ERR_INVALID_ARGUMENT);
  }
  // Every shard holds the same tables: the detections are prepared once, against rank 0's, and uploaded to every shard
  // before any shard's step starts.  The uploads only enqueue copies, and no policy has moved yet.
  std::vector<LandmarkDetection> prepared;
  if (const int st = ranks_[0]->filter().prepare_step_detections(detections, n, &prepared)) return st;
  for (Amcl* a : ranks_)
    if (const int st = a->filter().upload_detections(prepared)) return st;
  return Amcl::update_group(ranks_.data(), shards(), control, Filter::staged_detections(), 0, out);
}

int ShardedAmcl::update_begin(const double control[4], bb200_weigh_view* views) {
  error_.clear();
  return Amcl::update_group_begin(ranks_.data(), shards(), control, views);
}

int ShardedAmcl::update_end(bb200_update_result* out) {
  error_.clear();
  return Amcl::update_group_end(ranks_.data(), shards(), out);
}

int ShardedAmcl::merged_cells(double linear_resolution, double angular_resolution, std::vector<bb200_cluster_cell>* merged, uint64_t* n_particles) {
  static_assert(sizeof(bb200_cluster_cell) == sizeof(HostCell), "public and internal cell records must agree");
  const int shards = static_cast<int>(ranks_.size());
  std::vector<std::vector<HostCell>> cells(static_cast<size_t>(shards));
  std::vector<const bb200_cluster_cell*> ptrs;
  std::vector<uint64_t> counts, firsts;
  uint64_t total_cells = 0;
  *n_particles = 0;
  for (int r = 0; r < shards; ++r) {
    Filter& f = ranks_[static_cast<size_t>(r)]->filter();
    std::vector<HostCell>& c = cells[static_cast<size_t>(r)];
    if (f.size() > 0)
      if (const int st = f.cell_records(linear_resolution, angular_resolution, &c)) return st;
    const uint64_t n = c.size();
    ptrs.push_back(reinterpret_cast<const bb200_cluster_cell*>(c.data()));
    counts.push_back(n);
    firsts.push_back(f.first_index());
    total_cells += n;
    *n_particles += f.size();
  }
  if (*n_particles == 0) {
    error_ = "no particles";
    return static_cast<int>(BB200_ERR_STATE);
  }
  merged->resize(total_cells);
  uint64_t n_merged = 0;
  const int st = merge_cells(ptrs.data(), counts.data(), firsts.data(), shards, merged->data(), merged->size(), &n_merged);
  if (st != BB200_OK) return st;
  merged->resize(n_merged);
  return static_cast<int>(BB200_OK);
}

int ShardedAmcl::cluster_estimate(const bb200_cluster_param& p, bb200_estimate* out, uint32_t* n_cells, uint32_t* n_clusters) {
  error_.clear();
  std::vector<bb200_cluster_cell> merged;
  uint64_t n_particles = 0;
  const int st = merged_cells(p.linear_hash_resolution, p.angular_hash_resolution, &merged, &n_particles);
  if (st != BB200_OK) return st;
  const ClusterSelection sel = select_cluster(reinterpret_cast<const HostCell*>(merged.data()), merged.size(), n_particles, p.linear_hash_resolution,
                                              p.angular_hash_resolution, p.weight_cap_percentile);
  estimate_from_moments(sel.moments, ranks_[0]->filter().pivot(), out);  // every shard accumulates about the same pivot
  if (n_cells != nullptr) *n_cells = static_cast<uint32_t>(merged.size());
  if (n_clusters != nullptr) *n_clusters = sel.clusters;
  return static_cast<int>(BB200_OK);
}

int ShardedAmcl::get_particles(double* states, double* weights, uint64_t capacity) {
  error_.clear();
  uint64_t done = 0;
  for (Amcl* a : ranks_) {  // rank order is global particle order
    Filter& f = a->filter();
    const uint64_t n = std::min<uint64_t>(f.size(), capacity - done);
    const int st = f.get_particles(states != nullptr ? states + 4 * done : nullptr, weights != nullptr ? weights + done : nullptr, n);
    if (st != BB200_OK) return st;
    done += n;
    if (done >= capacity) break;
  }
  return static_cast<int>(BB200_OK);
}

int ShardedAmcl::particle_histogram(double linear_resolution, double angular_resolution, bb200_cluster_cell* bins, uint64_t capacity, uint64_t* n_bins,
                                    double* max_bin_weight) {
  error_.clear();
  std::vector<bb200_cluster_cell> merged;
  uint64_t n_particles = 0;
  const int st = merged_cells(linear_resolution, angular_resolution, &merged, &n_particles);
  if (st != BB200_OK) return st;
  if (n_bins != nullptr) *n_bins = merged.size();
  double top = 1e-3;  // beluga_ros/particle_cloud.hpp:197
  for (const bb200_cluster_cell& c : merged) top = c.weight > top ? c.weight : top;
  if (max_bin_weight != nullptr) *max_bin_weight = top;
  if (bins != nullptr) {
    if (capacity < merged.size()) {
      error_ = "histogram bin buffer too small (n_bins has the count)";
      return static_cast<int>(BB200_ERR_CAPACITY);
    }
    std::copy(merged.begin(), merged.end(), bins);
  }
  return static_cast<int>(BB200_OK);
}

int ShardedAmcl::sample_states(uint64_t count, uint32_t step, double* states_out) {
  error_.clear();
  const size_t shards = ranks_.size();
  std::vector<Filter*> f(shards);
  uint64_t n_particles = 0;
  for (size_t r = 0; r < shards; ++r) {
    f[r] = &ranks_[r]->filter();
    n_particles += f[r]->size();
  }
  const uint64_t max_particles = ranks_[0]->params().max_particles;
  if (n_particles == 0) {
    error_ = "no particles";
    return static_cast<int>(BB200_ERR_STATE);
  }
  if (count > max_particles) {
    error_ = "more samples than the filter capacity";
    return static_cast<int>(BB200_ERR_CAPACITY);
  }
  if (count > 0 && states_out == nullptr) {
    error_ = "states_out is null";
    return static_cast<int>(BB200_ERR_INVALID_ARGUMENT);
  }
  if (count == 0) return static_cast<int>(BB200_OK);
  // The global CDF: the one the last step left when it kept its particles, or one built as a sharded step builds it --
  // the exponent from the largest weight of all shards, the offsets from the shards' fixed-point totals in rank order.
  // Current CDFs quantised with different exponents were built shard by shard (e.g. bb200_filter_build_cdf on one shard):
  // together they are no global CDF.  With one exponent on every shard they are the global build's bit for bit, since
  // the global largest weight is some shard's largest weight.
  std::vector<uint64_t> totals(shards, 0);
  bool current = true, first = true;
  int exponent = 0;
  for (size_t r = 0; r < shards; ++r) {
    if (f[r]->size() == 0) continue;
    int e = 0;
    if (const int st = f[r]->current_cdf(&totals[r], &e)) return st;
    current = current && totals[r] != 0 && (first || e == exponent);
    exponent = e;
    first = false;
  }
  if (!current) {
    double wmax = 0.0;
    for (size_t r = 0; r < shards; ++r) {
      if (f[r]->size() == 0) continue;
      double w = 0.0;
      if (const int st = f[r]->max_weight(&w)) return st;
      wmax = w > wmax ? w : wmax;
    }
    for (size_t r = 0; r < shards; ++r)
      if (f[r]->size() > 0)
        if (const int st = f[r]->build_cdf(wmax, &totals[r], nullptr)) return st;
  }
  uint64_t total = 0;
  std::vector<uint64_t> offsets(shards, 0);
  for (size_t r = 0; r < shards; ++r) {
    offsets[r] = total;
    total += totals[r];
  }
  for (size_t r = 0; r < shards; ++r)
    if (const int st = f[r]->sample_range(count, step, total, offsets[r])) return st;
  for (Filter* s : f)  // every shard's draws have reached their slots' staging buffers
    if (const int st = s->synchronize()) return st;
  const uint64_t shard = max_particles / shards;  // slot j lies in the staging buffer of shard j / shard
  for (size_t r = 0; r < shards && r * shard < count; ++r)
    if (const int st = f[r]->staging_states(states_out + 4 * r * shard, std::min<uint64_t>(shard, count - r * shard))) return st;
  return static_cast<int>(BB200_OK);
}

int ShardedAmcl::cast_rays(const double* poses, uint64_t n_poses, const double* bearings_cs, uint64_t n_bearings, double max_range, double* ranges) {
  error_.clear();
  uint64_t n_rays = 0;
  if (const int st = ranks_[0]->filter().check_cast_rays(poses, n_poses, bearings_cs, n_bearings, ranges, &n_rays)) return st;
  if (n_rays == 0) return static_cast<int>(BB200_OK);
  // The poses are cut into contiguous ranges, one per shard, each cast on that shard's copy of the map; every shard
  // launches before any reads back, so shards on different devices cast at the same time.
  std::vector<Filter*> casters;
  for (Amcl* a : ranks_) casters.push_back(&a->filter());
  const uint64_t k = casters.size();
  auto first_pose = [&](uint64_t c) { return n_poses * c / k; };  // n_poses <= kMaxCastRays: no overflow
  for (uint64_t c = 0; c < k; ++c) {
    const uint64_t begin = first_pose(c), end = first_pose(c + 1);
    if (end > begin)
      if (const int st = casters[c]->enqueue_cast_rays(poses + 4 * begin, end - begin, bearings_cs, n_bearings, max_range)) return st;
  }
  for (uint64_t c = 0; c < k; ++c) {
    const uint64_t begin = first_pose(c), end = first_pose(c + 1);
    if (end > begin)
      if (const int st = casters[c]->finish_cast_rays(ranges + begin * n_bearings, (end - begin) * n_bearings)) return st;
  }
  return static_cast<int>(BB200_OK);
}

}  // namespace bb200
