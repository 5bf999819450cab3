#include "batch.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <initializer_list>

namespace bb200 {

namespace {

constexpr uint64_t kSliceAlign = 32;  // particles
static_assert(kBatchMaxParticles <= kBatchClusterMaxParticles, "the batch cluster estimate packs a member's particle index into 15 bits");

/// Moment-partial rows a member of `capacity` particles can need in the finish launch (whichever form it takes).
uint64_t finish_rows(uint64_t capacity) {
  return std::max<uint64_t>({resample_scatter_block_count(capacity), resample_block_count(capacity), moments_block_count(capacity)});
}

}  // namespace

int Batch::validate(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, std::string* error) {
  auto reject = [&](const std::string& m) {
    if (error != nullptr) *error = m;
    return static_cast<int>(BB200_ERR_INVALID_ARGUMENT);
  };
  if (params == nullptr || motions == nullptr) return reject("null argument");
  if (n_members < 1) return reject("a batch needs at least one member");
  for (int k = 0; k < n_members; ++k) {
    const bb200_amcl_param& p = params[k];
    const std::string who = "member " + std::to_string(k) + ": ";
    if (p.device != params[0].device) return reject(who + "all members of a batch share one device");
    if (p.max_particles == 0 || p.max_particles > kBatchMaxParticles) return reject(who + "max_particles must lie in [1, 32768]");
    if (p.min_particles != p.max_particles) return reject(who + "a batch member keeps a fixed particle count (min_particles == max_particles)");
    if (p.selective_resampling) return reject(who + "selective resampling is not supported in a batch");
    if (p.shard_first_index != 0 || p.shard_capacity != 0) return reject(who + "a batch member is not sharded");
    if (!(p.alpha_slow >= 0.0) || !(p.alpha_slow <= p.alpha_fast)) return reject(who + "need 0 <= alpha_slow <= alpha_fast");
    if (motions[k].model < BB200_MOTION_DIFFERENTIAL || motions[k].model > BB200_MOTION_STATIONARY) return reject(who + "unknown motion model");
  }
  return BB200_OK;
}

Batch::Batch(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members) {
  create_status_ = validate(params, motions, n_members, &error_);
  if (create_status_ != BB200_OK) return;
  uint64_t tiles = 0, rows = 0;
  members_.reserve(static_cast<size_t>(n_members));
  for (int k = 0; k < n_members; ++k) {
    members_.push_back(Member{AmclPolicy(params[k], motions[k])});
    Member& m = members_.back();
    // The CDF build reads weights and writes the CDF 16 bytes at a time from the slice's start: slices begin on whole
    // 256-byte lines.
    total_ = (total_ + kSliceAlign - 1) / kSliceAlign * kSliceAlign;
    m.offset = total_;
    m.capacity = params[k].max_particles;
    total_ += m.capacity;
    m.table_offset = table_total_;
    m.table_slots = 2;
    while (m.table_slots < 2 * m.capacity) m.table_slots <<= 1;
    table_total_ += m.table_slots;
    tiles += batch_scan_tiles(m.capacity);
    rows += finish_rows(m.capacity);
    record_ancestors_ = record_ancestors_ || params[k].record_ancestors != 0;
  }
  device_ = params[0].device;
  create_status_ = check_device(device_, &error_);
  if (create_status_ != BB200_OK) return;
  const size_t k1 = static_cast<size_t>(n_members) + 1;
  BB_TRY(cudaSetDevice(device_));
  BB_TRY(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  BB_TRY(dev_alloc(&states_[0], total_));
  BB_TRY(dev_alloc(&states_[1], total_));
  BB_TRY(dev_alloc(&weights_, total_));
  BB_TRY(dev_alloc(&cdf_, total_));
  if (record_ancestors_) BB_TRY(dev_alloc(&ancestors_, total_));
  BB_TRY(dev_alloc(&scalars_, members_.size()));
  BB_TRY(dev_alloc(&tile_state_, tiles));
  BB_TRY(dev_alloc(&partials_, rows * kMomentCount));
  BB_TRY(dev_alloc(&table_, members_.size()));
  BB_TRY(host_alloc(&table_host_, members_.size()));
  BB_TRY(dev_alloc(&first_, kBatchLaunches * k1));
  BB_TRY(host_alloc(&first_host_, kBatchLaunches * k1));
  BB_TRY(host_alloc(&summary_host_, members_.size()));
  BB_TRY(host_alloc(&ticket_host_, 1));
  BB_TRY(dev_alloc(&members_done_, 1));
  *ticket_host_ = 0;  // pinned allocations are recycled with their old contents
  BB_TRY(cudaMemsetAsync(scalars_, 0, members_.size() * sizeof(Scalars), stream_));
  BB_TRY(cudaMemsetAsync(members_done_, 0, sizeof(unsigned int), stream_));
  BB_TRY(cudaStreamSynchronize(stream_));
  created_ = true;
}

Batch::~Batch() {
  if (stream_ != nullptr) cudaStreamSynchronize(stream_);
  for (void* p : std::initializer_list<void*>{states_[0], states_[1], weights_, cdf_, ancestors_, scalars_, tile_state_, partials_, table_, first_,
                                              points_, hits_, map_table_, members_done_, cl_hashes_, cl_keys_, cl_first_, cl_ids_, cl_cell_of_, cl_sort_[0], cl_sort_[1],
                                              cl_starts_, cl_records_, cl_table_, cl_cells_, sm_table_, samples_})
    cudaFree(p);
  for (void* p : std::initializer_list<void*>{table_host_, first_host_, points_host_, summary_host_, ticket_host_, cl_table_host_, cl_cells_host_,
                                              cl_records_host_, sm_table_host_, samples_host_})
    cudaFreeHost(p);
  if (stream_ != nullptr) cudaStreamDestroy(stream_);
}

int Batch::member_ok(int member) const {
  if (member < 0 || member >= members()) {
    error_ = "member index out of range";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  return BB200_OK;
}

#define BB_MEMBER(member) do { error_.clear(); if (const int st_ = member_ok(member)) return st_; } while (0)

const Batch::MapEntry* Batch::find_map(int id) const {
  const auto it = maps_.find(id);
  if (it != maps_.end()) return &it->second;
  error_ = "unknown map id " + std::to_string(id);
  return nullptr;
}

int Batch::set_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob) {
  error_.clear();
  MapTables tables;
  const int st = prepare_likelihood_field_map(p, grid, prob, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Batch::set_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid) {
  error_.clear();
  MapTables tables;
  const int st = prepare_beam_map(p, grid, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Batch::add_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob, int* id) {
  error_.clear();
  MapTables tables;
  const int st = prepare_likelihood_field_map(p, grid, prob, &tables, &error_);
  return st != BB200_OK ? st : add_map(tables, id);
}

int Batch::add_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid, int* id) {
  error_.clear();
  MapTables tables;
  const int st = prepare_beam_map(p, grid, &tables, &error_);
  return st != BB200_OK ? st : add_map(tables, id);
}

int Batch::set_map(const MapTables& tables) {
  // The old maps go before the new one is uploaded, so that the device never holds both; a failed upload leaves the
  // batch without a map.
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  maps_.clear();
  map_table_current_ = false;
  for (Member& m : members_) m.map = -1;
  int id = -1;
  const int st = add_map(tables, &id);
  if (st != BB200_OK) return st;
  for (Member& m : members_) m.map = id;
  return BB200_OK;
}

int Batch::add_map(const MapTables& tables, int* id) {
  BB_CHECK(cudaSetDevice(device_));
  const int new_id = next_map_id_;
  MapEntry& e = maps_[new_id];
  const int st = e.map.upload(tables, stream_, &error_);
  launches_ += e.map.launches();
  if (st != BB200_OK) {
    maps_.erase(new_id);
    return st;
  }
  map_table_current_ = false;
  ++next_map_id_;
  *id = new_id;
  return BB200_OK;
}

int Batch::update_map(int member, int id) {
  BB_MEMBER(member);
  if (find_map(id) == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  members_[static_cast<size_t>(member)].map = id;
  return BB200_OK;
}

int Batch::member_map(int member, int* id) const {
  error_.clear();
  if (const int st = member_ok(member)) return st;
  *id = members_[static_cast<size_t>(member)].map;
  return BB200_OK;
}

int Batch::remove_map(int id) {
  error_.clear();
  if (find_map(id) == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  for (size_t k = 0; k < members_.size(); ++k)
    if (members_[k].map == id) return fail(BB200_ERR_STATE, "member " + std::to_string(k) + " reads map " + std::to_string(id));
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));  // nothing in flight reads its tables
  maps_.erase(id);
  map_table_current_ = false;
  return BB200_OK;
}

int Batch::get_likelihood_field(int id, float* out, uint64_t capacity) const {
  error_.clear();
  const MapEntry* e = find_map(id);
  if (e == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  const std::vector<float>& field = e->map.field_host;
  if (field.empty()) {
    error_ = "map " + std::to_string(id) + " is not a likelihood-field map";
    return BB200_ERR_STATE;
  }
  if (capacity < field.size()) {
    error_ = "capacity below the field's cells";
    return BB200_ERR_CAPACITY;
  }
  std::memcpy(out, field.data(), field.size() * sizeof(float));
  return BB200_OK;
}

int Batch::ensure_map_table() {
  if (map_table_current_) return BB200_OK;
  std::vector<BatchMap> host;
  host.reserve(maps_.size());
  for (auto& [id, e] : maps_) {
    const DeviceMap& d = e.map;
    e.slot = static_cast<int>(host.size());
    host.push_back(BatchMap{d.field, d.occupancy, d.beam, d.free_cells, d.n_free, d.grid_width, d.grid_resolution, d.grid_origin});
  }
  if (host.size() > map_table_capacity_) {
    BB_CHECK(cudaFree(map_table_));  // every batch call ends synchronised: no step reads the old table
    map_table_ = nullptr;
    map_table_capacity_ = 0;
    BB_CHECK(dev_alloc(&map_table_, host.size()));
    map_table_capacity_ = host.size();
  }
  // On the batch's stream, so that the step's launches follow the copy in order; the pageable source is staged before the
  // call returns.
  BB_CHECK(cudaMemcpyAsync(map_table_, host.data(), host.size() * sizeof(BatchMap), cudaMemcpyHostToDevice, stream_));
  map_table_current_ = true;
  return BB200_OK;
}

int Batch::initialize(int member, const double mean[3], const double cov[9]) {
  BB_MEMBER(member);
  Member& m = members_[static_cast<size_t>(member)];
  double transform[9];
  std::string message;
  if (!normal_transform(cov, transform, &message)) return fail(BB200_ERR_INVALID_ARGUMENT, message);
  BB_CHECK(cudaSetDevice(device_));
  m.cdf_total = 0;
  launch_initialize_normal(states_[m.cur] + m.offset, weights_ + m.offset, m.capacity, mean, transform, m.policy.params().seed, 0, stream_);
  ++launches_;
  BB_CHECK(cudaGetLastError());
  BB_CHECK(cudaStreamSynchronize(stream_));
  m.n = m.capacity;
  m.pivot[0] = mean[0];
  m.pivot[1] = mean[1];
  m.policy.force_update();  // amcl_core.hpp:136
  return BB200_OK;
}

int Batch::initialize_from_map(int member) {
  BB_MEMBER(member);
  Member& m = members_[static_cast<size_t>(member)];
  if (m.map < 0) return fail(BB200_ERR_STATE, "initialize_from_map needs a map (set_*_map or update_map first)");
  const DeviceMap& map = maps_.at(m.map).map;
  if (map.n_free == 0) return fail(BB200_ERR_STATE, "the map has no free cell to sample from");
  BB_CHECK(cudaSetDevice(device_));
  m.cdf_total = 0;
  launch_initialize_uniform(states_[m.cur] + m.offset, weights_ + m.offset, m.capacity, map.free_cells, map.n_free, map.grid_width,
                            map.grid_resolution, map.grid_origin, m.policy.params().seed, 0, stream_);
  ++launches_;
  BB_CHECK(cudaGetLastError());
  BB_CHECK(cudaStreamSynchronize(stream_));
  m.n = m.capacity;
  map.centre(m.pivot);
  m.policy.force_update();
  return BB200_OK;
}

int Batch::initialize_states(int member, const double* states, const double* weights, uint64_t n) {
  BB_MEMBER(member);
  Member& m = members_[static_cast<size_t>(member)];
  if (n > m.capacity) return fail(BB200_ERR_CAPACITY, "more particles than the member's max_particles");
  if (n > 0 && states == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "states is null");
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  m.cdf_total = 0;
  if (n > 0) {
    BB_CHECK(cudaMemcpy(states_[m.cur] + m.offset, states, n * sizeof(Pose2), cudaMemcpyHostToDevice));
    const std::vector<double> ones(weights == nullptr ? n : 0, 1.0);
    BB_CHECK(cudaMemcpy(weights_ + m.offset, weights != nullptr ? weights : ones.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    m.pivot[0] = states[2];
    m.pivot[1] = states[3];
  }
  m.n = n;
  m.policy.force_update();
  return BB200_OK;
}

int Batch::force_update(int member) {
  BB_MEMBER(member);
  members_[static_cast<size_t>(member)].policy.force_update();
  return BB200_OK;
}

int Batch::get_particles(int member, double* states, double* weights, uint64_t capacity) {
  BB_MEMBER(member);
  const Member& m = members_[static_cast<size_t>(member)];
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, m.n);
  if (states != nullptr && n > 0) BB_CHECK(cudaMemcpy(states, states_[m.cur] + m.offset, n * sizeof(Pose2), cudaMemcpyDeviceToHost));
  if (weights != nullptr && n > 0) BB_CHECK(cudaMemcpy(weights, weights_ + m.offset, n * sizeof(double), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

int Batch::ancestors(int member, int64_t* out, uint64_t capacity) {
  BB_MEMBER(member);
  const Member& m = members_[static_cast<size_t>(member)];
  if (!m.policy.params().record_ancestors) return fail(BB200_ERR_STATE, "the member was created without record_ancestors");
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, m.ancestors_n);
  if (out != nullptr && n > 0) BB_CHECK(cudaMemcpy(out, ancestors_ + m.offset, n * sizeof(int64_t), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

int Batch::cluster_estimate(int member, const bb200_cluster_param& p, bb200_estimate* out) {
  BB_MEMBER(member);
  std::vector<uint8_t> present(members_.size(), 0);
  present[static_cast<size_t>(member)] = 1;
  std::vector<bb200_estimate> all(members_.size());  // indexed by member
  const int st = cluster_estimates(p, present.data(), all.data(), nullptr, nullptr);
  if (st == BB200_OK) *out = all[static_cast<size_t>(member)];
  return st;
}

int Batch::ensure_cluster_scratch() {
  if (cl_cells_host_ != nullptr) return BB200_OK;
  const size_t k = members_.size();
  BB_CHECK(dev_alloc(&cl_hashes_, total_));
  BB_CHECK(dev_alloc(&cl_keys_, table_total_));
  BB_CHECK(dev_alloc(&cl_first_, table_total_));
  BB_CHECK(dev_alloc(&cl_ids_, table_total_));
  BB_CHECK(dev_alloc(&cl_cell_of_, total_));
  BB_CHECK(dev_alloc(&cl_sort_[0], total_));
  BB_CHECK(dev_alloc(&cl_sort_[1], total_));
  BB_CHECK(dev_alloc(&cl_starts_, total_ + k));
  BB_CHECK(dev_alloc(&cl_records_, total_));
  BB_CHECK(dev_alloc(&cl_table_, k));
  BB_CHECK(host_alloc(&cl_table_host_, k));
  BB_CHECK(dev_alloc(&cl_cells_, k));
  BB_CHECK(host_alloc(&cl_cells_host_, k));  // last: marks the scratch as allocated
  return BB200_OK;
}

int Batch::ensure_cluster_records(uint64_t cells) {
  if (cells <= cl_records_host_capacity_) return BB200_OK;
  cudaFreeHost(cl_records_host_);
  cl_records_host_ = nullptr;
  cl_records_host_capacity_ = 0;
  const uint64_t want = std::min<uint64_t>(total_, std::max<uint64_t>(4096, 2 * cells));
  BB_CHECK(host_alloc(&cl_records_host_, want));
  cl_records_host_capacity_ = want;
  return BB200_OK;
}

int Batch::cluster_estimates(const bb200_cluster_param& p, const uint8_t* present, bb200_estimate* out, uint32_t* n_cells, uint32_t* n_clusters) {
  error_.clear();
  if (!(p.linear_hash_resolution > 0.0) || !(p.angular_hash_resolution > 0.0) || !(p.weight_cap_percentile >= 0.0) ||
      !(p.weight_cap_percentile < 1.0))
    return fail(BB200_ERR_INVALID_ARGUMENT, "cluster parameters: resolutions must be positive and the percentile in [0, 1)");
  std::vector<uint32_t> selected;
  if (const int st = select_members(present, &selected)) return st;
  if (selected.empty()) return BB200_OK;
  if (const int st = cell_records(p.linear_hash_resolution, p.angular_hash_resolution, selected)) return st;

  // Host pass per member (Clusterizer::estimate's): the flood over the cells, then the estimate about the member's pivot.
  const HostCell* cells = reinterpret_cast<const HostCell*>(cl_records_host_);
  for (size_t j = 0; j < selected.size(); ++j) {
    const uint32_t k = selected[j];
    const Member& m = members_[k];
    const uint32_t count = cl_cells_host_[j];
    const ClusterSelection sel = select_cluster(cells, count, m.n, p.linear_hash_resolution, p.angular_hash_resolution, p.weight_cap_percentile);
    if (out != nullptr) estimate_from_moments(sel.moments, m.pivot, &out[k]);
    if (n_cells != nullptr) n_cells[k] = count;
    if (n_clusters != nullptr) n_clusters[k] = sel.clusters;
    cells += count;
  }
  return BB200_OK;
}

int Batch::select_members(const uint8_t* present, std::vector<uint32_t>* selected) {
  for (size_t k = 0; k < members_.size(); ++k) {
    if (present != nullptr && present[k] == 0) continue;
    if (members_[k].n == 0) return fail(BB200_ERR_STATE, "member " + std::to_string(k) + ": no particles");
    selected->push_back(static_cast<uint32_t>(k));
  }
  return BB200_OK;
}

int Batch::cell_records(double linear, double angular, const std::vector<uint32_t>& selected) {
  BB_CHECK(cudaSetDevice(device_));
  if (const int st = ensure_cluster_scratch()) return st;  // every batch call ends synchronised: the pinned buffers are free

  const uint32_t n_sel = static_cast<uint32_t>(selected.size());
  for (uint32_t j = 0; j < n_sel; ++j) {
    const uint32_t k = selected[j];
    const Member& m = members_[k];
    BatchClusterMember& c = cl_table_host_[j];
    c = BatchClusterMember{};
    c.offset = m.offset;
    c.table_offset = m.table_offset;
    c.starts_offset = m.offset + k;  // a member's cells + 1 starts end before the next member's slice begins
    c.n = static_cast<uint32_t>(m.n);
    c.table_mask = m.table_slots - 1;
    c.cur = static_cast<uint32_t>(m.cur);
    c.pivot_x = m.pivot[0];
    c.pivot_y = m.pivot[1];
  }
  cudaStream_t stream = stream_;
  BB_CHECK(cudaMemcpyAsync(cl_table_, cl_table_host_, n_sel * sizeof(BatchClusterMember), cudaMemcpyHostToDevice, stream));
  BatchClusterArgs a{};
  a.members = cl_table_;
  a.states[0] = states_[0];
  a.states[1] = states_[1];
  a.weights = weights_;
  a.linear = linear;
  a.angular = angular;
  a.hashes = cl_hashes_;
  a.keys = cl_keys_;
  a.first = cl_first_;
  a.ids = cl_ids_;
  a.cell_of = cl_cell_of_;
  a.sort_a = cl_sort_[0];
  a.sort_b = cl_sort_[1];
  a.starts = cl_starts_;
  a.records = cl_records_;
  a.cells = cl_cells_;
  launch_batch_cluster_cells(a, n_sel, stream);
  BB_LAUNCHED("batch_cluster_cells");
  BB_CHECK(cudaMemcpyAsync(cl_cells_host_, cl_cells_, n_sel * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  BB_CHECK(cudaStreamSynchronize(stream));  // 1: the cell counts size the records' read-back
  uint64_t total_cells = 0;
  for (uint32_t j = 0; j < n_sel; ++j) total_cells += cl_cells_host_[j];
  if (const int st = ensure_cluster_records(total_cells)) return st;
  launch_batch_cluster_compact(cl_table_, cl_cells_, cl_records_, n_sel, cl_records_host_, stream);
  BB_LAUNCHED("batch_cluster_compact");
  BB_CHECK(cudaStreamSynchronize(stream));  // 2: every record is in pinned memory
  static_assert(sizeof(HostCell) == sizeof(CellRecord), "record layouts must agree");
  return BB200_OK;
}

int Batch::particle_histograms(double linear, double angular, const uint8_t* present, bb200_cluster_cell* const* bins, const uint64_t* capacity,
                               uint64_t* n_bins, double* max_bin_weight) {
  error_.clear();
  if (!(linear > 0.0) || !(angular > 0.0)) return fail(BB200_ERR_INVALID_ARGUMENT, "histogram resolutions must be positive");
  if (bins != nullptr && capacity == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "capacity is null");
  std::vector<uint32_t> selected;
  if (const int st = select_members(present, &selected)) return st;
  if (selected.empty()) return BB200_OK;
  if (const int st = cell_records(linear, angular, selected)) return st;

  // Filter::particle_histogram's host half per member.
  static_assert(sizeof(bb200_cluster_cell) == sizeof(CellRecord), "public and internal cell records must agree");
  const CellRecord* cells = cl_records_host_;
  bool short_buffer = false;
  for (size_t j = 0; j < selected.size(); ++j) {
    const uint32_t k = selected[j];
    const uint32_t count = cl_cells_host_[j];
    double top = 1e-3;  // beluga_ros/particle_cloud.hpp:197
    for (uint32_t c = 0; c < count; ++c) top = cells[c].weight > top ? cells[c].weight : top;
    if (n_bins != nullptr) n_bins[k] = count;
    if (max_bin_weight != nullptr) max_bin_weight[k] = top;
    if (bins != nullptr && bins[k] != nullptr) {
      if (capacity[k] < count) {
        short_buffer = true;
      } else {
        std::memcpy(bins[k], cells, count * sizeof(CellRecord));
      }
    }
    cells += count;
  }
  if (short_buffer) return fail(BB200_ERR_CAPACITY, "histogram bin buffer too small for some member (n_bins has the counts)");
  return BB200_OK;
}

int Batch::ensure_samples(uint64_t draws) {
  if (sm_table_host_ == nullptr) {
    const size_t k = members_.size();
    sample_header_ = (k * sizeof(unsigned long long) + sizeof(Pose2) - 1) / sizeof(Pose2);
    BB_CHECK(dev_alloc(&sm_table_, k));
    BB_CHECK(host_alloc(&sm_table_host_, k));  // marks the table as allocated
  }
  if (draws <= samples_capacity_) return BB200_OK;
  cudaFree(samples_);
  cudaFreeHost(samples_host_);
  samples_ = samples_host_ = nullptr;
  samples_capacity_ = 0;
  const uint64_t want = std::min<uint64_t>(total_, std::max<uint64_t>(4096, 2 * draws));  // draws <= total_
  BB_CHECK(realloc_staged(&samples_, &samples_host_, sample_header_ + want));
  samples_capacity_ = want;
  return BB200_OK;
}

int Batch::sample_states(const uint64_t* counts, uint32_t step, const uint8_t* present, double* const* states_out) {
  error_.clear();
  // Filter::sample_states's checks per member, all before anything reaches the device.
  std::vector<uint32_t> drawn;  // selected members with something to draw, in member order
  uint64_t draws = 0;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (present != nullptr && present[k] == 0) continue;
    const Member& m = members_[k];
    const std::string who = "member " + std::to_string(k) + ": ";
    if (m.n == 0) return fail(BB200_ERR_STATE, who + "no particles");
    if (counts[k] > m.capacity) return fail(BB200_ERR_CAPACITY, who + "more samples than its max_particles");
    if (counts[k] > 0 && states_out[k] == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, who + "states_out is null");
    if (counts[k] == 0) continue;
    drawn.push_back(static_cast<uint32_t>(k));
    draws += counts[k];
  }
  if (drawn.empty()) return BB200_OK;
  BB_CHECK(cudaSetDevice(device_));
  if (const int st = ensure_samples(draws)) return st;  // every batch call ends synchronised: the pinned buffers are free

  const uint32_t n_sel = static_cast<uint32_t>(drawn.size());
  BatchSampleArgs a{};
  a.n_members = n_sel;
  uint64_t out_offset = 0;
  for (uint32_t j = 0; j < n_sel; ++j) {
    const uint32_t k = drawn[j];
    const Member& m = members_[k];
    BatchSampleMember& s = sm_table_host_[j];
    s = BatchSampleMember{};
    s.offset = m.offset;
    s.n = m.n;
    s.count = counts[k];
    s.out_offset = out_offset;
    s.seed = m.policy.params().seed;
    s.total = m.cdf_total;
    s.cur = m.cur;
    s.ceil_log2_count = ceil_log2_count(m.capacity);
    out_offset += s.count;
    uint32_t ctas[kSampleLaunches];
    batch_sample_ctas(s, s.total == 0, ctas);
    for (int l = 0; l < kSampleLaunches; ++l) {
      first_host_[static_cast<size_t>(l) * (n_sel + 1) + j] = a.ctas[l];  // the step's range buffers are free between calls
      a.ctas[l] += ctas[l];
    }
  }
  for (int l = 0; l < kSampleLaunches; ++l) first_host_[static_cast<size_t>(l) * (n_sel + 1) + n_sel] = a.ctas[l];
  cudaStream_t stream = stream_;
  BB_CHECK(cudaMemcpyAsync(sm_table_, sm_table_host_, n_sel * sizeof(BatchSampleMember), cudaMemcpyHostToDevice, stream));
  BB_CHECK(cudaMemcpyAsync(first_, first_host_, kSampleLaunches * (n_sel + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
  a.members = sm_table_;
  a.first = first_;
  a.step = step;
  a.states[0] = states_[0];
  a.states[1] = states_[1];
  a.weights = weights_;
  a.cdf = cdf_;
  a.scalars = scalars_;
  a.tile_state = tile_state_;
  a.partials = partials_;  // the step's moment rows are free between calls
  a.totals = reinterpret_cast<unsigned long long*>(samples_);
  a.out = samples_ + sample_header_;
  launches_ += static_cast<uint64_t>(launch_batch_sample(a, stream));
  BB_CHECK(cudaGetLastError());
  BB_CHECK(cudaMemcpyAsync(samples_host_, samples_, (sample_header_ + draws) * sizeof(Pose2), cudaMemcpyDeviceToHost, stream));
  BB_CHECK(cudaStreamSynchronize(stream));

  const unsigned long long* totals = reinterpret_cast<const unsigned long long*>(samples_host_);
  const Pose2* out = samples_host_ + sample_header_;
  for (uint32_t j = 0; j < n_sel; ++j) {
    const BatchSampleMember& s = sm_table_host_[j];
    members_[drawn[j]].cdf_total = totals[j];  // a rebuilt CDF is current until the member's particles or weights change
    std::memcpy(states_out[drawn[j]], out + s.out_offset, s.count * sizeof(Pose2));
  }
  return BB200_OK;
}

int Batch::ensure_points(uint64_t n_points) {
  if (n_points <= points_capacity_) return BB200_OK;
  BB_CHECK(cudaStreamSynchronize(stream_));
  points_capacity_ = 0;
  const uint64_t cap = std::max<uint64_t>(n_points + n_points / 2, 4096);
  BB_CHECK(realloc_staged(&points_, &points_host_, 2 * cap));
  points_capacity_ = cap;
  return BB200_OK;
}

bool Batch::ensure_hits(uint64_t words) {
  if (words <= hits_capacity_) return true;
  // Every batch call ends synchronised: nothing in flight reads the old buffer.
  cudaFree(hits_);
  hits_ = nullptr;
  hits_capacity_ = 0;
  // words is at most one pass's worth (the caller checks), so the slack never takes the buffer past that
  const uint64_t want = std::min<uint64_t>(std::max<uint64_t>(words + words / 2, 4096), kBeamHitPassBytes / sizeof(uint32_t));
  if (dev_alloc(&hits_, want) != cudaSuccess) {
    (void)cudaGetLastError();  // no room for the hit words: the fused kernel needs none
    return false;
  }
  hits_capacity_ = want;
  return true;
}

int Batch::update(const double* control_poses, const double* const* points_xy, const uint64_t* n_points, const uint8_t* present,
                  bb200_update_result* out) {
  error_.clear();
  const size_t count = members_.size();
  for (size_t k = 0; k < count; ++k) out[k] = bb200_update_result{};
  std::vector<AmclPolicy> before;
  before.reserve(count);
  for (const Member& m : members_) before.push_back(m.policy);
  auto rollback = [&](int st) {
    for (size_t k = 0; k < count; ++k) members_[k].policy = before[k];
    return st;
  };

  // Host half of every present member's Amcl::update (amcl_core.hpp:165-190).
  std::vector<bb200_step_plan> plans(count);
  std::vector<uint32_t> active;  // members that update in this step, in member order
  for (size_t k = 0; k < count; ++k) {
    if (present != nullptr && present[k] == 0) continue;
    members_[k].policy.plan_update(control_poses + 4 * k, members_[k].n, &plans[k]);
    if (plans[k].update) active.push_back(static_cast<uint32_t>(k));
  }
  if (active.empty()) return BB200_OK;

  uint64_t points_total = 0;
  uint32_t max_points = 0;
  int step_map = -1;            // the map every updating member reads, or -1 when they read several
  std::vector<int> forms(count, kBatchField);
  for (const uint32_t k : active)
    if (members_[k].map < 0) return rollback(fail(BB200_ERR_STATE, maps_.empty() ? "no map set" : "member " + std::to_string(k) + " has no map"));
  for (const uint32_t k : active) {
    if (n_points[k] > 0xffffffffull) return rollback(fail(BB200_ERR_INVALID_ARGUMENT, "too many points"));
    if (n_points[k] > 0 && points_xy[k] == nullptr) return rollback(fail(BB200_ERR_INVALID_ARGUMENT, "points_xy is null"));
    const int id = members_[k].map;
    const DeviceMap& map = maps_.at(id).map;
    if (plans[k].resample && plans[k].random_state_probability > 0.0 && map.n_free == 0)
      return rollback(fail(BB200_ERR_STATE, "recovery injection needs a map with free cells"));
    // The beam model walks a member's rays in two passes when its map allows it (the rule of the single filter).
    if (map.sensor == BB200_SENSOR_BEAM) forms[k] = beam_two_pass_map(map) ? kBatchBeamTwoPass : kBatchBeamFused;
    step_map = k == active.front() || step_map == id ? id : -1;
    points_total += n_points[k];
    max_points = std::max(max_points, static_cast<uint32_t>(n_points[k]));
  }
  int st = check(cudaSetDevice(device_), "cudaSetDevice");
  if (st == BB200_OK) st = ensure_points(points_total);  // the previous step has ended: the staging buffers are free
  if (st == BB200_OK && step_map < 0) st = ensure_map_table();
  if (st != BB200_OK) return rollback(st);

  // The step's member table and the concatenated scans.
  const uint32_t n_active = static_cast<uint32_t>(active.size());
  BatchStepArgs a{};
  a.n_members = n_active;
  uint64_t point_offset = 0, hit_words = 0;
  for (uint32_t j = 0; j < n_active; ++j) {
    const uint32_t k = active[j];
    const Member& m = members_[k];
    const bb200_step_plan& plan = plans[k];
    BatchMember& b = table_host_[j];
    b = BatchMember{};
    b.offset = m.offset;
    b.n = m.n;
    b.slots = m.capacity;
    b.seed = m.policy.params().seed;
    b.step = plan.step;
    b.resample = plan.resample;
    b.scheme = plan.opts.scheme;
    b.cur = m.cur;
    b.ceil_log2_count = ceil_log2_count(m.capacity);
    b.map = step_map < 0 ? maps_.at(m.map).slot : 0;
    b.random_state_probability = plan.random_state_probability;
    b.pivot_x = m.pivot[0];
    b.pivot_y = m.pivot[1];
    b.sampling = to_kernel_sampling(plan.sampling);
    b.point_offset = point_offset;
    b.n_points = static_cast<uint32_t>(n_points[k]);
    b.points_radius = scan_radius(points_xy[k], n_points[k]);
    if (n_points[k] > 0) std::memcpy(points_host_ + 2 * point_offset, points_xy[k], 2 * n_points[k] * sizeof(double));
    point_offset += n_points[k];
    b.hit_stride = (m.n + 31) / 32 * 32;
    if (forms[k] == kBatchBeamTwoPass) {
      b.hit_offset = hit_words;
      hit_words += b.hit_stride * n_points[k];
    }
  }
  // The two-pass members keep that form when their hit words fit under the single filter's bound for one pass and in
  // device memory; otherwise they take the fused kernel.
  if (hit_words > 0 && !(hit_words <= kBeamHitPassBytes / sizeof(uint32_t) && ensure_hits(hit_words)))
    for (const uint32_t k : active)
      if (forms[k] == kBatchBeamTwoPass) forms[k] = kBatchBeamFused;
  // The CTA ranges of every row: each member in the reweight row of its form.
  for (uint32_t j = 0; j < n_active; ++j) {
    const int form = forms[active[j]];
    a.forms |= 1 << form;
    uint32_t ctas[kBatchLaunches];
    batch_member_ctas(table_host_[j], form, ctas);
    for (int l = 0; l < kBatchLaunches; ++l) {
      first_host_[static_cast<size_t>(l) * (n_active + 1) + j] = a.ctas[l];
      a.ctas[l] += ctas[l];
    }
  }
  for (int l = 0; l < kBatchLaunches; ++l) first_host_[static_cast<size_t>(l) * (n_active + 1) + n_active] = a.ctas[l];

  cudaStream_t stream = stream_;
  for (const uint32_t k : active) members_[k].cdf_total = 0;  // from here on the step may have rewritten their CDFs
  seq_ = seq_ == 0x7fffffff ? 1 : seq_ + 1;
  *ticket_host_ = 0;
  st = check(cudaMemcpyAsync(table_, table_host_, n_active * sizeof(BatchMember), cudaMemcpyHostToDevice, stream), "upload member table");
  if (st == BB200_OK)
    st = check(cudaMemcpyAsync(first_, first_host_, kBatchLaunches * (n_active + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, stream), "upload ranges");
  if (st == BB200_OK && points_total > 0)
    st = check(cudaMemcpyAsync(points_, points_host_, 2 * points_total * sizeof(double), cudaMemcpyHostToDevice, stream), "upload points");
  if (st != BB200_OK) return rollback(st);
  a.members = table_;
  a.first = first_;
  a.max_points = max_points;
  a.states[0] = states_[0];
  a.states[1] = states_[1];
  a.weights = weights_;
  a.cdf = cdf_;
  a.ancestors = ancestors_;
  a.tile_state = tile_state_;
  a.scalars = scalars_;
  a.partials = partials_;
  a.points = points_;
  if (step_map >= 0) {
    const DeviceMap& map = maps_.at(step_map).map;
    a.field = map.field;
    a.free_cells = map.free_cells;
    a.n_free = map.n_free;
    a.grid_width = map.grid_width;
    a.grid_resolution = map.grid_resolution;
    a.grid_origin = map.grid_origin;
    a.occupancy = map.occupancy;
    a.beam = map.beam;
  } else {
    a.maps = map_table_;
  }
  a.hits = hits_;
  a.summary = summary_host_;
  a.members_done = members_done_;
  a.ticket = ticket_host_;
  a.seq = seq_;
  launches_ += static_cast<uint64_t>(launch_batch_step(a, stream));
  st = check(cudaGetLastError(), "batch step launch");
  if (st != BB200_OK) return rollback(st);

  // The last member to finish stores the ticket into pinned memory.
  const bool done = wait_for_ticket(ticket_host_, seq_, stream);
  if (!done) st = check(cudaStreamSynchronize(stream), "batch step");
  if (st == BB200_OK && !done && *static_cast<volatile int*>(ticket_host_) != seq_) st = fail(BB200_ERR_CUDA, "the batch step ended without its completion ticket");
  if (st != BB200_OK) return rollback(st);

  for (uint32_t j = 0; j < n_active; ++j) {
    const uint32_t k = active[j];
    Member& m = members_[k];
    const StepSummary& s = summary_host_[j];
    const bb200_step_plan& plan = plans[k];
    bb200_update_result& r = out[k];
    estimate_from_moments(s.moments, m.pivot, &r.estimate);
    pivot_to_estimate(r.estimate, m.pivot);
    if (plan.resample) {
      m.cur ^= 1;
      m.n = m.capacity;
      m.ancestors_n = m.n;
    } else {
      m.cdf_total = s.total;  // the step's scan, over the weights before normalisation
    }
    r.updated = 1;
    r.resampled = plan.resample;
    r.n_particles = m.n;
    r.random_state_probability = plan.random_state_probability;
    r.weight_sum = std::ldexp(static_cast<double>(s.total), -s.exponent);
    r.weights_degenerate = s.valid != 0 ? 0 : 1;
    m.policy.commit_update(r.resampled, plan.random_state_probability);
  }
  return BB200_OK;
}

}  // namespace bb200
