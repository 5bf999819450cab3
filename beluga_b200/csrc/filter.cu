#include "filter.hpp"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <initializer_list>

#include "cluster_host.hpp"

namespace bb200 {

MotionSampling to_kernel_sampling(const bb200_motion_sampling& s) {
  MotionSampling m{};
  m.model = s.model;
  for (int k = 0; k < 3; ++k) {
    m.mean[k] = s.mean[k];
    m.stddev[k] = s.stddev[k];
  }
  m.first_c = s.first_rotation[0];
  m.first_s = s.first_rotation[1];
  return m;
}

bool normal_transform(const double cov[9], double transform[9], std::string* error) {
  // isApprox(transpose) of Eigen: ||C - C^T||_F^2 <= 1e-24 * ||C||_F^2
  double diff2 = 0.0, norm2 = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double d = cov[3 * i + j] - cov[3 * j + i];
      diff2 += d * d;
      norm2 += cov[3 * i + j] * cov[3 * i + j];
    }
  if (!(diff2 <= 1e-24 * norm2)) {
    if (error) *error = "Invalid covariance matrix, it is not symmetric.";
    return false;
  }
  // Cyclic Jacobi on the symmetric 3x3; eigenvalues ascending like SelfAdjointEigenSolver.
  double a[3][3], v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) a[i][j] = cov[3 * i + j];
  for (int sweep = 0; sweep < 64; ++sweep) {
    if (a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2] == 0.0) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - s * vkq;
          v[k][q] = s * vkp + c * vkq;
        }
      }
  }
  int order[3] = {0, 1, 2};
  std::sort(order, order + 3, [&](int i, int j) { return a[i][i] < a[j][j]; });
  for (int j = 0; j < 3; ++j) {
    const double lambda = a[order[j]][order[j]];
    if (lambda < 0.0) {
      if (error) *error = "Invalid covariance matrix, it has negative eigenvalues.";
      return false;
    }
    for (int i = 0; i < 3; ++i) transform[3 * i + j] = v[i][order[j]] * std::sqrt(lambda);
  }
  return true;
}

int check_device(int device, std::string* error) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0)
    return reject(BB200_ERR_NO_DEVICE, "no CUDA device available (this backend has no CPU fallback)", error);
  if (device < 0 || device >= count) return reject(BB200_ERR_INVALID_ARGUMENT, "device ordinal out of range", error);
  return BB200_OK;
}

double scan_radius(const double* points_xy, uint64_t n_points) {
  double radius = 0.0;
  for (uint64_t i = 0; i < n_points; ++i) {
    const double r = std::fabs(points_xy[2 * i]) + std::fabs(points_xy[2 * i + 1]);
    radius = (r > radius || std::isnan(r)) ? r : radius;
  }
  return radius;
}

bool wait_for_ticket(const volatile int* word, int ticket, cudaStream_t stream) {
  for (uint32_t spins = 1; *word != ticket; ++spins)
    if ((spins & 0x3fffu) == 0 && cudaStreamQuery(stream) != cudaErrorNotReady) return false;  // ended without it, or failed
  std::atomic_thread_fence(std::memory_order_acquire);
  return true;
}

// ---------------------------------------------------------------------------------------------------

Filter::Filter(const bb200_filter_config& config) : config_(config), cluster_(config.capacity) {
  cluster_.mark = [this](const char* name) { mark(name); };
  create_status_ = check_device(config.device, &error_);
  if (create_status_ != BB200_OK) return;
  if (config.capacity == 0) {
    create_status_ = fail(BB200_ERR_INVALID_ARGUMENT, "capacity must be positive");
    return;
  }
  if (config_.global_count == 0) config_.global_count = config_.capacity;
  capacity_ = config.capacity;
  first_index_ = config.first_index;
  BB_TRY(cudaSetDevice(config.device));
  BB_TRY(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  BB_TRY(dev_alloc(&states_[0], capacity_));
  BB_TRY(dev_alloc(&states_[1], capacity_));
  BB_TRY(dev_alloc(&weights_, capacity_));
  BB_TRY(dev_alloc(&cdf_, capacity_));
  if (config.record_ancestors) BB_TRY(dev_alloc(&ancestors_, capacity_));
  BB_TRY(dev_alloc(&scalars_, 1));
  BB_TRY(cudaMallocHost(reinterpret_cast<void**>(&scalars_host_), sizeof(Scalars)));
  tile_capacity_ = scan_tile_count(capacity_) + 1;
  BB_TRY(dev_alloc(&tile_state_, tile_capacity_));
  partials_rows_ = std::max(std::max(resample_block_count(capacity_), moments_block_count(capacity_)), kSmCount * 8u);
  BB_TRY(dev_alloc(&partials_, static_cast<size_t>(partials_rows_) * kMomentCount));
  BB_TRY(dev_alloc(&results_, 16));
  BB_TRY(cudaMallocHost(reinterpret_cast<void**>(&results_host_), 16 * sizeof(double)));
  BB_TRY(dev_alloc(&sched_, 1));
  BB_TRY(dev_alloc(&bins_, capacity_));
  BB_TRY(dev_alloc(&bin_rank_, capacity_));
  BB_TRY(dev_alloc(&perm_, capacity_));
  BB_TRY(dev_alloc(&counters_, schedule_max_bins()));
  BB_TRY(dev_alloc(&sched_tiles_, schedule_tile_count()));
  BB_TRY(dev_alloc(&mail_, 1));  // its own allocation: exported to peer processes through CUDA IPC
  BB_TRY(dev_alloc(&shard_totals_, kMaxShards));
  BB_TRY(dev_alloc(&summary_, 1));
  BB_TRY(cudaMallocHost(reinterpret_cast<void**>(&summary_host_), sizeof(StepSummary)));
  std::memset(summary_host_, 0, sizeof(StepSummary));  // pinned allocations are recycled with their old contents (a stale completion ticket)
  BB_TRY(cudaMemsetAsync(mail_, 0, sizeof(ShardMail), stream_));
  BB_TRY(cudaMemsetAsync(summary_, 0, sizeof(StepSummary), stream_));
  BB_TRY(cudaMemsetAsync(scalars_, 0, sizeof(Scalars), stream_));
  BB_TRY(cudaStreamSynchronize(stream_));
  global_size_ = config_.global_count;
  created_ = true;
}

Filter::~Filter() {
  if (stream_ != nullptr) cudaStreamSynchronize(stream_);
  release_peers();
  for (auto& e : event_pool_) cudaEventDestroy(e);
  for (void* p : std::initializer_list<void*>{mail_, shard_totals_, summary_, states_[0], states_[1], weights_, cdf_, ancestors_, hashes_, scalars_,
                                              sched_, bins_, bin_rank_, perm_, counters_, sched_tiles_, tile_state_, partials_, results_, kld_keys_,
                                              kld_vals_, kld_flags_, kld_scan_, kld_tile_state_, kld_hashes_global_, points_, beam_hits_})
    cudaFree(p);
  for (void* p : std::initializer_list<void*>{summary_host_, scalars_host_, results_host_, points_host_}) cudaFreeHost(p);
  if (stream_ != nullptr && owns_stream_) cudaStreamDestroy(stream_);
}

void Filter::mark(const char* name) {
  if (!timing_) return;
  if (events_used_ == event_pool_.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    event_pool_.push_back(e);
  }
  cudaEvent_t e = event_pool_[events_used_++];
  cudaEventRecord(e, stream_);
  marks_.push_back(Mark{name, e});
}

void Filter::finish_marks() {
  if (!timing_ || marks_.empty()) {
    marks_.clear();
    events_used_ = 0;
    return;
  }
  if (std::string(marks_.back().name) != "end") mark("end");
  cudaEventSynchronize(marks_.back().event);
  for (size_t i = 0; i + 1 < marks_.size(); ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, marks_[i].event, marks_[i + 1].event);
    timings_.emplace_back(marks_[i].name, ms);
  }
  marks_.clear();
  events_used_ = 0;
}

int Filter::last_timings(const char** names, float* ms, int capacity) const {
  const int n = std::min<int>(capacity, static_cast<int>(timings_.size()));
  for (int i = 0; i < n; ++i) {
    names[i] = timings_[i].first;
    ms[i] = timings_[i].second;
  }
  return static_cast<int>(timings_.size());
}

int Filter::set_stream(void* stream) {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  if (owns_stream_ && stream_ != nullptr) cudaStreamDestroy(stream_);
  stream_ = static_cast<cudaStream_t>(stream);
  owns_stream_ = false;
  return BB200_OK;
}

// ---- stream-ordered operations (the blocking ones further down add the synchronisation and read-back) ----------

int Filter::enqueue_propagate_reweight(const bb200_motion_sampling* sampling, uint32_t step, const double* points_xy, uint64_t n_points) {
  // points_xy == nullptr: propagate only.  The pinned point staging buffer is overwritten: the caller has synchronised
  // since the previous upload.
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  const bool do_reweight = points_xy != nullptr;
  if (do_reweight && map_.sensor < 0) return fail(BB200_ERR_STATE, "no sensor model map set");
  if (do_reweight && n_points > 0xffffffffull) return fail(BB200_ERR_INVALID_ARGUMENT, "too many points");
  BB_CHECK(cudaSetDevice(config_.device));
  if (do_reweight) {
    const int st = upload_points(points_xy, n_points);
    if (st != BB200_OK) return st;
  }
  MotionSampling s{};
  if (sampling != nullptr) s = to_kernel_sampling(*sampling);
  mark("begin_step");
  launch_begin_step(scalars_, stream_);
  BB_LAUNCHED("begin_step");
  const int st = enqueue_propagate_reweight_kernels(sampling != nullptr ? &s : nullptr, step, do_reweight, n_points, false);
  cdf_valid_ = false;
  cloud_known_ = false;
  return st;
}

int Filter::enqueue_max_weight() {
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  BB_CHECK(cudaSetDevice(config_.device));
  launch_begin_step(scalars_, stream_);
  BB_LAUNCHED("begin_step");
  launch_max_weight(weights_, n_, scalars_, stream_);
  BB_LAUNCHED("max_weight");
  return BB200_OK;
}

int Filter::enqueue_build_cdf(double global_wmax) {
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  BB_CHECK(cudaSetDevice(config_.device));
  mark("prepare_cdf");
  launch_prepare_cdf(scalars_, global_wmax, config_.global_count, tile_state_, scan_tile_count(n_), stream_);
  BB_LAUNCHED("prepare_cdf");
  mark("quantize_scan");
  launch_quantize_scan(weights_, n_, cdf_, scalars_, tile_state_, stream_);
  BB_LAUNCHED("quantize_scan");
  cdf_valid_ = true;
  return BB200_OK;
}

int Filter::enqueue_resample_range(const bb200_resample_opts& o, uint64_t global_total, uint64_t cdf_offset, uint64_t slot_begin, uint64_t slot_end) {
  // Sharded filter: this rank produces the output slots [slot_begin, slot_end) -- exactly those whose
  // comb position falls inside its span of the global CDF -- into the staging buffer, in slot order.
  if (!cdf_valid_) return fail(BB200_ERR_STATE, "build_cdf must run before resample_range");
  if (o.scheme != BB200_RESAMPLE_SYSTEMATIC || o.min_particles < o.max_particles)
    return fail(BB200_ERR_STATE, "range resampling supports the systematic comb without KLD (multinomial or KLD on shards: bb200_amcl_join_shards / bb200_sharded_amcl)");
  if (o.random_state_probability > 0.0 && map_.n_free == 0) return fail(BB200_ERR_STATE, "recovery injection needs a map with free cells");
  if (slot_end < slot_begin || slot_end - slot_begin > capacity_) return fail(BB200_ERR_CAPACITY, "slot range exceeds the staging buffer");
  BB_CHECK(cudaSetDevice(config_.device));
  if (slot_end > slot_begin) {
    ResampleArgs a = make_resample_args(o, 0, slot_end - slot_begin, false);
    a.slot_first = slot_begin;  // global slot index
    a.global_total = global_total;
    a.cdf_offset = cdf_offset;
    a.weights_out = nullptr;  // the current weights stay untouched; adopt() writes the ones
    mark("resample_range");
    launch_resample(a, scalars_, partials_, stream_);
    BB_LAUNCHED("resample_range");
  }
  return BB200_OK;
}

int Filter::enqueue_adopt(uint64_t n) {
  // The caller has placed n particle states into the current state buffer, e.g. through an all-to-all: make them
  // the particle set with unit weights (make_from_state, particle_traits.hpp:105).
  if (n > capacity_) return fail(BB200_ERR_CAPACITY, "more particles than the filter capacity");
  BB_CHECK(cudaSetDevice(config_.device));
  cloud_known_ = false;
  n_ = n;
  cdf_valid_ = false;
  if (n > 0) {
    mark("fill_weights");
    launch_fill(weights_, n, 1.0, stream_);
    BB_LAUNCHED("fill_weights");
  }
  return BB200_OK;
}

int Filter::enqueue_moments(const double pivot[2]) {
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  BB_CHECK(cudaSetDevice(config_.device));
  return enqueue_moment_kernels(pivot);
}

int Filter::enqueue_moment_kernels(const double pivot[2]) {
  mark("moments");
  launch_moments(states_[cur_], weights_, n_, pivot[0], pivot[1], partials_, stream_);
  BB_LAUNCHED("moments");
  launch_reduce_partials(partials_, moments_block_count(n_), kMomentCount, results_, stream_);
  BB_LAUNCHED("reduce_partials");
  return BB200_OK;
}

void Filter::release_peers() {
  if (peers_ipc_) {  // unmap what cudaIpcOpenMemHandle mapped; local peers are plain pointers owned by their filters
    for (int r = 0; r < peer_world_; ++r) {
      if (r == peer_rank_) continue;
      for (int b = 0; b < 2; ++b)
        if (peer_states_[b][r] != nullptr) cudaIpcCloseMemHandle(peer_states_[b][r]);
      if (peer_mail_[r] != nullptr) cudaIpcCloseMemHandle(peer_mail_[r]);
      if (peer_kld_hashes_[r] != nullptr) cudaIpcCloseMemHandle(peer_kld_hashes_[r]);
    }
  }
  for (int r = 0; r < kMaxShards; ++r) {
    peer_states_[0][r] = peer_states_[1][r] = nullptr;
    peer_mail_[r] = nullptr;
    peer_kld_hashes_[r] = nullptr;
  }
  peer_world_ = 0;
  peers_ipc_ = false;
}

int Filter::leave_shards() {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  release_peers();
  return BB200_OK;
}

int Filter::enable_shard_kld() {
  if (kld_hashes_global_ != nullptr) return BB200_OK;
  if (peer_world_ != 0) return fail(BB200_ERR_STATE, "KLD on shards must be enabled before the shards are joined");
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(dev_alloc(&kld_hashes_global_, config_.global_count));  // one spatial hash per candidate slot of the WHOLE filter
  return BB200_OK;
}

int Filter::export_shard(void* out256) {
  BB_CHECK(cudaSetDevice(config_.device));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "four IPC handles are exported as 256 bytes");
  cudaIpcMemHandle_t h[4];
  std::memset(h, 0, sizeof(h));
  BB_CHECK(cudaIpcGetMemHandle(&h[0], states_[0]));
  BB_CHECK(cudaIpcGetMemHandle(&h[1], states_[1]));
  BB_CHECK(cudaIpcGetMemHandle(&h[2], mail_));
  if (kld_hashes_global_ != nullptr) BB_CHECK(cudaIpcGetMemHandle(&h[3], kld_hashes_global_));
  std::memcpy(out256, h, sizeof(h));
  return BB200_OK;
}

int Filter::join_shards_ipc(int world, int rank, const void* handles) {
  if (world < 1 || world > kMaxShards || rank < 0 || rank >= world) return fail(BB200_ERR_INVALID_ARGUMENT, "shard groups hold 1..8 ranks");
  if (peer_world_ != 0) return fail(BB200_ERR_STATE, "the peers' buffers are already mapped");
  if (config_.first_index != static_cast<uint64_t>(rank) * capacity_ || config_.global_count != static_cast<uint64_t>(world) * capacity_)
    return fail(BB200_ERR_INVALID_ARGUMENT, "shard r of R holds the global indices [r * capacity, (r + 1) * capacity) of R * capacity particles");
  BB_CHECK(cudaSetDevice(config_.device));
  const auto* all = static_cast<const cudaIpcMemHandle_t*>(handles);
  peers_ipc_ = true;
  peer_world_ = world;
  peer_rank_ = rank;
  for (int r = 0; r < world; ++r) {
    if (r == rank) {
      peer_states_[0][r] = states_[0];
      peer_states_[1][r] = states_[1];
      peer_mail_[r] = mail_;
      peer_kld_hashes_[r] = kld_hashes_global_;
      continue;
    }
    static const cudaIpcMemHandle_t kNoHandle{};
    void* p[4] = {nullptr, nullptr, nullptr, nullptr};
    for (int b = 0; b < 4; ++b) {
      if (b == 3 && (kld_hashes_global_ == nullptr || std::memcmp(&all[4 * r + 3], &kNoHandle, sizeof(kNoHandle)) == 0)) continue;  // no KLD on this filter
      const int st = check(cudaIpcOpenMemHandle(&p[b], all[4 * r + b], cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
      if (st != BB200_OK) {
        peer_states_[0][r] = static_cast<Pose2*>(p[0]);
        peer_states_[1][r] = static_cast<Pose2*>(p[1]);
        peer_mail_[r] = static_cast<ShardMail*>(p[2]);
        release_peers();
        return st;
      }
    }
    peer_states_[0][r] = static_cast<Pose2*>(p[0]);
    peer_states_[1][r] = static_cast<Pose2*>(p[1]);
    peer_mail_[r] = static_cast<ShardMail*>(p[2]);
    peer_kld_hashes_[r] = static_cast<unsigned long long*>(p[3]);
  }
  shard_kld_ = kld_hashes_global_ != nullptr;
  for (int r = 0; r < world; ++r) shard_kld_ = shard_kld_ && peer_kld_hashes_[r] != nullptr;
  split_posts_ = false;  // every rank has its own host thread: post and wait travel in one launch
  return BB200_OK;
}

int Filter::join_shards_local(Filter* const* filters, int world) {
  if (filters == nullptr || world < 1 || world > kMaxShards) return BB200_ERR_INVALID_ARGUMENT;
  for (int r = 0; r < world; ++r) {
    Filter* f = filters[r];
    if (f == nullptr || !f->ok()) return BB200_ERR_INVALID_ARGUMENT;
    if (f->peer_world_ != 0) return f->fail(BB200_ERR_STATE, "the peers' buffers are already mapped");
    if (f->capacity_ != filters[0]->capacity_ || f->config_.first_index != static_cast<uint64_t>(r) * f->capacity_ ||
        f->config_.global_count != static_cast<uint64_t>(world) * f->capacity_ || f->config_.seed != filters[0]->config_.seed)
      return f->fail(BB200_ERR_INVALID_ARGUMENT, "shard r of R holds the global indices [r * capacity, (r + 1) * capacity) of R * capacity particles, same seed");
  }
  for (int a = 0; a < world; ++a) {
    Filter* fa = filters[a];
    for (int b = 0; b < world; ++b) {
      const Filter* fb = filters[b];
      if (fa->config_.device != fb->config_.device) {
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, fa->config_.device, fb->config_.device) != cudaSuccess || !can)
          return fa->fail(BB200_ERR_CUDA, "no peer access between the devices of two shards");
        if (fa->check(cudaSetDevice(fa->config_.device), "cudaSetDevice") != BB200_OK) return BB200_ERR_CUDA;
        const cudaError_t e = cudaDeviceEnablePeerAccess(fb->config_.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fa->check(e, "cudaDeviceEnablePeerAccess");
        (void)cudaGetLastError();
      }
      fa->peer_states_[0][b] = fb->states_[0];
      fa->peer_states_[1][b] = fb->states_[1];
      fa->peer_mail_[b] = fb->mail_;
      fa->peer_kld_hashes_[b] = fb->kld_hashes_global_;
    }
    fa->shard_kld_ = true;
    for (int b = 0; b < world; ++b) fa->shard_kld_ = fa->shard_kld_ && filters[b]->kld_hashes_global_ != nullptr;
    fa->peer_world_ = world;
    fa->peer_rank_ = a;
    fa->peers_ipc_ = false;
    fa->split_posts_ = true;  // one thread enqueues all shards: every post must be enqueued before any wait that needs it
  }
  return BB200_OK;
}

int Filter::enqueue_exchange(int kind, bool post, bool wait) {
  ShardExchangeArgs a{};
  a.kind = kind;
  a.post = post ? 1 : 0;
  a.wait = wait ? 1 : 0;
  a.rank = peer_rank_;
  a.world = peer_world_;
  a.epoch = epoch_;
  for (int r = 0; r < peer_world_; ++r) a.peers[r] = peer_mail_[r];
  a.scalars = scalars_;
  a.results = results_;
  a.summary = summary_host_;  // pinned host memory: the step's results need no copy
  a.rank_totals = shard_totals_;
  a.ceil_log2_count = ceil_log2_count(config_.global_count);
  a.tile_state = tile_state_;
  a.n_tiles = scan_tile_count(n_);
  launch_shard_exchange(a, stream_);
  BB_LAUNCHED("shard_exchange");
  return BB200_OK;
}

int Filter::step_begin(const bb200_motion_sampling& sampling, uint32_t step, const double* points_xy, uint64_t n_points, const bb200_resample_opts& o,
                       bool resample_planned) {
  const uint64_t world = peer_world_ > 1 ? static_cast<uint64_t>(peer_world_) : 1;
  const bool kld = o.min_particles < o.max_particles;
  if (n_ == 0 && !(world > 1 && shard_kld_)) return fail(BB200_ERR_STATE, "no particles");  // a KLD-sized filter may leave a shard empty
  if (map_.sensor < 0) return fail(BB200_ERR_STATE, "no sensor model map set");
  if (kld && !(world > 1 && shard_kld_)) return fail(BB200_ERR_STATE, "the fused step does not run KLD on one GPU; use resample()");
  if (n_points > 0xffffffffull) return fail(BB200_ERR_INVALID_ARGUMENT, "too many points");
  if (o.random_state_probability > 0.0 && map_.n_free == 0) return fail(BB200_ERR_STATE, "recovery injection needs a map with free cells");
  if (world > 1) {
    if ((!shard_kld_ && n_ != capacity_) || n_ > capacity_ || o.max_particles != world * capacity_)
      return fail(BB200_ERR_STATE, "a sharded filter keeps `capacity` particles on every rank (fewer only under KLD)");
  } else if (o.max_particles == 0 || o.max_particles > capacity_) {
    return fail(BB200_ERR_CAPACITY, "max_particles exceeds the filter capacity");
  }
  BB_CHECK(cudaSetDevice(config_.device));
  const int st = upload_points(points_xy, n_points);
  if (st != BB200_OK) return st;
  step_ = StepContext{};
  summary_host_->error = 0;
  step_.active = true;
  step_.sampling = to_kernel_sampling(sampling);
  step_.step = step;
  step_.n_points = n_points;
  step_.opts = o;
  step_.resample_planned = resample_planned;
  return BB200_OK;
}

void Filter::step_abort() { step_.active = false; }

int Filter::step_phase(int phase) {
  if (!step_.active) return fail(BB200_ERR_STATE, "step_begin must run first");
  BB_CHECK(cudaSetDevice(config_.device));
  const bool sharded = peer_world_ > 1;
  const bb200_resample_opts& o = step_.opts;
  int st = BB200_OK;
  switch (phase) {
    case kPhaseReweight: {
      mark("begin_step");
      {
        const bool scheduled = n_ >= kScheduleMinParticles;
        const bool warm = map_.sensor != BB200_SENSOR_BEAM && map_.field.use_fixed && map_.bordered_bytes <= (96ull << 20);
        launch_begin_fused_step(scalars_, tile_state_, scan_tile_count(n_), sched_, scheduled ? counters_ : nullptr, schedule_max_bins(), sched_tiles_,
                                schedule_tile_count(), warm ? map_.field.bordered : nullptr, map_.bordered_bytes, stream_);
        BB_LAUNCHED("begin_step");
        st = enqueue_propagate_reweight_kernels(&step_.sampling, step_.step, true, step_.n_points, scheduled);
      }
      if (st != BB200_OK) return st;
      if (sharded) {
        ++epoch_;  // one sequence number per batch of exchanges
        if (split_posts_) {
          mark("exchange");
          st = enqueue_exchange(kExchangeWmax, true, false);
        }
      }
      return st;
    }
    case kPhaseCdf: {
      if (sharded) {
        mark("exchange_wmax");
        st = enqueue_exchange(kExchangeWmax, !split_posts_, true);  // global largest weight -> exponent; resets the scan state
        if (st != BB200_OK) return st;
      }
      mark("quantize_scan");
      // one GPU: the exponent comes from the shard's own largest weight inside the kernel (scan state reset by begin_step);
      // sharded: the exchange above has set the common exponent and reset the scan state
      launch_quantize_scan(weights_, n_, cdf_, scalars_, tile_state_, stream_, !sharded, config_.global_count);
      BB_LAUNCHED("quantize_scan");
      if (sharded) {
        if (step_.resample_planned) {  // the CDF holds what sampling needs; every new particle weighs 1 (overlaps the wait for the peers' totals)
          mark("fill_weights");
          launch_fill(weights_, capacity_, 1.0, stream_);
          BB_LAUNCHED("fill_weights");
          step_.weights_filled = true;
        }
        if (split_posts_) {
          mark("exchange");
          st = enqueue_exchange(kExchangeTotal, true, false);
        }
      }
      return st;
    }
    case kPhaseResample: {
      if (step_.resampled) return fail(BB200_ERR_STATE, "this step has already resampled");
      ResampleArgs a;
      if (sharded) {
        if (!step_.totals_exchanged) {
          mark("exchange_total");
          st = enqueue_exchange(kExchangeTotal, !split_posts_, true);  // every rank's fixed-point total -> CDF offsets
          if (st != BB200_OK) return st;
          step_.totals_exchanged = true;
        }
        const bool systematic = o.scheme == BB200_RESAMPLE_SYSTEMATIC;
        const uint64_t accepted = step_.kld_accepted;  // KLD on shards: the count take_while_kld settled on (0: fixed size)
        const uint64_t slots = accepted != 0 ? accepted : o.max_particles;
        a = make_resample_args(o, 0, systematic ? capacity_ : slots, false);
        a.slot_first = 0;
        a.weights_out = nullptr;
        a.ancestors = nullptr;
        a.peer_count = peer_world_;
        a.peer_shard = accepted != 0 ? (accepted + static_cast<uint64_t>(peer_world_) - 1) / static_cast<uint64_t>(peer_world_) : capacity_;
        a.rank_totals = shard_totals_;
        a.rank = peer_rank_;
        a.world = peer_world_;
        if (accepted != 0) {  // the comb still spans max_particles slots; only [0, accepted) are kept
          a.window_begin = 0;
          a.window_end = accepted;
          a.inject_mod = peer_world_;
        }
        if (!systematic) {  // draws are independent: walk all global slots, keep those landing in this rank's CDF span
          a.span_filter = 1;
          a.owner_first = first_index_;
          a.owner_count = capacity_;
        }
        for (int r = 0; r < peer_world_; ++r) a.peer_out[r] = peer_states_[cur_ ^ 1][r];
        if (!step_.weights_filled) {
          mark("fill_weights");
          launch_fill(weights_, capacity_, 1.0, stream_);  // the CDF holds what sampling needs; every new particle weighs 1
          BB_LAUNCHED("fill_weights");
          step_.weights_filled = true;
        }
        mark("resample_push");
      } else {
        a = make_resample_args(o, 0, o.max_particles, false);
        mark("resample");
      }
      // the last block sums the moments (one GPU: straight into pinned host memory, with the step's completion ticket)
      step_.poll_seq = 0;
      if (!sharded && !timing_) {
        step_seq_ = step_seq_ == 0x7fffffff ? 1 : step_seq_ + 1;
        step_.poll_seq = step_seq_;
        summary_host_->seq = 0;  // nothing of this filter is in flight: the previous step was seen to end
      }
      a.tail = StepTail{1, results_, sharded ? nullptr : summary_host_, step_.poll_seq};
      step_.partial_rows = launch_resample(a, scalars_, partials_, stream_);
      BB_LAUNCHED("resample");
      step_.resampled = true;
      if (sharded && split_posts_) {
        mark("exchange");
        st = enqueue_exchange(kExchangeMoments, true, false);
      }
      return st;
    }
    case kPhaseFinish: {
      if (sharded) {
        mark("exchange_moments");
        st = enqueue_exchange(kExchangeMoments, !split_posts_, true);  // also the barrier: the peers' stores into this rank's buffer are complete
        if (st != BB200_OK) return st;
      } else if (!step_.resampled) {  // kPhaseNormalize left the moments in results_: hand them to the host block
        mark("readback");
        launch_write_summary(results_, scalars_, summary_host_, stream_);
        BB_LAUNCHED("write_summary");
      }
      mark("end");
      return BB200_OK;
    }
    case kPhaseNormalize: {
      if (step_.normalized) return fail(BB200_ERR_STATE, "the weights of this step are already normalised");
      if (sharded) {
        mark("exchange");
        st = enqueue_exchange(kExchangeTotal, !split_posts_, true);
        if (st != BB200_OK) return st;
        step_.totals_exchanged = true;
      }
      uint32_t rows = 0;
      mark("normalize");
      launch_normalize(weights_, n_, scalars_, sharded ? ~0ull : 0ull, partials_, &rows, stream_);  // actions/normalize.hpp:82
      BB_LAUNCHED("normalize");
      st = enqueue_moment_kernels(pivot_);  // a KLD-sized shard may be empty here
      if (st != BB200_OK) return st;
      step_.normalized = true;
      if (sharded && split_posts_) {
        mark("exchange");
        st = enqueue_exchange(kExchangeMoments, true, false);
      }
      return st;
    }
    default:
      return fail(BB200_ERR_INVALID_ARGUMENT, "unknown step phase");
  }
}

int Filter::kld_sharded_candidates(uint64_t begin, uint64_t end) {
  if (!step_.active || !shard_kld_ || peer_world_ < 2) return fail(BB200_ERR_STATE, "KLD on shards: no step in progress on a KLD-enabled shard group");
  if (!step_.totals_exchanged) return fail(BB200_ERR_STATE, "KLD on shards: the totals exchange must run first");
  if (end <= begin || end > config_.global_count) return fail(BB200_ERR_INVALID_ARGUMENT, "KLD on shards: bad slot window");
  BB_CHECK(cudaSetDevice(config_.device));
  const bb200_resample_opts& o = step_.opts;
  if (kld_keys_ == nullptr) {  // the counting pass runs over ALL slots on every rank: tables sized for the whole filter
    const uint64_t n = config_.global_count;
    BB_CHECK(dev_alloc(&kld_flags_, n));
    BB_CHECK(dev_alloc(&kld_scan_, n));
    kld_table_size_ = 2;
    while (kld_table_size_ < 2 * n) kld_table_size_ <<= 1;
    BB_CHECK(dev_alloc(&kld_keys_, kld_table_size_));
    BB_CHECK(dev_alloc(&kld_vals_, kld_table_size_));
    BB_CHECK(dev_alloc(&kld_tile_state_, static_cast<size_t>(scan_tile_count(n)) + 1));
  }
  if (begin == 0) {
    mark("kld");
    launch_kld_clear(kld_keys_, kld_vals_, kld_table_size_, stream_);
  }
  const bool systematic = o.scheme == BB200_RESAMPLE_SYSTEMATIC;
  ResampleArgs a = make_resample_args(o, 0, std::min<uint64_t>(end - begin, capacity_), false);
  a.states_out = nullptr;
  a.weights_out = nullptr;
  a.ancestors = nullptr;
  a.rank_totals = shard_totals_;
  a.rank = peer_rank_;
  a.world = peer_world_;
  a.window_begin = begin;
  a.window_end = end;
  a.peer_hash_count = peer_world_;
  for (int r = 0; r < peer_world_; ++r) a.peer_hashes[r] = peer_kld_hashes_[r];
  a.inject_mod = peer_world_;
  a.slot_first = 0;
  if (!systematic) {
    a.span_filter = 1;
    a.slot_first = begin;
    a.slot_count = end - begin;
  }
  mark("kld_candidates");
  launch_resample(a, scalars_, partials_, stream_);
  BB_LAUNCHED("kld_candidates");
  ++epoch_;
  if (split_posts_) return enqueue_exchange(kExchangeKld, true, false);
  return BB200_OK;
}

int Filter::kld_sharded_count(uint64_t begin, uint64_t end, uint64_t k_before) {
  if (!step_.active || !shard_kld_) return fail(BB200_ERR_STATE, "KLD on shards: no step in progress");
  BB_CHECK(cudaSetDevice(config_.device));
  const bb200_resample_opts& o = step_.opts;
  mark("exchange_kld");
  const int st = enqueue_exchange(kExchangeKld, !split_posts_, true);  // every rank's hashes of this window have arrived
  if (st != BB200_OK) return st;
  mark("kld");
  KldArgs k{kld_hashes_global_ + begin, end - begin, begin, k_before, o.min_particles, o.kld_epsilon, o.kld_z};
  launch_kld_chunk(k, kld_keys_, kld_vals_, kld_table_size_, kld_flags_, kld_scan_, scalars_, kld_tile_state_, stream_);
  BB_LAUNCHED_N("kld", 5);
  BB_CHECK(cudaMemcpyAsync(scalars_host_, scalars_, sizeof(Scalars), cudaMemcpyDeviceToHost, stream_));
  return BB200_OK;
}

int Filter::kld_sharded_read(uint64_t* cutoff, uint64_t* new_buckets) {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  if (scalars_host_->exchange_error != 0) return fail(BB200_ERR_STATE, "shard exchange timed out during the KLD count");
  *cutoff = scalars_host_->kld_cutoff;
  *new_buckets = scalars_host_->pad[1];
  return BB200_OK;
}

int Filter::step_totals(uint64_t* rank_totals, int* exponent) {
  if (!step_.active || peer_world_ < 2) return fail(BB200_ERR_STATE, "no sharded step in progress");
  BB_CHECK(cudaSetDevice(config_.device));
  if (!step_.totals_exchanged) {
    mark("exchange_total");
    const int st = enqueue_exchange(kExchangeTotal, !split_posts_, true);
    if (st != BB200_OK) return st;
    step_.totals_exchanged = true;
  }
  if (rank_totals == nullptr) return BB200_OK;  // enqueue only
  BB_CHECK(cudaStreamSynchronize(stream_));
  if (summary_host_->error != 0) return fail(BB200_ERR_STATE, "shard exchange timed out");
  for (int r = 0; r < peer_world_; ++r) rank_totals[r] = summary_host_->rank_totals[r];
  if (exponent != nullptr) *exponent = summary_host_->exponent;
  return BB200_OK;
}

void Filter::step_set_kld_accepted(uint64_t accepted) { step_.kld_accepted = accepted; }

int Filter::step_end(bb200_estimate* est, double* weight_sum, uint64_t* new_size, double* sum_sq) {
  if (!step_.active) return fail(BB200_ERR_STATE, "step_begin must run first");
  BB_CHECK(cudaSetDevice(config_.device));
  // The resample kernel's last block stores the summary to pinned memory and then the step's ticket.  Everything later on
  // this stream is ordered behind that kernel anyway.
  const bool done = step_.poll_seq != 0 && step_.resampled && wait_for_ticket(&summary_host_->seq, step_.poll_seq, stream_);
  if (!done) BB_CHECK(cudaStreamSynchronize(stream_));
  step_.poll_seq = 0;
  finish_marks();
  const bool sharded = peer_world_ > 1;
  if (summary_host_->error != 0) {
    step_.active = false;
    return fail(BB200_ERR_STATE, "shard exchange timed out: a peer rank never posted its value for this step");
  }
  const double* moments = summary_host_->moments;
  step_.total = summary_host_->total;
  step_.exponent = summary_host_->exponent;
  weights_valid_ = summary_host_->valid != 0;
  if (step_.resampled) {
    cur_ ^= 1;
    n_ = sharded ? capacity_ : step_.opts.max_particles;
    if (sharded && step_.kld_accepted != 0) {  // the new set of `accepted` particles in equal contiguous shards
      const uint64_t shard = (step_.kld_accepted + static_cast<uint64_t>(peer_world_) - 1) / static_cast<uint64_t>(peer_world_);
      const uint64_t begin = std::min<uint64_t>(static_cast<uint64_t>(peer_rank_) * shard, step_.kld_accepted);
      n_ = std::min<uint64_t>(shard, step_.kld_accepted - begin);
      first_index_ = static_cast<uint64_t>(peer_rank_) * shard;
    } else if (sharded) {
      first_index_ = config_.first_index;
    }
    ancestors_n_ = n_;
    cdf_valid_ = false;
    step_.active = false;
  } else {
    cdf_valid_ = true;  // kPhaseResample may still follow (selective resampling)
    ++epoch_;           // ... as a new batch of exchanges
  }
  if (new_size != nullptr) *new_size = !sharded ? n_ : (step_.resampled && step_.kld_accepted != 0 ? step_.kld_accepted : global_size_);
  if (sharded && step_.resampled) global_size_ = step_.kld_accepted != 0 ? step_.kld_accepted : config_.global_count;
  if (weight_sum != nullptr) *weight_sum = std::ldexp(static_cast<double>(step_.total), -step_.exponent);
  if (sum_sq != nullptr) *sum_sq = moments[1];
  if (!weights_valid_) error_ = "no positive finite weight (uniform CDF substituted)";
  bb200_estimate local{};
  if (est == nullptr) est = &local;
  estimate_from_moments(moments, pivot_, est);
  pivot_to_estimate(*est, pivot_);
  cloud_ = *est;
  cloud_known_ = step_.resampled;  // unit weights: the estimate describes the raw cloud, the next step can predict its pose bins
  return BB200_OK;
}

int Filter::synchronize() {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  finish_marks();
  return BB200_OK;
}

int Filter::device_pointer(int which, void** ptr, uint64_t* bytes) {
  switch (which) {
    case 0: *ptr = states_[cur_]; *bytes = capacity_ * sizeof(Pose2); return BB200_OK;
    case 1: *ptr = weights_; *bytes = capacity_ * sizeof(double); return BB200_OK;
    case 2: *ptr = cdf_; *bytes = capacity_ * sizeof(unsigned long long); return BB200_OK;
    case 3: *ptr = states_[cur_ ^ 1]; *bytes = capacity_ * sizeof(Pose2); return BB200_OK;
    case 4: *ptr = scalars_; *bytes = sizeof(Scalars); return BB200_OK;
    case 5: *ptr = results_; *bytes = 16 * sizeof(double); return BB200_OK;
    default: return fail(BB200_ERR_INVALID_ARGUMENT, "unknown device pointer id");
  }
}

// ---- maps -----------------------------------------------------------------------------------------

int Filter::set_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& g, bool prob) {
  MapTables tables;
  const int st = prepare_likelihood_field_map(p, g, prob, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Filter::set_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& g) {
  MapTables tables;
  const int st = prepare_beam_map(p, g, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Filter::set_map(const MapTables& tables) {
  BB_CHECK(cudaSetDevice(config_.device));
  return map_.upload(tables, stream_, &error_);
}

int Filter::get_likelihood_field(float* out, uint64_t capacity) const {
  const std::vector<float>& field = map_.field_host;
  if (field.empty()) return BB200_ERR_STATE;
  if (capacity < field.size()) return BB200_ERR_CAPACITY;
  std::memcpy(out, field.data(), field.size() * sizeof(float));
  return BB200_OK;
}

// ---- particle access ---------------------------------------------------------------------------------

int Filter::set_particles(const double* states, const double* weights, uint64_t n) {
  if (n > capacity_) return fail(BB200_ERR_CAPACITY, "more particles than the filter capacity");
  if (n > 0 && states == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "states is null");
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  if (n > 0) {
    BB_CHECK(cudaMemcpy(states_[cur_], states, n * sizeof(Pose2), cudaMemcpyHostToDevice));
    if (weights != nullptr) {
      BB_CHECK(cudaMemcpy(weights_, weights, n * sizeof(double), cudaMemcpyHostToDevice));
    } else {
      const std::vector<double> ones(n, 1.0);
      BB_CHECK(cudaMemcpy(weights_, ones.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    }
  }
  n_ = n;
  cdf_valid_ = false;
  cloud_known_ = false;
  if (n > 0) {  // the covariance is accumulated about the pivot: keep it inside the cloud (no cancellation for far-away sets)
    pivot_[0] = states[2];
    pivot_[1] = states[3];
  }
  return BB200_OK;
}

int Filter::get_particles(double* states, double* weights, uint64_t capacity) {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, n_);
  if (states != nullptr && n > 0) BB_CHECK(cudaMemcpy(states, states_[cur_], n * sizeof(Pose2), cudaMemcpyDeviceToHost));
  if (weights != nullptr && n > 0) BB_CHECK(cudaMemcpy(weights, weights_, n * sizeof(double), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

int Filter::initialize_normal(const double mean[3], const double cov[9], uint64_t n) {
  if (n > capacity_) return fail(BB200_ERR_CAPACITY, "more particles than the filter capacity");
  double transform[9];
  std::string message;
  if (!normal_transform(cov, transform, &message)) return fail(BB200_ERR_INVALID_ARGUMENT, message);
  BB_CHECK(cudaSetDevice(config_.device));
  launch_initialize_normal(states_[cur_], weights_, n, mean, transform, config_.seed, first_index_, stream_);
  BB_LAUNCHED("initialize_normal");
  BB_CHECK(cudaStreamSynchronize(stream_));
  n_ = n;
  cdf_valid_ = false;
  pivot_[0] = mean[0];
  pivot_[1] = mean[1];
  {  // the cloud just drawn is N(mean, cov): the first step can predict its pose bins
    const Pose2 m = pose_from_xytheta(mean[0], mean[1], mean[2]);
    cloud_ = bb200_estimate{{m.c, m.s, m.x, m.y}, {cov[0], cov[1], cov[2], cov[3], cov[4], cov[5], cov[6], cov[7], cov[8]}};
    cloud_known_ = true;
  }
  return BB200_OK;
}

int Filter::initialize_uniform(uint64_t n) {
  if (n > capacity_) return fail(BB200_ERR_CAPACITY, "more particles than the filter capacity");
  if (map_.sensor < 0) return fail(BB200_ERR_STATE, "initialize_from_map needs a map (set_*_map first)");
  if (map_.n_free == 0) return fail(BB200_ERR_STATE, "the map has no free cell to sample from");
  BB_CHECK(cudaSetDevice(config_.device));
  launch_initialize_uniform(states_[cur_], weights_, n, map_.free_cells, map_.n_free, map_.grid_width, map_.grid_resolution, map_.grid_origin,
                            config_.seed, first_index_, stream_);
  BB_LAUNCHED("initialize_uniform");
  BB_CHECK(cudaStreamSynchronize(stream_));
  n_ = n;
  cdf_valid_ = false;
  cloud_known_ = false;
  map_.centre(pivot_);
  return BB200_OK;
}

// ---- per-step operations -----------------------------------------------------------------------------

int Filter::upload_points(const double* points_xy, uint64_t n_points) {
  if (n_points > points_capacity_) {
    points_capacity_ = 0;
    const uint64_t cap = std::max<uint64_t>(n_points, 2048);
    BB_CHECK(realloc_staged(&points_, &points_host_, 2 * cap));
    points_capacity_ = cap;
  }
  double range_sum = 0.0;
  for (uint64_t i = 0; i < n_points; ++i) {
    const double e = std::hypot(points_xy[2 * i], points_xy[2 * i + 1]);
    if (std::isfinite(e)) range_sum += e;
  }
  points_radius_ = scan_radius(points_xy, n_points);
  points_mean_range_ = n_points > 0 ? range_sum / static_cast<double>(n_points) : 1.0;  // lever arm of the heading in the schedule
  if (n_points > 0) {
    // The previous step's copy must have left the staging buffer before it is overwritten.
    std::memcpy(points_host_, points_xy, 2 * n_points * sizeof(double));
    BB_CHECK(cudaMemcpyAsync(points_, points_host_, 2 * n_points * sizeof(double), cudaMemcpyHostToDevice, stream_));
  }
  return BB200_OK;
}

bool Filter::predict_schedule(const MotionSampling& s, Schedule* grid) const {
  // The cloud after this step's propagate, from what the host already knows: the last estimate (the particles carry unit
  // weights, so it describes the raw cloud) composed with the motion means, spread widened by the motion noise.
  if (!cloud_known_) return false;
  const bb200_estimate& e = cloud_;
  const Pose2 mean = motion_apply(s.model, Pose2{e.mean[0], e.mean[1], e.mean[2], e.mean[3]}, s.mean[0], s.mean[1], s.mean[2], Rot2{s.first_c, s.first_s});
  double var_theta = std::max(e.cov[8], 0.0) + s.stddev[0] * s.stddev[0];
  double spread = s.stddev[1] * s.stddev[1];
  if (s.model == BB200_MOTION_DIFFERENTIAL) var_theta += s.stddev[2] * s.stddev[2];
  if (s.model != BB200_MOTION_DIFFERENTIAL) spread += s.stddev[2] * s.stddev[2];
  if (s.model != BB200_MOTION_STATIONARY) spread += s.mean[1] * s.mean[1] * var_theta;
  const double vx = e.cov[0] + spread, vy = e.cov[4] + spread;
  if (!std::isfinite(var_theta) || !std::isfinite(vx) || !std::isfinite(vy) || !std::isfinite(mean.x) || !std::isfinite(mean.y)) return false;
  const double r = std::exp(-0.5 * var_theta);
  schedule_from_moments(*grid, r * mean.c, r * mean.s, mean.x, mean.y, vx, vy, static_cast<double>(n_), points_mean_range_, 0.5 * map_.grid_resolution);
  return true;
}

int Filter::enqueue_propagate_reweight_kernels(const MotionSampling* sampling, uint32_t step, bool do_reweight, uint64_t n_points, bool counters_reset) {
  const bool scheduled = do_reweight && n_ >= kScheduleMinParticles;
  Schedule grid{};
  const uint32_t* perm = nullptr;
  if (scheduled && counters_reset && sampling != nullptr && predict_schedule(*sampling, &grid)) {
    // Bin grid predicted on the host: propagate histograms its own output, two more launches turn it into the order.
    mark("propagate");
    launch_propagate_binned(states_[cur_], n_, *sampling, config_.seed, step, first_index_, grid, bin_rank_, counters_, sched_, stream_);
    BB_LAUNCHED("propagate");
    mark("schedule");
    launch_finish_schedule(bin_rank_, n_, grid.n_bins, sched_, counters_, perm_, sched_tiles_, stream_);
    BB_LAUNCHED_N("schedule", 2);
    perm = perm_;
  } else if (sampling != nullptr || scheduled) {
    mark("propagate");
    launch_propagate(states_[cur_], n_, sampling != nullptr, sampling != nullptr ? *sampling : MotionSampling{}, config_.seed, step,
                     first_index_, scheduled ? sched_ : nullptr, stream_);
    BB_LAUNCHED_N("propagate", scheduled ? 2 : 1);
  }
  if (scheduled && perm == nullptr) {
    mark("schedule");
    launch_build_schedule(states_[cur_], n_, sched_, bins_, counters_, perm_, sched_tiles_, points_mean_range_, 0.5 * map_.grid_resolution, stream_);
    BB_LAUNCHED_N("schedule", 4);
    perm = perm_;
  }
  if (do_reweight) {
    if (map_.sensor == BB200_SENSOR_BEAM) {
      mark("reweight_beam");
      uint64_t pass = 0;
      if (n_points > 0 && beam_two_pass_map(map_)) {
        // hit words of one pass: at most kBeamHitPassBytes, whole warps of particles
        pass = std::min<uint64_t>(n_, std::max<uint64_t>(32, (kBeamHitPassBytes / (4ull * n_points)) / 32 * 32));
        const uint64_t words = beam_hit_words(pass, static_cast<uint32_t>(n_points));
        if (words > beam_hits_words_) {
          BB_CHECK(cudaStreamSynchronize(stream_));
          cudaFree(beam_hits_);
          beam_hits_ = nullptr;
          beam_hits_words_ = 0;
          // sized for the filter's capacity so that a growing particle count (KLD) does not reallocate every step
          const uint64_t pass_cap = std::min<uint64_t>(capacity_, std::max<uint64_t>(32, (kBeamHitPassBytes / (4ull * n_points)) / 32 * 32));
          const uint64_t want = beam_hit_words(std::max(pass, pass_cap), static_cast<uint32_t>(n_points));
          if (dev_alloc(&beam_hits_, want) == cudaSuccess) {
            beam_hits_words_ = want;
          } else {
            (void)cudaGetLastError();  // no room for the intermediate: the fused kernel needs none
            pass = 0;
          }
        }
      }
      if (pass > 0) {
        launch_reweight_beam_two_pass(states_[cur_], weights_, n_, perm, map_.occupancy, map_.beam, points_, static_cast<uint32_t>(n_points), beam_hits_, pass,
                                      scalars_, stream_);
        BB_LAUNCHED_N("reweight_beam", 2 * static_cast<int>((n_ + pass - 1) / pass));
      } else {
        launch_reweight_beam(states_[cur_], weights_, n_, perm, map_.occupancy, map_.beam, points_, static_cast<uint32_t>(n_points), scalars_, stream_);
        BB_LAUNCHED("reweight_beam");
      }
    } else {
      mark("reweight_lfm");
      launch_reweight_lfm(states_[cur_], weights_, n_, perm, map_.field, points_, points_host_, static_cast<uint32_t>(n_points),
                          points_radius_, scalars_, stream_);
      BB_LAUNCHED("reweight_lfm");
    }
  }
  return BB200_OK;
}

int Filter::propagate_reweight(const bb200_motion_sampling* sampling, uint32_t step, const double* points_xy, uint64_t n_points) {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));  // the pinned point staging buffer may still be read by the previous upload
  const int st = enqueue_propagate_reweight(sampling, step, points_xy, n_points);
  if (st != BB200_OK) return st;
  finish_marks();
  return BB200_OK;
}

int Filter::max_weight(double* wmax) {
  const int st = enqueue_max_weight();
  if (st != BB200_OK) return st;
  BB_CHECK(cudaMemcpyAsync(scalars_host_, scalars_, sizeof(Scalars), cudaMemcpyDeviceToHost, stream_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  double v;
  std::memcpy(&v, &scalars_host_->wmax_bits, sizeof(double));
  *wmax = v;
  return BB200_OK;
}

int Filter::build_cdf(double global_wmax, uint64_t* local_total, int* exponent) {
  int st = BB200_OK;
  if (global_wmax < 0.0) st = enqueue_max_weight();  // no global value: the exponent from this filter's own largest weight
  if (st == BB200_OK) st = enqueue_build_cdf(global_wmax);
  if (st != BB200_OK) return st;
  BB_CHECK(cudaMemcpyAsync(scalars_host_, scalars_, sizeof(Scalars), cudaMemcpyDeviceToHost, stream_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  finish_marks();
  if (local_total != nullptr) *local_total = scalars_host_->total;
  if (exponent != nullptr) *exponent = scalars_host_->exponent;
  // No positive finite weight (the reference would divide by zero in normalize.hpp:82): a uniform CDF
  // has been substituted and the weights are left as they are; reported through last_error only.
  weights_valid_ = scalars_host_->valid != 0;
  if (!weights_valid_) error_ = "no positive finite weight (uniform CDF substituted)";
  return BB200_OK;
}

int Filter::normalize_by(uint64_t global_total, double* local_sum_sq) {
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  if (!cdf_valid_) return fail(BB200_ERR_STATE, "build_cdf must run before normalize_by");
  BB_CHECK(cudaSetDevice(config_.device));
  uint32_t rows = 0;
  mark("normalize");
  launch_normalize(weights_, n_, scalars_, global_total, partials_, &rows, stream_);
  BB_LAUNCHED("normalize");
  launch_reduce_partials(partials_, rows, 1, results_, stream_);
  BB_LAUNCHED("reduce_partials");
  BB_CHECK(cudaMemcpyAsync(results_host_, results_, sizeof(double), cudaMemcpyDeviceToHost, stream_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  finish_marks();
  if (local_sum_sq != nullptr) *local_sum_sq = results_host_[0];
  return BB200_OK;
}

int Filter::normalize(double* factor, double* sum_sq) {
  uint64_t total = 0;
  int exponent = 0;
  const int st = build_cdf(-1.0, &total, &exponent);
  if (st != BB200_OK) return st;
  if (factor != nullptr) *factor = std::ldexp(static_cast<double>(total), -exponent);
  return normalize_by(total, sum_sq);
}

int Filter::ensure_cdf_ready() {
  if (cdf_valid_) return BB200_OK;
  return build_cdf(-1.0, nullptr, nullptr);
}

int Filter::moments(const double pivot[2], double out[9]) {
  const int st = enqueue_moments(pivot);
  if (st != BB200_OK) return st;
  BB_CHECK(cudaMemcpyAsync(results_host_, results_, kMomentCount * sizeof(double), cudaMemcpyDeviceToHost, stream_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  finish_marks();
  std::memcpy(out, results_host_, kMomentCount * sizeof(double));
  return BB200_OK;
}

int Filter::estimate(bb200_estimate* out) {
  double m[kMomentCount];
  const int st = moments(pivot_, m);
  if (st != BB200_OK) return st;
  estimate_from_moments(m, pivot_, out);
  pivot_to_estimate(*out, pivot_);
  return BB200_OK;
}

// ---- cluster-based estimate ---------------------------------------------------------------------

int Filter::cluster_estimate(const bb200_cluster_param& p, bb200_estimate* out, uint32_t* cluster_ids, uint64_t ids_capacity, uint32_t* n_cells,
                             uint32_t* n_clusters) {
  BB_CHECK(cudaSetDevice(config_.device));
  const int st = cluster_.estimate(states_[cur_], weights_, n_, pivot_, p, stream_, out, cluster_ids, ids_capacity, n_cells, n_clusters, &error_);
  if (st == BB200_OK) finish_marks();
  return st;
}

int Filter::particle_histogram(double linear_resolution, double angular_resolution, bb200_cluster_cell* bins, uint64_t capacity, uint64_t* n_bins,
                               double* max_bin_weight) {
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  if (!(linear_resolution > 0.0) || !(angular_resolution > 0.0)) return fail(BB200_ERR_INVALID_ARGUMENT, "histogram resolutions must be positive");
  BB_CHECK(cudaSetDevice(config_.device));
  std::vector<HostCell> host;
  const int st = cluster_.cell_records(states_[cur_], weights_, n_, pivot_, linear_resolution, angular_resolution, stream_, &host, &error_);
  if (st != BB200_OK) return st;
  finish_marks();
  if (n_bins != nullptr) *n_bins = host.size();
  double top = 1e-3;  // beluga_ros/particle_cloud.hpp:197
  for (const HostCell& c : host) top = c.weight > top ? c.weight : top;
  if (max_bin_weight != nullptr) *max_bin_weight = top;
  if (bins != nullptr) {
    if (capacity < host.size()) return fail(BB200_ERR_CAPACITY, "histogram bin buffer too small (n_bins has the count)");
    static_assert(sizeof(bb200_cluster_cell) == sizeof(HostCell), "public and internal cell records must agree");
    std::memcpy(bins, host.data(), host.size() * sizeof(HostCell));
  }
  return BB200_OK;
}

int Filter::sample_states(uint64_t count, uint32_t step, double* states_out) {
  // views::sample | take_exactly(count) (beluga_ros/particle_cloud.hpp:141-147): `count` states drawn by weight, the
  // particle set itself untouched.  Counter RNG: the multinomial draws of `step` (the caller picks a step the filter
  // does not use, e.g. 0xFFFFFFFF - publish count).
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  if (count > capacity_) return fail(BB200_ERR_CAPACITY, "more samples than the filter capacity");
  if (count > 0 && states_out == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "states_out is null");
  if (count == 0) return BB200_OK;
  int st = ensure_cdf_ready();
  if (st != BB200_OK && !cdf_valid_) return st;
  BB_CHECK(cudaSetDevice(config_.device));
  bb200_resample_opts o{};
  o.scheme = BB200_RESAMPLE_MULTINOMIAL;
  o.step = step;
  o.min_particles = o.max_particles = count;
  ResampleArgs a = make_resample_args(o, 0, count, false);
  a.weights_out = nullptr;  // the weights stay what they are
  a.ancestors = nullptr;
  launch_resample(a, scalars_, partials_, stream_);  // into the staging state buffer; no flip
  BB_LAUNCHED("sample_states");
  BB_CHECK(cudaMemcpyAsync(states_out, states_[cur_ ^ 1], count * sizeof(Pose2), cudaMemcpyDeviceToHost, stream_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  return BB200_OK;
}

ResampleArgs Filter::make_resample_args(const bb200_resample_opts& o, uint64_t slot_begin, uint64_t slot_end, bool with_hashes) const {
  ResampleArgs a{};
  a.states_in = states_[cur_];
  a.cdf = cdf_;
  a.n_in = n_;
  a.states_out = states_[cur_ ^ 1] + slot_begin;
  a.weights_out = weights_ + slot_begin;
  a.ancestors = ancestors_ != nullptr ? ancestors_ + slot_begin : nullptr;
  a.hashes = with_hashes ? hashes_ + slot_begin : nullptr;
  a.slot_first = first_index_ + slot_begin;
  a.slot_count = slot_end - slot_begin;
  a.total_slots = o.max_particles;
  a.scheme = o.scheme;
  a.seed = config_.seed;
  a.step = o.step;
  a.random_state_probability = o.random_state_probability;
  a.free_cells = map_.free_cells;
  a.n_free = map_.n_free;
  a.grid_width = map_.grid_width;
  a.grid_resolution = map_.grid_resolution;
  a.grid_origin = map_.grid_origin;
  for (int k = 0; k < 3; ++k) a.hash_resolution[k] = o.spatial_resolution[k];
  a.pivot_x = pivot_[0];
  a.pivot_y = pivot_[1];
  return a;
}

int Filter::resample(const bb200_resample_opts& o, uint64_t* new_size) {
  if (n_ == 0) return fail(BB200_ERR_STATE, "no particles");
  if (o.max_particles == 0 || o.max_particles > capacity_) return fail(BB200_ERR_CAPACITY, "max_particles exceeds the filter capacity");
  if (o.random_state_probability > 0.0 && map_.n_free == 0) return fail(BB200_ERR_STATE, "recovery injection needs a map with free cells");
  int st = ensure_cdf_ready();
  if (st != BB200_OK && !cdf_valid_) return st;
  BB_CHECK(cudaSetDevice(config_.device));
  // The weight array is reused for the output (all ones); the CDF already holds what sampling needs.
  uint64_t m = o.max_particles;
  if (o.min_particles >= o.max_particles) {
    // take_while_kld never stops before max when min == max (take_while_kld.hpp:86-87,136).
    mark("resample");
    launch_resample(make_resample_args(o, 0, o.max_particles, false), scalars_, partials_, stream_);
    BB_LAUNCHED("resample");
    BB_CHECK(cudaStreamSynchronize(stream_));
  } else {
    st = resample_kld(o, &m);
    if (st != BB200_OK) return st;
  }
  finish_marks();
  cur_ ^= 1;
  cloud_known_ = false;
  n_ = m;
  ancestors_n_ = n_;
  cdf_valid_ = false;
  if (new_size != nullptr) *new_size = n_;
  return BB200_OK;
}

int Filter::resample_range(const bb200_resample_opts& o, uint64_t global_total, uint64_t cdf_offset, uint64_t slot_begin, uint64_t slot_end) {
  const int st = enqueue_resample_range(o, global_total, cdf_offset, slot_begin, slot_end);
  if (st != BB200_OK) return st;
  BB_CHECK(cudaStreamSynchronize(stream_));
  finish_marks();
  return BB200_OK;
}

int Filter::adopt(uint64_t n, int from_staging) {
  const int st = enqueue_adopt(n);
  if (st != BB200_OK) return st;
  if (from_staging) cur_ ^= 1;  // the staging buffer holds the n states
  BB_CHECK(cudaStreamSynchronize(stream_));
  finish_marks();
  return BB200_OK;
}

int Filter::resample_kld(const bb200_resample_opts& o, uint64_t* accepted) {
  if (config_.global_count != capacity_ || first_index_ != 0) return fail(BB200_ERR_STATE, "KLD-adaptive resampling runs on a single shard");
  if (o.max_particles >= (1ull << 32)) return fail(BB200_ERR_CAPACITY, "KLD-adaptive resampling keeps 32-bit slot indices: max_particles must be below 2^32");
  if (hashes_ == nullptr) {
    BB_CHECK(dev_alloc(&hashes_, capacity_));
    BB_CHECK(dev_alloc(&kld_flags_, capacity_));
    BB_CHECK(dev_alloc(&kld_scan_, capacity_));
    kld_table_size_ = 2;
    while (kld_table_size_ < 2 * capacity_) kld_table_size_ <<= 1;
    BB_CHECK(dev_alloc(&kld_keys_, kld_table_size_));
    BB_CHECK(dev_alloc(&kld_vals_, kld_table_size_));
  }
  mark("kld");
  launch_kld_clear(kld_keys_, kld_vals_, kld_table_size_, stream_);
  const uint64_t max = o.max_particles;
  uint64_t begin = 0, k_before = 0;
  uint64_t end = std::min<uint64_t>(max, std::max<uint64_t>(2 * o.min_particles, 65536));
  *accepted = max;
  while (begin < max) {
    launch_resample(make_resample_args(o, begin, end, true), scalars_, partials_, stream_);
    BB_LAUNCHED("resample");
    KldArgs k{hashes_ + begin, end - begin, begin, k_before, o.min_particles, o.kld_epsilon, o.kld_z};
    launch_kld_chunk(k, kld_keys_, kld_vals_, kld_table_size_, kld_flags_, kld_scan_, scalars_, tile_state_, stream_);
    BB_LAUNCHED_N("kld", 5);
    BB_CHECK(cudaMemcpyAsync(scalars_host_, scalars_, sizeof(Scalars), cudaMemcpyDeviceToHost, stream_));
    BB_CHECK(cudaStreamSynchronize(stream_));
    if (scalars_host_->kld_cutoff != ~0ull) {
      // take_while drops the first element whose condition fails (take_while_kld.hpp:134-136).
      *accepted = std::min<uint64_t>(scalars_host_->kld_cutoff - 1, max);
      break;
    }
    k_before += scalars_host_->pad[1];
    begin = end;
    end = std::min<uint64_t>(max, end * 2);
  }
  return BB200_OK;
}

int Filter::step_resample(const bb200_motion_sampling& sampling, uint32_t step, const double* points_xy, uint64_t n_points,
                          const bb200_resample_opts& o, bb200_estimate* est, double* weight_sum, uint64_t* new_size) {
  int st = step_begin(sampling, step, points_xy, n_points, o, true);
  for (int phase = kPhaseReweight; st == BB200_OK && phase <= kPhaseFinish; ++phase) st = step_phase(phase);
  if (st != BB200_OK) {
    step_.active = false;
    return st;
  }
  return step_end(est, weight_sum, new_size, nullptr);
}

int Filter::ancestors(int64_t* out, uint64_t capacity) {
  if (ancestors_ == nullptr) return fail(BB200_ERR_STATE, "filter was created without record_ancestors");
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, ancestors_n_);
  if (n > 0) BB_CHECK(cudaMemcpy(out, ancestors_, n * sizeof(int64_t), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

int Filter::cdf(uint64_t* out, uint64_t capacity) {
  if (!cdf_valid_) return fail(BB200_ERR_STATE, "no CDF has been built for the current weights");
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, n_);
  if (n > 0) BB_CHECK(cudaMemcpy(out, cdf_, n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

}  // namespace bb200
