// Device-resident particle set of the CUDA MCL backend: buffers, its map (device_map.hpp) and the per-step
// kernel sequence behind the C ABI of include/beluga_b200.h.  Host-side counterpart of
// beluga::TupleVector<std::tuple<SE2d, Weight>> (reference: containers/tuple_vector.hpp:50-223)
// plus the actions/views that iterate it (propagate, reweight, normalize, sample, assign).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/beluga_b200.h"
#include "cluster.cuh"
#include "device_buffer.hpp"
#include "device_map.hpp"
#include "kernels.cuh"
#include "shard_link.hpp"
#include "state_blob.hpp"

namespace bb200 {

/// The particle arrays of a state blob, copied to the host.
struct ParticleArrays {
  std::vector<double> states, weights;
  std::vector<uint64_t> cdf;
  std::vector<int64_t> ancestors;
};

class Filter {
 public:
  explicit Filter(const bb200_filter_config& config);
  ~Filter();
  Filter(const Filter&) = delete;
  Filter& operator=(const Filter&) = delete;

  // Every method returns a bb200_status and records the message for last_error().
  int set_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob);
  int set_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid);
  /// A landmark map for LandmarkSensorModel2d (lp) or, with lp null, BearingSensorModel2d (bp).
  int set_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map);
  /// Prepares a step's detections on a landmark map and enqueues their upload; BB200_ERR_STATE on any other map.  The
  /// reweight of a step that passes staged_detections() as its points weighs them.  prepare_step_detections followed by
  /// upload_detections.
  int stage_detections(const bb200_landmark_detection* detections, uint64_t n);
  /// The host half of stage_detections: the detections prepared against this filter's landmark map (prepare_detections);
  /// BB200_ERR_STATE on any other map, BB200_ERR_INVALID_ARGUMENT for n >= 2^32 - 1.  Nothing reaches the device.
  int prepare_step_detections(const bb200_landmark_detection* detections, uint64_t n, std::vector<LandmarkDetection>* prepared);
  /// The device half: enqueues the upload of detections prepared against this map's tables (or an identical copy of
  /// them, as every shard of a filter holds) on this filter's stream, once the previous step's upload has left the
  /// pinned staging buffer.
  int upload_detections(const std::vector<LandmarkDetection>& prepared);
  /// The `points_xy` of a step on a landmark map: the reweight weighs the staged detections instead of points.
  static const double* staged_detections() { return &kStagedDetections; }
  /// Makes the prepared tables this filter's map (the upload half of set_*_map).
  int set_map(const MapTables& tables);
  int get_likelihood_field(float* out, uint64_t capacity) const;

  int set_particles(const double* states, const double* weights, uint64_t n);
  int get_particles(double* states, double* weights, uint64_t capacity);
  int initialize_normal(const double mean[3], const double cov[9], uint64_t n);
  /// n samples of MultivariateUniformDistribution over the free cells of the current map (initialize_from_map).
  int initialize_uniform(uint64_t n);
  uint64_t size() const { return n_; }

  int propagate_reweight(const bb200_motion_sampling* sampling, uint32_t step, const double* points_xy, uint64_t n_points);
  int max_weight(double* wmax);
  int build_cdf(double global_wmax, uint64_t* local_total, int* exponent);
  int normalize_by(uint64_t global_total, double* local_sum_sq);
  int normalize(double* factor, double* sum_sq);
  int resample(const bb200_resample_opts& o, uint64_t* new_size);
  int resample_range(const bb200_resample_opts& o, uint64_t global_total, uint64_t cdf_offset, uint64_t slot_begin, uint64_t slot_end);
  int adopt(uint64_t n, int from_staging);
  int ancestors(int64_t* out, uint64_t capacity);
  int cdf(uint64_t* out, uint64_t capacity);
  /// The particle set's part of a state blob: its scalars, and *size the blob's size with them.  With `arrays`, also its
  /// arrays (the CDF while it is current, the ancestors when `record_ancestors`) and the current CDF's total.
  int particle_set(ParticleSetState* set, ParticleArrays* arrays, uint64_t* size, bool record_ancestors);
  /// Makes the particle set of a decoded state this filter's (its params' max_particles fit the capacity).
  int restore_particle_set(const FilterState& s);
  int estimate(bb200_estimate* out);
  int moments(const double pivot[2], double out[9]);
  /// beluga::cluster_based_estimate (algorithm/cluster_based_estimation.hpp:415-432); cluster_ids
  /// (optional, one per particle) is the parity hook for ParticleClusterizer::operator() (:304-316).
  int cluster_estimate(const bb200_cluster_param& p, bb200_estimate* out, uint32_t* cluster_ids, uint64_t ids_capacity, uint32_t* n_cells,
                       uint32_t* n_clusters);
  /// Device-side histogram of the particle cloud over spatial-hash buckets (beluga_ros/particle_cloud.hpp:197-210): one
  /// record per occupied bucket in first-occurrence order.  bins may be null (count only).
  int particle_histogram(double linear_resolution, double angular_resolution, bb200_cluster_cell* bins, uint64_t capacity, uint64_t* n_bins,
                         double* max_bin_weight);
  /// The records of particle_histogram, in first-occurrence order, as the host vector the clusterizer returns.
  int cell_records(double linear_resolution, double angular_resolution, std::vector<HostCell>* host);
  /// `count` states drawn by weight without touching the set (views::sample | take_exactly, particle_cloud.hpp:141-147).
  int sample_states(uint64_t count, uint32_t step, double* states_out);
  /// Ray2d::cast (algorithm/raycasting.hpp:79-107) on the current map for n_poses sensor poses {cos, sin, x, y} (map frame)
  /// and n_bearings bearings {cos, sin}, pose major: ranges[i * n_bearings + j] = min(distance, max_range) on a hit, +inf on
  /// a miss.  One launch and one synchronisation (none without rays); the particle set is not touched.
  int cast_rays(const double* poses, uint64_t n_poses, const double* bearings, uint64_t n_bearings, double max_range, double* ranges);
  /// cast_rays in three parts, so that a caller holding filters on several devices keeps them all casting at once: the
  /// refusals (nothing reaches the device; *n_rays = n_poses * n_bearings), the upload and launch of n_rays > 0 rays, and
  /// the read-back of the ranges with the one synchronisation.
  int check_cast_rays(const double* poses, uint64_t n_poses, const double* bearings, uint64_t n_bearings, const double* ranges, uint64_t* n_rays);
  int enqueue_cast_rays(const double* poses, uint64_t n_poses, const double* bearings, uint64_t n_bearings, double max_range);
  int finish_cast_rays(double* ranges, uint64_t n_rays);

  // ---- sample_states over joined shards (bb200_sharded_amcl_sample_states) ----
  /// Enqueues the multinomial draws of `step` among the global slots [0, count) whose position lies in this shard's span
  /// [cdf_offset, cdf_offset + local total) of the global CDF (global_total): resample_range's multinomial form.  Slot j's
  /// state goes to the staging buffer of the shard that owns it (j / capacity), as the sharded resample pushes its
  /// particles; no weight, ancestor or particle of any shard changes.  The CDF must be current.
  int sample_range(uint64_t count, uint32_t step, uint64_t global_total, uint64_t cdf_offset);
  /// The local total and the fixed-point exponent of the current CDF; total 0 when the CDF is not current (or there are no
  /// particles).
  int current_cdf(uint64_t* total, int* exponent);
  /// The first n states of the staging buffer, after this filter's stream has drained.
  int staging_states(double* out, uint64_t n);

  /// The fused single-GPU step (propagate | reweight | normalize | resample | estimate with one host synchronisation) is
  /// step_begin, kPhaseReweight and then this: CDF, resample, moments, and the synchronisation (step_end).
  int finish_resample(bb200_estimate* est, double* weight_sum, uint64_t* new_size);

  // ---- a step whose sensor model the caller runs (bb200_amcl_update_begin / _end, bb200_sharded_amcl_update_begin / _end) ----
  /// The host half of a weighed step's begin: checks the step and allocates the factor buffer (and, on joined shards, the
  /// event of kPhaseApplyFactors) on first use.  Nothing reaches the device, so a driver of several shards runs it on
  /// every shard before weigh_propagate on any, and a refusal leaves every shard's particles as they were.  `injects`: the
  /// plan may inject random states, which needs a map with free cells.
  int weigh_prepare(const bb200_resample_opts& o, bool injects);
  /// The device half, after weigh_prepare: enqueues the reset and the propagate (the non-binned propagate_kernel: no
  /// pose-bin schedule); no host synchronisation.  `resample_planned`: kPhaseResample follows kPhaseCdf directly.  One
  /// filter: the step then ends as the fused step does (weigh_apply, then finish_resample); otherwise weigh_apply is
  /// followed by the blocking normalize / resample / estimate.  Joined shards: the step continues with kPhaseApplyFactors
  /// and the phases after it, as step_begin's does after kPhaseReweight.
  int weigh_propagate(const bb200_motion_sampling& sampling, uint32_t step, const bb200_resample_opts& o, bool resample_planned);
  /// Enqueues w *= factors over the particle set and the largest weight into the device scalars.
  int weigh_apply();
  /// Orders this filter's stream behind the end of `peer`'s kPhaseApplyFactors (a stream wait, no host synchronisation).
  int wait_for_factors(const Filter& peer);
  /// Whether a weighed step is open on this filter: the C ABI then refuses every call but the step's end and destroy.
  void set_weigh_open(bool open) { weigh_open_ = open; }
  bool weigh_open() const { return weigh_open_; }
  /// Device views of an open weighed step: the propagated states and the factors the caller writes, n of each.
  const double* weigh_states() const { return reinterpret_cast<const double*>(states_[cur_].get()); }
  double* weigh_factors() { return factors_.get(); }

  // Stream-ordered variants for callers that interleave collectives on the same stream (sharded
  // filters): nothing here synchronises with the host or reads results back.  Each blocking call
  // above is its variant here followed by the synchronisation and the read-back.
  int set_stream(void* stream);
  int enqueue_propagate_reweight(const bb200_motion_sampling* sampling, uint32_t step, const double* points_xy, uint64_t n_points);
  /// global_wmax < 0: the exponent from the wmax in the device scalars (all-reduced by the caller).
  int enqueue_build_cdf(double global_wmax);
  int enqueue_resample_range(const bb200_resample_opts& o, uint64_t global_total, uint64_t cdf_offset, uint64_t slot_begin, uint64_t slot_end);
  int enqueue_adopt(uint64_t n);
  int enqueue_moments(const double pivot[2]);   // raw moments stay in the device result block

  // ---- one filter over several shards, exchanges through peer memory (no NCCL, no host round trip) ----
  /// Export, join and leave go through the link; its views stay valid because the state buffers are never reallocated.
  ShardLink& link() { return link_; }
  cudaStream_t stream() const { return stream_; }
  /// The fused resampling step (propagate | reweight | normalize | resample | estimate), any number of shards.
  /// step_begin validates and stages the inputs; step_phase(1..4) only enqueues; step_end synchronises once.
  /// A driver holding several shards in one thread enqueues phase k of every shard before phase k+1 of any.
  int step_begin(const bb200_motion_sampling& sampling, uint32_t step, const double* points_xy, uint64_t n_points, const bb200_resample_opts& o,
                 bool resample_planned);
  enum StepPhase : int {
    kPhaseReweight = 1,   // begin_step | propagate | schedule | reweight                      (posts the shard's largest weight)
    kPhaseCdf = 2,        // common exponent | fixed-point CDF                                 (posts the shard's total)
    kPhaseResample = 3,   // resample (+ redistribution over peer memory) | moments of the new set (posts them)
    kPhaseFinish = 4,     // global moments, read-back
    kPhaseNormalize = 5,  // joined shards, instead of kPhaseResample on a step that keeps its particles: w /= S | moments
    kPhaseApplyFactors = 6  // a weighed step (weigh_propagate), instead of kPhaseReweight: w *= factors   (posts the shard's largest weight)
  };
  int step_phase(int phase);
  void step_abort();
  // KLD on shards (views/take_while_kld.hpp:72-137 over the globally ordered candidate stream).  After kPhaseCdf:
  //   step_totals            enqueues the exchange of the ranks' fixed-point totals
  //   kld_sharded_candidates hashes of this rank's candidates among the slots [begin, end) -> every rank's hash array
  //   kld_sharded_count      (after all ranks' candidates) distinct-bucket count over the window, on every rank alike
  //   kld_sharded_read       first failing count (~0: none in this window), new buckets of the window
  //   step_set_kld_accepted  the count the loop settled on; kPhaseResample then produces exactly those slots
  int step_totals();
  int kld_sharded_candidates(uint64_t begin, uint64_t end);
  int kld_sharded_count(uint64_t begin, uint64_t end, uint64_t k_before);
  int kld_sharded_read(uint64_t* cutoff, uint64_t* new_buckets);
  void step_set_kld_accepted(uint64_t accepted);
  uint64_t global_size() const { return link_.world() > 1 ? global_size_ : n_; }
  uint64_t first_index() const { return first_index_; }
  const double* pivot() const { return pivot_; }
  /// Synchronises and closes the batch of phases enqueued so far.  After kPhaseNormalize a caller may still run
  /// kPhaseResample + kPhaseFinish + step_end (selective resampling: the decision needs the effective sample size).
  int step_end(bb200_estimate* est, double* weight_sum, uint64_t* new_size, double* sum_sq);

  int synchronize();
  int device_pointer(int which, void** ptr, uint64_t* bytes);

  void set_timing(bool on) { timing_ = on; }
  void clear_timings() { timings_.clear(); }
  int last_timings(const char** names, float* ms, int capacity) const;
  uint64_t launch_count() const { return launches_ + map_.launches() + cluster_.launches(); }
  /// False when the last CDF was built from a weight set without any positive finite weight (uniform CDF substituted).
  bool last_weights_valid() const { return weights_valid_; }
  const char* last_error() const { return error_.c_str(); }
  void record_error(const std::string& message) const { error_ = message; }  // the C-ABI exception guard
  int fail_with(int status, const std::string& message) { return fail(status, message); }
  bool ok() const { return created_; }
  int create_status() const { return create_status_; }

 private:
  int fail(int status, const std::string& message) {
    error_ = message;
    return status;
  }
  int check(cudaError_t e, const char* what) { return cuda_check(e, what, &error_); }
  /// A joined shard's particle count against the plan's: `capacity` particles (fewer only under KLD), world * capacity in all.
  int check_shard_size(const bb200_resample_opts& o);
  int upload_points(const double* points_xy, uint64_t n_points);
  /// propagate | schedule | reweight on a staged step (points uploaded, scalars reset), no validation.
  int enqueue_propagate_reweight_kernels(const MotionSampling* sampling, uint32_t step, bool do_reweight, uint64_t n_points, bool counters_reset);
  int enqueue_max_weight();  // begin_step | max_weight: this filter's largest weight into the device scalars
  /// moments | reduce_partials about `pivot` into the device result block; unlike enqueue_moments, also on an empty set.
  int enqueue_moment_kernels(const double pivot[2]);
  bool predict_schedule(const MotionSampling& s, Schedule* grid) const;
  int ensure_cdf_ready();
  int resample_kld(const bb200_resample_opts& o, uint64_t* accepted);
  /// The KLD tables for `slots` candidate slots, all or none (the one-GPU hashes, or the shards' scan state).
  int ensure_kld_tables(uint64_t slots, bool sharded);
  /// The box injected states are drawn from on a landmark map (launch_resample), null on a grid map.
  const double* random_box() const { return map_.landmark_map() ? map_.box : nullptr; }
  ResampleArgs make_resample_args(const bb200_resample_opts& o, uint64_t slot_begin, uint64_t slot_end, bool with_hashes) const;
  void mark(const char* name);  // timing: record an event before the next kernel
  void finish_marks();
  bool use_device() const;

  struct StepContext {
    bool active{false};
    MotionSampling sampling{};
    uint32_t step{0};
    uint64_t n_points{0};
    bb200_resample_opts opts{};
    uint32_t partial_rows{1};
    bool resampled{false};   // kPhaseResample ran in the batch being closed
    bool normalized{false};  // kPhaseNormalize ran (weights are normalised, the CDF stays valid)
    bool resample_planned{false};  // kPhaseResample follows kPhaseCdf directly (every_n fired, no ESS decision in between)
    bool weights_filled{false};
    bool totals_exchanged{false};
    int poll_seq{0};  // != 0: the resample kernel stores this ticket to the pinned summary when the step is complete
    uint64_t kld_accepted{0};  // KLD on shards: particle count of the new set (0: fixed size)
    unsigned long long total{0};
    int exponent{0};
  };
  StepContext step_{};
  int enqueue_exchange(int kind, bool post, bool wait);

  bb200_filter_config config_{};
  bool created_{false};
  int create_status_{BB200_OK};
  mutable std::string error_;
  cudaStream_t stream_{nullptr};
  bool owns_stream_{true};
  PinnedBuffer<StepSummary> summary_host_;

  // particle set (ping-pong states for the resample gather)
  uint64_t capacity_{0}, n_{0};
  uint64_t first_index_{0};   // global index of local particle 0 (moves when a KLD-sized filter re-splits its particles)
  uint64_t global_size_{0};   // particles over all shards
  DeviceBuffer<Pose2> states_[2];
  int cur_{0};
  DeviceBuffer<double> weights_;
  DeviceBuffer<unsigned long long> cdf_;
  DeviceBuffer<long long> ancestors_;
  uint64_t ancestors_n_{0};
  bool cdf_valid_{false};
  bool weights_valid_{true};

  // scratch
  DeviceBuffer<Scalars> scalars_;
  PinnedBuffer<Scalars> scalars_host_;
  DeviceBuffer<unsigned long long> tile_state_;
  DeviceBuffer<double> partials_;
  DeviceBuffer<double> results_;      // kMomentCount + extras
  PinnedBuffer<double> results_host_;

  Clusterizer cluster_;

  // KLD scratch, allocated on first use for the slots of one pass (capacity_ on one GPU, global_count on shards)
  struct KldTables {
    DeviceBuffer<unsigned long long> hashes;      // one GPU: spatial hash of each candidate slot
    DeviceBuffer<uint32_t> flags, scan;
    DeviceBuffer<unsigned long long> keys;        // hash set of a power of two >= 2 * slots entries
    DeviceBuffer<unsigned int> vals;
    DeviceBuffer<unsigned long long> tile_state;  // shards: scan state of the count (one GPU uses tile_state_)
  };
  KldTables kld_;

  // measurement
  DeviceBuffer<double> points_;
  PinnedBuffer<double> points_host_;  // staging
  double points_radius_{0.0};
  static const double kStagedDetections;
  /// A step's measurement against the map's kind: points on a grid map, staged detections on a landmark map.
  int check_measurement(const double* points_xy) {
    if (map_.landmark_map() != (points_xy == staged_detections()))
      return fail(BB200_ERR_STATE, map_.landmark_map() ? "a landmark map weighs detections, not points" : "detections need a landmark map");
    return BB200_OK;
  }
  DeviceBuffer<LandmarkDetection> detections_;    // landmark maps: the staged detections ...
  PinnedBuffer<LandmarkDetection> detections_host_;
  uint32_t n_detections_{0};                      // ... and their count
  double points_mean_range_{1.0};

  // execution schedule (pose-sorted processing order of the reweight kernels)
  static constexpr uint64_t kScheduleMinParticles = 32768;
  DeviceBuffer<Schedule> sched_;
  DeviceBuffer<uint32_t> bins_;
  DeviceBuffer<uint2> bin_rank_;
  DeviceBuffer<uint32_t> perm_;
  DeviceBuffer<uint32_t> counters_;
  DeviceBuffer<unsigned long long> sched_tiles_;

  DeviceMap map_;
  DeviceBuffer<double> rays_;  // ray casts (grown on use): the poses, the bearings, then the ranges
  uint64_t cast_out_{0};       // offset of the last cast's ranges in rays_
  DeviceBuffer<uint32_t> beam_hits_;  // two-pass beam model: hit word per (beam, particle) of one pass
  DeviceBuffer<double> factors_;      // weighed steps: the caller's likelihood per particle (capacity_, allocated on the first)
  bool weigh_open_{false};
  cudaEvent_t factors_applied_{nullptr};  // weighed steps of shards: the end of kPhaseApplyFactors (created by the first)

  double pivot_[2]{0.0, 0.0};
  bb200_estimate cloud_{};     // last estimate, when it describes the raw (unit-weight) cloud
  bool cloud_known_{false};
  int step_seq_{0};

  // timing
  bool timing_{false};
  struct Mark {
    const char* name;
    cudaEvent_t event;
  };
  std::vector<Mark> marks_;
  std::vector<cudaEvent_t> event_pool_;
  size_t events_used_{0};
  std::vector<std::pair<const char*, float>> timings_;
  uint64_t launches_{0};

  // Declared last, so destroyed first: the peers' buffers mapped into this process are closed before this filter's own
  // buffers are freed.
  ShardLink link_{&error_};
};

/// bb200_motion_sampling -> the kernels' MotionSampling.
MotionSampling to_kernel_sampling(const bb200_motion_sampling& s);

/// BB200_ERR_NO_DEVICE without any CUDA device, BB200_ERR_INVALID_ARGUMENT for an ordinal out of range.
int check_device(int device, std::string* error);

/// Largest |x| + |y| of a scan's end points: bounds the cells the reweight kernels can reach.  A NaN sticks, which sends
/// the scan down the exact lookup path.
double scan_radius(const double* points_xy, uint64_t n_points);

/// Spins until the kernel that ends a step stores `ticket` into the pinned word: the host sees the end of the step a few
/// microseconds before a stream synchronisation would return.  The stream is queried now and then so that a failed launch
/// cannot hang the caller.  False when the stream ended (or failed) without the ticket being seen: the caller synchronises.
bool wait_for_ticket(const volatile int* word, int ticket, cudaStream_t stream);

/// Symmetric 3x3 covariance -> V * sqrt(Lambda) (multivariate_normal_distribution.hpp:109-126).
/// Returns false with a message for non-symmetric / negative-eigenvalue input.
bool normal_transform(const double cov[9], double transform[9], std::string* error);

}  // namespace bb200
