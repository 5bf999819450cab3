// K independent beluga::Amcl filters that share one device, stepped together: one call runs every updating member's step
// with a fixed sequence of launches (csrc/kernels.cuh: launch_batch_step) and one host synchronisation, whatever K is.
// Each member keeps the host half of a bb200_amcl (AmclPolicy) and a slice of the batch's particle buffers, and reads one
// of the batch's maps (a grid with its sensor model, the likelihood-field model or the beam model, or a landmark map with
// the landmark or bearing model).
#pragma once

#include <map>
#include <string>
#include <vector>

#include "amcl.hpp"
#include "cluster.cuh"
#include "device_buffer.hpp"
#include "device_map.hpp"
#include "state_blob.hpp"

namespace bb200 {

/// Largest particle count of a batch member: one member's kernels then run in at most 128 CTAs of each launch, and a
/// KLD-adaptive member's resample_kld takes one chunk (its first chunk of min(max, max(2 min, 65536)) slots is all of them).
constexpr uint64_t kBatchMaxParticles = 32768;

class Batch {
 public:
  /// flags (bb200_batch_flags): BB200_BATCH_ADAPTIVE lets members have min_particles < max_particles (KLD-adaptive
  /// particle counts, as a standalone filter), otherwise every member keeps a fixed count; BB200_BATCH_SELECTIVE lets
  /// members have selective_resampling.  The flags change validation only.
  Batch(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags = 0);
  ~Batch();
  Batch(const Batch&) = delete;
  Batch& operator=(const Batch&) = delete;

  /// The configurations a batch rejects, checked without touching a device (BB200_OK or BB200_ERR_INVALID_ARGUMENT).
  static int validate(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags, std::string* error);

  bool ok() const { return created_; }
  int create_status() const { return create_status_; }
  const char* last_error() const { return error_.c_str(); }
  void record_error(const std::string& message) const { error_ = message; }  // the C-ABI exception guard
  /// Slots, occupied and vacant: the length of every per-member array a call takes.
  int members() const { return static_cast<int>(members_.size()); }

  /// A new member in the lowest vacant slot, or in a new slot after the last; *member receives the slot.  The member is
  /// validated as create validates one under this batch's flags and device, and starts as a created member does: no map,
  /// no particles.  Every other member keeps its particles, weights, CDF, ancestors, policies and map: their live data
  /// moves to the new layout in one launch (none when no other member holds particles).
  int add_member(const bb200_amcl_param& params, const bb200_motion_param& motion, int* member);
  /// Makes slot `member` vacant and frees its share of the particle buffers (BB200_ERR_STATE for the last occupied slot).
  int remove_member(int member);
  int member_active(int member, int* active) const;
  /// The state blob (state_blob.hpp) of every member whose present[m] is non-zero (present == nullptr: every occupied
  /// slot).  size[m] receives the size of member m's blob; out[m] receives the blob when out and out[m] are set and
  /// capacity[m] holds it (BB200_ERR_CAPACITY, before anything reaches the device, when some selected buffer does not).
  /// One batch_relayout_kernel launch gathers every written member's arrays into one staging buffer, one copy brings it to
  /// pinned memory and one synchronisation ends the call, whatever K is; none of them when no written member holds data.
  int export_members(const uint8_t* present, void* const* out, const uint64_t* capacity, uint64_t* size);
  /// export_members with member `member` alone selected.
  int export_member(int member, void* out, uint64_t capacity, uint64_t* size);
  /// add_member with a history: the member of a state blob, validated as add_member validates it (the blob's device is
  /// not read), in the lowest vacant slot or a new one, reading map `map` (-1: none).  Its arrays reach the new layout
  /// with one copy and one launch more than add_member's; on failure the batch is unchanged.
  int import_member(const void* blob, uint64_t size, int map, int* member);
  /// Gives the members of a batch just created from these states' params and motions their particle sets and policies
  /// (bb200_amcl_batch_create_from_states): one copy and one launch, whatever K is.
  int restore_members(const std::vector<FilterState>& states);
  uint64_t launch_count() const { return launches_; }  // including the map uploads' (the beam model's normaliser tables)

  /// One map for every member: removes every map, adds this one and assigns every member to it.
  int set_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob);
  int set_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid);
  /// Adds a map without assigning it; *id receives its id (0, 1, ... over the batch's life, never reused).
  int add_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob, int* id);
  int add_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid, int* id);
  /// A landmark map for LandmarkSensorModel2d (lp) or, with lp null, BearingSensorModel2d (bp), prepared and checked as
  /// Filter::set_landmark_map prepares it: set_* for every member, add_* without assigning it.
  int set_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map);
  int add_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map, int* id);
  /// Replaces the staged detections of every member whose present[m] is non-zero (present == nullptr: every occupied
  /// slot) with detections[m][0, n[m]): a host copy, no device call.  A BB200_MEASUREMENT_LANDMARKS member weighs its
  /// staged detections in every step until they are replaced; remove_member drops them.
  int set_detections(const bb200_landmark_detection* const* detections, const uint64_t* n, const uint8_t* present);
  /// Amcl::update_map for one member: its particles and policies stay; its later steps read map `id`.
  int update_map(int member, int id);
  int member_map(int member, int* id) const;
  /// Frees map `id` (BB200_ERR_STATE while a member reads it).
  int remove_map(int id);
  int get_likelihood_field(int id, float* out, uint64_t capacity) const;
  int initialize(int member, const double mean[3], const double cov[9]);
  int initialize_from_map(int member);
  int initialize_states(int member, const double* states, const double* weights, uint64_t n);
  int force_update(int member);
  int get_particles(int member, double* states, double* weights, uint64_t capacity);
  /// Member m's current particle count.
  int member_size(int member, uint64_t* n) const;
  int ancestors(int member, int64_t* out, uint64_t capacity);
  /// The cluster estimate of one member: cluster_estimates with that member alone selected.
  int cluster_estimate(int member, const bb200_cluster_param& p, bb200_estimate* out);
  /// beluga::cluster_based_estimate of every member whose present[m] is non-zero (present == nullptr: all of them): two
  /// kernel launches and two host synchronisations whatever K and the cell counts are.  out[m], n_cells[m] and
  /// n_clusters[m] (either may be nullptr) are written for selected members only.
  int cluster_estimates(const bb200_cluster_param& p, const uint8_t* present, bb200_estimate* out, uint32_t* n_cells, uint32_t* n_clusters);
  /// Filter::particle_histogram of every selected member: the device half of cluster_estimates with these resolutions (two
  /// launches, two synchronisations).  n_bins[m] and max_bin_weight[m] (either may be nullptr) are written for selected
  /// members; bins[m] (bins or bins[m] nullptr: counts only) receives member m's bins when capacity[m] holds them, and
  /// BB200_ERR_CAPACITY is returned when some selected member's buffer does not.
  int particle_histograms(double linear, double angular, const uint8_t* present, bb200_cluster_cell* const* bins, const uint64_t* capacity,
                          uint64_t* n_bins, double* max_bin_weight);
  /// Filter::sample_states(counts[m], step, states_out[m]) for every selected member with counts[m] > 0, one launch when
  /// every such member's CDF is current and four when some CDF has to be rebuilt, and one host synchronisation.  No particle
  /// set changes.
  int sample_states(const uint64_t* counts, uint32_t step, const uint8_t* present, double* const* states_out);
  /// Filter::cast_rays for every selected member on its own map, or on map map_ids[m] when map_ids is set and the entry is
  /// not -1: n_poses[m] x n_bearings[m] rays from poses[m] along bearings[m] up to max_range[m] into ranges[m].  One launch
  /// (none without rays) and one host synchronisation, whatever K and the maps are.  Every check is made before anything
  /// reaches the device, and no member changes.
  int cast_rays(const uint8_t* present, const int* map_ids, const double* const* poses, const uint64_t* n_poses, const double* const* bearings,
                const uint64_t* n_bearings, const double* max_range, double* const* ranges);
  /// Amcl::update for every member whose present[m] is non-zero (present == nullptr: all of them).  Atomic for the whole
  /// batch: when the device half fails, every member's host state is rolled back.
  int update(const double* control_poses, const double* const* points_xy, const uint64_t* n_points, const uint8_t* present,
             bb200_update_result* out);
  /// update with each member's measurement as base-frame points, a laser scan or a point cloud
  /// (bb200_amcl_batch_update_measurements): every present member's measurement is checked first, and scans and clouds
  /// are converted on the device by one more launch.
  int update_measurements(const double* control_poses, const bb200_measurement* measurements, const uint8_t* present, bb200_update_result* out);
  /// update_measurements, then the cluster estimate of every member that updated, byte-identical to cluster_estimates
  /// over those members right after it (bb200_amcl_batch_update_clustered): three more launches after the step
  /// (batch_cluster_table, batch_cluster_cells, batch_cluster_select) and the step's one synchronisation, plus one launch
  /// and one synchronisation when some member falls back to the host pass.  clustered[m], n_cells[m] and n_clusters[m]
  /// (either may be nullptr) are written for the members with out[m].updated.
  int update_clustered(const double* control_poses, const bb200_measurement* measurements, const uint8_t* present, const bb200_cluster_param& p,
                       bb200_update_result* out, bb200_estimate* clustered, uint32_t* n_cells, uint32_t* n_clusters);

  /// The first half of update_measurements / update_clustered for a step in which some members are weighed by the caller
  /// (kind BB200_MEASUREMENT_WEIGHTS; bb200_amcl_batch_update_begin): the policies' decisions, the conversion of scans
  /// and clouds, the propagate and the built-in reweight of the other members are enqueued, and views[m] gives member m's
  /// propagated states and its slice of the factor buffer.  Nothing is synchronised; the step stays open until update_end.
  int update_begin(const double* control_poses, const bb200_measurement* measurements, const uint8_t* present, bb200_weigh_view* views);
  /// The second half: w *= factor for the weighed members, then the rest of the step and, with `cluster`, the cluster
  /// estimates as update_clustered computes them; the step's one synchronisation.  Atomic as update.
  int update_end(const bb200_cluster_param* cluster, bb200_update_result* out, bb200_estimate* clustered, uint32_t* n_cells, uint32_t* n_clusters);
  /// Whether a step is open (update_begin .. update_end): the C ABI then refuses every other call but destroy.
  bool step_open() const { return open_.open; }

 private:
  /// Where update_clustered's step writes the cluster estimates.
  struct ClusteredOut {
    const bb200_cluster_param* p;
    bb200_estimate* estimates;
    uint32_t* n_cells;
    uint32_t* n_clusters;
  };
  struct Member {
    AmclPolicy policy;     // in a vacant slot, its last occupant's (never read)
    bool active{true};     // false: a vacant slot
    uint64_t offset{0};    // first particle in the batch buffers
    uint64_t capacity{0};  // max_particles
    uint64_t n{0};
    int cur{0};            // state buffer holding the particles
    double pivot[2]{0.0, 0.0};
    uint64_t ancestors_n{0};
    uint64_t table_offset{0};  // its hash table in the cluster scratch
    uint32_t table_slots{0};   // a power of two >= 2 * capacity
    int map{-1};               // id of the map it reads (-1: none)
    // Total of the CDF in its cdf_ slice while that CDF is the one a standalone filter would sample from (Filter's
    // cdf_valid_): set by a step that kept the particles (normalised, or selective with a high effective sample size)
    // and by a rebuild in sample_states; 0 (stale) after a resampling step, an initialisation or a failed step.
    unsigned long long cdf_total{0};
    // The beam directions of the last scan it passed (update_measurements), kept until the scan geometry changes: the
    // key, the kept readings' indices and their (cos, sin) on the device.
    struct ScanTable {
      bool valid{false};
      uint64_t n_ranges{0}, max_beams{0};
      uint32_t angle_min_bits{0}, angle_increment_bits{0};
      std::vector<uint64_t> indices;
      DeviceBuffer<double2> directions;
    };
    ScanTable scan;
    // The detections a BB200_MEASUREMENT_LANDMARKS step weighs (set_detections), as given: their category slices are
    // resolved against the member's map at step time.
    std::vector<bb200_landmark_detection> detections;
    bool detections_staged{false};
  };
  struct MapEntry {
    DeviceMap map;
    int slot{0};  // its entry in the device map table
  };
  /// Where the occupied slots' data lie in the batch buffers, and the sizes of the buffers that hold it.
  struct Layout {
    std::vector<uint64_t> offset, table_offset;  // per slot (vacant: 0)
    std::vector<uint32_t> table_slots;
    uint64_t total{0}, table_total{0}, tiles{0}, rows{0};
    bool record_ancestors{false};
  };
  /// The buffers a layout and the slot count size: the particle slices, the step's scan tiles, finish rows, per-member
  /// scalars and tables.
  struct Storage {
    DeviceBuffer<Pose2> states[2];
    DeviceBuffer<double> weights;
    DeviceBuffer<unsigned long long> cdf;
    DeviceBuffer<long long> ancestors;
    DeviceBuffer<Scalars> scalars;
    DeviceBuffer<unsigned long long> tile_state;
    DeviceBuffer<double> partials;
    MirroredBuffer<BatchMember> table;
    MirroredBuffer<uint32_t> first;
    PinnedBuffer<StepSummary> summary_host;
  };
  /// The layout of the slots' params (nullptr: vacant): particle slices 32-aligned in slot order, hash tables back to back,
  /// and the tiles and rows of every occupied slot.  The one rule of the constructor and of every membership change.
  static Layout lay_out(const std::vector<const bb200_amcl_param*>& slots);
  /// The checks validate makes on member k (a member of a batch on `device` with `flags`).
  static int validate_member(const bb200_amcl_param& p, const bb200_motion_param& motion, int k, int device, uint32_t flags, std::string* error);
  int allocate(const Layout& layout, size_t slots, Storage* s);
  void adopt(Storage&& s);
  /// Assigns every occupied member its place in `layout`.
  void place(const Layout& layout);
  /// The device half of a membership change to `slots`: new buffers, every surviving member's live data moved into them
  /// (batch_relayout_kernel), the old buffers freed and the scratch sized by the old layout dropped.  A survivor is a slot
  /// occupied now and in `slots`.  On failure the batch is unchanged.
  /// `arrival` (nullable): a member joining in slot arrival->slot with the arrays of a decoded state, moved into the new
  /// buffers before they are adopted (unpack).
  struct Arrival {
    size_t slot;
    const FilterState* state;
  };
  int relayout(const std::vector<const bb200_amcl_param*>& slots, Layout* layout, const Arrival* arrival = nullptr);
  /// add_member, or with `state` import_member: a member with these params in the lowest vacant slot or a new one after
  /// the last, validated, then given its place by a relayout (with `state`'s arrays and reading map `map`).
  int join(const bb200_amcl_param& params, const bb200_motion_param& motion, const FilterState* state, int map, int* member);
  /// The scalars of member m's state blob.
  static ParticleSetState particle_set(const Member& m);
  /// Member m as the member a decoded state describes: its policy, count, pivot, CDF total and ancestors count (its
  /// particles go to state buffer 0).
  static void adopt_state(Member& m, const FilterState& s);
  /// The arrays of states[j] into the staging buffer (host), one copy to the device, then one batch_relayout_kernel launch
  /// into the buffers `*_to` at offsets to[j] (none when no state holds arrays).  Nothing is synchronised.
  int unpack(const std::vector<const FilterState*>& states, const std::vector<uint64_t>& to, Pose2* states_to, double* weights_to,
             unsigned long long* cdf_to, long long* ancestors_to);
  /// One batch_relayout_kernel launch over `moves` (non-empty) with the ends in `a`; its table goes through the transfer scratch.
  int launch_moves(const std::vector<BatchRelayoutMember>& moves, BatchRelayoutArgs a);
  /// BB200_ERR_INVALID_ARGUMENT when present (nullptr: every occupied slot) selects a vacant slot.
  int check_present(const uint8_t* present);
  /// check_present, then every selected member's measurement as the single filter checks it (BB200_ERR_INVALID_ARGUMENT);
  /// with `weighed_by_caller`, BB200_MEASUREMENT_WEIGHTS members are taken as they are.
  int check_measurements(const bb200_measurement* in, const uint8_t* present, bool weighed_by_caller);
  bool selected_member(const uint8_t* present, size_t k) const { return members_[k].active && (present == nullptr || present[k] != 0); }
  int fail(int status, const std::string& message) {
    error_ = message;
    return status;
  }
  int check(cudaError_t e, const char* what) { return cuda_check(e, what, &error_); }
  int member_ok(int member) const;
  const MapEntry* find_map(int id) const;
  int ensure_scan_table(Member& m, const bb200_laser_scan& scan);
  /// The step of update and update_measurements: in[m] is member m's measurement, already checked when it is a scan or a cloud.
  /// With `clustered`, the step also selects every updated member's cluster estimate on the device (update_clustered).
  int step(const double* control_poses, const bb200_measurement* in, const uint8_t* present, bb200_update_result* out,
           const ClusteredOut* clustered = nullptr);
  /// The halves of step: plans, uploads and launch_batch_step_head (views: written for update_begin), then the tail
  /// launches, the synchronisation and the commit.  Between the two the step is open_.
  int step_begin(const double* control_poses, const bb200_measurement* in, const uint8_t* present, bb200_weigh_view* views);
  int step_end(const ClusteredOut* clustered, bb200_update_result* out);
  /// A step between step_begin and step_end: the policies to put back on failure, the plans, the updating members and
  /// the launch arguments.
  struct OpenStep {
    bool open{false};
    std::vector<AmclPolicy> before;
    std::vector<bb200_step_plan> plans;
    std::vector<uint32_t> active;
    bool kld{false};
    BatchStepArgs args{};
  };
  OpenStep open_;
  DeviceBuffer<double> factors_;  // weighed members' factors, laid out like weights_ (grown by the first such step)
  bool ensure_hits(uint64_t words);
  int set_map(const MapTables& tables);
  int add_map(const MapTables& tables, int* id);
  int ensure_map_table();
  int ensure_cluster_scratch();
  /// The cluster scratch, whose hashes and tables a KLD count reuses, and the step's KLD parameter table.
  int ensure_kld_scratch();
  int ensure_cluster_records(uint64_t cells);
  /// The cluster scratch and the selection's: rehash schedules, per-member scratch, tables and results.
  int ensure_select_scratch();
  /// The members whose present[m] is non-zero (present == nullptr: all of them), in member order; BB200_ERR_STATE when one
  /// of them has no particles.
  int select_members(const uint8_t* present, std::vector<uint32_t>* selected);
  /// Clusterizer::cell_records of every member in `selected` (non-empty): their records back to back in cl_records_host_,
  /// member selected[j]'s count in cl_.cells.host[j].  Two launches and two host synchronisations.
  int cell_records(double linear, double angular, const std::vector<uint32_t>& selected);
  /// Member k's row of the cluster table: its slice, hash table, count, state buffer and pivot as they are now.
  BatchClusterMember cluster_member(uint32_t k) const;
  /// The arguments of batch_cluster_cells over the cluster table at these resolutions.
  BatchClusterArgs cluster_args(double linear, double angular) const;

  std::vector<Member> members_;  // by slot
  uint32_t flags_{0};
  int device_{0};
  cudaStream_t stream_{nullptr};
  std::map<int, MapEntry> maps_;  // by id
  int next_map_id_{0};
  DeviceBuffer<BatchMap> map_table_;  // one entry per map (MapEntry::slot), for steps whose members read several maps
  bool map_table_current_{false};     // the table and the slots match maps_
  bool created_{false};
  int create_status_{BB200_OK};
  mutable std::string error_;
  bool record_ancestors_{false};

  uint64_t total_{0};
  DeviceBuffer<Pose2> states_[2];
  DeviceBuffer<double> weights_;
  DeviceBuffer<unsigned long long> cdf_;
  DeviceBuffer<long long> ancestors_;
  DeviceBuffer<Scalars> scalars_;
  DeviceBuffer<unsigned long long> tile_state_;
  DeviceBuffer<double> partials_;
  MirroredBuffer<BatchMember> table_;
  // kBatchRows x (K + 1): the step's rows, then those of batch_points_kernel, batch_kld_kernel, batch_resampled_moments_kernel
  // and batch_ess_kernel
  MirroredBuffer<uint32_t> first_;
  MirroredBuffer<double> points_;   // (x, y) pairs
  MirroredBuffer<LandmarkDetection> detections_;  // the step's prepared detections, every kBatchLandmark member's in member order
  // Scans and clouds of update_measurements (the table allocated on first use): batch_points_kernel's member table and
  // the raw measurements (kept ranges, or x, y, z per cloud point).
  MirroredBuffer<BatchPointsMember> inputs_;
  MirroredBuffer<float> input_;
  DeviceBuffer<uint32_t> hits_;   // beam model, two-pass form: the step's hit words (grows only)
  PinnedBuffer<StepSummary> summary_host_;  // one per member of the step's table
  PinnedBuffer<int> ticket_host_;
  DeviceBuffer<unsigned int> members_done_;
  int seq_{0};
  uint64_t launches_{0};

  // Cluster estimate scratch (allocated on first use): per-member slices of the particle-sized buffers, and the hash
  // tables back to back.
  uint64_t table_total_{0};
  struct ClusterBuffers {
    DeviceBuffer<unsigned long long> hashes;
    DeviceBuffer<unsigned long long> keys;
    DeviceBuffer<unsigned int> first;
    DeviceBuffer<uint32_t> ids;
    DeviceBuffer<uint32_t> cell_of;
    DeviceBuffer<uint32_t> sort[2];
    DeviceBuffer<uint32_t> starts;
    DeviceBuffer<CellRecord> records;
    MirroredBuffer<BatchClusterMember> table;
    MirroredBuffer<uint32_t> cells;
  };
  ClusterBuffers cl_;
  PinnedBuffer<CellRecord> cl_records_host_;  // written by the compaction kernel
  // KLD parameters of a step's members (allocated on first use, one entry per member of the step's table).  The count
  // itself runs in the cluster scratch: per-slot hashes in cl_.hashes, bucket sets in cl_.keys and cl_.first.
  MirroredBuffer<BatchKldMember> kld_;
  // The device selection of update_clustered (allocated on first use): the probed rehash schedules, one scratch slice per
  // member (select_scratch_bytes of its max_particles, at offsets[k]), the post-step table inputs and the results.
  struct SelectBuffers {
    DeviceBuffer<uint32_t> schedule_start;
    DeviceBuffer<RehashStep> schedule;
    DeviceBuffer<unsigned char> scratch;
    std::vector<uint64_t> offsets;
    MirroredBuffer<BatchClusterPost> post;
    PinnedBuffer<BatchClusterResult> results;
  };
  SelectBuffers sel_;

  // Pose-sample scratch: the member table (allocated on first use), and the draws after a header of one CDF total per
  // member, so that one copy brings both back.
  MirroredBuffer<BatchSampleMember> sm_table_;
  // Moves and state blob transfers (grown on use): the move table and CTA prefix of every batch_relayout_kernel launch
  // (one entry per moved member), and the staging buffer that holds a transfer's members' arrays (StageLayout, batch.cu).
  struct TransferBuffers {
    DeviceBuffer<BatchRelayoutMember> table;
    DeviceBuffer<uint32_t> first;
    MirroredBuffer<unsigned char> stage;
  };
  TransferBuffers xfer_;
  MirroredBuffer<Pose2> samples_;
  // Ray-cast scratch (grown on use): the member table, and every casting member's poses, then bearings, then ranges.
  struct RayBuffers {
    MirroredBuffer<BatchRayMember> table;
    MirroredBuffer<double> data;
  };
  RayBuffers rays_;
};

}  // namespace bb200
