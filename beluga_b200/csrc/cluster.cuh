// Device side of the cluster-based estimate (reference: beluga/algorithm/cluster_based_estimation.hpp).
//
// The reference groups the particles into spatial-hash cells (make_cluster_map, :141-161), then
// runs a priority-queue flood over the cells (assign_clusters, :205-253) and finally estimates
// mean/covariance per cluster (estimate_clusters, :351-398).  Everything per PARTICLE runs here on
// the device and produces one CellRecord per occupied cell; the per-CELL flood (sequential, order
// dependent, a few thousand cells) runs on the host (cluster_host.hpp).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "cluster_host.hpp"
#include "cluster_select.cuh"
#include "device_buffer.hpp"
#include "kernels.cuh"

namespace bb200 {

/// What the host pass needs to know about one occupied cell; cells are numbered in the order in
/// which the particle sequence first touches them (the insertion order of the reference's map).
struct CellRecord {
  Pose2 representative;         // state of the first particle that fell into the cell (ClusterCell::representative_state)
  unsigned long long hash;      // spatial hash of the cell
  unsigned int first_index;     // index of that first particle
  unsigned int count;           // ClusterCell::num_particles
  double weight;                // sum of the particle weights in particle order (ClusterCell::weight before normalisation)
  double moments[kMomentCount]; // raw moments of the cell's particles about the pivot (layout of kMomentCount)
};
static_assert(sizeof(CellRecord) == 128, "CellRecord is copied to the host as raw bytes");

/// Scratch buffers of the clusterizer (owned by Clusterizer, sized for its `capacity` particles).
struct ClusterScratch {
  DeviceBuffer<unsigned long long> hashes;  // [capacity]
  DeviceBuffer<unsigned long long> keys;    // [table size]: a power of two >= 2 * capacity
  DeviceBuffer<unsigned int> first;         // [table size] smallest particle index per key
  DeviceBuffer<uint32_t> slot_of;           // [capacity] table slot of each particle's cell
  DeviceBuffer<uint32_t> flags;             // [capacity] first-occurrence flags, scanned in place
  DeviceBuffer<uint32_t> cell_of;           // [capacity] dense cell id per particle
  DeviceBuffer<uint32_t> starts;            // [capacity + 1] cell counts, scanned in place into segment starts
  DeviceBuffer<uint32_t> keys_a, keys_b;    // radix sort ping-pong: keys and particle indices
  DeviceBuffer<uint32_t> idx_a, idx_b;
  DeviceBuffer<uint32_t> histogram;         // [256 * sort tiles]
  DeviceBuffer<unsigned long long> tile_state;
  DeviceBuffer<unsigned long long> words;   // [4]: scan ticket, cell count, spare
  DeviceBuffer<CellRecord> records;         // grows with the cell count
};

uint32_t cluster_sort_tiles(uint64_t n);

/// hashes -> hash set (key -> smallest particle index) -> first-occurrence flags -> dense cell ids
/// base; leaves the number of occupied cells in scratch.words[1].
void launch_cluster_cells_begin(const Pose2* states, uint64_t n, double linear_resolution, double angular_resolution, const ClusterScratch& s,
                                cudaStream_t stream);

/// Cell id per particle, cell sizes and the stable sort of the particle indices by cell (particle order
/// preserved inside a cell).  `cells` = value read back from words[1].  Returns the buffer holding the
/// sorted particle indices and the number of kernels launched.
const uint32_t* launch_cluster_sort(uint64_t n, uint32_t cells, const ClusterScratch& s, cudaStream_t stream, int* launches);
/// One CellRecord per cell from the sorted indices.
void launch_cluster_records(const Pose2* states, const double* weights, const uint32_t* sorted_idx, uint32_t cells, double pivot_x, double pivot_y,
                            const ClusterScratch& s, cudaStream_t stream);

// ---- every selected member of a batch at once ------------------------------------------------------------------------

/// Largest member a batch cluster estimate handles: a member's particle index then fits in 15 bits.
constexpr uint32_t kBatchClusterMaxParticles = 32768;

/// One selected member of a batch cluster estimate.  Its scratch is its own slice of each buffer.
struct BatchClusterMember {
  uint64_t offset;         // first particle in the batch buffers; also its record slice (cells <= particles)
  uint64_t table_offset;   // first slot of its hash table
  uint64_t starts_offset;  // first of its cells + 1 segment starts
  uint32_t n;              // particles (> 0)
  uint32_t table_mask;     // table slots - 1 (a power of two minus one)
  uint32_t cur;            // state buffer holding the particles
  uint32_t pad;
  double pivot_x, pivot_y; // the member's moment pivot
};

struct BatchClusterArgs {
  const BatchClusterMember* members;  // one per CTA
  const Pose2* states[2];
  const double* weights;
  double linear, angular;             // spatial-hash resolutions
  unsigned long long* hashes;         // [particles]
  unsigned long long* keys;           // [table slots]
  unsigned int* first;                // [table slots] smallest particle index per key
  uint32_t* ids;                      // [table slots] cell id of the key's cell
  uint32_t* cell_of;                  // [particles]
  uint32_t* sort_a;                   // [particles] sort ping-pong
  uint32_t* sort_b;
  uint32_t* starts;                   // [particles + members]
  CellRecord* records;                // [particles] member slices
  uint32_t* cells;                    // [selected members] occupied cells
};

/// One CTA per selected member: hash set, first-occurrence numbering, stable sort by cell and one CellRecord per cell,
/// written to the member's record slice; cells[j] receives member j's cell count.  One launch.
void launch_batch_cluster_cells(const BatchClusterArgs& a, uint32_t n_members, cudaStream_t stream);
/// Member j's cells[j] records to out[cells[0] + ... + cells[j - 1]]: the records of all members back to back.  One launch.
void launch_batch_cluster_compact(const BatchClusterMember* members, const uint32_t* cells, const CellRecord* records, uint32_t n_members,
                                  CellRecord* out, cudaStream_t stream);

// ---- the cluster estimate of every member that a batch step updated, selected on the device -----------------------
// After the step: batch_cluster_table_kernel turns the pre-step member table into the post-step one (state buffer, count
// and pivot, from the step's summaries), batch_cluster_cells_kernel runs on it, and batch_cluster_select_kernel restates
// select_cluster per member (cluster_select.cuh), one CTA each.

static_assert(kBatchClusterMaxParticles == kSelectMaxCells, "the rehash schedules cover every count a batch member can reach");

/// What the table kernel needs besides the pre-step BatchClusterMember: how the step may have changed the member.
struct BatchClusterPost {
  uint64_t scratch_offset;  // bytes: the member's selection scratch when it does not fit in shared memory
  uint32_t capacity;        // max_particles: the count after a fixed-size resample
  int mode;                 // 0: kept its particles, 1: resampled, 2: the step decides (StepSummary::resampled)
  int kld;                  // 1: a resample keeps StepSummary::accepted particles
  int pad;
};

/// One member's selection, written to pinned memory.  fallback: the device cannot promise the host's bits (a NaN cell
/// weight, or a neighbour heading at an angular bucket edge); the host then runs select_cluster on the member's records.
struct BatchClusterResult {
  uint32_t found;
  uint32_t clusters;
  uint32_t cells;
  uint32_t fallback;
  double moments[kMomentCount];  // of the heaviest cluster, or of every cell
};

struct BatchSelectArgs {
  BatchClusterMember* members;        // pre-step table in, post-step table out (table kernel); one per CTA
  const BatchClusterPost* post;
  const StepSummary* summary;         // the step's, one per member of its table (pinned)
  uint32_t n_members;
  const CellRecord* records;          // the member slices batch_cluster_cells_kernel wrote
  const uint32_t* cells;              // their cell counts
  const unsigned long long* keys;     // their bucket sets: key -> cell id
  const uint32_t* ids;
  const uint32_t* schedule_start;     // RehashTable::start, by n / 5
  const RehashStep* schedule;         // RehashTable::steps
  unsigned char* scratch;             // BatchClusterPost::scratch_offset
  double linear, angular, percentile;
  Pose2 adjacent[6];                  // ParticleClusterizer::adjacent_grid_cells_, rot_exp on the host
  BatchClusterResult* results;        // one per member (pinned)
};

/// One launch each.
void launch_batch_cluster_table(const BatchSelectArgs& a, cudaStream_t stream);
void launch_batch_cluster_select(const BatchSelectArgs& a, cudaStream_t stream);

/// The clusterizer of a filter: scratch for up to `capacity` particles on one device, allocated on first use,
/// run over any particle set of that size in that device's memory.  Every call works on the current device, ordered on
/// `stream`, and returns a bb200_status with the message in *error.
class Clusterizer {
 public:
  explicit Clusterizer(uint64_t capacity) : capacity_(capacity) {}
  Clusterizer(const Clusterizer&) = delete;
  Clusterizer& operator=(const Clusterizer&) = delete;

  /// Per-particle half of the clusterizer, also the device-side histogram of the particle cloud: one record per occupied
  /// cell in first-occurrence order, raw moments about `pivot`, copied to *host.
  int cell_records(const Pose2* states, const double* weights, uint64_t n, const double pivot[2], double linear_resolution, double angular_resolution,
                   cudaStream_t stream, std::vector<HostCell>* host, std::string* error);
  /// beluga::cluster_based_estimate (algorithm/cluster_based_estimation.hpp:415-432) of the n particles, the moments taken
  /// about `pivot`; cluster_ids (optional, one per particle) is the parity hook for ParticleClusterizer::operator() (:304-316).
  int estimate(const Pose2* states, const double* weights, uint64_t n, const double pivot[2], const bb200_cluster_param& p, cudaStream_t stream,
               bb200_estimate* out, uint32_t* cluster_ids, uint64_t ids_capacity, uint32_t* n_cells, uint32_t* n_clusters, std::string* error);
  uint64_t launches() const { return launches_; }

  /// Called with each stage's timing label before its launches and with "end" after the last copy (a filter's timing marks).
  std::function<void(const char*)> mark;

 private:
  int ensure_scratch(uint32_t cells, std::string* error);

  uint64_t capacity_;
  ClusterScratch s_;  // allocated (all but the records) once `hashes` is set
  uint64_t launches_{0};
};

}  // namespace bb200
