// ---- batches of filters ----------------------------------------------------------------------------------
// Each kernel below runs, per CTA, the block body of the single-filter kernel it stands for, on the CTA's member.
#include "bucket_set.cuh"
#include "cdf.cuh"
#include "kld.cuh"
#include "raycast.cuh"
#include "resample.cuh"
#include "reweight_beam.cuh"
#include "reweight_landmark_block.cuh"
#include "reweight_lfm.cuh"

#include <algorithm>

namespace bb200 {

namespace {

/// The member owning CTA `cta` of `launch` (the last one whose range starts at or before it: members without CTAs in this
/// launch have empty ranges), the CTA's index inside that range and the range's length.
template <class Args>
__device__ __forceinline__ uint32_t batch_member_of(const Args& s, int launch, uint32_t cta, uint32_t& local, uint32_t& count) {
  const uint32_t* first = s.first + static_cast<size_t>(launch) * (s.n_members + 1);
  uint32_t lo = 0, hi = s.n_members;  // first[lo] <= cta < first[hi]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(first + mid) <= cta) {
      lo = mid;
    } else {
      hi = mid;
    }
  }
  const uint32_t begin = __ldg(first + lo);
  local = cta - begin;
  count = __ldg(first + lo + 1) - begin;
  return lo;
}

/// A member's current (which = 0) or staging (which = 1) state buffer; a select, not an indexed load from the parameters.
__device__ __forceinline__ Pose2* batch_states(const BatchStepArgs& s, const BatchMember& m, int which) {
  return ((m.cur ^ which) != 0 ? s.states[1] : s.states[0]) + m.offset;
}

// Where a member's map views come from: the parameter block when every member of the step reads one map (kTable false:
// the views stay in the constant bank, as in the single-filter kernels), the batch's map table otherwise.
template <bool kTable>
__device__ __forceinline__ const FieldView& batch_field(const BatchStepArgs& s, const BatchMember& m) {
  if constexpr (kTable) return s.maps[m.map].field;
  else return s.field;
}
template <bool kTable>
__device__ __forceinline__ const OccupancyView& batch_occupancy(const BatchStepArgs& s, const BatchMember& m) {
  if constexpr (kTable) return s.maps[m.map].occupancy;
  else return s.occupancy;
}
template <bool kTable>
__device__ __forceinline__ const BeamParams& batch_beam(const BatchStepArgs& s, const BatchMember& m) {
  if constexpr (kTable) return s.maps[m.map].beam;
  else return s.beam;
}
/// Recovery injection's free cells and grid geometry.
template <bool kTable>
__device__ __forceinline__ void batch_recovery_map(const BatchStepArgs& s, const BatchMember& m, ResampleArgs& a) {
  if constexpr (kTable) {
    const BatchMap& map = s.maps[m.map];
    a.free_cells = map.free_cells;
    a.n_free = map.n_free;
    a.grid_width = map.grid_width;
    a.grid_resolution = map.grid_resolution;
    a.grid_origin = map.grid_origin;
  } else {
    a.free_cells = s.free_cells;
    a.n_free = s.n_free;
    a.grid_width = s.grid_width;
    a.grid_resolution = s.grid_resolution;
    a.grid_origin = s.grid_origin;
  }
}

/// A member's landmark model constants, landmarks and box (landmark.model 0: a grid map).
template <bool kTable>
__device__ __forceinline__ const LandmarkParams& batch_landmark(const BatchStepArgs& s, const BatchMember& m) {
  if constexpr (kTable) return s.maps[m.map].landmark;
  else return s.landmark;
}
template <bool kTable>
__device__ __forceinline__ const LandmarkPoint* batch_landmarks(const BatchStepArgs& s, const BatchMember& m) {
  if constexpr (kTable) return s.maps[m.map].landmarks;
  else return s.landmarks;
}
template <bool kTable>
__device__ __forceinline__ BoxSpace batch_box(const BatchStepArgs& s, const BatchMember& m) {
  const double* b = kTable ? s.maps[m.map].box : s.box;
  return BoxSpace{b[0], b[1], b[2], b[3]};
}

/// The per-step scalars of every member (what begin_fused_step_kernel resets for one filter) and the scan state.
template <class Args>
__device__ __forceinline__ void batch_reset_grid(const Args& s, uint32_t scan_tiles) {
  const uint32_t stride = gridDim.x * 256;
  for (uint32_t t = blockIdx.x * 256 + threadIdx.x; t < s.n_members; t += stride) {
    Scalars* sc = s.scalars + t;
    sc->wmax_bits = 0;
    sc->tile_ticket = 0;
    sc->total = 0;
    sc->exponent = 0;
    sc->valid = 0;
    sc->blocks_done = 0;
  }
  for (uint32_t t = blockIdx.x * 256 + threadIdx.x; t < scan_tiles; t += stride) s.tile_state[t] = 0;
}

__global__ void __launch_bounds__(256) batch_begin_kernel(BatchStepArgs s) { batch_reset_grid(s, s.ctas[kBatchScan]); }

/// propagate_kernel's per-particle body (counter RNG keyed by the member's seed, local index and step).
__global__ void __launch_bounds__(kPrThreads) batch_propagate_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const BatchMember& m = s.members[batch_member_of(s, kBatchPropagate, blockIdx.x, local, count)];
  const uint64_t i = static_cast<uint64_t>(local) * kPrThreads + threadIdx.x;
  if (i < m.n) {
    Pose2* states = batch_states(s, m, 0);
    store_pose(states + i, propagate_one(load_pose(states + i), m.sampling, m.seed, i, m.step));
  }
}

/// One CTA of reweight_lfm_fixed_kernel (or, for maps beyond kFixedMaxSide, reweight_lfm_kernel) per 256 particles of a
/// member; each member's scan is staged into shared memory in kChunkBeams-point chunks.  The kernel is chosen per member
/// (by its map), so it is uniform within a CTA.
template <bool kTable>
__global__ void __launch_bounds__(kRwThreads, kRwBlocksPerSm) batch_reweight_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchReweight, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  const Pose2* states = batch_states(s, m, 0);
  const double2* points = reinterpret_cast<const double2*>(s.points) + m.point_offset;
  const uint64_t slot_base = static_cast<uint64_t>(local) * kRwThreads;
  const FieldView& field = batch_field<kTable>(s, m);
  if (field.use_fixed) {
    reweight_lfm_fixed_block(states, s.weights + m.offset, m.n, nullptr, field, points, m.n_points, m.points_radius, s.scalars + k, slot_base);
  } else {
    reweight_lfm_block(states, s.weights + m.offset, m.n, nullptr, field, points, m.n_points, m.points_radius, s.scalars + k, slot_base);
  }
}

// batch_member_ctas sizes every reweight row (kBatchReweight, kBatchReweightWalk, kBatchReweightBeam) with kRwThreads: one
// CTA per 256 particles in every reweight form.
static_assert(kWalkThreads == kRwThreads && kMixThreads == kRwThreads && kBeamThreads == kRwThreads,
              "batch_member_ctas sizes every reweight row of a batch step with kRwThreads");

/// beam_walk_kernel per member: the whole member in one pass, its hit words beam-major at hits + hit_offset.
template <bool kTable>
__global__ void __launch_bounds__(kWalkThreads, kWalkBlocksPerSm) batch_beam_walk_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const BatchMember& m = s.members[batch_member_of(s, kBatchReweightWalk, blockIdx.x, local, count)];
  const double2* points = reinterpret_cast<const double2*>(s.points) + m.point_offset;
  beam_walk_block(batch_states(s, m, 0), m.n, 0, m.n, nullptr, batch_occupancy<kTable>(s, m), batch_beam<kTable>(s, m).beam_max_range, points,
                  m.n_points, s.hits + m.hit_offset, m.hit_stride, local);
}

/// beam_mixture_kernel per member over the words batch_beam_walk_kernel wrote; the largest weight into the member's scalars.
template <bool kTable>
__global__ void __launch_bounds__(kMixThreads) batch_beam_mixture_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchReweightWalk, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  const double2* points = reinterpret_cast<const double2*>(s.points) + m.point_offset;
  beam_mixture_block(batch_states(s, m, 0), s.weights + m.offset, m.n, 0, m.n, nullptr, batch_occupancy<kTable>(s, m), batch_beam<kTable>(s, m),
                     points, m.n_points, s.hits + m.hit_offset, m.hit_stride, s.scalars + k, local);
}

/// reweight_beam_kernel per member (maps the walk cannot take, or a step whose hit words would not fit).
template <bool kTable>
__global__ void __launch_bounds__(kBeamThreads, kBeamBlocksPerSm) batch_reweight_beam_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchReweightBeam, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  const double2* points = reinterpret_cast<const double2*>(s.points) + m.point_offset;
  reweight_beam_block(batch_states(s, m, 0), s.weights + m.offset, m.n, nullptr, batch_occupancy<kTable>(s, m), batch_beam<kTable>(s, m), points,
                      m.n_points, s.scalars + k, local);
}

/// reweight_landmark_kernel per kBatchLandmark member: its detections at detections + point_offset.  The model is the
/// member's map's, so it is uniform within a CTA.
template <bool kTable>
__global__ void __launch_bounds__(kLandmarkThreads) batch_reweight_landmark_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchLandmarkRow, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  const LandmarkParams& params = batch_landmark<kTable>(s, m);
  const LandmarkDetection* detections = s.detections + m.point_offset;
  if (params.model == BB200_SENSOR_BEARING) {
    reweight_landmark_block<BB200_SENSOR_BEARING>(batch_states(s, m, 0), s.weights + m.offset, m.n, params, batch_landmarks<kTable>(s, m), detections,
                                                  m.n_points, s.scalars + k, local);
  } else {
    reweight_landmark_block<BB200_SENSOR_LANDMARK>(batch_states(s, m, 0), s.weights + m.offset, m.n, params, batch_landmarks<kTable>(s, m), detections,
                                                   m.n_points, s.scalars + k, local);
  }
}

/// apply_factors_kernel per weighed member: w *= factor over the member's slice, the largest weight into its scalars.
__global__ void __launch_bounds__(kMaxThreads) batch_weigh_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchWeighRow, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  apply_factors_block(s.weights + m.offset, s.factors + m.offset, m.n, s.scalars + k, local, count);
}

/// quantize_scan_kernel per member: the exponent from the member's own largest weight, its own look-back state.
__global__ void __launch_bounds__(kQsThreads) batch_scan_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchScan, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  quantize_scan_tile(s.weights + m.offset, m.n, s.cdf + m.offset, s.scalars + k, s.tile_state + (blockIdx.x - local), local, 1,
                     m.ceil_log2_count);
}

/// The end of a member's step: its summary block, then -- from the last member to get there -- the step's ticket.
struct BatchTail {
  StepSummary* summary;
  unsigned int* members_done;
  uint32_t n_members;
  int* ticket;
  int seq;
  unsigned long long accepted;  // StepSummary::accepted
  int resampled;                // StepSummary::resampled
};
__device__ __forceinline__ bool tail_enabled(const BatchTail&) { return true; }
__device__ __forceinline__ void tail_publish(const BatchTail& tail, const double* v, Scalars* scalars) {
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) tail.summary->moments[k] = v[k];
  scalars->blocks_done = 0;
  tail.summary->accepted = tail.accepted;
  tail.summary->resampled = tail.resampled;
  tail.summary->total = scalars->total;
  tail.summary->exponent = scalars->exponent;
  tail.summary->valid = scalars->valid;
  tail.summary->error = 0;
  __threadfence_system();  // this member's summary before its arrival
  if (atomicAdd(tail.members_done, 1u) + 1u == tail.n_members) {
    __threadfence_system();  // every member's summary (each fenced before its arrival) before the ticket
    *tail.members_done = 0;
    *reinterpret_cast<volatile int*>(tail.ticket) = tail.seq;  // the host polls this word
    __threadfence_system();
  }
}

/// normalize_kernel's blocks (launch_normalize's partition, moments_block_count(n) blocks) for each member that runs the
/// effective-sample-size test; the last of a member's blocks to arrive sums their rows as reduce_partials_kernel does and
/// stores on_effective_size_drop's decision, ESS = 1 / sum w~^2 < n / 2, in scalars->ess_resample (a sum that is not
/// positive, NaN included, gives ESS 0: resample).  The same double arithmetic as Amcl::update_device on the host.
__global__ void __launch_bounds__(kStreamThreads) batch_ess_kernel(BatchStepArgs s) {
  __shared__ double s_red[kStreamThreads / kWarp];
  __shared__ int s_last;
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchEssRow, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  Scalars* scalars = s.scalars + k;
  double* rows = s.partials + (blockIdx.x - local);  // one sum of squares per CTA
  normalize_block(s.weights + m.offset, m.n, scalars, 0, rows, RangeBlocks{local, count});
  if (threadIdx.x == 0) {
    __threadfence();  // the row before the arrival count
    s_last = atomicAdd(&scalars->blocks_done, 1u) + 1u == count ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double v = 0.0;
  for (uint32_t r = threadIdx.x; r < count; r += kStreamThreads) v = v + __ldcg(rows + r);
  const double sum_sq = block_sum<kStreamThreads>(v, s_red);
  if (threadIdx.x == 0) {
    const double ess = sum_sq > 0.0 ? 1.0 / sum_sq : 0.0;
    scalars->ess_resample = ess < static_cast<double>(m.n) * 0.5 ? 1 : 0;
    scalars->blocks_done = 0;  // free for the arrivals of the finish launch
  }
}

/// A step that keeps its particles: normalize_kernel's w /= S (unless batch_ess_kernel has divided already) and
/// moments_kernel's rows over the same partition (moments_block_count blocks), the rows summed like
/// reduce_partials_kernel does.
__device__ __forceinline__ void normalize_moments_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, double px,
                                                        double py, Scalars* scalars, double* __restrict__ moment_partials, uint32_t block,
                                                        uint32_t grid, const BatchTail& tail, bool divide) {
  __shared__ double s_red[kMomentCount * kStreamThreads / kWarp];
  const double factor = scalbn(static_cast<double>(scalars->total), -scalars->exponent);
  const bool valid = divide && scalars->valid != 0 && factor > 0.0;
  double m[kMomentCount];
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) m[k] = 0.0;
  for (uint64_t i = static_cast<uint64_t>(block) * kStreamThreads + threadIdx.x; i < n; i += static_cast<uint64_t>(grid) * kStreamThreads) {
    double w = weights[i];
    if (valid) {
      w = w / factor;  // actions/normalize.hpp:82
      weights[i] = w;
    }
    accumulate_moments(m, load_pose(states + i), w, px, py);
  }
  finish_block_moments<kStreamThreads>(m, s_red, moment_partials, scalars, block, grid, tail);
}

/// Per member: resample_scatter_kernel or resample_kernel (recovery injection, multinomial draws) on a resampling step,
/// normalisation otherwise; then the member's moments, summed by its last CTA.  A member that resamples under KLD draws
/// every one of its max_particles slots with their spatial hashes, as Filter::resample_kld's one chunk does, and leaves
/// its summary to batch_resampled_moments_kernel.  A member that ran the effective-sample-size test follows its
/// decision: it draws and leaves its summary to that kernel too (Filter::resample, then Filter::estimate), or it sums the
/// moments of the weights batch_ess_kernel normalised (Filter::estimate).  Its range fits either partition; the CTAs
/// beyond the one it takes only leave.  kBox: some member of the step reads a landmark map, and such a member's injected
/// states come from its map's box (resample_box_kernel's body).
template <bool kTable, bool kBox>
__global__ void __launch_bounds__(kRsThreads) batch_finish_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchFinish, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  Scalars* scalars = s.scalars + k;
  double* partials = s.partials + static_cast<size_t>(blockIdx.x - local) * kMomentCount;
  const bool ess = m.resample == kBatchResampleEss;
  const BatchTail tail{s.summary + k, s.members_done, s.n_members, s.ticket, s.seq, 0, m.resample == 1 ? 1 : 0};
  if (!m.resample || (ess && scalars->ess_resample == 0)) {
    const uint32_t grid = ess ? moments_blocks(m.n) : count;
    if (local >= grid) return;
    normalize_moments_block(batch_states(s, m, 0), s.weights + m.offset, m.n, m.pivot_x, m.pivot_y, scalars, partials, local, grid, tail, !ess);
    return;
  }
  ResampleArgs a{};
  a.states_in = batch_states(s, m, 0);
  a.cdf = s.cdf + m.offset;
  a.n_in = m.n;
  a.states_out = batch_states(s, m, 1);
  a.weights_out = s.weights + m.offset;
  a.ancestors = s.ancestors != nullptr ? s.ancestors + m.offset : nullptr;
  a.slot_count = m.slots;
  a.total_slots = m.slots;
  a.scheme = m.scheme;
  a.seed = m.seed;
  a.step = m.step;
  a.random_state_probability = m.random_state_probability;
  batch_recovery_map<kTable>(s, m, a);
  a.pivot_x = m.pivot_x;
  a.pivot_y = m.pivot_y;
  if (m.kld) {  // launch_resample with hashes: always the per-slot form
    const BatchKldMember& q = s.kld[k];
    a.hashes = s.hashes + m.offset;
    for (int d = 0; d < 3; ++d) a.hash_resolution[d] = q.hash_resolution[d];
  }
  // systematic, nothing drawn per slot and no hashes: launch_resample's scatter form
  const bool scatter = !m.kld && m.scheme == 1 && m.random_state_probability <= 0.0;
  if (m.kld || ess) {  // a.tail is the disabled one (no summary, no arrival): batch_resampled_moments_kernel publishes
    const uint32_t grid = scatter ? resample_scatter_blocks(m.n) : resample_blocks(m.slots);
    if (local >= grid) return;
    if (scatter) {
      resample_scatter_block(a, scalars, partials, local, grid, a.tail);
    } else if (kBox && batch_landmark<kTable>(s, m).model != 0) {
      resample_block<StepTail, true>(a, scalars, partials, local, grid, a.tail, batch_box<kTable>(s, m));
    } else {
      resample_block(a, scalars, partials, local, grid, a.tail);
    }
  } else if (scatter) {
    resample_scatter_block(a, scalars, partials, local, count, tail);
  } else if (kBox && batch_landmark<kTable>(s, m).model != 0) {
    resample_block<BatchTail, true>(a, scalars, partials, local, count, tail, batch_box<kTable>(s, m));
  } else {
    resample_block(a, scalars, partials, local, count, tail);
  }
}

// ---- KLD-adaptive members (Filter::resample_kld's one chunk, then Filter::estimate) ---------------------------------
// A member holds at most kBatchMaxParticles = 32768 particles, so resample_kld's first chunk, min(max, max(2 min, 65536))
// slots, is all of them: one draw (batch_finish_kernel), one count with no buckets before it, accepted =
// min(cutoff - 1, max).  The count is kld_check_kernel's: a bucket set that keeps each bucket's smallest slot makes "slot
// j is the first of its bucket" an order-independent fact, so k after every slot is a prefix sum of those flags in slot
// order, and the cutoff is the smallest count whose condition fails.

constexpr int kBatchKldThreads = 1024;
constexpr int kBatchKldWarps = kBatchKldThreads / kWarp;

/// Whether a member of the step drew a new particle set: every resampling member, except a selective one whose effective
/// sample size stayed at n / 2 or above.
__device__ __forceinline__ bool batch_resampled(const BatchMember& m, const Scalars* scalars) {
  return m.resample == 1 || (m.resample == kBatchResampleEss && scalars->ess_resample != 0);
}

/// One CTA per KLD member: clear its bucket set, insert every slot's hash, then flag first occurrences and scan them
/// chunk by chunk in slot order; scalars->kld_cutoff receives the first failing count (~0 when every count passes).  A
/// selective member that kept its particles has nothing to count.
__global__ void __launch_bounds__(kBatchKldThreads) batch_kld_kernel(BatchStepArgs s) {
  __shared__ uint32_t s_warp[kBatchKldWarps];
  __shared__ unsigned long long s_min[kBatchKldWarps];
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchKldRow, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  if (!batch_resampled(m, s.scalars + k)) return;
  const BatchKldMember& q = s.kld[k];
  const unsigned long long* hashes = s.hashes + m.offset;
  unsigned long long* keys = s.keys + q.table_offset;
  unsigned int* vals = s.vals + q.table_offset;
  const uint64_t mask = q.table_mask;
  const uint32_t slots = static_cast<uint32_t>(m.slots);
  const int tid = threadIdx.x, lane = tid % kWarp, warp = tid / kWarp;

  for (uint64_t t = tid; t <= mask; t += kBatchKldThreads) {  // launch_kld_clear
    keys[t] = bucket_set::kEmpty;
    vals[t] = ~0u;
  }
  __syncthreads();
  for (uint32_t j = tid; j < slots; j += kBatchKldThreads) bucket_set::insert_min(keys, vals, mask, hashes[j], j);  // kld_insert_kernel
  __syncthreads();
  unsigned long long failing = ~0ull, k_before = 0;
  for (uint32_t base = 0; base < slots; base += kBatchKldThreads) {
    const uint32_t j = base + tid;
    bool head = false;
    if (j < slots) head = vals[bucket_set::find(keys, mask, hashes[j])] == j;  // kld_flag_kernel
    const unsigned heads = __ballot_sync(0xffffffffu, head);
    if (lane == 0) s_warp[warp] = __popc(heads);
    __syncthreads();
    unsigned long long before = k_before;
    for (int w = 0; w < kBatchKldWarps; ++w) {
      const uint32_t c = s_warp[w];
      if (w < warp) before += c;
      k_before += c;
    }
    // kld_check_kernel: k = buckets up to and including slot j
    if (j < slots && !kld_count_allowed(j + 1ull, before + __popc(heads & ((1u << lane) - 1u)) + (head ? 1u : 0u), q.min_particles,
                                        q.two_epsilon, q.z))
      failing = j + 1ull;
    // Counts only grow: once a chunk holds a failing count, no later chunk holds a smaller one.  (Also the barrier
    // before the next chunk writes s_warp.)
    if (__syncthreads_or(failing != ~0ull)) break;
  }
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) {
    const unsigned long long o = __shfl_down_sync(0xffffffffu, failing, off);
    failing = o < failing ? o : failing;
  }
  if (lane == 0) s_min[warp] = failing;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kBatchKldWarps; ++w) failing = s_min[w] < failing ? s_min[w] : failing;
    s.scalars[k].kld_cutoff = failing;
  }
}

/// Filter::estimate after Filter::resample: moments_kernel over the new particle set of a member that resampled under KLD
/// or after the effective-sample-size test (unit weights, the partition of moments_block_count(accepted) blocks), summed
/// like reduce_partials_kernel by the last of those CTAs, which publishes the member's summary.  accepted is the KLD count
/// of a KLD member and max_particles otherwise.  Each such member has moments_block_count(max_particles) CTAs; those
/// beyond moments_block_count(accepted) only leave, and so do all of those of a selective member that kept its particles
/// (batch_finish_kernel published its summary).
__global__ void __launch_bounds__(kStreamThreads) batch_resampled_moments_kernel(BatchStepArgs s) {
  __shared__ double s_red[kMomentCount * kStreamThreads / kWarp];
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchMomentsRow, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  Scalars* scalars = s.scalars + k;
  if (!batch_resampled(m, scalars)) return;
  uint64_t accepted = m.slots;
  if (m.kld) {
    const unsigned long long cutoff = scalars->kld_cutoff;
    // take_while drops the first element whose condition fails (take_while_kld.hpp:134-136)
    accepted = cutoff != ~0ull ? (cutoff - 1 < m.slots ? cutoff - 1 : m.slots) : m.slots;
  }
  const uint32_t grid = moments_blocks(accepted);
  if (local >= grid) return;
  const Pose2* states = batch_states(s, m, 1);  // the new set (the host flips cur once the step has ended)
  double v[kMomentCount];
#pragma unroll
  for (int c = 0; c < kMomentCount; ++c) v[c] = 0.0;
  for (uint64_t i = static_cast<uint64_t>(local) * kStreamThreads + threadIdx.x; i < accepted; i += static_cast<uint64_t>(grid) * kStreamThreads)
    accumulate_moments(v, load_pose(states + i), 1.0, m.pivot_x, m.pivot_y);  // the draw wrote w = 1 to every slot
  const BatchTail tail{s.summary + k, s.members_done, s.n_members, s.ticket, s.seq, m.kld ? accepted : 0, 1};
  finish_block_moments<kStreamThreads>(v, s_red, s.partials + static_cast<size_t>(blockIdx.x - local) * kMomentCount, scalars, local, grid, tail);
}

// ---- pose samples of a batch (Filter::sample_states per member) --------------------------------------------------
// A member whose CDF is stale gets the CDF Filter::build_cdf would build: scalars and scan state reset, the largest weight
// (max_weight_kernel's block body), then the quantise + scan with the exponent derived from it exactly as prepare_cdf
// derives it (a degenerate weight set gets the uniform CDF).

__global__ void __launch_bounds__(256) batch_sample_reset_kernel(BatchSampleArgs s) { batch_reset_grid(s, s.ctas[kSampleScan]); }

__global__ void __launch_bounds__(kMaxThreads) batch_sample_max_kernel(BatchSampleArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kSampleMax, blockIdx.x, local, count);
  const BatchSampleMember& m = s.members[k];
  max_weight_block(s.weights + m.offset, m.n, s.scalars + k, local, count);
}

__global__ void __launch_bounds__(kQsThreads) batch_sample_scan_kernel(BatchSampleArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kSampleScan, blockIdx.x, local, count);
  const BatchSampleMember& m = s.members[k];
  quantize_scan_tile(s.weights + m.offset, m.n, s.cdf + m.offset, s.scalars + k, s.tile_state + (blockIdx.x - local), local, 1,
                     m.ceil_log2_count);
}

/// resample_kernel's multinomial draws of `count` slots without weights, ancestors or tail, into the member's run of `out`.
__global__ void __launch_bounds__(kRsThreads) batch_sample_kernel(BatchSampleArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kSampleDraw, blockIdx.x, local, count);
  const BatchSampleMember& m = s.members[k];
  Scalars* scalars = s.scalars + k;
  ResampleArgs a{};
  a.states_in = (m.cur != 0 ? s.states[1] : s.states[0]) + m.offset;
  a.cdf = s.cdf + m.offset;
  a.n_in = m.n;
  a.states_out = s.out + m.out_offset;
  a.slot_count = m.count;
  a.total_slots = m.count;
  a.global_total = m.total;  // 0: the rebuilt CDF's, in scalars->total
  a.scheme = BB200_RESAMPLE_MULTINOMIAL;
  a.seed = m.seed;
  a.step = s.step;
  resample_block(a, scalars, s.partials + static_cast<size_t>(blockIdx.x - local) * kMomentCount, local, count, a.tail);
  if (local == 0 && threadIdx.x == 0) s.totals[k] = m.total != 0 ? m.total : scalars->total;
}

// ---- scans and point clouds of a batch step (before the step's launches) -------------------------------------------

constexpr int kPtThreads = 256;
constexpr uint32_t kBatchCloudPointsPerCta = 16 * kPtThreads;

/// Bit pattern of |x| + |y| that orders like scan_radius's result (filter.cu): non-negative doubles order like their bits,
/// and every NaN becomes the one pattern above +inf, so that the largest pattern is NaN when some term is.
__device__ __forceinline__ unsigned long long radius_bits(double x, double y) {
  const double r = fabs(x) + fabs(y);
  return isnan(r) ? 0x7ff8000000000000ull : static_cast<unsigned long long>(__double_as_longlong(r));
}

/// The largest of every thread's `bits`, in thread 0.
__device__ __forceinline__ unsigned long long block_max_bits(unsigned long long bits) {
  __shared__ unsigned long long s_max[kPtThreads / kWarp];
#pragma unroll
  for (int o = kWarp / 2; o > 0; o >>= 1) bits = max(bits, __shfl_xor_sync(0xffffffffu, bits, o));
  if ((threadIdx.x & (kWarp - 1)) == 0) s_max[threadIdx.x / kWarp] = bits;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kPtThreads / kWarp; ++w) bits = max(bits, s_max[w]);
  return bits;
}

/// A scan member (one CTA): bb200_scan_to_points's loop over the kept beams with the directions given, the survivors
/// compacted in beam order, chunk by chunk; n_points and points_radius of the member follow.
__device__ __forceinline__ void scan_points_block(const BatchPointsMember& in, const float* __restrict__ ranges, double2* __restrict__ out,
                                                  BatchMember& m) {
  __shared__ uint32_t s_warp[kPtThreads / kWarp];
  const uint32_t lane = threadIdx.x & (kWarp - 1), warp = threadIdx.x / kWarp;
  const double* o = in.origin;
  uint32_t kept = 0;
  unsigned long long bits = 0;
  for (uint64_t base = 0; base < in.count; base += kPtThreads) {
    const uint64_t i = base + threadIdx.x;
    bool keep = false;
    double px = 0.0, py = 0.0;
    if (i < in.count) {
      const double r = static_cast<double>(ranges[i]);
      keep = !(isnan(r) || !(r >= in.min_range) || !(r <= in.max_range));  // laser_scan.hpp:80-84
      if (keep) {
        const double2 d = in.directions[i];
        const double x = r * d.x, y = r * d.y;
        px = x;
        py = y;
        if (in.has_origin) {  // origin * (x, y, 0), keep (x, y)  (beluga_ros/src/amcl.cpp:59-61)
          px = (o[0] * x + o[1] * y) + o[3];
          py = (o[4] * x + o[5] * y) + o[7];
        }
      }
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    uint32_t before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kPtThreads / kWarp; ++w) {
      before += w < static_cast<int>(warp) ? s_warp[w] : 0u;
      total += s_warp[w];
    }
    if (keep) {
      out[kept + before + __popc(ballot & ((1u << lane) - 1u))] = make_double2(px, py);
      bits = max(bits, radius_bits(px, py));
    }
    kept += total;
    __syncthreads();  // every warp has read s_warp before the next chunk writes it
  }
  bits = block_max_bits(bits);
  if (threadIdx.x == 0) {
    m.n_points = kept;
    m.points_radius = __longlong_as_double(static_cast<long long>(bits));
  }
}

/// CTA `local` of a cloud member: cloud_to_points (c_api.cu) on its kBatchCloudPointsPerCta points, from the packed floats;
/// the member's points_radius (0 when the step began) takes the CTA's largest term.
__device__ __forceinline__ void cloud_points_block(const BatchPointsMember& in, const float* __restrict__ xyz, double2* __restrict__ out,
                                                   BatchMember& m, uint32_t local) {
  const double* o = in.origin;
  unsigned long long bits = 0;
  const uint64_t end = min(static_cast<uint64_t>(in.count), (static_cast<uint64_t>(local) + 1) * kBatchCloudPointsPerCta);
  for (uint64_t i = static_cast<uint64_t>(local) * kBatchCloudPointsPerCta + threadIdx.x; i < end; i += kPtThreads) {
    const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    double px = x, py = y;
    if (in.has_origin) {
      px = ((o[0] * x + o[1] * y) + o[2] * z) + o[3];
      py = ((o[4] * x + o[5] * y) + o[6] * z) + o[7];
    }
    out[i] = make_double2(px, py);
    bits = max(bits, radius_bits(px, py));
  }
  bits = block_max_bits(bits);
  if (threadIdx.x == 0 && bits != 0) atomicMax(reinterpret_cast<unsigned long long*>(&m.points_radius), bits);
}

__global__ void __launch_bounds__(kPtThreads) batch_points_kernel(BatchPointsArgs s) {
  uint32_t local, count;
  const uint32_t j = batch_member_of(s, 0, blockIdx.x, local, count);
  const BatchPointsMember& in = s.inputs[j];
  BatchMember& m = s.members[j];
  double2* out = reinterpret_cast<double2*>(s.points) + m.point_offset;
  if (in.kind == kBatchInputScan) {
    scan_points_block(in, s.input + in.input_offset, out, m);
  } else {
    cloud_points_block(in, s.input + in.input_offset, out, m, local);
  }
}

// ---- membership changes: the surviving members' live data, from the old layout to the new one ------------------

constexpr int kRelayoutThreads = 256;

__global__ void __launch_bounds__(kRelayoutThreads) batch_relayout_kernel(BatchRelayoutArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, 0, blockIdx.x, local, count);
  const BatchRelayoutMember& m = s.members[k];
  const uint64_t i = static_cast<uint64_t>(local) * kRelayoutThreads + threadIdx.x;
  if (i < m.n) {
    const Pose2* from = (m.cur != 0 ? s.states_from[1] : s.states_from[0]) + m.from;
    s.states_to[m.to + i] = from[i];
    s.weights_to[m.to + i] = s.weights_from[m.from + i];
  }
  if (i < m.cdf_n) s.cdf_to[m.to + i] = s.cdf_from[m.from + i];
  if (i < m.ancestors_n) s.ancestors_to[m.to + i] = s.ancestors_from[m.from + i];
}

// ---- ray casts: each member's rays on its map --------------------------------------------------------------------

__global__ void __launch_bounds__(kRayThreads) batch_cast_rays_kernel(BatchRayArgs s) {
  uint32_t local, count;
  const BatchRayMember& m = s.members[batch_member_of(s, 0, blockIdx.x, local, count)];
  const OccupancyView grid = m.grid;
  cast_rays_block(grid, s.poses + m.pose_offset, s.bearings + m.bearing_offset, m.n_bearings, m.n_rays, m.max_range, s.ranges + m.ray_offset, local);
}

template <bool kTable>
int launch_batch_step_head_from(const BatchStepArgs& s, cudaStream_t stream) {
  const uint32_t reset = std::max(s.n_members, s.ctas[kBatchScan]);
  batch_begin_kernel<<<std::max(1u, std::min((reset + 255u) / 256u, kSmCount * 4u)), 256, 0, stream>>>(s);
  batch_propagate_kernel<<<s.ctas[kBatchPropagate], kPrThreads, 0, stream>>>(s);
  int launches = 2;
  if (s.forms & (1 << kBatchField)) {
    const size_t smem = static_cast<size_t>(std::min(s.max_points, kChunkBeams)) * sizeof(double2);
    batch_reweight_kernel<kTable><<<s.ctas[kBatchReweight], kRwThreads, smem, stream>>>(s);
    launches += 1;
  }
  if (s.forms & (1 << kBatchBeamTwoPass)) {
    batch_beam_walk_kernel<kTable><<<s.ctas[kBatchReweightWalk], kWalkThreads, 0, stream>>>(s);
    batch_beam_mixture_kernel<kTable><<<s.ctas[kBatchReweightWalk], kMixThreads, 0, stream>>>(s);
    launches += 2;
  }
  if (s.forms & (1 << kBatchBeamFused)) {
    batch_reweight_beam_kernel<kTable><<<s.ctas[kBatchReweightBeam], kBeamThreads, 0, stream>>>(s);
    launches += 1;
  }
  if (s.forms & (1 << kBatchLandmark)) {
    batch_reweight_landmark_kernel<kTable><<<s.landmark_ctas, kLandmarkThreads, 0, stream>>>(s);
    launches += 1;
  }
  return launches;
}

template <bool kTable>
int launch_batch_step_tail_from(const BatchStepArgs& s, cudaStream_t stream) {
  int launches = 2;
  if (s.weigh_ctas > 0) {
    batch_weigh_kernel<<<s.weigh_ctas, kMaxThreads, 0, stream>>>(s);
    launches += 1;
  }
  batch_scan_kernel<<<s.ctas[kBatchScan], kQsThreads, 0, stream>>>(s);
  if (s.ess_ctas > 0) {
    batch_ess_kernel<<<s.ess_ctas, kStreamThreads, 0, stream>>>(s);
    launches += 1;
  }
  if (s.landmark_maps) {
    batch_finish_kernel<kTable, true><<<s.ctas[kBatchFinish], kRsThreads, 0, stream>>>(s);
  } else {
    batch_finish_kernel<kTable, false><<<s.ctas[kBatchFinish], kRsThreads, 0, stream>>>(s);
  }
  if (s.kld != nullptr) {
    batch_kld_kernel<<<s.post_ctas[0], kBatchKldThreads, 0, stream>>>(s);
    launches += 1;
  }
  if (s.kld != nullptr || s.ess_ctas > 0) {
    batch_resampled_moments_kernel<<<s.post_ctas[1], kStreamThreads, 0, stream>>>(s);
    launches += 1;
  }
  return launches;
}

}  // namespace

uint32_t batch_scan_tiles(uint64_t n) { return scan_tile_count(n); }

void batch_member_ctas(const BatchMember& m, int form, uint32_t out[kBatchLaunches]) {
  out[kBatchPropagate] = static_cast<uint32_t>((m.n + kPrThreads - 1) / kPrThreads);
  out[kBatchReweight] = out[kBatchReweightWalk] = out[kBatchReweightBeam] = 0;
  if (form != kBatchWeighed && form != kBatchLandmark) out[batch_reweight_row(form)] = static_cast<uint32_t>((m.n + kRwThreads - 1) / kRwThreads);
  out[kBatchScan] = scan_tile_count(m.n);
  // the partition launch_resample / launch_moments would use for a single filter of this size
  if (!m.resample) {
    out[kBatchFinish] = moments_block_count(m.n);
    return;
  }
  const uint32_t draw = m.scheme == 1 && m.random_state_probability <= 0.0 && !m.kld ? resample_scatter_block_count(m.n) : resample_block_count(m.slots);
  // a selective member's range fits the draw and the moments of the weights it keeps, whichever the device decides
  out[kBatchFinish] = m.resample == kBatchResampleEss ? std::max(draw, moments_block_count(m.n)) : draw;
}

void batch_post_ctas(const BatchMember& m, uint32_t out[3]) {
  const bool ess = m.resample == kBatchResampleEss;
  out[0] = m.kld ? 1u : 0u;
  out[1] = m.kld || ess ? moments_blocks(m.slots) : 0u;
  out[2] = ess ? moments_blocks(m.n) : 0u;  // launch_normalize's partition
}

uint32_t batch_weigh_ctas(const BatchMember& m) { return static_cast<uint32_t>(std::min<uint64_t>((m.n + kMaxThreads - 1) / kMaxThreads, kStreamMaxBlocks)); }

uint32_t batch_landmark_ctas(const BatchMember& m) { return static_cast<uint32_t>((m.n + kLandmarkThreads - 1) / kLandmarkThreads); }

int launch_batch_step_head(const BatchStepArgs& s, cudaStream_t stream) {
  return s.maps != nullptr ? launch_batch_step_head_from<true>(s, stream) : launch_batch_step_head_from<false>(s, stream);
}

int launch_batch_step_tail(const BatchStepArgs& s, cudaStream_t stream) {
  return s.maps != nullptr ? launch_batch_step_tail_from<true>(s, stream) : launch_batch_step_tail_from<false>(s, stream);
}

uint32_t batch_points_ctas(const BatchPointsMember& m) {
  if (m.kind == kBatchInputScan) return 1;
  if (m.kind == kBatchInputCloud)
    return std::max(1u, static_cast<uint32_t>((static_cast<uint64_t>(m.count) + kBatchCloudPointsPerCta - 1) / kBatchCloudPointsPerCta));
  return 0;
}

int launch_batch_points(const BatchPointsArgs& s, cudaStream_t stream) {
  batch_points_kernel<<<s.ctas, kPtThreads, 0, stream>>>(s);
  return 1;
}

void batch_sample_ctas(const BatchSampleMember& m, bool rebuilt, uint32_t out[kSampleLaunches]) {
  out[kSampleMax] = rebuilt ? static_cast<uint32_t>(std::min<uint64_t>((m.n + kMaxThreads - 1) / kMaxThreads, kStreamMaxBlocks)) : 0u;  // launch_max_weight's grid
  out[kSampleScan] = rebuilt ? scan_tile_count(m.n) : 0u;
  out[kSampleDraw] = resample_block_count(m.count);
}

int launch_batch_sample(const BatchSampleArgs& s, cudaStream_t stream) {
  int launches = 1;
  if (s.ctas[kSampleScan] > 0) {
    const uint32_t reset = std::max(s.n_members, s.ctas[kSampleScan]);
    batch_sample_reset_kernel<<<std::max(1u, std::min((reset + 255u) / 256u, kSmCount * 4u)), 256, 0, stream>>>(s);
    batch_sample_max_kernel<<<s.ctas[kSampleMax], kMaxThreads, 0, stream>>>(s);
    batch_sample_scan_kernel<<<s.ctas[kSampleScan], kQsThreads, 0, stream>>>(s);
    launches += 3;
  }
  batch_sample_kernel<<<s.ctas[kSampleDraw], kRsThreads, 0, stream>>>(s);
  return launches;
}

uint32_t batch_relayout_ctas(const BatchRelayoutMember& m) {
  const uint64_t n = std::max({m.n, m.cdf_n, m.ancestors_n});
  return static_cast<uint32_t>((n + kRelayoutThreads - 1) / kRelayoutThreads);
}

int launch_batch_relayout(const BatchRelayoutArgs& s, cudaStream_t stream) {
  batch_relayout_kernel<<<s.ctas, kRelayoutThreads, 0, stream>>>(s);
  return 1;
}

int launch_batch_cast_rays(const BatchRayArgs& s, cudaStream_t stream) {
  batch_cast_rays_kernel<<<s.ctas, kRayThreads, 0, stream>>>(s);
  return 1;
}

}  // namespace bb200
