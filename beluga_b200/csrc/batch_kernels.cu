// ---- batches of filters ----------------------------------------------------------------------------------
// Each kernel below runs, per CTA, the block body of the single-filter kernel it stands for, on the CTA's member.
#include "cdf.cuh"
#include "resample.cuh"
#include "reweight_beam.cuh"
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
};
__device__ __forceinline__ bool tail_enabled(const BatchTail&) { return true; }
__device__ __forceinline__ void tail_publish(const BatchTail& tail, const double* v, Scalars* scalars) {
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) tail.summary->moments[k] = v[k];
  scalars->blocks_done = 0;
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

/// A step that keeps its particles: normalize_kernel's w /= S and moments_kernel's rows over the same partition
/// (moments_block_count blocks), the rows summed like reduce_partials_kernel does.
__device__ __forceinline__ void normalize_moments_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, double px,
                                                        double py, Scalars* scalars, double* __restrict__ moment_partials, uint32_t block,
                                                        uint32_t grid, const BatchTail& tail) {
  __shared__ double s_red[kMomentCount * kStreamThreads / kWarp];
  const double factor = scalbn(static_cast<double>(scalars->total), -scalars->exponent);
  const bool valid = scalars->valid != 0 && factor > 0.0;
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
/// normalisation otherwise; then the member's moments, summed by its last CTA.
template <bool kTable>
__global__ void __launch_bounds__(kRsThreads) batch_finish_kernel(BatchStepArgs s) {
  uint32_t local, count;
  const uint32_t k = batch_member_of(s, kBatchFinish, blockIdx.x, local, count);
  const BatchMember& m = s.members[k];
  Scalars* scalars = s.scalars + k;
  double* partials = s.partials + static_cast<size_t>(blockIdx.x - local) * kMomentCount;
  const BatchTail tail{s.summary + k, s.members_done, s.n_members, s.ticket, s.seq};
  if (!m.resample) {
    normalize_moments_block(batch_states(s, m, 0), s.weights + m.offset, m.n, m.pivot_x, m.pivot_y, scalars, partials, local, count, tail);
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
  if (m.scheme == 1 && m.random_state_probability <= 0.0) {  // systematic, nothing drawn per slot: launch_resample's scatter form
    resample_scatter_block(a, scalars, partials, local, count, tail);
  } else {
    resample_block(a, scalars, partials, local, count, tail);
  }
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

template <bool kTable>
int launch_batch_step_from(const BatchStepArgs& s, cudaStream_t stream) {
  const uint32_t reset = std::max(s.n_members, s.ctas[kBatchScan]);
  batch_begin_kernel<<<std::max(1u, std::min((reset + 255u) / 256u, kSmCount * 4u)), 256, 0, stream>>>(s);
  batch_propagate_kernel<<<s.ctas[kBatchPropagate], kPrThreads, 0, stream>>>(s);
  int launches = 4;
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
  batch_scan_kernel<<<s.ctas[kBatchScan], kQsThreads, 0, stream>>>(s);
  batch_finish_kernel<kTable><<<s.ctas[kBatchFinish], kRsThreads, 0, stream>>>(s);
  return launches;
}

}  // namespace

uint32_t batch_scan_tiles(uint64_t n) { return scan_tile_count(n); }

void batch_member_ctas(const BatchMember& m, int form, uint32_t out[kBatchLaunches]) {
  out[kBatchPropagate] = static_cast<uint32_t>((m.n + kPrThreads - 1) / kPrThreads);
  out[kBatchReweight] = out[kBatchReweightWalk] = out[kBatchReweightBeam] = 0;
  out[batch_reweight_row(form)] = static_cast<uint32_t>((m.n + kRwThreads - 1) / kRwThreads);
  out[kBatchScan] = scan_tile_count(m.n);
  // the partition launch_resample / launch_moments would use for a single filter of this size
  if (!m.resample) {
    out[kBatchFinish] = moments_block_count(m.n);
  } else if (m.scheme == 1 && m.random_state_probability <= 0.0) {
    out[kBatchFinish] = resample_scatter_block_count(m.n);
  } else {
    out[kBatchFinish] = resample_block_count(m.slots);
  }
}

int launch_batch_step(const BatchStepArgs& s, cudaStream_t stream) {
  return s.maps != nullptr ? launch_batch_step_from<true>(s, stream) : launch_batch_step_from<false>(s, stream);
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

}  // namespace bb200
