// Block bodies of the resample (resample.cu), shared with the batch kernels: the per-slot and the scatter form, the raw
// moments of the new set and the last block's sum of them.
#pragma once

#include "propagate.cuh"

namespace bb200 {

namespace {

constexpr int kStreamThreads = 256;

/// Blocks of moments_kernel over n particles (moments_block_count), on the host and on the device.
BB_HD uint32_t moments_blocks(uint64_t n) {
  const uint64_t blocks = (n + kStreamThreads - 1) / kStreamThreads;
  return static_cast<uint32_t>(blocks < 1 ? 1 : blocks > kStreamMaxBlocks ? kStreamMaxBlocks : blocks);
}

// ---- normalize -------------------------------------------------------------------------------------

/// The block index and block count a block body runs with: the launch's own (a single-filter kernel; read where they are
/// used, so that the kernel compiles as it did with the body written inside it) ...
struct LaunchBlocks {
  __device__ __forceinline__ uint32_t block() const { return blockIdx.x; }
  __device__ __forceinline__ uint32_t grid() const { return gridDim.x; }
};
/// ... or a batch member's range of the launch.
struct RangeBlocks {
  uint32_t index, count;
  __device__ __forceinline__ uint32_t block() const { return index; }
  __device__ __forceinline__ uint32_t grid() const { return count; }
};

/// One block of normalize_kernel: w /= S (S = T * 2^-e, T = global_total, or scalars->global_total when it is ~0, or
/// scalars->total when it is 0) when the weights are valid, and the block's sum of w^2 into partials[block].
template <class Blocks>
__device__ __forceinline__ void normalize_block(double* __restrict__ weights, uint64_t n, const Scalars* scalars, unsigned long long global_total,
                                                double* __restrict__ partials, const Blocks& blocks) {
  __shared__ double s_red[kStreamThreads / kWarp];
  // S = T * 2^-e: the normalisation factor derived from the exact integer total.
  // 0: single GPU, the total is on the device; ~0: sharded, the sum of the ranks' totals is on the device
  const unsigned long long t = global_total == ~0ull ? scalars->global_total : (global_total != 0 ? global_total : scalars->total);
  const double factor = scalbn(static_cast<double>(t), -scalars->exponent);
  const bool valid = scalars->valid != 0 && factor > 0.0;
  double sq = 0.0;
  for (uint64_t i = static_cast<uint64_t>(blocks.block()) * kStreamThreads + threadIdx.x; i < n;
       i += static_cast<uint64_t>(blocks.grid()) * kStreamThreads) {
    double w = weights[i];
    if (valid) {
      w = w / factor;  // actions/normalize.hpp:82
      weights[i] = w;
    }
    sq = sq + w * w;
  }
  const double total = block_sum<kStreamThreads>(sq, s_red);
  if (threadIdx.x == 0) partials[blocks.block()] = total;
}

// ---- resample -------------------------------------------------------------------------------------

constexpr int kRsThreads = 256;
// (CTAs per SM, particles per thread and round) = (3, 2) was chosen by a sweep at 1M on a B200, carried over to the H100
// without re-measuring.
constexpr int kRsBlocksPerSm = 3;  // resident CTAs per SM the kernel is compiled for (register cap)
constexpr int kRsUnroll = 2;       // particles per thread and round

/// Blocks of resample_kernel over `slots` output slots (resample_block_count), on the host and on the device.
BB_HD uint32_t resample_blocks(uint64_t slots) {
  const uint64_t blocks = (slots + kRsThreads - 1) / kRsThreads;
  return static_cast<uint32_t>(blocks < 1 ? 1 : blocks > kSmCount * 16 ? kSmCount * 16 : blocks);
}
/// Blocks of resample_scatter_kernel over n_in particles (resample_scatter_block_count), on the host and on the device.
BB_HD uint32_t resample_scatter_blocks(uint64_t n_in) {
  // one pass over the input particles; a few particles per thread amortise the block reduction of the moments
  const uint64_t blocks = (n_in + kRsThreads - 1) / kRsThreads;
  return static_cast<uint32_t>(blocks < 1 ? 1 : blocks > kSmCount * kRsBlocksPerSm ? kSmCount * kRsBlocksPerSm : blocks);
}

/// Smallest i in [0, n) with cdf[i] > t.
__device__ __forceinline__ uint64_t cdf_upper_bound(const unsigned long long* __restrict__ cdf, uint64_t n, unsigned long long t) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(cdf + mid) > t) {
      hi = mid;
    } else {
      lo = mid + 1;
    }
  }
  return lo < n ? lo : n - 1;  // unreachable clamp (t < total by construction)
}

__device__ __forceinline__ void accumulate_moments(double* m, const Pose2& st, double w, double px, double py) {
  const double dx = st.x - px, dy = st.y - py;
  m[0] += w;
  m[1] += w * w;
  m[2] += w * st.c;
  m[3] += w * st.s;
  m[4] += w * dx;
  m[5] += w * dy;
  m[6] += w * dx * dx;
  m[7] += w * dx * dy;
  m[8] += w * dy * dy;
}

template <int kThreads>
__device__ __forceinline__ void store_block_moments(double* m, double* scratch /* kMomentCount * kThreads/32 */, double* __restrict__ partials_row) {
  block_sum_many<kThreads, kMomentCount>(m, scratch);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < kMomentCount; ++k) partials_row[k] = m[k];
  }
}

/// Stores the block's raw moments and, when the launch carries a StepTail, lets the LAST block to arrive add the
/// per-block rows up in a fixed order (thread-strided over the rows, then the block tree: the same sum for any
/// arrival order) -- the reduce_partials launch and the read-back copies of the fused step folded into the resample.
/// With tail.summary set (single GPU: pinned host memory, written straight over PCIe) the host finds the step's
/// results after its one stream synchronisation.
/// What the last block of a single filter's resample does with the summed moments (thread 0).
__device__ __forceinline__ bool tail_enabled(const StepTail& tail) { return tail.enabled != 0; }
__device__ __forceinline__ void tail_publish(const StepTail& tail, const double* v, Scalars* scalars) {
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) {
    tail.results[k] = v[k];
    if (tail.summary != nullptr) tail.summary->moments[k] = v[k];
  }
  scalars->blocks_done = 0;
  if (tail.summary != nullptr) {
    tail.summary->total = scalars->total;
    tail.summary->exponent = scalars->exponent;
    tail.summary->valid = scalars->valid;
    tail.summary->error = 0;
    __threadfence_system();
    if (tail.seq != 0) {  // the host polls this word instead of synchronising with the stream
      *reinterpret_cast<volatile int*>(&tail.summary->seq) = tail.seq;
      __threadfence_system();
    }
  }
}

/// `block` of `grid` blocks that produce one particle set's moments (a batch member's blocks are a slice of the launch).
template <int kThreads, class Tail>
__device__ __forceinline__ void finish_block_moments(double* m, double* scratch, double* __restrict__ moment_partials, Scalars* scalars,
                                                     uint32_t block, uint32_t grid, const Tail& tail) {
  store_block_moments<kThreads>(m, scratch, moment_partials + static_cast<size_t>(block) * kMomentCount);
  if (!tail_enabled(tail)) return;
  __shared__ int s_last;
  if (threadIdx.x == 0) {
    __threadfence();  // the row above before the arrival count
    s_last = atomicAdd(&scalars->blocks_done, 1u) + 1u == grid ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double v[kMomentCount];
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) v[k] = 0.0;
  for (uint32_t r = threadIdx.x; r < grid; r += kThreads) {
    const double* row = moment_partials + static_cast<size_t>(r) * kMomentCount;
#pragma unroll
    for (int k = 0; k < kMomentCount; ++k) v[k] = v[k] + __ldcg(row + k);  // nine independent loads per row
  }
  block_sum_many<kThreads, kMomentCount>(v, scratch);
  if (threadIdx.x == 0) tail_publish(tail, v, scalars);
}

/// Block `block` of `grid` of the per-slot resample (resample_kernel; resample_box_kernel with kBox, whose injected
/// states come from a landmark map's box).
template <class Tail, bool kBox = false>
__device__ __forceinline__ void resample_block(const ResampleArgs& a, Scalars* __restrict__ scalars, double* __restrict__ moment_partials,
                                               uint32_t block, uint32_t grid, const Tail& tail, const BoxSpace& box = BoxSpace{}) {
  __shared__ double s_red[kMomentCount * kRsThreads / kWarp];
  unsigned long long total = a.global_total != 0 ? a.global_total : scalars->total;
  unsigned long long cdf_offset = a.cdf_offset, span_end = 0;
  uint64_t slot_first = a.slot_first, slot_count = a.slot_count;
  if (a.rank_totals != nullptr) {  // offsets = exclusive prefix of the ranks' totals (distributed.py: cdf_offsets)
    total = 0;
    cdf_offset = 0;
    for (int r = 0; r < a.world; ++r) {
      const unsigned long long t = a.rank_totals[r];
      if (r < a.rank) cdf_offset += t;
      total += t;
    }
    span_end = cdf_offset + a.rank_totals[a.rank];
  }
  unsigned long long stride = 0, offset = 0;
  if (a.scheme == 1) {
    // Systematic comb: stride = T / M, offset uniform in [0, stride).
    stride = total / a.total_slots;
    offset = mulhi64(counter_draw(a.seed, 0, a.step, kStreamSystematic).a, stride);
    if (a.rank_totals != nullptr) {
      // The slots whose comb position offset + j*stride lies in [cdf_offset, span_end) (distributed.py: slot_ranges).
      auto first_slot_at_or_after = [&](unsigned long long position) -> uint64_t {
        if (position <= offset) return 0;
        const unsigned long long j = (position - offset + stride - 1) / stride;
        return j < a.total_slots ? j : a.total_slots;
      };
      slot_first = first_slot_at_or_after(cdf_offset);
      uint64_t slot_end = a.rank + 1 == a.world ? a.total_slots : first_slot_at_or_after(span_end);
      // KLD on shards: only the slots of the current window [window_begin, window_end) -- the chunk being counted, or
      // [0, accepted count) for the final pass -- are produced.
      if (a.window_end > a.window_begin) {
        slot_first = slot_first < a.window_begin ? a.window_begin : slot_first;
        slot_end = slot_end > a.window_end ? a.window_end : slot_end;
      }
      slot_count = slot_end > slot_first ? slot_end - slot_first : 0;
    }
  }
  double m[kMomentCount];
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) m[k] = 0.0;

  for (uint64_t local = static_cast<uint64_t>(block) * kRsThreads + threadIdx.x; local < slot_count;
       local += static_cast<uint64_t>(grid) * kRsThreads) {
    const uint64_t j = slot_first + local;
    Pose2 st;
    long long ancestor = -1;
    bool inject = false;
    Draw d{0, 0};
    if (a.random_state_probability > 0.0 || a.scheme == 0) d = counter_draw(a.seed, j, a.step, kStreamResample);
    // random_intersperse.hpp:93-100: one coin per ADVANCE of the view -- slot 0, the element begin() yields, is never injected
    if (a.random_state_probability > 0.0) inject = j > 0 && uniform01(d.a) < a.random_state_probability;
    unsigned long long t = 0;
    if (!inject) t = a.scheme == 1 ? offset + j * stride : mulhi64(d.b, total);
    if (a.span_filter != 0) {
      // an injected state belongs to the slot's owner; with a particle count that is still being decided (KLD on shards)
      // slots are dealt round robin instead
      const bool my_slot = a.inject_mod > 0 ? (j % static_cast<uint64_t>(a.inject_mod) == static_cast<uint64_t>(a.rank))
                                            : (j >= a.owner_first && j - a.owner_first < a.owner_count);
      const bool mine = inject ? my_slot : (t >= cdf_offset && t - cdf_offset < scalars->total);
      if (!mine) continue;
    }
    if (inject) {
      if constexpr (kBox) {
        st = random_box_state(box, a.seed, j, a.step);
      } else {
        st = random_free_state(FreeSpace{a.free_cells, a.n_free, a.grid_width, a.grid_resolution, a.grid_origin},
                               counter_draw(a.seed, j, a.step, kStreamRandomState));
      }
    } else {
      const uint64_t idx = cdf_upper_bound(a.cdf, a.n_in, t - cdf_offset);  // the caller guarantees t lies in this shard's span
      ancestor = static_cast<long long>(idx);
      st = load_pose(a.states_in + idx);
    }
    if (a.peer_hash_count > 0) {
      // KLD on shards, counting pass: only the candidate's spatial hash is needed, and every rank needs it -- the
      // ranks then count distinct buckets over the same globally ordered hash stream and reach the same cutoff.
      const unsigned long long h = spatial_hash(st, a.hash_resolution[0], a.hash_resolution[1], a.hash_resolution[2]);
      for (int r = 0; r < a.peer_hash_count; ++r) a.peer_hashes[r][j] = h;
      continue;
    }
    if (a.peer_count > 0) {
      const uint64_t owner = j / a.peer_shard;  // P2P store over NVLink (or a local store when owner == this rank)
      store_pose(a.peer_out[owner] + (j - owner * a.peer_shard), st);
    } else {
      store_pose(a.states_out + local, st);
    }
    if (a.weights_out != nullptr) a.weights_out[local] = 1.0;  // make_from_state (particle_traits.hpp:105)
    if (a.ancestors != nullptr) a.ancestors[local] = ancestor;
    if (a.hashes != nullptr) a.hashes[local] = spatial_hash(st, a.hash_resolution[0], a.hash_resolution[1], a.hash_resolution[2]);
    accumulate_moments(m, st, 1.0, a.pivot_x, a.pivot_y);
  }
  finish_block_moments<kRsThreads>(m, s_red, moment_partials, scalars, block, grid, tail);
}

// ---- resample, scatter form (systematic comb on one GPU) ----------------------------------------------
// With the comb t_j = offset + j * stride the slots that pick particle i are exactly those with
// cdf[i-1] <= t_j < cdf[i]: a contiguous slot range [ja, jb) that follows from two integer divisions.
// So instead of a binary search per SLOT (20 dependent probes of the CDF) every PARTICLE reads its two
// CDF entries and stores its state jb - ja times.  Same ancestors as resample_kernel by construction
// (the parity tests compare them with the oracle's lower_bound search); the raw moments are summed per
// particle (count * term) instead of per slot, which moves the estimate at rounding level only.

/// Number of slots j with offset + j * stride < position, i.e. ceil((position - offset) / stride) capped at total_slots, with
/// the division replaced by a multiplication with magic = floor((2^64 - 1) / stride): the high word of x * magic is the
/// quotient or one below it (x < 2^64, so the error of the reciprocal costs less than 1); one remainder check makes it
/// exact.  A 64-bit division is ~150 instructions; this is 8.
__device__ __forceinline__ uint64_t comb_slots_before_magic(unsigned long long position, unsigned long long offset, unsigned long long stride,
                                                           unsigned long long magic, uint64_t total_slots) {
  if (position <= offset) return 0;
  const unsigned long long x = position - offset + stride - 1;
  unsigned long long j = __umul64hi(x, magic);
  if (x - j * stride >= stride) ++j;
  return j < total_slots ? j : total_slots;
}

/// Block `block` of `grid` of the scatter-form resample (resample_scatter_kernel).
template <class Tail>
__device__ __forceinline__ void resample_scatter_block(const ResampleArgs& a, Scalars* __restrict__ scalars, double* __restrict__ moment_partials,
                                                       uint32_t block, uint32_t grid, const Tail& tail) {
  __shared__ double s_red[kMomentCount * kRsThreads / kWarp];
  __shared__ unsigned long long s_comb[3];
  // One GPU: the local CDF is the global one.  Sharded (rank_totals set): positions shift by the totals of
  // the lower ranks and every copy goes to the rank that owns its slot, over NVLink peer memory.
  unsigned long long total = scalars->total, cdf_offset = 0;
  if (a.rank_totals != nullptr) {
    total = 0;
    for (int r = 0; r < a.world; ++r) {
      const unsigned long long t = a.rank_totals[r];
      if (r < a.rank) cdf_offset += t;
      total += t;
    }
  }
  if (threadIdx.x == 0) {  // the two 64-bit divisions of the comb, once per block
    const unsigned long long st = total / a.total_slots;
    s_comb[0] = st;
    s_comb[1] = mulhi64(counter_draw(a.seed, 0, a.step, kStreamSystematic).a, st);
    s_comb[2] = ~0ull / (st != 0 ? st : 1ull);
  }
  __syncthreads();
  const unsigned long long stride = s_comb[0], offset = s_comb[1], magic = s_comb[2];
  // the comb spans total_slots; only the slots below window_end (KLD: the accepted count) are produced
  const uint64_t slot_limit = a.window_end > 0 ? a.window_end : a.total_slots;
  const int lane = threadIdx.x % kWarp;
  double m[kMomentCount];
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) m[k] = 0.0;

  auto store_copy = [&](uint64_t j, const Pose2& st, uint64_t ancestor) {
    if (a.peer_count > 0) {
      const uint64_t owner = j / a.peer_shard;
      store_pose(a.peer_out[owner] + (j - owner * a.peer_shard), st);
    } else {
      store_pose(a.states_out + j, st);
      if (a.weights_out != nullptr) a.weights_out[j] = 1.0;  // make_from_state (particle_traits.hpp:105)
      if (a.ancestors != nullptr) a.ancestors[j] = static_cast<long long>(ancestor);
    }
  };

  // kRsUnroll particles per thread and round: their CDF reads, divisions and state loads are independent, so one thread keeps
  // several 32-byte gathers in flight (the kernel is bound by the latency of cdf -> state -> store, not by bandwidth).
  // Every thread runs the same number of rounds: whole warps stay together for the cooperative stores.
  constexpr uint64_t kOwnCopies = 4;  // up to this many copies a thread stores itself
  const uint64_t per_round = static_cast<uint64_t>(grid) * kRsThreads * kRsUnroll;
  const uint64_t rounds = (a.n_in + per_round - 1) / per_round;
  for (uint64_t round = 0; round < rounds; ++round) {
    const uint64_t first = round * per_round + static_cast<uint64_t>(block) * kRsThreads * kRsUnroll + threadIdx.x;
    uint64_t ja[kRsUnroll], copies[kRsUnroll];
#pragma unroll
    for (int u = 0; u < kRsUnroll; ++u) {
      const uint64_t i = first + static_cast<uint64_t>(u) * kRsThreads;
      ja[u] = 0;
      copies[u] = 0;
      if (i < a.n_in) {
        ja[u] = comb_slots_before_magic(cdf_offset + (i > 0 ? __ldg(a.cdf + i - 1) : 0ull), offset, stride, magic, slot_limit);
        copies[u] = comb_slots_before_magic(cdf_offset + __ldg(a.cdf + i), offset, stride, magic, slot_limit) - ja[u];
      }
    }
    Pose2 st[kRsUnroll];
#pragma unroll
    for (int u = 0; u < kRsUnroll; ++u) {
      st[u] = Pose2{1.0, 0.0, 0.0, 0.0};
      if (copies[u] > 0) st[u] = load_pose(a.states_in + first + static_cast<uint64_t>(u) * kRsThreads);
    }
#pragma unroll
    for (int u = 0; u < kRsUnroll; ++u) {
      const uint64_t i = first + static_cast<uint64_t>(u) * kRsThreads;
      if (copies[u] > 0) {
        const double c = static_cast<double>(copies[u]), dx = st[u].x - a.pivot_x, dy = st[u].y - a.pivot_y;
        m[0] += c;  // every copy has weight 1: sum w = sum w^2 = copies
        m[1] += c;
        m[2] += c * st[u].c;
        m[3] += c * st[u].s;
        m[4] += c * dx;
        m[5] += c * dy;
        m[6] += c * (dx * dx);
        m[7] += c * (dx * dy);
        m[8] += c * (dy * dy);
      }
      if (copies[u] <= kOwnCopies) {
        for (uint64_t j = ja[u]; j < ja[u] + copies[u]; ++j) store_copy(j, st[u], i);
      }
    }
    // Heavy particles: the warp stores their copies together, 32 slots per round.
#pragma unroll
    for (int u = 0; u < kRsUnroll; ++u) {
      unsigned heavy = __ballot_sync(0xffffffffu, copies[u] > kOwnCopies);
      while (heavy != 0u) {
        const int src = __ffs(heavy) - 1;
        heavy &= heavy - 1u;
        const uint64_t hja = __shfl_sync(0xffffffffu, ja[u], src), hcopies = __shfl_sync(0xffffffffu, copies[u], src);
        const uint64_t hi = __shfl_sync(0xffffffffu, first + static_cast<uint64_t>(u) * kRsThreads, src);
        Pose2 hs;
        hs.c = __shfl_sync(0xffffffffu, st[u].c, src);
        hs.s = __shfl_sync(0xffffffffu, st[u].s, src);
        hs.x = __shfl_sync(0xffffffffu, st[u].x, src);
        hs.y = __shfl_sync(0xffffffffu, st[u].y, src);
        for (uint64_t j = hja + lane; j < hja + hcopies; j += kWarp) store_copy(j, hs, hi);
      }
    }
  }
  finish_block_moments<kRsThreads>(m, s_red, moment_partials, scalars, block, grid, tail);
}

}  // namespace

}  // namespace bb200
