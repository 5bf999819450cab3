// Initialisation, the motion update and the execution schedule of the reweight kernels.
#include "cdf.cuh"
#include "propagate.cuh"

namespace bb200 {

namespace {

// ---- initialize_normal (a16) ---------------------------------------------------------------------
// MultivariateNormalDistribution<SE2d>: (x, y, theta) = mean + T * delta, SE2(exp(theta), (x, y))
// (random/multivariate_normal_distribution.hpp:96-103, multivariate_distribution_traits.hpp:110-112).

struct NormalInit {
  double mean[3];
  double t[9];
};

__global__ void __launch_bounds__(256) initialize_normal_kernel(Pose2* states, double* weights, uint64_t n, NormalInit p, uint64_t seed,
                                                                uint64_t first_index) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double d0, d1, d2, unused;
  box_muller(counter_draw(seed, first_index + i, 0, kStreamInit0), d0, d1);
  box_muller(counter_draw(seed, first_index + i, 0, kStreamInit1), d2, unused);
  double v[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) v[r] = p.mean[r] + (p.t[3 * r + 0] * d0 + p.t[3 * r + 1] * d1 + p.t[3 * r + 2] * d2);
  const Rot2 r = rot_exp(v[2]);
  states[i] = Pose2{r.c, r.s, v[0], v[1]};
  weights[i] = 1.0;
}

// initialize_from_map (a16; beluga_ros/include/beluga_ros/amcl.hpp:192-209): max_particles samples of the map
// distribution, weights 1.  Counter stream 6 at step 0, keyed by the global particle index.
__global__ void __launch_bounds__(256) initialize_uniform_kernel(Pose2* states, double* weights, uint64_t n, FreeSpace fs, uint64_t seed,
                                                                 uint64_t first_index) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  store_pose(states + i, random_free_state(fs, counter_draw(seed, first_index + i, 0, kStreamRandomState)));
  weights[i] = 1.0;
}

// ---- propagate (a2 + a6) --------------------------------------------------------------------------
// One thread per particle, original order.  Also accumulates the first and second moments of the
// propagated cloud (block reduction + double atomics); they only feed the execution schedule below,
// never a result, so their summation order does not matter.

__global__ void __launch_bounds__(kPrThreads) propagate_kernel(Pose2* __restrict__ states, uint64_t n, int do_propagate, MotionSampling sampling,
                                                               uint64_t seed, uint32_t step, uint64_t first_index, Schedule* __restrict__ sched) {
  __shared__ double s_red[6 * kPrThreads / kWarp];
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * kPrThreads + threadIdx.x;
  double m[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (i < n) {
    Pose2 st = load_pose(states + i);
    if (do_propagate) {
      st = propagate_one(st, sampling, seed, first_index + i, step);
      store_pose(states + i, st);
    }
    m[0] = st.c, m[1] = st.s, m[2] = st.x, m[3] = st.y, m[4] = st.x * st.x, m[5] = st.y * st.y;
  }
  if (sched != nullptr) {
    block_sum_many<kPrThreads, 6>(m, s_red);
    if (threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < 6; ++k) atomicAdd(&sched->sums[k], m[k]);
    }
  }
}

// ---- execution schedule ---------------------------------------------------------------------------
// The likelihood-field lookup of beam k lands, for two particles, in nearby cells only if their poses
// are close (x, y, and theta scaled by the beam range).  The posterior is wide, so in index order the
// 32 lanes of a warp gather from ~31 distinct 32-byte sectors and the kernel is bound by L2 sector
// bandwidth.  The reweight kernels therefore walk the particles in the order
// of a counting sort over a 3-D grid of pose bins.  This only permutes WHICH THREAD handles a
// particle: weights are written back to the particle's own slot, so every result is independent of it.

constexpr uint32_t kMaxBins = kScheduleMaxBins;

__global__ void schedule_reset_kernel(Schedule* sched) {
  for (int k = 0; k < 6; ++k) sched->sums[k] = 0.0;
  sched->tile_ticket = 0;
}

__global__ void schedule_params_kernel(Schedule* sched, uint64_t n, double mean_range, double min_bin) {
  const double inv_n = 1.0 / static_cast<double>(n);
  const double mx = sched->sums[2] * inv_n, my = sched->sums[3] * inv_n;
  schedule_from_moments(*sched, sched->sums[0] * inv_n, sched->sums[1] * inv_n, mx, my, sched->sums[4] * inv_n - mx * mx,
                        sched->sums[5] * inv_n - my * my, static_cast<double>(n), mean_range, min_bin);
}

__device__ __forceinline__ uint32_t schedule_bin(const Schedule& g, const Pose2& st) {
  // heading relative to the mean as u = 2 tan(dtheta / 2): monotone in dtheta, one division instead of an atan2
  const double cr = st.c * g.c0 + st.s * g.s0, sr = st.s * g.c0 - st.c * g.s0;
  const double u = cr > -0.4 ? 2.0 * sr / (1.0 + cr) : (sr >= 0.0 ? 1e6 : -1e6);
  // CDF value of each coordinate (single precision: the bin only decides which thread handles the particle)
  const float zt = static_cast<float>(u) * g.kt, zx = static_cast<float>(st.x - g.mx) * g.kx, zy = static_cast<float>(st.y - g.my) * g.ky;
  const float ft = __fdividef(static_cast<float>(g.nt), 1.0f + __expf(-zt));  // exp overflow -> 0, underflow -> count: the edge bins
  const float fx = __fdividef(static_cast<float>(g.nx), 1.0f + __expf(-zx));
  const float fy = __fdividef(static_cast<float>(g.ny), 1.0f + __expf(-zy));
  const int bt = min(max(__float2int_rz(ft), 0), static_cast<int>(g.nt) - 1);  // NaN converts to 0
  int bx = min(max(__float2int_rz(fx), 0), static_cast<int>(g.nx) - 1);
  int by = min(max(__float2int_rz(fy), 0), static_cast<int>(g.ny) - 1);
  // Boustrophedon order: every other row runs backwards in x and every other plane backwards in y, so that consecutive
  // bins are always neighbours (a warp crossing a row end would otherwise span the whole cloud).
  if (bt & 1) by = static_cast<int>(g.ny) - 1 - by;
  const uint32_t row = static_cast<uint32_t>(bt) * g.ny + static_cast<uint32_t>(by);
  if (row & 1u) bx = static_cast<int>(g.nx) - 1 - bx;
  return row * g.nx + static_cast<uint32_t>(bx);
}

/// propagate with the histogram of the execution schedule fused in (the bin grid comes from the host's prediction).
__global__ void __launch_bounds__(kPrThreads) propagate_binned_kernel(Pose2* __restrict__ states, uint64_t n, MotionSampling sampling, uint64_t seed,
                                                                      uint32_t step, uint64_t first_index, Schedule grid,
                                                                      uint2* __restrict__ bin_rank, uint32_t* __restrict__ counters) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * kPrThreads + threadIdx.x;
  if (i < n) {
    const Pose2 st = propagate_one(load_pose(states + i), sampling, seed, first_index + i, step);
    store_pose(states + i, st);
    const uint32_t b = schedule_bin(grid, st);
    // The particle's arrival rank inside its bin: the scatter pass then needs no second round of atomics.  (Which
    // particle gets which rank varies from run to run; it only permutes the execution order inside a bin.)
    const uint32_t rank = atomicAdd(counters + b, 1u);
    bin_rank[i] = make_uint2(b, rank);
  }
}

constexpr int kPlaceItems = 4;  // particles per thread: the bin-offset gathers of one thread are independent
__global__ void __launch_bounds__(256) schedule_place_kernel(const uint2* __restrict__ bin_rank, uint64_t n, const uint32_t* __restrict__ offsets,
                                                             uint32_t* __restrict__ perm) {
  const uint64_t first = static_cast<uint64_t>(blockIdx.x) * (256 * kPlaceItems) + threadIdx.x;
  uint2 br[kPlaceItems];
  uint32_t off[kPlaceItems];
#pragma unroll
  for (int k = 0; k < kPlaceItems; ++k) {
    const uint64_t i = first + static_cast<uint64_t>(k) * 256;
    br[k] = i < n ? __ldcs(bin_rank + i) : make_uint2(0u, 0u);
  }
#pragma unroll
  for (int k = 0; k < kPlaceItems; ++k) off[k] = __ldg(offsets + br[k].x);
#pragma unroll
  for (int k = 0; k < kPlaceItems; ++k) {
    const uint64_t i = first + static_cast<uint64_t>(k) * 256;
    if (i < n) perm[off[k] + br[k].y] = static_cast<uint32_t>(i);
  }
}

__global__ void __launch_bounds__(256) schedule_histogram_kernel(const Pose2* __restrict__ states, uint64_t n, const Schedule* __restrict__ sched,
                                                                 uint32_t* __restrict__ bins, uint32_t* __restrict__ counters) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  const uint32_t b = schedule_bin(*sched, load_pose(states + i));
  bins[i] = b;
  atomicAdd(counters + b, 1u);
}

__global__ void __launch_bounds__(256) schedule_scatter_kernel(const uint32_t* __restrict__ bins, uint64_t n, uint32_t* __restrict__ offsets,
                                                               uint32_t* __restrict__ perm) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  perm[atomicAdd(offsets + bins[i], 1u)] = static_cast<uint32_t>(i);
}

}  // namespace

void launch_initialize_normal(Pose2* states, double* weights, uint64_t n, const double mean[3], const double transform[9], uint64_t seed,
                              uint64_t first_index, cudaStream_t stream) {
  if (n == 0) return;
  NormalInit p;
  for (int i = 0; i < 3; ++i) p.mean[i] = mean[i];
  for (int i = 0; i < 9; ++i) p.t[i] = transform[i];
  initialize_normal_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(states, weights, n, p, seed, first_index);
}

void launch_initialize_uniform(Pose2* states, double* weights, uint64_t n, const uint32_t* free_cells, uint64_t n_free, int grid_width,
                               double grid_resolution, const Pose2& grid_origin, uint64_t seed, uint64_t first_index, cudaStream_t stream) {
  if (n == 0) return;
  const FreeSpace fs{free_cells, n_free, grid_width, grid_resolution, grid_origin};
  initialize_uniform_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(states, weights, n, fs, seed, first_index);
}

void launch_propagate(Pose2* states, uint64_t n, bool do_propagate, const MotionSampling& sampling, uint64_t seed, uint32_t step,
                      uint64_t first_index, Schedule* sched, cudaStream_t stream) {
  if (n == 0) return;
  if (sched != nullptr) schedule_reset_kernel<<<1, 1, 0, stream>>>(sched);
  propagate_kernel<<<static_cast<unsigned>((n + kPrThreads - 1) / kPrThreads), kPrThreads, 0, stream>>>(states, n, do_propagate ? 1 : 0, sampling,
                                                                                                      seed, step, first_index, sched);
}

void launch_propagate_binned(Pose2* states, uint64_t n, const MotionSampling& sampling, uint64_t seed, uint32_t step, uint64_t first_index,
                             const Schedule& grid, uint2* bin_rank, uint32_t* counters, Schedule* /*sched*/, cudaStream_t stream) {
  if (n == 0) return;
  propagate_binned_kernel<<<static_cast<unsigned>((n + kPrThreads - 1) / kPrThreads), kPrThreads, 0, stream>>>(
      states, n, sampling, seed, step, first_index, grid, bin_rank, counters);
}

uint32_t schedule_max_bins() { return kMaxBins; }
uint32_t schedule_tile_count() { return (kMaxBins + kScanTile - 1) / kScanTile; }

void launch_build_schedule(const Pose2* states, uint64_t n, Schedule* sched, uint32_t* bins, uint32_t* counters, uint32_t* perm,
                           unsigned long long* tile_state, double mean_range, double min_bin, cudaStream_t stream) {
  if (n == 0) return;
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  cudaMemsetAsync(counters, 0, kMaxBins * sizeof(uint32_t), stream);
  cudaMemsetAsync(tile_state, 0, schedule_tile_count() * sizeof(unsigned long long), stream);
  schedule_params_kernel<<<1, 1, 0, stream>>>(sched, n, mean_range, min_bin);
  schedule_histogram_kernel<<<blocks, 256, 0, stream>>>(states, n, sched, bins, counters);
  launch_scan_u32_prepared(counters, counters, kMaxBins, &sched->tile_ticket, tile_state, nullptr, stream);
  schedule_scatter_kernel<<<blocks, 256, 0, stream>>>(bins, n, counters, perm);
}

void launch_finish_schedule(const uint2* bin_rank, uint64_t n, uint32_t n_bins, Schedule* sched, uint32_t* counters, uint32_t* perm,
                            unsigned long long* tile_state, cudaStream_t stream) {
  if (n == 0) return;
  // (Scanning the counters in the tail of propagate_binned_kernel -- its last block -- was tried: one SM reading 250 KB
  // in dependent 16-byte steps was several times slower than sixteen look-back tiles on a B200.)
  const unsigned blocks = static_cast<unsigned>((n + 256 * kPlaceItems - 1) / (256 * kPlaceItems));
  launch_scan_u32_prepared(counters, counters, n_bins, &sched->tile_ticket, tile_state, nullptr, stream);
  schedule_place_kernel<<<blocks, 256, 0, stream>>>(bin_rank, n, counters, perm);
}

}  // namespace bb200
