// Resample (per-slot and scatter form), normalisation, raw moments and the fixed-order reductions of one filter.
#include "resample.cuh"

#include <algorithm>

namespace bb200 {

namespace {

// ---- normalize -------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kStreamThreads) normalize_kernel(double* __restrict__ weights, uint64_t n, const Scalars* scalars,
                                                                   unsigned long long global_total, double* __restrict__ partials) {
  normalize_block(weights, n, scalars, global_total, partials, LaunchBlocks{});
}

// ---- resample -------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kRsThreads) resample_kernel(ResampleArgs a, Scalars* __restrict__ scalars, double* __restrict__ moment_partials) {
  resample_block(a, scalars, moment_partials, blockIdx.x, gridDim.x, a.tail);
}

__global__ void __launch_bounds__(kRsThreads) resample_box_kernel(ResampleArgs a, Scalars* __restrict__ scalars, double* __restrict__ moment_partials,
                                                                  BoxSpace box) {
  resample_block<StepTail, true>(a, scalars, moment_partials, blockIdx.x, gridDim.x, a.tail, box);
}

__global__ void __launch_bounds__(kRsThreads, kRsBlocksPerSm) resample_scatter_kernel(ResampleArgs a, Scalars* __restrict__ scalars,
                                                                     double* __restrict__ moment_partials) {
  resample_scatter_block(a, scalars, moment_partials, blockIdx.x, gridDim.x, a.tail);
}

// ---- moments / reductions -------------------------------------------------------------------------

__global__ void __launch_bounds__(kStreamThreads) moments_kernel(const Pose2* __restrict__ states, const double* __restrict__ weights, uint64_t n,
                                                                 double px, double py, double* __restrict__ moment_partials) {
  __shared__ double s_red[kMomentCount * kStreamThreads / kWarp];
  double m[kMomentCount];
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) m[k] = 0.0;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kStreamThreads + threadIdx.x; i < n; i += static_cast<uint64_t>(gridDim.x) * kStreamThreads) {
    accumulate_moments(m, load_pose(states + i), weights[i], px, py);
  }
  store_block_moments<kStreamThreads>(m, s_red, moment_partials + static_cast<size_t>(blockIdx.x) * kMomentCount);
}

__global__ void __launch_bounds__(256) reduce_partials_kernel(const double* __restrict__ partials, uint32_t n_partials, int width, double* __restrict__ out) {
  // One block per column; fixed summation order (thread-strided, then the block tree).
  __shared__ double s_red[256 / kWarp];
  const int k = blockIdx.x;
  double v = 0.0;
  for (uint32_t r = threadIdx.x; r < n_partials; r += 256) v = v + partials[static_cast<size_t>(r) * width + k];
  const double total = block_sum<256>(v, s_red);
  if (threadIdx.x == 0) out[k] = total;
}

__global__ void __launch_bounds__(256) fill_kernel(double* __restrict__ out, uint64_t n, double value) {
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x; i < n; i += static_cast<uint64_t>(gridDim.x) * 256) out[i] = value;
}

}  // namespace

void launch_normalize(double* weights, uint64_t n, const Scalars* scalars, unsigned long long global_total, double* partials,
                      uint32_t* n_partials, cudaStream_t stream) {
  const unsigned blocks = static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>((n + kStreamThreads - 1) / kStreamThreads, kStreamMaxBlocks)));
  *n_partials = blocks;
  normalize_kernel<<<blocks, kStreamThreads, 0, stream>>>(weights, n, scalars, global_total, partials);
}

uint32_t resample_block_count(uint64_t slots) { return resample_blocks(slots); }

uint32_t resample_scatter_block_count(uint64_t n_in) { return resample_scatter_blocks(n_in); }

uint32_t launch_resample(const ResampleArgs& args, Scalars* scalars, double* moment_partials, cudaStream_t stream) {
  // The whole set on one GPU with the systematic comb and nothing per slot to draw: scatter form.
  // (Sharded with peer memory and device-side totals: the same, every copy stored into its owner's buffer.)
  const bool plain = args.scheme == 1 && args.random_state_probability <= 0.0 && args.hashes == nullptr && args.span_filter == 0 &&
                     args.peer_hash_count == 0 && args.window_begin == 0 &&
                     args.global_total == 0 && args.cdf_offset == 0 && args.slot_first == 0;
  const bool scatter = plain && ((args.peer_count == 0 && args.rank_totals == nullptr && args.slot_count == args.total_slots) ||
                                 (args.peer_count > 0 && args.rank_totals != nullptr));
  if (scatter) {
    const uint32_t blocks = resample_scatter_block_count(args.n_in);
    resample_scatter_kernel<<<blocks, kRsThreads, 0, stream>>>(args, scalars, moment_partials);
    return blocks;
  }
  const uint32_t blocks = resample_block_count(args.slot_count);
  resample_kernel<<<blocks, kRsThreads, 0, stream>>>(args, scalars, moment_partials);
  return blocks;
}

uint32_t launch_resample(const ResampleArgs& args, const double* box, Scalars* scalars, double* moment_partials, cudaStream_t stream) {
  if (box == nullptr || args.random_state_probability <= 0.0) return launch_resample(args, scalars, moment_partials, stream);
  const uint32_t blocks = resample_block_count(args.slot_count);
  resample_box_kernel<<<blocks, kRsThreads, 0, stream>>>(args, scalars, moment_partials, BoxSpace{box[0], box[1], box[2], box[3]});
  return blocks;
}

uint32_t moments_block_count(uint64_t n) { return moments_blocks(n); }

void launch_moments(const Pose2* states, const double* weights, uint64_t n, double pivot_x, double pivot_y, double* moment_partials,
                    cudaStream_t stream) {
  moments_kernel<<<moments_block_count(n), kStreamThreads, 0, stream>>>(states, weights, n, pivot_x, pivot_y, moment_partials);
}

void launch_fill(double* out, uint64_t n, double value, cudaStream_t stream) {
  if (n == 0) return;
  fill_kernel<<<static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, kStreamMaxBlocks)), 256, 0, stream>>>(out, n, value);
}

void launch_reduce_partials(const double* partials, uint32_t n_partials, int width, double* out, cudaStream_t stream) {
  reduce_partials_kernel<<<width, 256, 0, stream>>>(partials, n_partials, width, out);
}

}  // namespace bb200
