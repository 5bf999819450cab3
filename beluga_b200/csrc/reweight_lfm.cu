// Likelihood-field reweight of one filter: the general kernel (maps beyond kFixedMaxSide), the fixed-point kernel with
// the scan staged in shared memory, and the persistent fixed-point kernel with the scan in the constant bank.
#include "reweight_lfm.cuh"

#include <cstring>

#include <algorithm>

namespace bb200 {

namespace {

__global__ void __launch_bounds__(kRwThreads, kRwGeneralBlocksPerSm)
    reweight_lfm_kernel(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, const uint32_t* __restrict__ perm,
                        FieldView field, const double2* __restrict__ points, uint32_t n_points, double points_radius,
                        Scalars* __restrict__ scalars) {
  reweight_lfm_block(states, weights, n, perm, field, points, n_points, points_radius, scalars, static_cast<uint64_t>(blockIdx.x) * kRwThreads);
}

/// Scan points as a kernel parameter: they sit in the constant bank -- no shared-memory load per beam and no L1
/// data-pipe traffic.  Both loops read them with register-indexed LDC.64, two per beam.  30 KB of the 32 KB parameter
/// space; longer scans take the shared-memory (TMA) variant.
constexpr uint32_t kParamBeams = 1920;
struct ScanParam {
  double2 p[kParamBeams];
};

/// Scan in the constant bank: nothing is shared between the warps of a CTA, so the grid is persistent
/// (CTAs/SM x SM count) and every WARP draws the next 32 particles of the schedule from a global
/// ticket counter.  A CTA-per-256-particles grid loses time to its slowest warp (each CTA holds its
/// SM slot until the last of its warps is through 1080 beams) and to the partial last wave.
/// P = 2: lane l of a 64-slot task weighs the particles of slots l and l + 32 in one loop: each scan point is read once
/// for both, and the loop control is shared.  Each gather instruction still covers 32 consecutive slots (a few pose bins,
/// so a few table lines); adjacent slots (2l, 2l + 1) spread one instruction over twice as many bins and are slower.
template <int P>
__global__ void __launch_bounds__(kRwThreads, P == 1 ? kRwBlocksPerSm : kRwPairBlocksPerSm)
    reweight_lfm_fixed_param_kernel(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, const uint32_t* __restrict__ perm,
                                    FieldView field, uint32_t n_points, double points_radius, Scalars* __restrict__ scalars,
                                    const __grid_constant__ ScanParam scan) {
  const int lane = threadIdx.x % kWarp;
  constexpr int kTask = kWarp * P;  // a task = the next kWarp * P particles of the schedule
  const unsigned long long n_tasks = (n + kTask - 1) / kTask;
  unsigned long long* ticket_counter = &scalars->work_ticket;
  unsigned long long ticket = __shfl_sync(0xffffffffu, lane == 0 ? atomicAdd(ticket_counter, 1ull) : 0ull, 0);
  unsigned long long best = 0ull;
  while (ticket < n_tasks) {
    // Draw the next ticket now; its round trip to L2 hides behind this task's beams.
    const unsigned long long next = lane == 0 ? atomicAdd(ticket_counter, 1ull) : 0ull;
    bool active[P];  // idle slots of the last task walk the beams with a dummy pose
    uint64_t i[P];
    uint32_t margin_start[P];
    FixedPose q[P];
    double acc[P];
#pragma unroll
    for (int k = 0; k < P; ++k) {
      const uint64_t slot = ticket * kTask + static_cast<uint64_t>(k) * kWarp + lane;
      active[k] = slot < n;
      i[k] = slot_particle(perm, slot, active[k]);
    }
    bool inside = fixed_pose_setup(field, states, i[0], active[0], points_radius, q[0], margin_start[0]);
#pragma unroll
    for (int k = 1; k < P; ++k) inside &= fixed_pose_setup(field, states, i[k], active[k], points_radius, q[k], margin_start[k]);
    const FixedGrid grid = fixed_grid_setup(field, inside);
#pragma unroll
    for (int k = 0; k < P; ++k) acc[k] = field.init;
    fixed_sum<P>(field, states, grid, q, margin_start, i, active, scan.p, n_points, acc);
#pragma unroll
    for (int k = 0; k < P; ++k) {
      if (active[k]) {
        const unsigned long long bits = store_reweighted(field, weights, i[k], weights[i[k]], acc[k]);
        best = bits > best ? bits : best;
      }
    }
    ticket = __shfl_sync(0xffffffffu, next, 0);
  }
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) {
    const unsigned long long o = __shfl_down_sync(0xffffffffu, best, off);
    best = o > best ? o : best;
  }
  if (lane == 0) {
    if (best != 0ull) atomicMax(&scalars->wmax_bits, best);
    // The last warp out rewinds the ticket counter for the next launch.
    const unsigned long long warps = static_cast<unsigned long long>(gridDim.x) * (kRwThreads / kWarp);
    if (atomicAdd(&scalars->work_done, 1ull) + 1ull == warps) {
      scalars->work_done = 0ull;
      *ticket_counter = 0ull;
    }
  }
}

__global__ void __launch_bounds__(kRwThreads, kRwBlocksPerSm)
    reweight_lfm_fixed_kernel(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, const uint32_t* __restrict__ perm,
                              FieldView field, const double2* __restrict__ points, uint32_t n_points, double points_radius,
                              Scalars* __restrict__ scalars) {
  reweight_lfm_fixed_block(states, weights, n, perm, field, points, n_points, points_radius, scalars, static_cast<uint64_t>(blockIdx.x) * kRwThreads);
}

}  // namespace

uint32_t fixed_index_bias(uint32_t border_pitch) { return kFixedBiasY * (4u * border_pitch) + kFixedBiasX; }

int sm_count() {
  static thread_local int cached_device = -1, cached = 0;
  int device = 0;
  cudaGetDevice(&device);
  if (device != cached_device) {
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, device);
    cached_device = device;
  }
  return cached > 0 ? cached : static_cast<int>(kSmCount);
}

void launch_reweight_lfm(const Pose2* states, double* weights, uint64_t n, const uint32_t* perm, const FieldView& field,
                         const double* points_xy_device, const double* points_xy_host, uint32_t n_points, double points_radius, Scalars* scalars,
                         cudaStream_t stream) {
  if (n == 0) return;
  const unsigned blocks = static_cast<unsigned>((n + kRwThreads - 1) / kRwThreads);
  const size_t smem = static_cast<size_t>(n_points < kChunkBeams ? n_points : kChunkBeams) * sizeof(double2);
  const double2* points = reinterpret_cast<const double2*>(points_xy_device);
  if (field.use_fixed) {
    static thread_local ScanParam scan;  // launch parameters are copied at launch time
    if (points_xy_host != nullptr && n_points <= kParamBeams) {
      std::memcpy(scan.p, points_xy_host, static_cast<size_t>(n_points) * sizeof(double2));
      // Two particles per thread halve the warps with work: worth it only while the pair tasks still fill every resident
      // warp kRwPairFill times over (811 009 particles and more on a 132-SM H100).
      const uint64_t pair_tasks = (n + 2 * kWarp - 1) / (2 * kWarp);
      const uint64_t pair_warps = static_cast<uint64_t>(sm_count()) * kRwPairBlocksPerSm * (kRwThreads / kWarp);
      if (pair_tasks >= kRwPairFill * pair_warps) {
        const unsigned ctas_needed = static_cast<unsigned>((n + 2 * kRwThreads - 1) / (2 * kRwThreads));
        const unsigned persistent = std::min<unsigned>(static_cast<unsigned>(sm_count()) * kRwPairBlocksPerSm, ctas_needed);
        reweight_lfm_fixed_param_kernel<2><<<persistent, kRwThreads, 0, stream>>>(states, weights, n, perm, field, n_points, points_radius, scalars, scan);
      } else {
        const unsigned ctas_needed = static_cast<unsigned>((n + kRwThreads - 1) / kRwThreads);
        const unsigned persistent = std::min<unsigned>(static_cast<unsigned>(sm_count()) * kRwBlocksPerSm, ctas_needed);
        reweight_lfm_fixed_param_kernel<1><<<persistent, kRwThreads, 0, stream>>>(states, weights, n, perm, field, n_points, points_radius, scalars, scan);
      }
    } else {
      reweight_lfm_fixed_kernel<<<blocks, kRwThreads, smem, stream>>>(states, weights, n, perm, field, points, n_points, points_radius, scalars);
    }
  } else {
    reweight_lfm_kernel<<<blocks, kRwThreads, smem, stream>>>(states, weights, n, perm, field, points, n_points, points_radius, scalars);
  }
}

}  // namespace bb200
