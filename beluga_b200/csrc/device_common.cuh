// Device building blocks shared by the kernel sources: fixed-order block reductions, the rule for which weights can be
// selected, the mbarrier / TMA bulk-copy helpers and the 32-byte state load and store.
#pragma once

#include <cfloat>

#include "kernels.cuh"

namespace bb200 {

namespace {

constexpr int kWarp = 32;

/// Grid cap of the grid-stride streaming launches (normalise, moments, largest weight, fill).
constexpr uint32_t kStreamMaxBlocks = kSmCount * 8;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---- fixed-order block reductions --------------------------------------------------------------

template <int kThreads>
__device__ __forceinline__ double block_sum(double v, double* scratch /* kThreads/32 doubles */) {
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) v = v + __shfl_down_sync(0xffffffffu, v, off);
  const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  __syncthreads();  // scratch may still be read by a previous call
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  double total = 0.0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 0; w < kThreads / kWarp; ++w) total = total + scratch[w];
  }
  return total;  // valid in thread 0
}

/// Fixed-order block sums of K values at once: warp tree per value, one shared-memory round for all
/// of them, then thread 0 adds the per-warp partials in warp order.  Two barriers instead of 2K.
template <int kThreads, int K>
__device__ __forceinline__ void block_sum_many(double* v /* K values, in/out: totals valid in thread 0 */, double* scratch /* K * kThreads/32 */) {
  constexpr int kWarps = kThreads / kWarp;
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int off = kWarp / 2; off > 0; off >>= 1) v[k] = v[k] + __shfl_down_sync(0xffffffffu, v[k], off);
  }
  const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) scratch[k * kWarps + warp] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double total = 0.0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) total = total + scratch[k * kWarps + w];
      v[k] = total;
    }
  }
}

template <int kThreads>
__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, unsigned long long* scratch) {
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) {
    const unsigned long long o = __shfl_down_sync(0xffffffffu, v, off);
    v = o > v ? o : v;
  }
  const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  unsigned long long m = 0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 0; w < kThreads / kWarp; ++w) m = scratch[w] > m ? scratch[w] : m;
  }
  return m;
}

/// The one rule for which weights can be selected: 0 < w <= DBL_MAX.  Zero, negative, NaN and +-inf weights never enter
/// the largest weight and quantise to 0 (a +inf weight would otherwise saturate to 2^64 - 1 and wrap the CDF).
__device__ __forceinline__ bool weight_selectable(double w) { return w > 0.0 && w <= DBL_MAX; }

/// Positive finite weights order like their bit patterns; anything else counts as 0.
__device__ __forceinline__ unsigned long long weight_order_bits(double w) {
  return weight_selectable(w) ? static_cast<unsigned long long>(__double_as_longlong(w)) : 0ull;
}

// ---- TMA 1-D bulk copy of the scan points into shared memory ------------------------------------

__device__ __forceinline__ void mbarrier_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarrier_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbarrier_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_global, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst_smem)),
               "l"(src_global), "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}
__device__ __forceinline__ void mbarrier_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "BB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra BB_DONE;\n"
      "bra BB_WAIT;\n"
      "BB_DONE:\n"
      "}\n" ::"r"(smem_addr(bar)),
      "r"(parity)
      : "memory");
}

// ---- 32-byte states ------------------------------------------------------------------------------

__device__ __forceinline__ Pose2 load_pose(const Pose2* p) {
  const double2 a = *reinterpret_cast<const double2*>(p);
  const double2 b = *(reinterpret_cast<const double2*>(p) + 1);
  return Pose2{a.x, a.y, b.x, b.y};
}
__device__ __forceinline__ void store_pose(Pose2* p, const Pose2& v) {
  *reinterpret_cast<double2*>(p) = make_double2(v.c, v.s);
  *(reinterpret_cast<double2*>(p) + 1) = make_double2(v.x, v.y);
}

}  // namespace

}  // namespace bb200
