// Block body of the landmark and bearing reweight (reweight_landmark.cu), shared with the batch kernels.  Apart from
// reweight_landmark.cuh, which the host probe compiles without CUDA.
#pragma once

#include "device_common.cuh"
#include "reweight_landmark.cuh"

namespace bb200 {

namespace {

constexpr int kLandmarkThreads = 256;
constexpr uint32_t kLandmarkDetChunk = 32;   // detections staged per shared-memory chunk (2 KB)
constexpr uint32_t kLandmarkChunk = 256;     // candidates staged per shared-memory chunk (8 KB)

// One thread per particle, block `block` of a grid of kLandmarkThreads-thread blocks.  Every particle of a CTA walks the
// same detections and the same candidate slices, so the shared-memory reads are broadcasts and the search loop does not
// diverge.  The first minimum of each slice is kept (std::min_element), the factors are multiplied in libstdc++'s
// grouping of four, and w *= that product.
template <int kModel>
__device__ __forceinline__ void reweight_landmark_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n,
                                                        const LandmarkParams& params, const LandmarkPoint* __restrict__ landmarks,
                                                        const LandmarkDetection* __restrict__ detections, uint32_t n_detections,
                                                        Scalars* __restrict__ scalars, uint32_t block) {
  __shared__ LandmarkDetection s_det[kLandmarkDetChunk];
  __shared__ LandmarkPoint s_lm[kLandmarkChunk];
  __shared__ unsigned long long s_red[kLandmarkThreads / kWarp];
  const uint64_t i = static_cast<uint64_t>(block) * kLandmarkThreads + threadIdx.x;
  const bool active = i < n;
  Pose2 st{1.0, 0.0, 0.0, 0.0};
  double w = 0.0;
  if (active) {
    st = load_pose(states + i);
    w = weights[i];
  }
  const LandmarkFrame f = landmark_frame(st, params);
  ProductByFours prod;
  for (uint32_t base = 0; base < n_detections; base += kLandmarkDetChunk) {
    const uint32_t count = min(kLandmarkDetChunk, n_detections - base);
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < count; k += kLandmarkThreads) s_det[k] = detections[base + k];
    __syncthreads();
    for (uint32_t k = 0; k < count; ++k) {
      const LandmarkDetection& d = s_det[k];
      const Vec3 query = kModel == BB200_SENSOR_BEARING ? Vec3{0.0, 0.0, 0.0} : lm_query(f, d);
      uint32_t best = d.begin;
      double best_key = 0.0;
      for (uint32_t first = d.begin; first < d.end; first += kLandmarkChunk) {
        const uint32_t chunk = min(kLandmarkChunk, d.end - first);
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < chunk; j += kLandmarkThreads) s_lm[j] = landmarks[first + j];
        __syncthreads();
        for (uint32_t j = 0; j < chunk; ++j) {
          const double key = landmark_key<kModel>(f, d, query, s_lm[j]);
          if (first + j == d.begin || landmark_better<kModel>(key, best_key)) best = first + j, best_key = key;
        }
      }
      const bool found = d.end > d.begin;
      prod.push(landmark_factor<kModel>(f, d, found, found ? landmarks[best] : LandmarkPoint{0.0, 0.0, 0.0, 0.0}, params));
    }
  }
  if (active) {
    w = w * prod.finish();
    weights[i] = w;
  }
  const unsigned long long m = block_max_u64<kLandmarkThreads>(active ? weight_order_bits(w) : 0ull, s_red);
  if (threadIdx.x == 0 && m != 0) atomicMax(&scalars->wmax_bits, m);
}

}  // namespace

}  // namespace bb200
