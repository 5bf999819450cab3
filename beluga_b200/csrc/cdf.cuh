// Block bodies of the fixed-point CDF build (cdf.cu), shared with the batch kernels: the largest weight, the
// quantise + scan tile and the decoupled look-back scan machinery.
#pragma once

#include "device_common.cuh"

namespace bb200 {

namespace {

constexpr int kMaxThreads = 512;

/// Block `block` of `grid` of max_weight_kernel: the largest positive finite weight into scalars->wmax_bits.
__device__ __forceinline__ void max_weight_block(const double* __restrict__ weights, uint64_t n, Scalars* scalars, uint32_t block, uint32_t grid) {
  __shared__ unsigned long long s_red[kMaxThreads / kWarp];
  unsigned long long m = 0;
  for (uint64_t i = static_cast<uint64_t>(block) * kMaxThreads + threadIdx.x; i < n; i += static_cast<uint64_t>(grid) * kMaxThreads) {
    const unsigned long long b = weight_order_bits(weights[i]);
    m = b > m ? b : m;
  }
  m = block_max_u64<kMaxThreads>(m, s_red);
  if (threadIdx.x == 0 && m != 0) atomicMax(&scalars->wmax_bits, m);
}

/// Block `block` of `grid` of apply_factors_kernel: w_i = w_i * factors_i, the multiply of the built-in reweight
/// (store_reweighted), and the largest selectable product into scalars->wmax_bits.  24 bytes per particle.
__device__ __forceinline__ void apply_factors_block(double* __restrict__ weights, const double* __restrict__ factors, uint64_t n, Scalars* scalars,
                                                    uint32_t block, uint32_t grid) {
  __shared__ unsigned long long s_red[kMaxThreads / kWarp];
  unsigned long long m = 0;
  for (uint64_t i = static_cast<uint64_t>(block) * kMaxThreads + threadIdx.x; i < n; i += static_cast<uint64_t>(grid) * kMaxThreads) {
    const double updated = weights[i] * factors[i];
    weights[i] = updated;
    const unsigned long long b = weight_order_bits(updated);
    m = b > m ? b : m;
  }
  m = block_max_u64<kMaxThreads>(m, s_red);
  if (threadIdx.x == 0 && m != 0) atomicMax(&scalars->wmax_bits, m);
}

// ---- fixed-point CDF ------------------------------------------------------------------------------
// q_i = floor(w_i * 2^e) with e chosen so that the largest weight lands in [2^(P-1), 2^P),
// P = min(52, 62 - ceil(log2(N_global))): the total stays below 2^62 and integer addition is
// associative, so the CDF is identical for any scan order, tile size or number of ranks.

constexpr int kScanThreads = 512;
constexpr int kScanItems = 8;
constexpr uint32_t kScanTile = kScanThreads * kScanItems;
// tile_state word: [63:62] flag (0 empty, 1 aggregate, 2 inclusive prefix), [61:0] value
constexpr unsigned long long kFlagAggregate = 1ull << 62, kFlagPrefix = 2ull << 62, kValueMask = (1ull << 62) - 1;

__device__ __forceinline__ void prepare_cdf_scalars(Scalars* s, double wmax, int ceil_log2_count) {
  int ex = 0;
  const bool ok = weight_selectable(wmax);
  if (ok) (void)frexp(wmax, &ex);
  const int p = min(52, 62 - ceil_log2_count);
  s->exponent = p - ex;
  s->valid = ok ? 1 : 0;
  s->tile_ticket = 0;
  s->total = 0;
}

/// Inclusive scan of per-thread totals across the block (warp shuffles + one smem hop).
template <int kThreads>
__device__ __forceinline__ unsigned long long block_inclusive_scan_u64(unsigned long long v, unsigned long long* warp_sums,
                                                                        unsigned long long& block_total) {
  const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
#pragma unroll
  for (int off = 1; off < kWarp; off <<= 1) {
    const unsigned long long o = __shfl_up_sync(0xffffffffu, v, off);
    if (lane >= off) v += o;
  }
  if (lane == kWarp - 1) warp_sums[warp] = v;
  __syncthreads();
  if (warp == 0) {
    unsigned long long ws = lane < kThreads / kWarp ? warp_sums[lane] : 0ull;
#pragma unroll
    for (int off = 1; off < kWarp; off <<= 1) {
      const unsigned long long o = __shfl_up_sync(0xffffffffu, ws, off);
      if (lane >= off) ws += o;
    }
    if (lane < kThreads / kWarp) warp_sums[lane] = ws;
  }
  __syncthreads();
  block_total = warp_sums[kThreads / kWarp - 1];
  return v + (warp > 0 ? warp_sums[warp - 1] : 0ull);
}

/// Decoupled look-back: returns the exclusive prefix of this tile and publishes its inclusive one.
/// Warp 0 inspects 32 predecessors per round (one coalesced read of the tile words) instead of walking
/// them one L2 round trip at a time.
__device__ __forceinline__ unsigned long long lookback_exclusive_prefix(unsigned long long* tile_state, uint32_t tile,
                                                                         unsigned long long tile_total, unsigned long long* s_prefix) {
  if (threadIdx.x < kWarp) {
    const int lane = threadIdx.x;
    unsigned long long exclusive = 0;
    if (tile == 0) {
      if (lane == 0) atomicExch(&tile_state[0], kFlagPrefix | tile_total);
    } else {
      if (lane == 0) atomicExch(&tile_state[tile], kFlagAggregate | tile_total);
      int32_t window = static_cast<int32_t>(tile) - 1;  // newest predecessor of this round
      for (;;) {
        const int32_t look = window - lane;
        unsigned long long word;
        do {  // tiles before tile 0 count as a published prefix of zero
          word = look >= 0 ? *reinterpret_cast<volatile unsigned long long*>(&tile_state[look]) : (2ull << 62);
        } while (__any_sync(0xffffffffu, (word >> 62) == 0));
        const unsigned prefixes = __ballot_sync(0xffffffffu, (word >> 62) == 2);
        const int last = prefixes != 0 ? __ffs(prefixes) - 1 : kWarp - 1;  // nearest tile that already knows its prefix
        unsigned long long v = lane <= last ? (word & kValueMask) : 0ull;
#pragma unroll
        for (int off = kWarp / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        exclusive += v;
        if (prefixes != 0) break;
        window -= kWarp;
      }
      if (lane == 0) atomicExch(&tile_state[tile], kFlagPrefix | (exclusive + tile_total));
    }
    if (lane == 0) *s_prefix = exclusive;
  }
  __syncthreads();
  return *s_prefix;
}

// Tile of the CDF build: 256 threads x 8 consecutive weights (two 32-byte sectors per thread, read and written with
// 16-byte accesses).  The quantisation is a multiplication by 2^e (exact, like scalbn, wherever the result is >= 1),
// split into two power-of-two factors so that each stays a normal double for any exponent.
constexpr int kQsThreads = 256;
constexpr int kQsItems = 8;  // 16 halves the tiles per byte but was slower at 12.5M on a B200 (not re-measured on the H100)
constexpr uint32_t kQsTile = kQsThreads * kQsItems;

__device__ __forceinline__ double pow2_double(int e) {  // |e| <= 1000
  return __longlong_as_double(static_cast<long long>(e + 1023) << 52);
}
__device__ __forceinline__ unsigned long long quantize_mul(double w, double f1, double f2) {
  return weight_selectable(w) ? __double2ull_rd((w * f1) * f2) : 0ull;
}

/// derive_exponent: the fused step -- the exponent comes from scalars->wmax_bits here (no prepare_cdf launch; the
/// tile holding element 0 publishes exponent / valid for the host); otherwise scalars->exponent / valid are given.
/// One tile of the CDF build; `tile` counts from the set's first weight.
__device__ __forceinline__ void quantize_scan_tile(const double* __restrict__ weights, uint64_t n, unsigned long long* __restrict__ cdf,
                                                   Scalars* scalars, unsigned long long* tile_state, uint32_t tile, int derive_exponent,
                                                   int ceil_log2_count) {
  __shared__ unsigned long long s_warp[kQsThreads / kWarp];
  __shared__ unsigned long long s_prefix;
  int exponent, valid_flag;
  if (derive_exponent) {  // every thread derives the exponent itself: a broadcast load and a few integer operations
    const double wmax = __longlong_as_double(static_cast<long long>(scalars->wmax_bits));
    int ex = 0;
    const bool ok = weight_selectable(wmax);
    if (ok) (void)frexp(wmax, &ex);
    exponent = min(52, 62 - ceil_log2_count) - ex;
    valid_flag = ok ? 1 : 0;
    if (tile == 0 && threadIdx.x == 0) {
      scalars->exponent = exponent;
      scalars->valid = valid_flag;
    }
  } else {
    exponent = scalars->exponent;
    valid_flag = scalars->valid;
  }
  const int e1 = exponent / 2;
  const double f1 = pow2_double(e1), f2 = pow2_double(exponent - e1);
  const bool valid = valid_flag != 0;

  const uint64_t base = static_cast<uint64_t>(tile) * (kQsThreads * kQsItems) + static_cast<uint64_t>(threadIdx.x) * kQsItems;
  unsigned long long q[kQsItems];
  unsigned long long local = 0;
  if (base + kQsItems <= n) {
    const double2* src = reinterpret_cast<const double2*>(weights + base);
#pragma unroll
    for (int k = 0; k < kQsItems / 2; ++k) {
      const double2 w = __ldcs(src + k);  // read once: streaming
      // Degenerate weight set (no positive finite weight): fall back to a uniform CDF.
      q[2 * k] = valid ? quantize_mul(w.x, f1, f2) : (1ull << 20);
      q[2 * k + 1] = valid ? quantize_mul(w.y, f1, f2) : (1ull << 20);
      local += q[2 * k] + q[2 * k + 1];
    }
  } else {
#pragma unroll
    for (int k = 0; k < kQsItems; ++k) {
      const uint64_t idx = base + k;
      q[k] = idx < n ? (valid ? quantize_mul(weights[idx], f1, f2) : (1ull << 20)) : 0ull;
      local += q[k];
    }
  }
  unsigned long long tile_total;
  const unsigned long long inclusive = block_inclusive_scan_u64<kQsThreads>(local, s_warp, tile_total);
  const unsigned long long prefix = lookback_exclusive_prefix(tile_state, tile, tile_total, &s_prefix);
  unsigned long long running = prefix + inclusive - local;
  if (base + kQsItems <= n) {
    ulonglong2* dst = reinterpret_cast<ulonglong2*>(cdf + base);
#pragma unroll
    for (int k = 0; k < kQsItems / 2; ++k) {
      ulonglong2 v;
      running += q[2 * k];
      v.x = running;
      running += q[2 * k + 1];
      v.y = running;
      dst[k] = v;
    }
  } else {
#pragma unroll
    for (int k = 0; k < kQsItems; ++k) {
      const uint64_t idx = base + k;
      running += q[k];
      if (idx < n) cdf[idx] = running;
    }
  }
  if (base <= n - 1 && n - 1 < base + kQsItems) scalars->total = prefix + inclusive;  // thread holding the last element
}

}  // namespace

}  // namespace bb200
