// Block bodies of the likelihood-field reweight (reweight_lfm.cu), shared with the batch kernels: the general lookup,
// the fixed-point cell lookup and the shared-memory (TMA) staging of the scan.
#pragma once

#include "device_common.cuh"

namespace bb200 {

namespace {

// ---- reweight (likelihood field; a3 + a5) --------------------------------------------------------

// Fixed-point kernels, measured with bench.py (reweight_lfm_fixed_param_kernel, 1M x 1080 beams) on an H100 80GB HBM3
// (SXM): at a 400 W power limit 3 CTAs/SM -> 1.12 ms, 4 -> 1.47 ms, 5 -> 1.80 ms; at 700 W, 3 CTAs/SM with unroll 1 ->
// 0.99 ms, unroll 2 -> 0.99 ms (slightly slower, and the shared-memory kernels spill).  6 CTAs/SM spills in every kernel.
// The two-particle param kernel (slots l, l + 32) at a 400 W power limit, 1M: 2 CTAs/SM -> 1.046-1.050 ms, 3 -> 1.069-1.072
// ms, against 1.141-1.178 ms for the one-particle kernel (DESIGN section 4, item 8).  kRwThreads is the B200's choice.
constexpr int kRwThreads = 256;  // x kRwBlocksPerSm CTAs per SM
constexpr int kRwBlocksPerSm = 3;
constexpr int kRwPairBlocksPerSm = 2;  // the two-particle variant of reweight_lfm_fixed_param_kernel (126 registers)
constexpr uint64_t kRwPairFill = 6;      // pair tasks per resident warp below which one particle per thread is faster
constexpr int kRwUnroll = 1;  // iterations of the fixed-point kernels' eight-beam loop body unrolled
// The general kernel (reweight_lfm_kernel, maps beyond kFixedMaxSide) keeps the B200 sweep's (4 CTAs/SM, unroll 2).
constexpr int kRwGeneralBlocksPerSm = 4;
constexpr int kRwGeneralUnroll = 2;  // groups of four beams in flight per thread
constexpr uint32_t kChunkBeams = 2048; // beams staged per shared-memory chunk (32 KB), multiple of 4

/// floor(g) as int32 for |g| < 2^31: one F2I.F64.FLOOR (saturating).
__device__ __forceinline__ int floor_to_int_fast(double g) { return __double2int_rd(g); }

template <bool kFast>
__device__ __forceinline__ double field_lookup(const FieldView& f, double px, double py, double c, double s, double tx, double ty) {
  // likelihood_field_model.hpp:82-83 -- two products, one difference/sum, one offset; each rounded.
  const double x = (px * c - py * s) + tx;
  const double y = (px * s + py * c) + ty;
  // regular_grid.hpp:75-78 -- floor(p * inv_resolution) cast to int.
  const double gx = x * f.inv_resolution;
  const double gy = y * f.inv_resolution;
  int xi, yi;
  if (kFast) {
    xi = floor_to_int_fast(gx);
    yi = floor_to_int_fast(gy);
  } else {
    // General path: saturating conversion; non-finite coordinates fall outside the grid.
    const double fx = floor(gx), fy = floor(gy);
    xi = (fx >= 0.0 && fx < 2147483647.0) ? static_cast<int>(fx) : -1;
    yi = (fy >= 0.0 && fy < 2147483647.0) ? static_cast<int>(fy) : -1;
  }
  // dense_grid.hpp:92-96 contains().  Out-of-grid end points read the spare cell that holds
  // f(unknown_space_occupancy_prob), so the load is unconditional (no divergent branch).
  const bool inside = static_cast<unsigned>(xi) < static_cast<unsigned>(f.width) && static_cast<unsigned>(yi) < static_cast<unsigned>(f.height);
  const uint32_t ux = static_cast<uint32_t>(xi), uy = static_cast<uint32_t>(yi);
  uint32_t idx = (((uy >> 2) * static_cast<uint32_t>(f.tiles_x) + (ux >> 2)) << 4) | ((uy & 3u) << 2) | (ux & 3u);
  idx = inside ? idx : f.spare_index;
  return __ldg(f.tiled + idx);
}

/// acc + the sum of lookup(pts[b]) over b < count in libstdc++ std::transform_reduce's order (numeric:439-462): groups of
/// four, acc + ((f0+f1)+(f2+f3)), then one at a time.  kUnroll: groups per unrolled iteration (1 compiles as no pragma does).
template <int kUnroll, class Lookup>
__device__ __forceinline__ double transform_reduce_exact(const double2* pts, uint32_t count, double acc, Lookup lookup) {
  uint32_t b = 0;
#pragma unroll kUnroll
  for (; b + 4 <= count; b += 4) {
    const double2 p0 = pts[b], p1 = pts[b + 1], p2 = pts[b + 2], p3 = pts[b + 3];
    const double f0 = lookup(p0), f1 = lookup(p1), f2 = lookup(p2), f3 = lookup(p3);
    acc = acc + ((f0 + f1) + (f2 + f3));
  }
  for (; b < count; ++b) acc = acc + lookup(pts[b]);
  return acc;
}

/// The particle in schedule slot `slot` (perm: the schedule's order, nullptr for the identity); idle slots read particle 0.
__device__ __forceinline__ uint64_t slot_particle(const uint32_t* __restrict__ perm, uint64_t slot, bool active) {
  return active ? (perm != nullptr ? perm[slot] : slot) : 0;
}

/// transform = world_to_likelihood_field * state (likelihood_field_model.hpp:70-74); idle threads use the identity.
__device__ __forceinline__ Pose2 field_frame_pose(const FieldView& f, const Pose2* __restrict__ states, uint64_t i, bool active) {
  return pose_mul(f.world_to_field, active ? load_pose(states + i) : Pose2{1.0, 0.0, 0.0, 0.0});
}

/// Stores particle i's new weight, its weight w times the likelihood its sum of field values gives (actions/reweight.hpp:54-60),
/// and returns the new weight's order bits.  w is weights[i] itself or a copy read earlier.
__device__ __forceinline__ unsigned long long store_reweighted(const FieldView& f, double* __restrict__ weights, uint64_t i, const double& w,
                                                               double sum) {
  const double likelihood = f.exp_epilogue ? exp(sum) : sum;
  const double updated = w * likelihood;
  weights[i] = updated;
  return weight_order_bits(updated);
}

/// Block-wide max of the weight bit patterns without a closing barrier: every warp folds its max
/// into a shared word and the last warp to arrive publishes the block's value.  Warps that finish
/// their beams early retire instead of idling at a __syncthreads.
__device__ __forceinline__ void publish_weight_max(unsigned long long bits, unsigned long long* s_max, unsigned int* s_arrived,
                                                   unsigned int n_warps, Scalars* scalars) {
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) {
    const unsigned long long o = __shfl_down_sync(0xffffffffu, bits, off);
    bits = o > bits ? o : bits;
  }
  if (threadIdx.x % kWarp == 0) {
    atomicMax(s_max, bits);
    __threadfence_block();
    if (atomicAdd(s_arrived, 1u) + 1u == n_warps) {
      const unsigned long long m = atomicMax(s_max, 0ull);  // read the final value
      if (m != 0) atomicMax(&scalars->wmax_bits, m);
    }
  }
}

/// The shared-memory body of one CTA's reweight: the scan goes to shared memory in kChunkBeams-point chunks by TMA bulk
/// copy (completion on an mbarrier), `chunk(pts, count)` runs on each chunk, and the order bits that `weight_bits()`
/// returns after the last one go into the block's weight max.
template <class Chunk, class WeightBits>
__device__ __forceinline__ void staged_scan_block(const double2* __restrict__ points, uint32_t n_points, Scalars* __restrict__ scalars,
                                                  Chunk chunk, WeightBits weight_bits) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double2* s_pts = reinterpret_cast<double2*>(smem_raw);
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ unsigned long long s_max;
  __shared__ unsigned int s_arrived;
  if (threadIdx.x == 0) {
    s_max = 0ull;
    s_arrived = 0u;
    mbarrier_init(&s_bar, 1);
    mbarrier_init_fence();
  }
  __syncthreads();  // barrier and s_max initialised
  uint32_t phase = 0;
  for (uint32_t base = 0; base < n_points; base += kChunkBeams) {
    const uint32_t count = min(kChunkBeams, n_points - base);
    if (threadIdx.x == 0) {
      const uint32_t bytes = count * static_cast<uint32_t>(sizeof(double2));
      mbarrier_expect_tx(&s_bar, bytes);
      bulk_copy_g2s(s_pts, points + base, bytes, &s_bar);
    }
    mbarrier_wait(&s_bar, phase);
    phase ^= 1u;
    chunk(s_pts, count);
    if (base + kChunkBeams < n_points) __syncthreads();  // s_pts is about to be overwritten by the next chunk
  }
  publish_weight_max(weight_bits(), &s_max, &s_arrived, kRwThreads / kWarp, scalars);
}

/// One CTA of the general likelihood-field reweight: the particles in schedule slots [slot_base, slot_base + kRwThreads).
__device__ __forceinline__ void reweight_lfm_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n,
                                                   const uint32_t* __restrict__ perm, const FieldView& field, const double2* __restrict__ points,
                                                   uint32_t n_points, double points_radius, Scalars* __restrict__ scalars, uint64_t slot_base) {
  const uint64_t slot = slot_base + threadIdx.x;
  const bool active = slot < n;
  const uint64_t i = slot_particle(perm, slot, active);
  const double w = active ? weights[i] : 0.0;
  const Pose2 t = field_frame_pose(field, states, i, active);
  // Fast floor is exact while every |coordinate * inv_resolution| stays below 2^30.
  const double reach = (points_radius + fmax(fabs(t.x), fabs(t.y))) * field.inv_resolution;
  const bool fast = reach < 1073741824.0;  // false for NaN
  double acc = field.init;
  staged_scan_block(
      points, n_points, scalars,
      [&](const double2* pts, uint32_t count) {
        if (!active) return;
        acc = fast ? transform_reduce_exact<kRwGeneralUnroll>(pts, count, acc, [&](double2 p) { return field_lookup<true>(field, p.x, p.y, t.c, t.s, t.x, t.y); })
                   : transform_reduce_exact<kRwGeneralUnroll>(pts, count, acc, [&](double2 p) { return field_lookup<false>(field, p.x, p.y, t.c, t.s, t.x, t.y); });
      },
      [&] { return active ? store_reweighted(field, weights, i, w, acc) : 0ull; });
}

// ---- reweight, fixed-point cell lookup ----------------------------------------------------------------
// Same result as reweight_lfm_kernel, two thirds of the instructions per beam.  The reference rounds
// after every operation of   x = (px*c - py*s) + tx;  cell = floor(x * inv_resolution)   (4 mul, 4 add,
// 2 mul and 2 floor conversions per beam, all on the FP64 pipe).  The CELL is all that matters, so the
// kernel evaluates   g = fma(px, c*inv, fma(-py, s*inv, tx*inv + 1))   (2 fma per coordinate; the +1 is
// the border cell), which differs from the reference's value by d <= 11 * 2^13 * 2^-53 < 2^-36 cells
// while every term stays below 2^13 cells, and adds 1.5*2^20 (y): in the sum's bit pattern the low word is
// the fraction of g in units of 2^-32 (round to nearest) and the low 20 bits of the high word are
// 2^19 + floor(g).  If the fraction word is not zero, g is at least 2^-33 > d away from an integer and
// floor(reference value) = floor(g) exactly.  x adds 1.5*2^18 instead, so its high word carries
// floor(4g) -- x already shifted into the place the 4x4-tile index wants it -- and a non-zero fraction
// word puts g at least 2^-35 > d from an integer.  A thread that ever sees a zero fraction word (2^-32 per
// coordinate, about once every two steps among a million particles) or a particle out of the 2^13 range
// redoes its beams with the reference's own operation sequence; nothing else in the loop branches.
// Out-of-grid end points clamp (one DPX add-min per coordinate, which also strips the bias) to the
// one-cell border holding the unknown-space value, so the load is unconditional.  A warp whose particles all keep their
// end points inside the grid (fixed_pose_setup) needs neither: it runs the loop with fixed_lookup<true>.

constexpr double kFixedMagicX = 393216.0;   // 1.5 * 2^18: ulp 2^-34; high word = 0x41180000 + floor(4 g)    for |g| < 2^17
constexpr double kFixedMagicY = 1572864.0;  // 1.5 * 2^20: ulp 2^-32; high word = 0x41380000 + floor(g)      for |g| < 2^19
constexpr uint32_t kFixedBiasX = 0x41180000u, kFixedBiasY = 0x41380000u;
// The magic constants ride in the FMAs' addend (per-particle offsets ox, oy below), which saves the two additions per beam
// but lets THREE roundings at the magic's ulp into the word instead of one (the offset sum and both FMAs): the computed
// fixed-point value is within 3 half-ulps + 2^-36 cells of the reference's.  Two ulps of guard are added to the offset so
// that the reference's value lies in (computed - 4.07 ulp, computed + 0.07 ulp): the high word is the reference's cell
// whenever the fraction word is at least 5.  tests/test_fixed_point_lookup_model.py replays this with exact rationals,
// including end points a hair (2^-36 .. 2^-30 cells) either side of a cell edge at arbitrary headings.
constexpr double kFixedGuardX = 1.16415321826934814453125e-10; // 2^-33 = 2 ulp of kFixedMagicX
constexpr double kFixedGuardY = 4.656612873077392578125e-10;   // 2^-31 = 2 ulp of kFixedMagicY
constexpr uint32_t kFixedAmbiguous = 4u;  // fraction words 0..4: the cell is not decided (5 * 2^-32 per coordinate)

struct FixedPose {
  double cx, sx;         // cos, sin of the field-frame heading, times 1/resolution
  double ox, oy;         // field-frame position in cells, plus the border cell, plus magic constant and guard
};

/// The table geometry, held once per thread however many particles it weighs.
struct FixedGrid {
  uint32_t x_max, y_max; // 4 (width + 1) + 3, height + 1: largest 4 * padded x (+ 2 fraction bits) and padded y
  uint32_t row_pitch;    // 4 * 2^kx: elements per row of cells (four rows of tiles' worth per tile row)
  bool in_grid;          // warp-uniform: every end point of every particle of the warp lies inside the grid
};

/// `margin` collects the smallest fraction word seen (<= kFixedAmbiguous: a coordinate too close to a cell edge to call).
/// x arrives as 4 * padded x with two fraction bits below it, y as padded y: the element index
///   (y >> 2) * 16 * tiles_per_row  +  (x >> 2) * 16 + (x & 3) * 4 + (y & 3)
/// is then one bit-select (y's low two bits replace x's fraction bits), one mask and one multiply-add.
/// kInGrid: the warp's end points all lie inside the grid, so the clamp is the identity and is left out, and so is the
/// bias: both bias words are multiples of 4, so the biased words give the index plus fixed_index_bias(pitch) (mod 2^32),
/// and `table` is the base moved back by that much (FieldView::bordered_biased).
template <bool kInGrid>
__device__ __forceinline__ double fixed_lookup(const double* __restrict__ table, const FixedGrid& g, const FixedPose& q, double px, double py,
                                               uint32_t& margin) {
  const double gx = fma(px, q.cx, fma(-py, q.sx, q.ox));  // gx + 1 + magic + guard
  const double gy = fma(px, q.sx, fma(py, q.cx, q.oy));   // gy + 1 + magic + guard
  margin = __vimin3_u32(margin, static_cast<uint32_t>(__double2loint(gx)), static_cast<uint32_t>(__double2loint(gy)));
  uint32_t ux = static_cast<uint32_t>(__double2hiint(gx));  // bias + 4 * padded x + 2 fraction bits
  uint32_t uy = static_cast<uint32_t>(__double2hiint(gy));  // bias + padded y
  if (!kInGrid) {
    // min(word - bias, max): a negative coordinate wraps to a huge unsigned and clamps to the far border,
    // which holds the same unknown-space value as the near one.
    ux = __viaddmin_u32(ux, 0u - kFixedBiasX, g.x_max);
    uy = __viaddmin_u32(uy, 0u - kFixedBiasY, g.y_max);
  }
  uint32_t low;  // (ux & ~3) | (uy & 3) as ONE bit-select (the compiler splits it into two operations)
  asm("lop3.b32 %0, %1, 3, %2, 0xB8;" : "=r"(low) : "r"(ux), "r"(uy));
  const uint32_t idx = (uy & ~3u) * g.row_pitch + low;
  return __ldg(table + idx);
}

/// The reference's operation sequence (field_lookup) against the bordered layout.
__device__ __forceinline__ double bordered_lookup_exact(const FieldView& f, double px, double py, double c, double s, double tx, double ty) {
  const double x = (px * c - py * s) + tx;
  const double y = (px * s + py * c) + ty;
  const double fx = floor(x * f.inv_resolution), fy = floor(y * f.inv_resolution);
  // saturating: anything outside [-1, side] (NaN included) lands on the border
  const int xi = (fx >= 0.0 && fx < static_cast<double>(f.width)) ? static_cast<int>(fx) : -1;
  const int yi = (fy >= 0.0 && fy < static_cast<double>(f.height)) ? static_cast<int>(fy) : -1;
  return __ldg(f.bordered + bordered_index(static_cast<uint32_t>(xi + 1), static_cast<uint32_t>(yi + 1), f.border_kx));
}

// A thread weighs P particles (q[k], acc[k], margin[k]; one FixedGrid) against every point it reads, each particle's sum in
// libstdc++ transform_reduce's order (transform_reduce_exact).

/// f[j][k]: the table value at point b + j for particle k.
template <int P, bool kInGrid>
__device__ __forceinline__ void fixed_group(double (&f)[4][P], const double2* pts, uint32_t b, const FieldView& field,
                                            const FixedGrid& grid, const FixedPose (&q)[P], uint32_t (&margin)[P]) {
  const double* table = kInGrid ? field.bordered_biased : field.bordered;
  const double2 p0 = pts[b], p1 = pts[b + 1], p2 = pts[b + 2], p3 = pts[b + 3];
#pragma unroll
  for (int k = 0; k < P; ++k) {
    f[0][k] = fixed_lookup<kInGrid>(table, grid, q[k], p0.x, p0.y, margin[k]);
    f[1][k] = fixed_lookup<kInGrid>(table, grid, q[k], p1.x, p1.y, margin[k]);
    f[2][k] = fixed_lookup<kInGrid>(table, grid, q[k], p2.x, p2.y, margin[k]);
    f[3][k] = fixed_lookup<kInGrid>(table, grid, q[k], p3.x, p3.y, margin[k]);
  }
}

template <int P>
__device__ __forceinline__ void fixed_add(double (&acc)[P], const double (&f)[4][P]) {
#pragma unroll
  for (int k = 0; k < P; ++k) acc[k] = acc[k] + ((f[0][k] + f[1][k]) + (f[2][k] + f[3][k]));
}

/// The fixed-point sums of pts[0, count) onto acc, from FieldView::bordered_biased for kInGrid, else from bordered.
template <int P, bool kInGrid>
__device__ __forceinline__ void fixed_beams(const double2* pts, uint32_t count, const FieldView& field, const FixedGrid& grid,
                                            const FixedPose (&q)[P], double (&acc)[P], uint32_t (&margin)[P]) {
  uint32_t b = 0;
  if (4 <= count) {
    // Software pipeline: the loads of the next four beams are issued before the previous four are summed (a warp issues
    // in order: summing first would leave it with four loads in flight, then none).  Two groups per iteration, loaded
    // alternately into f and g: no register copies between groups.
    double f[4][P], g[4][P];
    fixed_group<P, kInGrid>(f, pts, 0, field, grid, q, margin);
    b = 4;
#pragma unroll kRwUnroll
    for (; b + 8 <= count; b += 8) {
      fixed_group<P, kInGrid>(g, pts, b, field, grid, q, margin);
      fixed_add<P>(acc, f);
      fixed_group<P, kInGrid>(f, pts, b + 4, field, grid, q, margin);
      fixed_add<P>(acc, g);
    }
    if (b + 4 <= count) {
      fixed_group<P, kInGrid>(g, pts, b, field, grid, q, margin);
      fixed_add<P>(acc, f);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int k = 0; k < P; ++k) f[j][k] = g[j][k];
      }
      b += 4;
    }
    fixed_add<P>(acc, f);
  }
  for (; b < count; ++b) {
    const double2 p = pts[b];
#pragma unroll
    for (int k = 0; k < P; ++k) acc[k] = acc[k] + fixed_lookup<kInGrid>(kInGrid ? field.bordered_biased : field.bordered, grid, q[k], p.x, p.y, margin[k]);
  }
}

/// Adds the field values of pts[0, count) to the P sums acc: the fixed-point loop, then the reference's own operation
/// sequence from the sum it started with for a particle whose margin ends at or below kFixedAmbiguous.  `pts` is the
/// ScanParam in the constant bank or a chunk in shared memory.
template <int P>
__device__ __forceinline__ void fixed_sum(const FieldView& field, const Pose2* __restrict__ states, const FixedGrid& grid,
                                          const FixedPose (&q)[P], const uint32_t (&margin_start)[P], const uint64_t (&i)[P],
                                          const bool (&active)[P], const double2* pts, uint32_t count, double (&acc)[P]) {
  double acc_before[P];
  uint32_t margin[P];
#pragma unroll
  for (int k = 0; k < P; ++k) acc_before[k] = acc[k], margin[k] = margin_start[k];
  if (grid.in_grid) {
    fixed_beams<P, true>(pts, count, field, grid, q, acc, margin);
  } else {
    fixed_beams<P, false>(pts, count, field, grid, q, acc, margin);
  }
#pragma unroll
  for (int k = 0; k < P; ++k) {
    if (margin[k] <= kFixedAmbiguous) {  // a coordinate within ~2^-30 cells of a cell edge, or a particle out of range
      const Pose2 t = field_frame_pose(field, states, i[k], active[k]);
      acc[k] = transform_reduce_exact<1>(pts, count, acc_before[k],
                                         [&](double2 p) { return bordered_lookup_exact(field, p.x, p.y, t.c, t.s, t.x, t.y); });
    }
  }
}

/// Per-particle constants of the fixed-point evaluation.  Returns whether every end point of the particle stays inside
/// the grid.
__device__ __forceinline__ bool fixed_pose_setup(const FieldView& field, const Pose2* __restrict__ states, uint64_t i, bool active,
                                                 double points_radius, FixedPose& q, uint32_t& margin_start) {
  const Pose2 t = field_frame_pose(field, states, i, active);
  const double inv = field.inv_resolution;
  // The error bound above needs every term of g below 2^13 cells.
  const double reach = (points_radius + fmax(fabs(t.x), fabs(t.y))) * inv + 2.0;
  margin_start = reach < 8100.0 ? 0xFFFFFFFFu : 0u;  // 0 also for NaN: straight to the exact sequence
  q.cx = t.c * inv, q.sx = t.s * inv;
  q.ox = (t.x * inv + 1.0) + (kFixedMagicX + kFixedGuardX);
  q.oy = (t.y * inv + 1.0) + (kFixedMagicY + kFixedGuardY);
  // points_radius bounds |px| + |py|, so every end point lies within points_radius * inv cells of (t.x, t.y) in each
  // coordinate, give or take rounding far below the two cells added.  A square inside [0, width) x [0, height) keeps every
  // reference cell inside the grid (reach < 8100 then holds too: width, height <= kFixedMaxSide).  False for NaN.
  const double cells = points_radius * inv + 2.0;
  const double gx = t.x * inv, gy = t.y * inv;
  return gx - cells >= 0.0 && gx + cells < static_cast<double>(field.width) && gy - cells >= 0.0 &&
         gy + cells < static_cast<double>(field.height);
}

/// The table geometry, and whether every particle of the warp (`inside`: all of this thread's) keeps its end points in the grid.
__device__ __forceinline__ FixedGrid fixed_grid_setup(const FieldView& field, bool inside) {
  FixedGrid g;
  g.x_max = field.border_x_max;
  g.y_max = field.border_y_max;
  g.row_pitch = 4u * field.border_pitch;
  g.in_grid = __all_sync(0xffffffffu, inside) && field.bordered_biased != nullptr;
  return g;
}

/// Scan staged in shared memory by TMA (scans longer than kParamBeams points): one CTA per kRwThreads particles, the
/// schedule slots [slot_base, slot_base + kRwThreads).
__device__ __forceinline__ void reweight_lfm_fixed_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n,
                                                         const uint32_t* __restrict__ perm, const FieldView& field, const double2* __restrict__ points,
                                                         uint32_t n_points, double points_radius, Scalars* __restrict__ scalars, uint64_t slot_base) {
  const uint64_t slot = slot_base + threadIdx.x;
  const bool active[1] = {slot < n};
  const uint64_t i[1] = {slot_particle(perm, slot, active[0])};
  uint32_t margin_start[1];
  FixedPose q[1];
  const FixedGrid grid = fixed_grid_setup(field, fixed_pose_setup(field, states, i[0], active[0], points_radius, q[0], margin_start[0]));
  double acc[1] = {field.init};
  staged_scan_block(
      points, n_points, scalars,
      [&](const double2* pts, uint32_t count) { fixed_sum<1>(field, states, grid, q, margin_start, i, active, pts, count, acc); },
      [&] { return active[0] ? store_reweighted(field, weights, i[0], weights[i[0]], acc[0]) : 0ull; });
}

}  // namespace

}  // namespace bb200
