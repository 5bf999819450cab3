// Block bodies of the beam-model reweight (reweight_beam.cu), shared with the batch kernels: the fused kernel's ray walk
// and mixture, and the two passes (walk, mixture) of the two-pass form.
#pragma once

#include "device_common.cuh"

namespace bb200 {

namespace {

// ---- reweight (beam model; a4 + a5) -----------------------------------------------------------
// BeamSensorModel (sensor/beam_model.hpp:104-150): one thread per particle, beams in the inner
// loop, so the lanes of a warp (neighbouring particles, same beam) walk rays of similar length.
// Ray casting is Ray2d::cast (algorithm/raycasting.hpp:79-107) over the standard Bresenham2i
// iterator (algorithm/raycasting/bresenham.hpp:84-160) on the int8 occupancy grid.

struct BeamRay {
  double far_x, far_y;  // bearing.unit_complex() * max_range  (raycasting.hpp:83)
  double z;             // measured range (beam_model.hpp:116)
  double short_decay;   // exp(-lambda_short * z) of the short-reading term (:137-141)
};

/// The largest span, in cells along either axis, for which the reference's int Bresenham arithmetic (bresenham.hpp:84-160)
/// cannot overflow: error + dyspan <= 4 * span < 2^31.
constexpr int kMaxRaySpan = (1 << 29) - 1;

/// regular_grid.hpp:75-78 for the source cell of a ray: floor(p * inv_resolution), or -1 when that is NaN or outside
/// [0, 2^31).  Such a source lies outside every grid (the reference's cast<int>() gives INT_MIN there on x86-64), so
/// every ray from it is a miss.
__device__ __forceinline__ int source_cell(double p, double inv_resolution) {
  const double c = floor(p * inv_resolution);
  return c >= 0.0 && c < 0x1p31 ? static_cast<int>(c) : -1;
}

/// The far-end cell of coordinate e (regular_grid.hpp:75-78, raycasting.hpp:81-85) as a span from the source cell s,
/// clamped to +-kMaxRaySpan.  Within the clamp this is the reference's span exactly (floor(e * inv_resolution) and s are
/// integers below 2^53); beyond it the reference's arithmetic overflows, and the far end is pulled back per axis.  A ray
/// with a non-finite end point is a miss: the caller decides that (for NaN this still returns a span within the clamp).
__device__ __forceinline__ int far_span(double e, double inv_resolution, int s) {
  const double span = floor(e * inv_resolution) - static_cast<double>(s);
  return static_cast<int>(fmin(fmax(span, -static_cast<double>(kMaxRaySpan)), static_cast<double>(kMaxRaySpan)));
}

/// One ray of Ray2d::cast (raycasting.hpp:79-107) over the standard Bresenham2i iterator (bresenham.hpp:84-160) as a
/// state machine (ray_step is one dependent load of the free-distance map plus a closed-form advance of the
/// iterator; the walk is bound by that load's latency).
struct RayWalk {
  int x, y;            // iterator position: x along the longer axis (swapped when `reversed`)
  int xstep, ystep;
  int xspan, dxspan, dyspan;
  int error, step;
  uint32_t recip;      // floor((2^32 - 1) / dxspan): quotients below 2^8 come out exact or one low
  bool reversed, small_span, active;
  int hit_x, hit_y;    // cell of the first non-free cell (valid when hit)
  bool hit;
};

__device__ __forceinline__ void ray_begin(RayWalk& w, int sx, int sy, int fx, int fy) {
  int xspan = fx - sx, xstep = 1;
  if (xspan < 0) {
    xspan = -xspan;
    xstep = -1;
  }
  int yspan = fy - sy, ystep = 1;
  if (yspan < 0) {
    yspan = -yspan;
    ystep = -1;
  }
  w.x = sx, w.y = sy;
  w.reversed = false;
  if (xspan < yspan) {  // iterate along the longer axis (bresenham.hpp:99-105)
    int t = w.x; w.x = w.y; w.y = t;
    t = xspan; xspan = yspan; yspan = t;
    t = xstep; xstep = ystep; ystep = t;
    w.reversed = true;
  }
  w.xstep = xstep, w.ystep = ystep;
  w.xspan = xspan, w.dxspan = 2 * xspan, w.dyspan = 2 * yspan;
  w.small_span = xspan < (1 << 22);  // then error + 255 * dyspan stays below 2^32
  w.recip = xspan > 0 ? 0xFFFFFFFFu / static_cast<uint32_t>(w.dxspan) : 0u;
  w.error = xspan;
  w.step = 0;
  w.active = true;
  w.hit = false;
  w.hit_x = w.hit_y = 0;
}

/// One iteration: inspect the current cell, then jump as far as the free-distance map allows.
__device__ __forceinline__ void ray_step(RayWalk& w, const OccupancyView& g) {
  const int cx = w.reversed ? w.y : w.x, cy = w.reversed ? w.x : w.y;
  if (!(static_cast<unsigned>(cx) < static_cast<unsigned>(g.width) && static_cast<unsigned>(cy) < static_cast<unsigned>(g.height))) {
    w.active = false;  // take_while(cell_is_valid), raycasting.hpp:86-87: a miss
    return;
  }
  const int d = __ldg(g.free_distance + (static_cast<size_t>(cy) * static_cast<size_t>(g.width) + static_cast<size_t>(cx)));
  if (d == 0) {  // !free_at: first non-free cell on the line
    w.hit = true;
    w.hit_x = cx, w.hit_y = cy;
    w.active = false;
    return;
  }
  // Every cell within Chebyshev distance d - 1 is free and the line moves at most one cell per step in each axis,
  // so the next d - 1 cells cannot stop the ray: advance d steps of the iterator (bresenham.hpp:122-160, standard
  // variant) in closed form.  error stays in (0, dxspan].
  const int k = min(d, w.xspan - w.step);
  if (k == 0) {  // the far end cell was free too: sentinel reached (bresenham.hpp:179)
    w.active = false;
    return;
  }
  w.step += k;
  w.x += k * w.xstep;
  int m;  // floor((t - 1) / dxspan) with t = error + k * dyspan
  if (w.small_span) {
    // 32-bit: t - 1 < 2^32 and the quotient is at most k <= 255, so the high word of (t - 1) * floor((2^32 - 1) / dxspan)
    // is the quotient or one below it; one remainder check makes it exact.  (A 64-bit division costs more than the
    // rest of the loop; an FP64 reciprocal needs two conversions on the quarter-rate pipe.)
    const uint32_t tm1 = static_cast<uint32_t>(w.error) + static_cast<uint32_t>(k) * static_cast<uint32_t>(w.dyspan) - 1u;
    uint32_t q = __umulhi(tm1, w.recip);
    uint32_t r = tm1 - q * static_cast<uint32_t>(w.dxspan);
    if (r >= static_cast<uint32_t>(w.dxspan)) {
      ++q;
      r -= static_cast<uint32_t>(w.dxspan);
    }
    m = static_cast<int>(q);
    w.error = static_cast<int>(r) + 1;  // t - m * dxspan
  } else {
    const long long t = static_cast<long long>(w.error) + static_cast<long long>(k) * w.dyspan;
    m = static_cast<int>((t - 1) / w.dxspan);
    w.error = static_cast<int>(t - static_cast<long long>(m) * w.dxspan);
  }
  w.y += m * w.ystep;
}

/// Distance in metres from the source cell centroid to the ray's hit cell (clamped to max_range), or -1 on a miss;
/// d2 = squared cell distance of that cell (only meaningful on a hit).
__device__ __forceinline__ double ray_result(const RayWalk& w, const OccupancyView& g, int sx, int sy, double max_range, unsigned long long& d2) {
  if (!w.hit) return -1.0;
  const double dxm = (static_cast<double>(w.hit_x) + 0.5) * g.resolution - (static_cast<double>(sx) + 0.5) * g.resolution;
  const double dym = (static_cast<double>(w.hit_y) + 0.5) * g.resolution - (static_cast<double>(sy) + 0.5) * g.resolution;
  const long long ix = static_cast<long long>(w.hit_x) - sx, iy = static_cast<long long>(w.hit_y) - sy;
  d2 = static_cast<unsigned long long>(ix * ix + iy * iy);
  return fmin(sqrt(dxm * dxm + dym * dym), max_range);
}

/// beam_model.hpp:128-135: the two normalisers as functions of z_mean.
__device__ __forceinline__ double2 beam_normalisers(const BeamParams& p, double z_mean) {
  const double sqrt2 = sqrt(2.);
  const double eta_hit = 2. / (erf((p.beam_max_range - z_mean) / (sqrt2 * p.sigma_hit)) - erf(-z_mean / (sqrt2 * p.sigma_hit)));
  const double eta_short = 1. / (1. - exp(-p.lambda_short * z_mean));
  return make_double2(eta_hit, eta_short);
}

/// The four-term mixture cubed (beam_model.hpp:125-147); short_decay = exp(-lambda_short * z), a per-beam constant.
__device__ __forceinline__ double beam_pz3(const BeamParams& p, double z, double short_decay, double z_mean, double n, double eta_hit, double eta_short) {
  const double d = (z - z_mean) / p.sigma_hit;
  double pz = p.z_hit * eta_hit * n * exp(-(d * d) / 2.);
  if (z < z_mean) pz += p.z_short * p.lambda_short * eta_short * short_decay;
  if (z < p.beam_max_range) {
    pz += p.z_rand / p.beam_max_range;
  } else {
    pz += p.z_max;
  }
  return pz * pz * pz;
}

constexpr int kBeamThreads = 256;
constexpr int kBeamBlocksPerSm = 3;  // chosen on a B200, not re-measured on the H100
constexpr uint32_t kBeamChunk = 1024;  // rays staged per shared-memory chunk (32 KB), multiple of 4

/// One CTA of the fused beam reweight: the particles in schedule slots [block * kBeamThreads, (block + 1) * kBeamThreads).
__device__ __forceinline__ void reweight_beam_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n,
                                                    const uint32_t* __restrict__ perm, const OccupancyView& grid, const BeamParams& params,
                                                    const double2* __restrict__ points, uint32_t n_points, Scalars* __restrict__ scalars,
                                                    uint32_t block) {
  __shared__ BeamRay s_rays[kBeamChunk];
  __shared__ unsigned long long s_red[kBeamThreads / kWarp];
  const uint64_t slot = static_cast<uint64_t>(block) * kBeamThreads + threadIdx.x;
  const bool active = slot < n;
  const uint64_t i = active ? (perm != nullptr ? perm[slot] : slot) : 0;

  Pose2 st{1.0, 0.0, 0.0, 0.0};
  double w = 0.0;
  if (active) {
    st = load_pose(states + i);
    w = weights[i];
  }
  // Ray2d: source pose in the grid frame and its cell (raycasting.hpp:67-70).
  const Pose2 src = pose_mul(grid.world_to_grid, st);
  const int sx = source_cell(src.x, grid.inv_resolution), sy = source_cell(src.y, grid.inv_resolution);
  const double n_norm = 1. / (sqrt(2. * 3.14159265358979323846) * params.sigma_hit);  // beam_model.hpp:107

  // The mixture value of one beam given its ray walk (beam_model.hpp:116-147).
  auto beam_value = [&](const BeamRay& ray, const RayWalk& walk) {
    unsigned long long d2 = 0;
    const double hit = ray_result(walk, grid, sx, sy, params.beam_max_range, d2);
    const double z_mean = hit >= 0.0 ? hit : params.beam_max_range;  // value_or(beam_max_range)
    double2 eta;
    if (params.eta != nullptr) {
      // hit within range: the entry of its cell distance; miss or clamped to the range: the last entry
      const bool in_table = hit >= 0.0 && hit < params.beam_max_range && d2 + 1 < params.eta_entries;
      eta = __ldg(params.eta + (in_table ? static_cast<uint32_t>(d2) : params.eta_entries - 1u));
    } else {
      eta = beam_normalisers(params, z_mean);
    }
    return beam_pz3(params, ray.z, ray.short_decay, z_mean, n_norm, eta.x, eta.y);
  };
  auto begin_walk = [&](RayWalk& walk, const BeamRay& ray) {
    // far end = r1 * t2 + t1 (raycasting.hpp:81-85)
    const double ex = (src.c * ray.far_x - src.s * ray.far_y) + src.x;
    const double ey = (src.s * ray.far_x + src.c * ray.far_y) + src.y;
    ray_begin(walk, sx, sy, sx + far_span(ex, grid.inv_resolution, sx), sy + far_span(ey, grid.inv_resolution, sy));
    if (!(isfinite(ex) && isfinite(ey))) walk.active = false;  // e.g. a NaN heading: the end point lies outside the grid, a miss
  };
  auto walk_ray = [&](const BeamRay& ray) {
    RayWalk walk;
    begin_walk(walk, ray);
    while (walk.active) ray_step(walk, grid);
    return beam_value(ray, walk);
  };

  double acc = 0.0;
  for (uint32_t base = 0; base < n_points; base += kBeamChunk) {
    const uint32_t count = min(kBeamChunk, n_points - base);
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < count; b += kBeamThreads) {
      const double2 p = points[base + b];
      const double z = sqrt(p.x * p.x + p.y * p.y);                      // beam_model.hpp:116
      const double bx = p.x / z, by = p.y / z;                            // :120-123
      s_rays[b] = BeamRay{bx * params.beam_max_range, by * params.beam_max_range, z, exp(-params.lambda_short * z)};
    }
    __syncthreads();
    if (active) {
      uint32_t b = 0;
      for (; b + 4 <= count; b += 4) {  // transform_reduce grouping (numeric:439-462)
        const double f0 = walk_ray(s_rays[b]), f1 = walk_ray(s_rays[b + 1]), f2 = walk_ray(s_rays[b + 2]), f3 = walk_ray(s_rays[b + 3]);
        acc = acc + ((f0 + f1) + (f2 + f3));
      }
      for (; b < count; ++b) acc = acc + walk_ray(s_rays[b]);
    }
  }
  if (active) {
    w = w * acc;
    weights[i] = w;
  }
  const unsigned long long m = block_max_u64<kBeamThreads>(active ? weight_order_bits(w) : 0ull, s_red);
  if (threadIdx.x == 0 && m != 0) atomicMax(&scalars->wmax_bits, m);
}

// ---- beam model in two passes ----------------------------------------------------------------------
// The fused kernel above carries the ray walk (integer, one dependent load per iteration) and the mixture (FP64:
// sqrt, exp, three dozen constants) in one register allocation: 78 registers and a long instruction stream per
// beam.  Split: the WALK writes the hit cell of every (particle, beam) as one 32-bit word -- beam-major, so a
// warp's 32 particles store and later load consecutive words -- and the MIXTURE reads it back.  4 bytes per ray each
// way (2.9 GB at 1M x 720: under a millisecond of HBM time) buy a 40-register walk kernel at twice the occupancy
// and a branch-free mixture loop.  Hit words: 0xFFFFFFFF = miss, else cy << 16 | cx (grids up to 65535 cells a side).

constexpr uint32_t kHitMiss = 0xFFFFFFFFu;
constexpr int kWalkBlocksPerSm = 8;  // resident CTAs per SM the walk is compiled for (register cap; the loop is latency-bound, so
                                     // warps beat registers even with a few spills); chosen by a sweep at C3 on a B200, not
                                     // re-measured on the H100
constexpr int kWalkThreads = 256;
constexpr uint32_t kWalkChunk = 1024;  // far ends staged per shared-memory chunk (16 KB)

/// The walk against the PADDED free-distance map (one border cell of zeros all round, 2^pad_shift bytes per row): a
/// jump of k <= d cells can at most land on the border, so the loop needs no bounds test -- a zero either is the first
/// non-free cell or the border (= the ray left the grid: a miss, raycasting.hpp:86-87), told apart after the loop.  The
/// iterator state is the linear cell index, advanced by k * (major stride) + m * (minor stride), so the x/y swap of the
/// steep case (bresenham.hpp:99-105) costs nothing per iteration.  Spans stay below 2^22 (checked by the launcher), so
/// the 32-bit reciprocal quotient of ray_step is the only path.  16 instructions per iteration instead of 45.
/// (Walking 2 or 4 rays per thread together was slower at C3 on a B200, not re-measured on the H100 --
/// the per-ray state machine and its activity flags cost more than the second load chain hides.)
/// One CTA of the walk: pass-local particles [block * kWalkThreads, (block + 1) * kWalkThreads) of the pass at slot_base.
/// `grid` by value: taken by reference, ptxas schedules beam_walk_kernel differently (same registers and spills).
__device__ __forceinline__ void beam_walk_block(const Pose2* __restrict__ states, uint64_t n, uint64_t slot_base, uint64_t slot_count,
                                                const uint32_t* __restrict__ perm, OccupancyView grid, double beam_max_range,
                                                const double2* __restrict__ points, uint32_t n_points, uint32_t* __restrict__ hits,
                                                uint64_t hit_stride, uint32_t block) {
  __shared__ double2 s_far[kWalkChunk];
  const uint64_t local = static_cast<uint64_t>(block) * kWalkThreads + threadIdx.x;
  const uint64_t slot = slot_base + local;
  const bool active = local < slot_count && slot < n;
  const uint64_t i = active ? (perm != nullptr ? perm[slot] : slot) : 0;
  // Ray2d: source pose in the grid frame and its cell (raycasting.hpp:67-70).
  const Pose2 src = pose_mul(grid.world_to_grid, active ? load_pose(states + i) : Pose2{1.0, 0.0, 0.0, 0.0});
  const int sx = source_cell(src.x, grid.inv_resolution), sy = source_cell(src.y, grid.inv_resolution);
  // A source outside the grid sees nothing: the first cell already fails cell_is_valid.  Nor does a non-finite heading: its
  // end points are not finite, so they lie outside the grid.
  const bool source_inside = static_cast<unsigned>(sx) < static_cast<unsigned>(grid.width) && static_cast<unsigned>(sy) < static_cast<unsigned>(grid.height) &&
                             isfinite(src.c) && isfinite(src.s);
  const int shift = grid.pad_shift;
  const int pitch = 1 << shift;
  const uint8_t* __restrict__ map = grid.free_padded;
  const int source_index = ((sy + 1) << shift) + (sx + 1);
  for (uint32_t base = 0; base < n_points; base += kWalkChunk) {
    const uint32_t count = min(kWalkChunk, n_points - base);
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < count; b += kWalkThreads) {
      const double2 p = points[base + b];
      const double z = sqrt(p.x * p.x + p.y * p.y);                                    // beam_model.hpp:116
      s_far[b] = make_double2((p.x / z) * beam_max_range, (p.y / z) * beam_max_range);  // :120-123, raycasting.hpp:83
    }
    __syncthreads();
    if (!active) continue;
    for (uint32_t b = 0; b < count; ++b) {
      uint32_t word = kHitMiss;
      // far end = r1 * t2 + t1 (raycasting.hpp:81-85)
      const double2 f = s_far[b];
      const double ex = (src.c * f.x - src.s * f.y) + src.x;
      const double ey = (src.s * f.x + src.c * f.y) + src.y;
      // From a source inside the grid with a finite heading, an end point is NaN exactly when the beam's bearing is (a
      // zero or non-finite scan point): it lies outside the grid, a miss.
      if (source_inside && ex == ex && ey == ey) {
        // far_span without its clamp: finite far ends lie within 2^21 cells of a source inside a grid of at most 65535
        // cells a side, so the floor fits an int and the spans stay far below kMaxRaySpan
        int span = __double2int_rd(ex * grid.inv_resolution) - sx, minor = __double2int_rd(ey * grid.inv_resolution) - sy;
        int stride_major = 1, stride_minor = pitch;
        if (span < 0) {
          span = -span;
          stride_major = -1;
        }
        if (minor < 0) {
          minor = -minor;
          stride_minor = -pitch;
        }
        if (span < minor) {  // iterate along the longer axis (bresenham.hpp:99-105)
          int t = span; span = minor; minor = t;
          t = stride_major; stride_major = stride_minor; stride_minor = t;
        }
        const uint32_t dxspan = 2u * static_cast<uint32_t>(span), dyspan = 2u * static_cast<uint32_t>(minor);
        const uint32_t recip = span > 0 ? 0xFFFFFFFFu / dxspan : 0u;
        int index = source_index;
        uint32_t err1 = static_cast<uint32_t>(span) - 1u;  // error - 1, error in (0, dxspan] (span == 0: never used)
        int remaining = span;
        for (;;) {
          const int d = __ldg(map + index);
          if (d == 0) {  // first non-free cell on the line, or the border
            const int cx = (index & (pitch - 1)) - 1, cy = (index >> shift) - 1;
            if (static_cast<unsigned>(cx) < static_cast<unsigned>(grid.width) && static_cast<unsigned>(cy) < static_cast<unsigned>(grid.height))
              word = (static_cast<uint32_t>(cy) << 16) | static_cast<uint32_t>(cx);
            break;
          }
          // Every cell within Chebyshev distance d - 1 is free and the line moves at most one cell per step in each axis:
          // advance d steps of the iterator (bresenham.hpp:122-160, standard variant) in closed form.
          const int k = min(d, remaining);
          if (k == 0) break;  // the far end cell was free too: sentinel reached (bresenham.hpp:179)
          remaining -= k;
          const uint32_t tm1 = err1 + static_cast<uint32_t>(k) * dyspan;  // t - 1, t = error + k * dyspan < 2^32
          uint32_t q = __umulhi(tm1, recip);                              // floor((t - 1) / dxspan) or one below
          uint32_t r = tm1 - q * dxspan;
          if (r >= dxspan) {
            ++q;
            r -= dxspan;
          }
          err1 = r;  // new error - 1
          index += k * stride_major + static_cast<int>(q) * stride_minor;
        }
      }
      __stcs(hits + static_cast<uint64_t>(base + b) * hit_stride + local, word);  // written once, read once: streaming
    }
  }
}

constexpr int kMixThreads = 256;
constexpr uint32_t kMixChunk = 2048;

/// One CTA of the mixture over the hit words beam_walk_block wrote for the same block of the same pass.
__device__ __forceinline__ void beam_mixture_block(const Pose2* __restrict__ states, double* __restrict__ weights, uint64_t n, uint64_t slot_base,
                                                   uint64_t slot_count, const uint32_t* __restrict__ perm, const OccupancyView& grid,
                                                   const BeamParams& params, const double2* __restrict__ points, uint32_t n_points,
                                                   const uint32_t* __restrict__ hits, uint64_t hit_stride, Scalars* __restrict__ scalars,
                                                   uint32_t block) {
  __shared__ double2 s_beam[kMixChunk];  // {z, exp(-lambda_short * z)}
  __shared__ unsigned long long s_red[kMixThreads / kWarp];
  const uint64_t local = static_cast<uint64_t>(block) * kMixThreads + threadIdx.x;
  const uint64_t slot = slot_base + local;
  const bool active = local < slot_count && slot < n;
  const uint64_t i = active ? (perm != nullptr ? perm[slot] : slot) : 0;
  const Pose2 src = pose_mul(grid.world_to_grid, active ? load_pose(states + i) : Pose2{1.0, 0.0, 0.0, 0.0});
  const int sx = source_cell(src.x, grid.inv_resolution), sy = source_cell(src.y, grid.inv_resolution);
  const double source_x = (static_cast<double>(sx) + 0.5) * grid.resolution, source_y = (static_cast<double>(sy) + 0.5) * grid.resolution;
  const double n_norm = 1. / (sqrt(2. * 3.14159265358979323846) * params.sigma_hit);  // beam_model.hpp:107

  auto value = [&](uint32_t word, const double2& beam) {
    const bool hit_cell = word != kHitMiss;
    const int cx = static_cast<int>(word & 0xFFFFu), cy = static_cast<int>(word >> 16);
    // distance between the centroids of the source cell and the hit cell (raycasting.hpp:91-104), clamped to the range
    const double dxm = (static_cast<double>(cx) + 0.5) * grid.resolution - source_x;
    const double dym = (static_cast<double>(cy) + 0.5) * grid.resolution - source_y;
    const double hit = fmin(sqrt(dxm * dxm + dym * dym), params.beam_max_range);
    const double z_mean = hit_cell ? hit : params.beam_max_range;  // value_or(beam_max_range)
    double2 eta;
    if (params.eta != nullptr) {
      const long long ix = static_cast<long long>(cx) - sx, iy = static_cast<long long>(cy) - sy;
      const unsigned long long d2 = static_cast<unsigned long long>(ix * ix + iy * iy);
      const bool in_table = hit_cell && hit < params.beam_max_range && d2 + 1 < params.eta_entries;
      eta = __ldg(params.eta + (in_table ? static_cast<uint32_t>(d2) : params.eta_entries - 1u));
    } else {
      eta = beam_normalisers(params, z_mean);
    }
    return beam_pz3(params, beam.x, beam.y, z_mean, n_norm, eta.x, eta.y);
  };

  double acc = 0.0;
  for (uint32_t base = 0; base < n_points; base += kMixChunk) {
    const uint32_t count = min(kMixChunk, n_points - base);
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < count; b += kMixThreads) {
      const double2 p = points[base + b];
      const double z = sqrt(p.x * p.x + p.y * p.y);  // beam_model.hpp:116
      s_beam[b] = make_double2(z, exp(-params.lambda_short * z));
    }
    __syncthreads();
    if (!active) continue;
    const uint32_t* h = hits + static_cast<uint64_t>(base) * hit_stride + local;
    uint32_t b = 0;
    for (; b + 4 <= count; b += 4) {  // transform_reduce grouping (numeric:439-462)
      const uint32_t w0 = __ldcs(h + static_cast<uint64_t>(b) * hit_stride), w1 = __ldcs(h + static_cast<uint64_t>(b + 1) * hit_stride);
      const uint32_t w2 = __ldcs(h + static_cast<uint64_t>(b + 2) * hit_stride), w3 = __ldcs(h + static_cast<uint64_t>(b + 3) * hit_stride);
      const double f0 = value(w0, s_beam[b]), f1 = value(w1, s_beam[b + 1]), f2 = value(w2, s_beam[b + 2]), f3 = value(w3, s_beam[b + 3]);
      acc = acc + ((f0 + f1) + (f2 + f3));
    }
    for (; b < count; ++b) acc = acc + value(__ldcs(h + static_cast<uint64_t>(b) * hit_stride), s_beam[b]);
  }
  double w = 0.0;
  if (active) {
    w = weights[i] * acc;  // actions/reweight.hpp:54-60
    weights[i] = w;
  }
  const unsigned long long m = block_max_u64<kMixThreads>(active ? weight_order_bits(w) : 0ull, s_red);
  if (threadIdx.x == 0 && m != 0) atomicMax(&scalars->wmax_bits, m);
}

}  // namespace

}  // namespace bb200
