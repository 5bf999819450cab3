// Cluster-based estimate, device side (see cluster.cuh).  Hand-written sm_90a kernels:
//   cluster_insert / cluster_flag   spatial hash per particle, hash set "cell -> first particle"
//   cluster_cell_of                 dense cell id per particle (cells numbered by first occurrence)
//   radix_histogram / radix_scatter stable LSD radix sort of the particle indices by cell id
//   cluster_cells                   one warp per cell: ordered weight sum, moments, representative
//   batch_cluster_cells / _compact  the same stages for every selected member of a batch, one CTA per member
// Nothing here uses floating-point atomics: every sum has a fixed order, so results are reproducible
// run to run and the per-cell weight is the reference's sequential sum bit for bit.
#include "bucket_set.cuh"
#include "cluster.cuh"
#include "device_common.cuh"

#include <algorithm>
#include <utility>

namespace bb200 {

namespace {

// ---- cells -------------------------------------------------------------------------------------------

/// spatial_hash<SE2d>{linear, linear, angular} (cluster_based_estimation.hpp:321-325) of every state,
/// inserted into an open-addressing set that keeps the smallest particle index per cell.
__global__ void __launch_bounds__(256) cluster_insert_kernel(const Pose2* __restrict__ states, uint64_t n, double linear, double angular,
                                                             unsigned long long* __restrict__ hashes, unsigned long long* keys,
                                                             unsigned int* first, uint64_t mask) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  const unsigned long long hash = spatial_hash(load_pose(states + i), linear, linear, angular);
  hashes[i] = hash;
  bucket_set::insert_min(keys, first, mask, hash, static_cast<unsigned int>(i));
}

/// flags[i] = 1 when particle i is the first of its cell (try_emplace inserted, :151-156).
__global__ void __launch_bounds__(256) cluster_flag_kernel(const unsigned long long* __restrict__ hashes, uint64_t n,
                                                           const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ first,
                                                           uint64_t mask, uint32_t* __restrict__ slot_of, uint32_t* __restrict__ flags) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  const uint64_t pos = bucket_set::find(keys, mask, hashes[i]);
  slot_of[i] = static_cast<uint32_t>(pos);
  flags[i] = first[pos] == static_cast<unsigned int>(i) ? 1u : 0u;
}

/// cell id = number of first occurrences before the cell's first particle; also the cell sizes.
__global__ void __launch_bounds__(256) cluster_cell_of_kernel(const uint32_t* __restrict__ slot_of, const unsigned int* __restrict__ first,
                                                              const uint32_t* __restrict__ exclusive, uint64_t n, uint32_t* __restrict__ cell_of,
                                                              uint32_t* counts) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  const uint32_t cell = exclusive[first[slot_of[i]]];
  cell_of[i] = cell;
  atomicAdd(counts + cell, 1u);
}

// ---- stable radix sort of (cell id, particle index) ----------------------------------------------
// LSD, 8 bits per pass, tiles of 2048 keys.  Stability (equal keys keep their input order) is what
// leaves every cell's particles in particle order after the last pass.

constexpr int kSortThreads = 256;
constexpr int kSortItems = 8;
constexpr int kSortTile = kSortThreads * kSortItems;
constexpr int kRadix = 256;

__global__ void __launch_bounds__(kSortThreads) radix_histogram_kernel(const uint32_t* __restrict__ keys, uint32_t n, int shift, uint32_t tiles,
                                                                      uint32_t* __restrict__ histogram) {
  __shared__ uint32_t s_hist[kRadix];
  s_hist[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t base = blockIdx.x * kSortTile;
#pragma unroll
  for (int r = 0; r < kSortItems; ++r) {
    const uint32_t e = base + r * kSortThreads + threadIdx.x;
    if (e < n) atomicAdd(&s_hist[(keys[e] >> shift) & (kRadix - 1)], 1u);
  }
  __syncthreads();
  histogram[threadIdx.x * tiles + blockIdx.x] = s_hist[threadIdx.x];  // digit-major: one scan gives every (digit, tile) base
}

__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ idx_in,
                                                                    uint32_t n, int shift, uint32_t tiles, const uint32_t* __restrict__ bases,
                                                                    uint32_t* __restrict__ keys_out, uint32_t* __restrict__ idx_out) {
  constexpr int kWarps = kSortThreads / kWarp;
  __shared__ uint32_t s_base[kRadix];            // next free output position per digit for this tile
  __shared__ uint32_t s_count[kWarps][kRadix];   // keys per (warp, digit) in the current round
  const int warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  s_base[threadIdx.x] = bases[threadIdx.x * tiles + blockIdx.x];
  const uint32_t base = blockIdx.x * kSortTile;
  for (int r = 0; r < kSortItems; ++r) {
#pragma unroll
    for (int w = 0; w < kWarps; ++w) s_count[w][threadIdx.x] = 0;
    __syncthreads();
    const uint32_t e = base + r * kSortThreads + threadIdx.x;
    const bool valid = e < n;
    const uint32_t key = valid ? keys_in[e] : 0u;
    const uint32_t digit = valid ? ((key >> shift) & (kRadix - 1)) : kRadix;  // invalid lanes form their own group
    const unsigned peers = __match_any_sync(0xffffffffu, digit);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) s_count[warp][digit] = __popc(peers);
    __syncthreads();
    // Thread d turns the per-warp counts of digit d into offsets (warp order = element order).
    {
      uint32_t running = s_base[threadIdx.x];
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        const uint32_t c = s_count[w][threadIdx.x];
        s_count[w][threadIdx.x] = running;
        running += c;
      }
      s_base[threadIdx.x] = running;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = s_count[warp][digit] + rank;
      keys_out[pos] = key;
      idx_out[pos] = idx_in != nullptr ? idx_in[e] : e;
    }
    __syncthreads();
  }
}

// ---- one record per cell ---------------------------------------------------------------------------

constexpr int kCellThreads = 128;

/// The record of one cell, built by one warp: sorted_idx[begin, end) are the cell's particles in particle order.  Each lane
/// gathers every 32nd particle, the moments meet in a fixed xor-shuffle tree, and the weight is the reference's sequential
/// sum.  The single-filter and the batch kernels both build their records here, so the two agree bit for bit.
__device__ __forceinline__ void cell_record_warp(const Pose2* states, const double* weights, const unsigned long long* hashes,
                                                 const uint32_t* sorted_idx, uint32_t begin, uint32_t end, double px, double py,
                                                 CellRecord* record) {
  const int lane = threadIdx.x % kWarp;
  double m[kMomentCount];
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) m[k] = 0.0;
  bool unit = true;
  auto add = [&](const Pose2& st, double w) {
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
    unit = unit && w == 1.0;
  };
  uint32_t p = begin + lane;
  for (; p + 3 * kWarp < end; p += 4 * kWarp) {  // four gathers in flight per lane
    const uint32_t i0 = sorted_idx[p], i1 = sorted_idx[p + kWarp], i2 = sorted_idx[p + 2 * kWarp], i3 = sorted_idx[p + 3 * kWarp];
    const double w0 = weights[i0], w1 = weights[i1], w2 = weights[i2], w3 = weights[i3];
    const Pose2 s0 = load_pose(states + i0), s1 = load_pose(states + i1), s2 = load_pose(states + i2), s3 = load_pose(states + i3);
    add(s0, w0);
    add(s1, w1);
    add(s2, w2);
    add(s3, w3);
  }
  for (; p < end; p += kWarp) {
    const uint32_t i = sorted_idx[p];
    add(load_pose(states + i), weights[i]);
  }
#pragma unroll
  for (int k = 0; k < kMomentCount; ++k) {
#pragma unroll
    for (int off = kWarp / 2; off > 0; off >>= 1) m[k] = m[k] + __shfl_xor_sync(0xffffffffu, m[k], off);
  }
  unit = __all_sync(0xffffffffu, unit);

  // ClusterCell::weight: `entry.weight += weight` in particle order (:153).  With unit weights (the
  // state after every resample) all partial sums are integers, so the count is that sum exactly;
  // otherwise the warp replays the sequential chain, 32 weights per coalesced load.
  double total = static_cast<double>(end - begin);
  if (!unit) {
    total = 0.0;
    double w = begin + lane < end ? weights[sorted_idx[begin + lane]] : 0.0;
    for (uint32_t base = begin; base < end; base += kWarp) {
      const uint32_t q = base + kWarp + lane;  // the next 32 weights travel while this batch is added up
      const double w_next = q < end ? weights[sorted_idx[q]] : 0.0;
      const int valid = static_cast<int>(min(static_cast<uint32_t>(kWarp), end - base));
      for (int k = 0; k < valid; ++k) total = total + __shfl_sync(0xffffffffu, w, k);
      w = w_next;
    }
  }
  if (lane == 0) {
    const uint32_t first = sorted_idx[begin];  // particle order inside the cell: the cell's earliest particle
    CellRecord r;
    r.hash = hashes[first];
    r.first_index = first;
    r.count = end - begin;
    r.weight = total;
    r.representative = load_pose(states + first);
#pragma unroll
    for (int k = 0; k < kMomentCount; ++k) r.moments[k] = m[k];
    *record = r;
  }
}

__global__ void __launch_bounds__(kCellThreads) cluster_cells_kernel(const Pose2* __restrict__ states, const double* __restrict__ weights,
                                                                    const unsigned long long* __restrict__ hashes,
                                                                    const uint32_t* __restrict__ sorted_idx, const uint32_t* __restrict__ starts,
                                                                    uint32_t cells, double px, double py, CellRecord* __restrict__ records) {
  const uint32_t cell = (blockIdx.x * kCellThreads + threadIdx.x) / kWarp;
  if (cell >= cells) return;  // whole warps leave together
  cell_record_warp(states, weights, hashes, sorted_idx, starts[cell], starts[cell + 1], px, py, records + cell);
}

// ---- every selected member of a batch: one CTA per member -------------------------------------------
// The CTA runs the whole per-particle half of its member (at most kBatchClusterMaxParticles particles) with the
// single-filter stages as block-wide loops: hash set, first-occurrence numbering in particle order, stable LSD sort of
// the particle indices by cell, segment starts, one record per cell.  A member's scratch is its own slice of the batch
// buffers, so no CTA waits for another.

constexpr int kBatchCellThreads = 1024;
constexpr int kBatchCellWarps = kBatchCellThreads / kWarp;
constexpr int kIndexBits = 15;  // particle index inside a member: < kBatchClusterMaxParticles
static_assert(kBatchClusterMaxParticles == (1u << kIndexBits), "sort values pack (cell, particle index) into 30 bits");

__global__ void __launch_bounds__(kBatchCellThreads) batch_cluster_cells_kernel(const BatchClusterArgs a) {
  __shared__ uint32_t s_warp[kBatchCellWarps];            // head flags per warp in the current chunk
  __shared__ uint32_t s_base[kRadix];                     // digit counts, then the next free output position per digit
  __shared__ uint32_t s_count[kBatchCellWarps][kRadix];   // keys per (warp, digit) in the current chunk
  const BatchClusterMember mb = a.members[blockIdx.x];
  const uint32_t n = mb.n;
  const Pose2* states = (mb.cur != 0 ? a.states[1] : a.states[0]) + mb.offset;
  const double* weights = a.weights + mb.offset;
  unsigned long long* hashes = a.hashes + mb.offset;
  unsigned long long* keys = a.keys + mb.table_offset;
  unsigned int* first = a.first + mb.table_offset;
  uint32_t* ids = a.ids + mb.table_offset;
  uint32_t* cell_of = a.cell_of + mb.offset;
  uint32_t* starts = a.starts + mb.starts_offset;
  const uint64_t mask = mb.table_mask;
  const int tid = threadIdx.x, lane = tid % kWarp, warp = tid / kWarp;
  const unsigned lanes_below = (1u << lane) - 1u;

  for (uint64_t s = tid; s <= mask; s += kBatchCellThreads) {
    keys[s] = bucket_set::kEmpty;
    first[s] = ~0u;
  }
  __syncthreads();
  // spatial_hash<SE2d>{linear, linear, angular} of every state into the set "cell -> smallest particle index".
  for (uint32_t i = tid; i < n; i += kBatchCellThreads) {
    const unsigned long long hash = spatial_hash(load_pose(states + i), a.linear, a.linear, a.angular);
    hashes[i] = hash;
    bucket_set::insert_min(keys, first, mask, hash, i);
  }
  __syncthreads();
  // Cells numbered by first occurrence: chunk by chunk in particle order, a cell's first particle takes the next number.
  uint32_t cells = 0;
  for (uint32_t base = 0; base < n; base += kBatchCellThreads) {
    const uint32_t i = base + tid;
    uint32_t pos = 0;
    bool head = false;
    if (i < n) {
      pos = static_cast<uint32_t>(bucket_set::find(keys, mask, hashes[i]));
      head = first[pos] == i;
      cell_of[i] = pos;  // the slot for now, the cell id below
    }
    const unsigned heads = __ballot_sync(0xffffffffu, head);
    if (lane == 0) s_warp[warp] = __popc(heads);
    __syncthreads();
    uint32_t before = cells;
    for (int w = 0; w < kBatchCellWarps; ++w) {
      const uint32_t c = s_warp[w];
      if (w < warp) before += c;
      cells += c;
    }
    if (head) ids[pos] = before + __popc(heads & lanes_below);
    __syncthreads();
  }
  // Sort values (cell << 15 | particle index), in particle order.
  uint32_t* in = a.sort_a + mb.offset;
  uint32_t* out = a.sort_b + mb.offset;
  for (uint32_t i = tid; i < n; i += kBatchCellThreads) {
    const uint32_t cell = ids[cell_of[i]];
    cell_of[i] = cell;
    in[i] = cell << kIndexBits | i;
  }
  __syncthreads();
  // Stable LSD radix sort by cell, 8 bits per pass: the order of a stable sort of the particle indices by cell, which is
  // also the order of the unique keys cell * 2^15 + index.  The last pass keeps the particle index only.
  const int passes = cells > kRadix ? 2 : 1;
  for (int pass = 0; pass < passes; ++pass) {
    const int shift = kIndexBits + 8 * pass;
    const bool last = pass == passes - 1;
    if (tid < kRadix) s_base[tid] = 0;
    __syncthreads();
    for (uint32_t i = tid; i < n; i += kBatchCellThreads) atomicAdd(&s_base[(in[i] >> shift) & (kRadix - 1)], 1u);
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the 256 digit counts, 8 per lane
      constexpr int kPer = kRadix / kWarp;
      uint32_t v[kPer], sum = 0;
#pragma unroll
      for (int k = 0; k < kPer; ++k) {
        v[k] = s_base[lane * kPer + k];
        sum += v[k];
      }
      uint32_t incl = sum;
#pragma unroll
      for (int off = 1; off < kWarp; off <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += o;
      }
      uint32_t running = incl - sum;
#pragma unroll
      for (int k = 0; k < kPer; ++k) {
        s_base[lane * kPer + k] = running;
        running += v[k];
      }
    }
    __syncthreads();
    for (uint32_t base = 0; base < n; base += kBatchCellThreads) {
      for (int k = tid; k < kBatchCellWarps * kRadix; k += kBatchCellThreads) (&s_count[0][0])[k] = 0;
      __syncthreads();
      const uint32_t e = base + tid;
      const bool valid = e < n;
      const uint32_t v = valid ? in[e] : 0u;
      const uint32_t digit = valid ? ((v >> shift) & (kRadix - 1)) : kRadix;  // invalid lanes form their own group
      const unsigned peers = __match_any_sync(0xffffffffu, digit);
      const uint32_t rank = __popc(peers & lanes_below);
      if (valid && rank == 0) s_count[warp][digit] = __popc(peers);
      __syncthreads();
      if (tid < kRadix) {  // thread d turns the per-warp counts of digit d into offsets (warp order = element order)
        uint32_t running = s_base[tid];
        for (int w = 0; w < kBatchCellWarps; ++w) {
          const uint32_t c = s_count[w][tid];
          s_count[w][tid] = running;
          running += c;
        }
        s_base[tid] = running;
      }
      __syncthreads();
      if (valid) out[s_count[warp][digit] + rank] = last ? (v & (kBatchClusterMaxParticles - 1)) : v;
      __syncthreads();
    }
    uint32_t* t = in;
    in = out;
    out = t;
  }
  const uint32_t* sorted = in;
  // Segment starts: a cell begins where the sorted sequence changes cell.
  for (uint32_t p = tid; p < n; p += kBatchCellThreads) {
    const uint32_t cell = cell_of[sorted[p]];
    if (p == 0 || cell != cell_of[sorted[p - 1]]) starts[cell] = p;
  }
  if (tid == 0) starts[cells] = n;
  __syncthreads();
  CellRecord* records = a.records + mb.offset;
  for (uint32_t c = warp; c < cells; c += kBatchCellWarps)
    cell_record_warp(states, weights, hashes, sorted, starts[c], starts[c + 1], mb.pivot_x, mb.pivot_y, records + c);
  if (tid == 0) a.cells[blockIdx.x] = cells;
}

/// Member j's records move from its slice to out[cells of members 0 .. j-1 ...]: one CTA per member, 16 bytes per thread.
constexpr int kCompactThreads = 256;

__global__ void __launch_bounds__(kCompactThreads) batch_cluster_compact_kernel(const BatchClusterMember* __restrict__ members,
                                                                                 const uint32_t* __restrict__ cells, const CellRecord* __restrict__ records,
                                                                                 CellRecord* __restrict__ out) {
  __shared__ uint64_t s_sum[kCompactThreads / kWarp];
  uint64_t sum = 0;
  for (uint32_t j = threadIdx.x; j < blockIdx.x; j += kCompactThreads) sum += cells[j];
#pragma unroll
  for (int off = kWarp / 2; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if (threadIdx.x % kWarp == 0) s_sum[threadIdx.x / kWarp] = sum;
  __syncthreads();
  uint64_t dst = 0;
#pragma unroll
  for (int w = 0; w < kCompactThreads / kWarp; ++w) dst += s_sum[w];
  constexpr int kWords = sizeof(CellRecord) / sizeof(double2);
  const double2* src = reinterpret_cast<const double2*>(records + members[blockIdx.x].offset);
  double2* to = reinterpret_cast<double2*>(out + dst);
  const uint64_t words = static_cast<uint64_t>(cells[blockIdx.x]) * kWords;
  for (uint64_t k = threadIdx.x; k < words; k += kCompactThreads) to[k] = src[k];
}

int bits_for(uint32_t values) {  // bits needed to represent 0 .. values-1
  int b = 0;
  while (b < 32 && (1ull << b) < values) ++b;
  return b;
}

}  // namespace

uint32_t cluster_sort_tiles(uint64_t n) { return static_cast<uint32_t>((n + kSortTile - 1) / kSortTile); }

void launch_cluster_cells_begin(const Pose2* states, uint64_t n, double linear_resolution, double angular_resolution, const ClusterScratch& s,
                                cudaStream_t stream) {
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  const uint64_t table_size = s.keys.size();
  cudaMemsetAsync(s.keys.get(), 0xFF, table_size * sizeof(unsigned long long), stream);
  cudaMemsetAsync(s.first.get(), 0xFF, table_size * sizeof(unsigned int), stream);
  cluster_insert_kernel<<<blocks, 256, 0, stream>>>(states, n, linear_resolution, angular_resolution, s.hashes.get(), s.keys.get(), s.first.get(),
                                                    table_size - 1);
  cluster_flag_kernel<<<blocks, 256, 0, stream>>>(s.hashes.get(), n, s.keys.get(), s.first.get(), table_size - 1, s.slot_of.get(), s.flags.get());
  launch_scan_u32(s.flags.get(), s.flags.get(), static_cast<uint32_t>(n), s.words.get() + 0, s.tile_state.get(), s.words.get() + 1, stream);
}

const uint32_t* launch_cluster_sort(uint64_t n, uint32_t cells, const ClusterScratch& s, cudaStream_t stream, int* launches) {
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  const uint32_t n32 = static_cast<uint32_t>(n);
  cudaMemsetAsync(s.starts.get(), 0, (static_cast<size_t>(cells) + 1) * sizeof(uint32_t), stream);
  cluster_cell_of_kernel<<<blocks, 256, 0, stream>>>(s.slot_of.get(), s.first.get(), s.flags.get(), n, s.cell_of.get(), s.starts.get());
  launch_scan_u32(s.starts.get(), s.starts.get(), cells + 1, s.words.get() + 0, s.tile_state.get(), nullptr, stream);

  const uint32_t tiles = cluster_sort_tiles(n);
  const int passes = std::max(1, (bits_for(cells) + 7) / 8);
  const uint32_t* keys_in = s.cell_of.get();
  const uint32_t* idx_in = nullptr;  // first pass: the identity
  uint32_t* keys_out = s.keys_a.get();
  uint32_t* idx_out = s.idx_a.get();
  for (int pass = 0; pass < passes; ++pass) {
    radix_histogram_kernel<<<tiles, kSortThreads, 0, stream>>>(keys_in, n32, 8 * pass, tiles, s.histogram.get());
    launch_scan_u32(s.histogram.get(), s.histogram.get(), kRadix * tiles, s.words.get() + 0, s.tile_state.get(), nullptr, stream);
    radix_scatter_kernel<<<tiles, kSortThreads, 0, stream>>>(keys_in, idx_in, n32, 8 * pass, tiles, s.histogram.get(), keys_out, idx_out);
    keys_in = keys_out;
    idx_in = idx_out;
    keys_out = keys_out == s.keys_a.get() ? s.keys_b.get() : s.keys_a.get();
    idx_out = idx_out == s.idx_a.get() ? s.idx_b.get() : s.idx_a.get();
  }
  if (launches != nullptr) *launches = 2 + 3 * passes;
  return idx_in;
}

void launch_cluster_records(const Pose2* states, const double* weights, const uint32_t* sorted_idx, uint32_t cells, double pivot_x, double pivot_y,
                            const ClusterScratch& s, cudaStream_t stream) {
  const unsigned cell_blocks = static_cast<unsigned>((static_cast<uint64_t>(cells) * kWarp + kCellThreads - 1) / kCellThreads);
  cluster_cells_kernel<<<cell_blocks, kCellThreads, 0, stream>>>(states, weights, s.hashes.get(), sorted_idx, s.starts.get(), cells, pivot_x, pivot_y,
                                                                  s.records.get());
}

void launch_batch_cluster_cells(const BatchClusterArgs& a, uint32_t n_members, cudaStream_t stream) {
  batch_cluster_cells_kernel<<<n_members, kBatchCellThreads, 0, stream>>>(a);
}

void launch_batch_cluster_compact(const BatchClusterMember* members, const uint32_t* cells, const CellRecord* records, uint32_t n_members,
                                  CellRecord* out, cudaStream_t stream) {
  batch_cluster_compact_kernel<<<n_members, kCompactThreads, 0, stream>>>(members, cells, records, out);
}

// ---- Clusterizer -------------------------------------------------------------------------------------

int Clusterizer::ensure_scratch(uint32_t cells, std::string* error) {
  auto check = [error](cudaError_t e, const char* what) { return cuda_check(e, what, error); };
  if (s_.hashes.get() == nullptr) {  // then the records are not allocated either
    const uint64_t capacity = capacity_;
    if (capacity >= (1ull << 31)) return reject(BB200_ERR_CAPACITY, "cluster estimate: more than 2^31 particles per filter", error);
    uint64_t table = 2;
    while (table < 2 * capacity) table <<= 1;
    const uint32_t tiles = cluster_sort_tiles(capacity);
    ClusterScratch c;
    BB_CHECK(c.keys.allocate(table));
    BB_CHECK(c.first.allocate(table));
    BB_CHECK(c.slot_of.allocate(capacity));
    BB_CHECK(c.flags.allocate(capacity));
    BB_CHECK(c.cell_of.allocate(capacity));
    BB_CHECK(c.starts.allocate(capacity + 1));
    BB_CHECK(c.keys_a.allocate(capacity));
    BB_CHECK(c.keys_b.allocate(capacity));
    BB_CHECK(c.idx_a.allocate(capacity));
    BB_CHECK(c.idx_b.allocate(capacity));
    BB_CHECK(c.histogram.allocate(static_cast<size_t>(256) * tiles));
    BB_CHECK(c.tile_state.allocate(static_cast<size_t>(scan_tile_count(std::max<uint64_t>(capacity + 1, 256ull * tiles)) + 1)));
    BB_CHECK(c.words.allocate(4));
    BB_CHECK(c.hashes.allocate(capacity));
    s_ = std::move(c);
  }
  BB_CHECK(s_.records.grow(cells, std::min<uint64_t>(capacity_, std::max<uint64_t>(1024, 2ull * cells))));
  return BB200_OK;
}

int Clusterizer::cell_records(const Pose2* states, const double* weights, uint64_t n, const double pivot[2], double linear_resolution,
                              double angular_resolution, cudaStream_t stream, std::vector<HostCell>* host, std::string* error) {
  // spatial hash -> first-occurrence numbering of the occupied cells -> stable sort of the particle indices by cell -> one
  // record per cell (representative = first particle, count, weight summed in particle order, raw moments).
  auto check = [error](cudaError_t e, const char* what) { return cuda_check(e, what, error); };
  auto stage = [this](const char* name) { if (mark) mark(name); };
  {
    const int st = ensure_scratch(0, error);
    if (st != BB200_OK) return st;
  }
  stage("cluster_cells");
  launch_cluster_cells_begin(states, n, linear_resolution, angular_resolution, s_, stream);
  BB_LAUNCHED_N("cluster_cells_begin", 3);
  unsigned long long cells64 = 0;
  BB_CHECK(cudaMemcpyAsync(&cells64, s_.words.get() + 1, sizeof(cells64), cudaMemcpyDeviceToHost, stream));
  BB_CHECK(cudaStreamSynchronize(stream));
  const uint32_t cells = static_cast<uint32_t>(cells64);
  {
    const int st = ensure_scratch(cells, error);
    if (st != BB200_OK) return st;
  }
  stage("cluster_sort");
  int sort_launches = 0;
  const uint32_t* sorted = launch_cluster_sort(n, cells, s_, stream, &sort_launches);
  BB_LAUNCHED_N("cluster_sort", sort_launches);
  stage("cluster_records");
  launch_cluster_records(states, weights, sorted, cells, pivot[0], pivot[1], s_, stream);
  BB_LAUNCHED("cluster_records");
  host->resize(cells);
  static_assert(sizeof(HostCell) == sizeof(CellRecord), "record layouts must agree");
  BB_CHECK(cudaMemcpyAsync(host->data(), s_.records.get(), static_cast<size_t>(cells) * sizeof(CellRecord), cudaMemcpyDeviceToHost, stream));
  BB_CHECK(cudaStreamSynchronize(stream));
  stage("end");
  return BB200_OK;
}

int Clusterizer::estimate(const Pose2* states, const double* weights, uint64_t n, const double pivot[2], const bb200_cluster_param& p, cudaStream_t stream,
                          bb200_estimate* out, uint32_t* cluster_ids, uint64_t ids_capacity, uint32_t* n_cells, uint32_t* n_clusters, std::string* error) {
  auto check = [error](cudaError_t e, const char* what) { return cuda_check(e, what, error); };
  if (n == 0) return reject(BB200_ERR_STATE, "no particles", error);
  if (n > capacity_) return reject(BB200_ERR_CAPACITY, "cluster estimate: more particles than the scratch holds", error);
  if (const char* why = cluster_param_error(p)) return reject(BB200_ERR_INVALID_ARGUMENT, why, error);
  if (cluster_ids != nullptr && ids_capacity < n) return reject(BB200_ERR_CAPACITY, "cluster id buffer too small", error);
  std::vector<HostCell> host;
  {
    const int st = cell_records(states, weights, n, pivot, p.linear_hash_resolution, p.angular_hash_resolution, stream, &host, error);
    if (st != BB200_OK) return st;
  }
  const uint32_t cells = static_cast<uint32_t>(host.size());
  const ClusterSelection sel = select_cluster(host.data(), host.size(), n, p.linear_hash_resolution, p.angular_hash_resolution, p.weight_cap_percentile);
  if (out != nullptr) estimate_from_moments(sel.moments, pivot, out);
  if (n_cells != nullptr) *n_cells = cells;
  if (n_clusters != nullptr) *n_clusters = sel.clusters;
  if (cluster_ids != nullptr) {
    std::vector<uint32_t> cell_of(n);
    BB_CHECK(cudaMemcpy(cell_of.data(), s_.cell_of.get(), n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (uint64_t i = 0; i < n; ++i) cluster_ids[i] = sel.cluster_of_cell[cell_of[i]];
  }
  return BB200_OK;
}


}  // namespace bb200
