// The cluster estimate of every member a batch step updated, selected on the device (see cluster.cuh):
//   batch_cluster_table    the post-step member table from the step's summaries
//   batch_cluster_select   select_cluster per member, one CTA each: the parallel part (normalised weights, percentile
//                          cap, six neighbours per cell through the member's bucket set, the map's bucket of every cell),
//                          then one thread runs the order-defining part (cluster_select.cuh)
#include "bucket_set.cuh"
#include "cluster.cuh"
#include "device_common.cuh"

namespace bb200 {

namespace {

/// beluga_ros's update then cluster estimate: the state the step leaves, as Batch::step commits it on the host.
__global__ void __launch_bounds__(128) batch_cluster_table_kernel(const BatchSelectArgs a) {
  const uint32_t j = blockIdx.x * 128 + threadIdx.x;
  if (j >= a.n_members) return;
  BatchClusterMember m = a.members[j];
  const BatchClusterPost p = a.post[j];
  const StepSummary& s = a.summary[j];
  const bool resampled = p.mode == 1 || (p.mode == 2 && s.resampled != 0);
  if (resampled) {
    m.cur ^= 1u;
    m.n = p.kld ? static_cast<uint32_t>(s.accepted) : p.capacity;
  }
  // estimate_from_moments then pivot_to_estimate: the mean's position, kept when both coordinates are finite
  const double x = m.pivot_x + s.moments[4] / s.moments[0];
  const double y = m.pivot_y + s.moments[5] / s.moments[0];
  if (isfinite(x) && isfinite(y)) {
    m.pivot_x = x;
    m.pivot_y = y;
  }
  a.members[j] = m;
}

constexpr int kSelectThreads = 256;
constexpr uint32_t kSelectSmem = 96u << 10;  // a member whose selection fits runs it in shared memory

/// The cell id of `hash` in a member's bucket set, kSelectNone when no particle fell into that cell (map.find == end).
__device__ __forceinline__ uint32_t find_cell(const unsigned long long* keys, const uint32_t* ids, uint64_t mask, unsigned long long hash) {
  const unsigned long long key = bucket_set::key_of(hash);
  for (uint64_t pos = bucket_set::probe_start(key, mask);; pos = (pos + 1) & mask) {
    const unsigned long long k = keys[pos];
    if (k == key) return ids[pos];
    if (k == bucket_set::kEmpty) return kSelectNone;
  }
}

/// Doubles as unsigned keys in the order of operator< (the NaN-free values the cap is taken from).
__device__ __forceinline__ unsigned long long order_key(double v) {
  const unsigned long long u = static_cast<unsigned long long>(__double_as_longlong(v));
  return (u >> 63) != 0 ? ~u : u | (1ull << 63);
}
__device__ __forceinline__ double from_order_key(unsigned long long k) {
  return __longlong_as_double(static_cast<long long>((k >> 63) != 0 ? k & ~(1ull << 63) : ~k));
}

__global__ void __launch_bounds__(kSelectThreads) batch_cluster_select_kernel(const BatchSelectArgs a) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  __shared__ uint32_t s_hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ uint32_t s_rank;
  const uint32_t j = blockIdx.x;
  const int tid = threadIdx.x;
  const BatchClusterMember mb = a.members[j];
  const uint32_t c = a.cells[j];
  const CellRecord* cells = a.records + mb.offset;
  const RehashStep* schedule = a.schedule + a.schedule_start[mb.n / 5];
  uint32_t max_buckets = 0;
  const int phases = rehash_phases(schedule, c, &max_buckets);
  const SelectLayout l = select_layout(c, phases, max_buckets);
  unsigned char* base = l.bytes <= kSelectSmem ? s_dyn : a.scratch + a.post[j].scratch_offset;
  double* capped = reinterpret_cast<double*>(base + l.capped);
  uint32_t* neighbors = reinterpret_cast<uint32_t*>(base + l.neighbors);
  uint32_t* bkt = reinterpret_cast<uint32_t*>(base + l.bkt);

  // normalize_and_cap_weights, first loop: weight / particles per cell
  bool fallback = false;
  for (uint32_t i = tid; i < c; i += kSelectThreads) {
    const double w = cells[i].weight / static_cast<double>(cells[i].count);
    capped[i] = w;
    fallback = fallback || isnan(w);  // nth_element over NaNs depends on its partition order
  }
  const int64_t nth = static_cast<int64_t>(static_cast<double>(c) * a.percentile);
  fallback = __syncthreads_or(fallback) || (c > 0 && nth >= static_cast<int64_t>(c));
  if (!fallback && c > 0) {
    // calculate_percentile_threshold: the nth smallest value (the same under any exact selection), by radix select
    unsigned long long prefix = 0;
    uint32_t rank = static_cast<uint32_t>(nth);
    for (int shift = 56; shift >= 0; shift -= 8) {
      s_hist[tid] = 0;
      __syncthreads();
      const unsigned long long high = shift == 56 ? 0ull : ~0ull << (shift + 8);
      for (uint32_t i = tid; i < c; i += kSelectThreads) {
        const unsigned long long key = order_key(capped[i]);
        if ((key & high) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        uint32_t r = rank;
        for (uint32_t d = 0; d < 256; ++d) {
          if (r < s_hist[d]) {
            s_prefix = prefix | (static_cast<unsigned long long>(d) << shift);
            s_rank = r;
            break;
          }
          r -= s_hist[d];
        }
      }
      __syncthreads();
      prefix = s_prefix;
      rank = s_rank;
    }
    const double cap = from_order_key(prefix);
    for (uint32_t i = tid; i < c; i += kSelectThreads) capped[i] = cap < capped[i] ? cap : capped[i];  // std::min(weight, cap)
  }
  // The six neighbours of every cell (adjacent_grid_cells_, :289-293), resolved to cell ids.
  const unsigned long long* keys = a.keys + mb.table_offset;
  const uint32_t* ids = a.ids + mb.table_offset;
  for (uint32_t t = tid; t < 6 * c; t += kSelectThreads) {
    const uint32_t i = t / 6, s = t % 6;
    const Pose2 q = pose_mul(cells[i].representative, a.adjacent[s]);
    fallback = fallback || heading_near_bucket_edge(q.s, q.c, a.angular);
    neighbors[t] = find_cell(keys, ids, mb.table_mask, spatial_hash(q, a.linear, a.linear, a.angular));
  }
  // The bucket of every cell in each bucket count the map passes through.
  for (int ph = 0; ph < phases; ++ph) {
    const unsigned long long buckets = schedule[ph].buckets;
    for (uint32_t i = tid; i < c; i += kSelectThreads) bkt[static_cast<uint64_t>(ph) * c + i] = static_cast<uint32_t>(cells[i].hash % buckets);
  }
  BatchClusterResult* out = a.results + j;
  if (__syncthreads_or(fallback)) {
    if (tid == 0) {
      out->found = 0;
      out->clusters = 0;
      out->cells = c;
      out->fallback = 1;
    }
    return;
  }
  if (tid != 0) return;
  uint32_t* next = reinterpret_cast<uint32_t*>(base + l.next);
  uint32_t* before = reinterpret_cast<uint32_t*>(base + l.before);
  uint32_t* order = reinterpret_cast<uint32_t*>(base + l.order);
  map_order(schedule, bkt, c, next, before, order);
  const SelectOutcome o = select_in_order(cells, c, order, capped, neighbors, reinterpret_cast<SelectQueued*>(base + l.heap),
                                          reinterpret_cast<uint32_t*>(base + l.cluster));
  out->found = o.found;
  out->clusters = o.clusters;
  out->cells = c;
  out->fallback = 0;
  for (int k = 0; k < kMomentCount; ++k) out->moments[k] = o.moments[k];
}

}  // namespace

void launch_batch_cluster_table(const BatchSelectArgs& a, cudaStream_t stream) {
  batch_cluster_table_kernel<<<(a.n_members + 127) / 128, 128, 0, stream>>>(a);
}

void launch_batch_cluster_select(const BatchSelectArgs& a, cudaStream_t stream) {
  cudaFuncSetAttribute(batch_cluster_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSelectSmem);
  batch_cluster_select_kernel<<<a.n_members, kSelectThreads, kSelectSmem, stream>>>(a);
}

}  // namespace bb200
