// Start of a filter step: the reset of the per-step scalars (and, in the fused step, of the scan and schedule state).
#include "kernels.cuh"

#include <algorithm>

namespace bb200 {

namespace {

// ---- begin_step ----------------------------------------------------------------------------------

__global__ void begin_step_kernel(Scalars* s) {
  s->wmax_bits = 0;
  s->tile_ticket = 0;
  s->total = 0;
  s->exponent = 0;
  s->valid = 0;
  s->kld_cutoff = ~0ull;
  s->work_ticket = 0;  // normally rewound by the persistent reweight kernel itself; a step starts clean regardless
  s->work_done = 0;
  s->blocks_done = 0;
}

/// The fused step's reset: the scalars above plus the scan state of the CDF build and -- when the execution schedule
/// is rebuilt this step -- the bin counters, the schedule's scan state and its moment sums.  One launch instead of a
/// scalar kernel, two memsets and a reset kernel.
struct StepReset {
  Scalars* scalars;
  unsigned long long* tile_state;
  uint32_t n_tiles;
  Schedule* sched;             // nullable
  uint32_t* counters;          // nullable
  uint32_t n_counters;
  unsigned long long* sched_tiles;
  uint32_t n_sched_tiles;
  const char* prefetch;        // nullable: a table the step is about to gather from (pulled into L2 while propagate runs)
  uint64_t prefetch_lines;     // its size in 128-byte lines
};

__global__ void __launch_bounds__(256) begin_fused_step_kernel(StepReset r) {
  const uint32_t t = blockIdx.x * 256 + threadIdx.x, stride = gridDim.x * 256;
  if (t == 0) {
    Scalars* s = r.scalars;
    s->wmax_bits = 0;
    s->tile_ticket = 0;
    s->total = 0;
    s->exponent = 0;
    s->valid = 0;
    s->kld_cutoff = ~0ull;
    s->work_ticket = 0;
    s->work_done = 0;
    s->blocks_done = 0;
    if (r.sched != nullptr) {
      for (int k = 0; k < 6; ++k) r.sched->sums[k] = 0.0;
      r.sched->tile_ticket = 0;
    }
  }
  for (uint32_t k = t; k < r.n_tiles; k += stride) r.tile_state[k] = 0;
  if (r.counters != nullptr) {
    uint4* c4 = reinterpret_cast<uint4*>(r.counters);  // device allocations are 256-byte aligned; n_counters is a multiple of 4
    for (uint32_t k = t; k < r.n_counters / 4; k += stride) c4[k] = make_uint4(0u, 0u, 0u, 0u);
    for (uint32_t k = t; k < r.n_sched_tiles; k += stride) r.sched_tiles[k] = 0;
  }
  // The likelihood table is gathered from at random by the reweight kernel; after an L2 flush (or a map-sized
  // working set) its first touches would be demand misses to HBM, paid at full latency by warps that have nothing
  // else to do when a shard is small.  Streaming it into L2 now costs a few microseconds of HBM bandwidth that the
  // FP64-bound propagate kernel does not use.
  for (uint64_t k = t; k < r.prefetch_lines; k += stride) asm volatile("prefetch.global.L2 [%0];" ::"l"(r.prefetch + k * 128));
}

}  // namespace

int ceil_log2_count(uint64_t n) {
  int b = 0;
  while ((uint64_t{1} << b) < n) ++b;
  return b;
}

void launch_begin_step(Scalars* scalars, cudaStream_t stream) { begin_step_kernel<<<1, 1, 0, stream>>>(scalars); }

void launch_begin_fused_step(Scalars* scalars, unsigned long long* tile_state, uint32_t n_tiles, Schedule* sched, uint32_t* counters,
                             uint32_t n_counters, unsigned long long* sched_tiles, uint32_t n_sched_tiles, const void* prefetch,
                             uint64_t prefetch_bytes, cudaStream_t stream) {
  const StepReset r{scalars, tile_state, n_tiles, sched, counters, (n_counters + 3u) & ~3u, sched_tiles, n_sched_tiles,
                    static_cast<const char*>(prefetch), prefetch != nullptr ? prefetch_bytes / 128 : 0};
  const uint64_t work = std::max<uint64_t>(std::max(n_tiles, counters != nullptr ? r.n_counters / 4 : 0u), r.prefetch_lines / 8);
  const unsigned blocks = static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>((work + 255u) / 256u, kSmCount * 4u)));
  begin_fused_step_kernel<<<blocks, 256, 0, stream>>>(r);
}

}  // namespace bb200
