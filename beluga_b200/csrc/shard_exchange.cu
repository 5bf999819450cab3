// ---- shard exchange ------------------------------------------------------------------------------------
// One single-CTA kernel posts this rank's step scalar into every rank's mail block and/or waits for the peers' (see
// ShardMail in kernels.cuh).
#include "cdf.cuh"

namespace bb200 {

namespace {

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

constexpr unsigned long long kExchangeTimeoutNs = 4000000000ull;  // 4 s: a peer that has not posted by then never will

__global__ void __launch_bounds__(256) shard_exchange_kernel(ShardExchangeArgs a) {
  __shared__ unsigned long long s_u[kMaxShards];
  __shared__ double s_d[kMaxShards][kMomentCount];
  __shared__ int s_timeout;
  const int t = threadIdx.x;
  if (t == 0) s_timeout = 0;
  __syncthreads();
  if (a.post && t < a.world) {
    // my value -> entry [kind][my rank] of rank t's block
    volatile ShardMailEntry* dst = &a.peers[t]->e[a.kind][a.rank];
    if (a.kind == kExchangeWmax) {
      dst->u[0] = a.scalars->wmax_bits;
    } else if (a.kind == kExchangeTotal) {
      dst->u[0] = a.scalars->total;
    } else if (a.kind == kExchangeMoments) {
#pragma unroll
      for (int k = 0; k < kMomentCount; ++k) dst->d[k] = a.results[k];
    }
    __threadfence_system();  // the payload -- and every earlier store of this stream, e.g. the states pushed to the peers -- before the flag
    dst->seq = a.epoch;
  }
  if (a.wait) {
    if (t < a.world) {
      const volatile ShardMailEntry* src = &a.peers[a.rank]->e[a.kind][t];
      const unsigned long long t0 = global_timer_ns();
      bool ok = true;
      while (src->seq != a.epoch) {
        if (global_timer_ns() - t0 > kExchangeTimeoutNs) {
          ok = false;
          break;
        }
        __nanosleep(64);
      }
      __threadfence_system();
      if (!ok) atomicExch(&s_timeout, 1);
      s_u[t] = src->u[0];
      if (a.kind == kExchangeMoments) {
#pragma unroll
        for (int k = 0; k < kMomentCount; ++k) s_d[t][k] = src->d[k];
      }
    }
    __syncthreads();
    if (t == 0) {
      if (s_timeout) {
        a.scalars->exchange_error = 1;
        a.summary->error = 1;
      }
      if (a.kind == kExchangeWmax) {
        unsigned long long m = 0;
        for (int r = 0; r < a.world; ++r) m = s_u[r] > m ? s_u[r] : m;  // positive doubles order like their bit patterns
        a.scalars->wmax_bits = m;
        prepare_cdf_scalars(a.scalars, __longlong_as_double(static_cast<long long>(m)), a.ceil_log2_count);
        a.summary->exponent = a.scalars->exponent;
        a.summary->valid = a.scalars->valid;
      } else if (a.kind == kExchangeTotal) {
        unsigned long long total = 0;
        for (int r = 0; r < a.world; ++r) {
          a.rank_totals[r] = s_u[r];
          a.summary->rank_totals[r] = s_u[r];
          total += s_u[r];
        }
        a.summary->total = total;
        a.scalars->global_total = total;
      } else if (a.kind == kExchangeMoments) {
        for (int k = 0; k < kMomentCount; ++k) {  // rank order: the same sum on every rank
          double v = 0.0;
          for (int r = 0; r < a.world; ++r) v = v + s_d[r][k];
          a.results[k] = v;
          a.summary->moments[k] = v;
        }
      }
    }
    if (a.kind == kExchangeWmax && a.tile_state != nullptr) {
      for (uint32_t k = t; k < a.n_tiles; k += blockDim.x) a.tile_state[k] = 0;
    }
  }
}

}  // namespace

void launch_shard_exchange(const ShardExchangeArgs& args, cudaStream_t stream) { shard_exchange_kernel<<<1, 256, 0, stream>>>(args); }

}  // namespace bb200
