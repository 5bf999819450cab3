// The KLD condition of views::take_while_kld, shared by the single filter's chunked count (kld.cu) and the batch's
// one-CTA count per member (batch_kernels.cu).
#pragma once

#include <cstdint>

namespace bb200 {

namespace {

/// kld_condition target size (views/take_while_kld.hpp:73-80), same operation order as the reference.
__device__ __forceinline__ bool kld_count_allowed(unsigned long long count, unsigned long long k, unsigned long long min_count, double two_epsilon, double z) {
  if (count <= min_count || k <= 2ull) return true;
  const double common = 2. / static_cast<double>(9 * (k - 1));
  const double base = 1. - common + sqrt(common) * z;
  const double result = (static_cast<double>(k - 1) / two_epsilon) * base * base * base;
  const double target = ceil(result);
  return target >= 18446744073709551615.0 || count <= static_cast<unsigned long long>(target);
}

}  // namespace

}  // namespace bb200
