// A caller's device sensor model for test_weighed_adaptor.cpp: a Gaussian position fix, L = exp(-|p - fix|^2 / (2 sigma^2)),
// one thread per particle on the stream the weighed step hands out.
#include <cuda_runtime.h>

#include <cstdint>

namespace {

__global__ void position_fix_kernel(const double* states, std::uint64_t n, double fx, double fy, double inv_two_var, double* factors) {
  const std::uint64_t i = static_cast<std::uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double dx = states[4 * i + 2] - fx, dy = states[4 * i + 3] - fy;
  factors[i] = exp(-(dx * dx + dy * dy) * inv_two_var);
}

}  // namespace

void launch_position_fix(void* stream, const double* states, std::uint64_t n, double fx, double fy, double sigma, double* factors) {
  const unsigned blocks = static_cast<unsigned>((n + 255) / 256);
  position_fix_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(states, n, fx, fy, 1.0 / (2.0 * sigma * sigma), factors);
}
