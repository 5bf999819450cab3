// The one owner of the library's CUDA memory: every device (cudaMalloc) and pinned host (cudaMallocHost) buffer of Filter,
// Batch, Clusterizer and DeviceMap is a Buffer, freed by its destructor.  A buffer never zeroes its memory and never
// synchronises: whoever frees memory that a stream may still read synchronises that stream first.
//
// Buffers allocated on first use come in groups.  A group is allocated into a local struct of Buffers and moved into its
// owner only when every allocation has succeeded, so that a failure leaves the owner as it was and frees the attempt.
#pragma once

#include <cuda_runtime_api.h>

#include <cstddef>
#include <utility>

namespace bb200 {

enum class Memory { kDevice, kPinned };

template <class T, Memory M>
class Buffer {
 public:
  Buffer() = default;
  ~Buffer() { reset(); }
  Buffer(Buffer&& other) noexcept : p_(std::exchange(other.p_, nullptr)), n_(std::exchange(other.n_, 0)) {}
  Buffer& operator=(Buffer&& other) noexcept {
    if (this != &other) {
      reset();
      p_ = std::exchange(other.p_, nullptr);
      n_ = std::exchange(other.n_, 0);
    }
    return *this;
  }
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;

  T* get() const { return p_; }
  size_t size() const { return n_; }  // elements

  /// Drops the old contents and allocates `count` elements, at least one, so that an empty table still has an address.
  /// On failure the buffer is empty (null, size 0).
  cudaError_t allocate(size_t count) {
    reset();
    const size_t n = count > 1 ? count : 1;
    void* p = nullptr;
    const cudaError_t e = M == Memory::kDevice ? cudaMalloc(&p, n * sizeof(T)) : cudaMallocHost(&p, n * sizeof(T));
    if (e != cudaSuccess) return e;
    p_ = static_cast<T*>(p);
    n_ = n;
    return cudaSuccess;
  }
  /// Room for `count` elements: when the buffer holds fewer, allocate(max(count, room)), which drops the contents.
  cudaError_t grow(size_t count, size_t room = 0) { return count > n_ ? allocate(count > room ? count : room) : cudaSuccess; }

 private:
  void reset() {
    if (p_ != nullptr) {
      if (M == Memory::kDevice) {
        cudaFree(p_);
      } else {
        cudaFreeHost(p_);
      }
    }
    p_ = nullptr;
    n_ = 0;
  }

  T* p_{nullptr};
  size_t n_{0};
};

template <class T>
using DeviceBuffer = Buffer<T, Memory::kDevice>;
template <class T>
using PinnedBuffer = Buffer<T, Memory::kPinned>;

/// A device buffer and its pinned twin: a table the host fills and uploads, or one the device fills and the host reads.
/// Callers fill host.get() and hand device.get() to launchers; the pair only sizes both halves together and copies
/// between them.
template <class T>
struct MirroredBuffer {
  DeviceBuffer<T> device;
  PinnedBuffer<T> host;

  /// Elements both halves hold: after a failed grow the pair is short, and the next grow retries the half that failed.
  size_t size() const { return device.size() < host.size() ? device.size() : host.size(); }
  /// Buffer::grow on the device half, then on the pinned half; the first error.
  cudaError_t grow(size_t count, size_t room = 0) {
    const cudaError_t e = device.grow(count, room);
    return e != cudaSuccess ? e : host.grow(count, room);
  }
  /// One cudaMemcpyAsync of elements [first, first + count) from the pinned half to the device half, or back.
  cudaError_t to_device(size_t first, size_t count, cudaStream_t stream) const {
    return cudaMemcpyAsync(device.get() + first, host.get() + first, count * sizeof(T), cudaMemcpyHostToDevice, stream);
  }
  cudaError_t to_host(size_t first, size_t count, cudaStream_t stream) const {
    return cudaMemcpyAsync(host.get() + first, device.get() + first, count * sizeof(T), cudaMemcpyDeviceToHost, stream);
  }
};

}  // namespace bb200
