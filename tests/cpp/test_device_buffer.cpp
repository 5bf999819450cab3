// csrc/device_buffer.hpp without a GPU: the four CUDA allocation functions are defined here over malloc, count the live
// allocations of each kind and fail the k-th call on request, and cudaMemcpyAsync records each copy it is asked for.
// Prints one line per failed check; exit status 0 when all checks pass.
#include "../../beluga_b200/csrc/device_buffer.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <utility>
#include <vector>

namespace {

std::map<void*, size_t> device_live, pinned_live;  // live allocations of each kind -> bytes
int alloc_calls = 0;   // allocation calls so far
int fail_call = -1;    // index of the allocation call that fails (-1: none)
int bad_frees = 0;     // frees of a pointer that is not live in that kind (double frees, wrong kind, null)
int failures = 0;

struct Copy {
  void* dst;
  const void* src;
  size_t bytes;
  cudaMemcpyKind kind;
  cudaStream_t stream;
};
std::vector<Copy> copies;                  // every cudaMemcpyAsync call, in order
cudaError_t copy_result = cudaSuccess;  // what cudaMemcpyAsync returns

cudaError_t fake_alloc(void** p, size_t bytes, std::map<void*, size_t>& live) {
  if (alloc_calls++ == fail_call) return cudaErrorMemoryAllocation;  // *p stays as it was, like the runtime's
  *p = std::malloc(bytes);
  live[*p] = bytes;
  return cudaSuccess;
}

cudaError_t fake_free(void* p, std::map<void*, size_t>& live) {
  if (live.erase(p) != 1) {
    ++bad_frees;
    return cudaErrorInvalidValue;
  }
  std::free(p);
  return cudaSuccess;
}

size_t live_count() { return device_live.size() + pinned_live.size(); }

#define EXPECT(cond)                                                   \
  do {                                                                 \
    if (!(cond)) {                                                     \
      std::printf("%s:%d: check failed: %s\n", __FILE__, __LINE__, #cond); \
      ++failures;                                                      \
    }                                                                  \
  } while (0)

}  // namespace

cudaError_t cudaMalloc(void** p, size_t bytes) { return fake_alloc(p, bytes, device_live); }
cudaError_t cudaFree(void* p) { return fake_free(p, device_live); }
cudaError_t cudaMallocHost(void** p, size_t bytes) { return fake_alloc(p, bytes, pinned_live); }
cudaError_t cudaFreeHost(void* p) { return fake_free(p, pinned_live); }
cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t stream) {
  copies.push_back(Copy{dst, src, bytes, kind, stream});
  return copy_result;
}

using bb200::DeviceBuffer;
using bb200::MirroredBuffer;
using bb200::PinnedBuffer;

namespace {

void test_kinds_and_sizes() {
  {
    DeviceBuffer<double> d;
    PinnedBuffer<int> h;
    EXPECT(d.get() == nullptr && d.size() == 0 && live_count() == 0);
    EXPECT(d.allocate(10) == cudaSuccess && d.size() == 10 && device_live.count(d.get()) == 1 && device_live[d.get()] == 10 * sizeof(double));
    EXPECT(h.allocate(3) == cudaSuccess && h.size() == 3 && pinned_live.count(h.get()) == 1 && pinned_live[h.get()] == 3 * sizeof(int));
    EXPECT(device_live.size() == 1 && pinned_live.size() == 1);
    EXPECT(d.allocate(0) == cudaSuccess && d.size() == 1 && device_live[d.get()] == sizeof(double));  // an empty table still has an address
    EXPECT(device_live.size() == 1);  // the old contents went
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

void test_move() {
  {
    DeviceBuffer<uint32_t> a;
    EXPECT(a.allocate(8) == cudaSuccess);
    uint32_t* p = a.get();
    DeviceBuffer<uint32_t> b(std::move(a));
    EXPECT(a.get() == nullptr && a.size() == 0 && b.get() == p && b.size() == 8 && live_count() == 1);
    DeviceBuffer<uint32_t> c;
    EXPECT(c.allocate(4) == cudaSuccess && live_count() == 2);
    c = std::move(b);  // c's own buffer is freed, b's moves over
    EXPECT(b.get() == nullptr && b.size() == 0 && c.get() == p && c.size() == 8 && live_count() == 1);
    DeviceBuffer<uint32_t>& alias = c;
    c = std::move(alias);
    EXPECT(c.get() == p && c.size() == 8 && live_count() == 1);
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

void test_grow() {
  {
    DeviceBuffer<double> b;
    EXPECT(b.grow(0) == cudaSuccess && b.get() == nullptr && alloc_calls == 0);  // nothing needed: nothing allocated
    EXPECT(b.grow(10) == cudaSuccess && b.size() == 10);
    double* p = b.get();
    const int calls = alloc_calls;
    EXPECT(b.grow(10, 1000) == cudaSuccess && b.get() == p && alloc_calls == calls);  // room enough: no reallocation
    EXPECT(b.grow(11, 64) == cudaSuccess && b.size() == 64 && live_count() == 1);     // the growth policy's room
    EXPECT(b.grow(100, 64) == cudaSuccess && b.size() == 100 && live_count() == 1);   // never less than asked for
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

void test_failure_leaves_empty() {
  {
    DeviceBuffer<double> d;
    PinnedBuffer<double> h;
    EXPECT(d.allocate(5) == cudaSuccess && h.allocate(5) == cudaSuccess);
    fail_call = alloc_calls;
    EXPECT(d.allocate(7) == cudaErrorMemoryAllocation && d.get() == nullptr && d.size() == 0);
    fail_call = alloc_calls;
    EXPECT(h.grow(9) == cudaErrorMemoryAllocation && h.get() == nullptr && h.size() == 0);
    fail_call = -1;
    EXPECT(live_count() == 0);
    EXPECT(d.grow(3) == cudaSuccess && d.size() == 3 && live_count() == 1);  // an empty buffer grows again
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

// A group of buffers allocated on first use, the way Filter, Batch and Clusterizer allocate their lazy scratch: into a
// local struct, moved into the owner only when every allocation has succeeded.
struct Group {
  DeviceBuffer<unsigned long long> keys;
  DeviceBuffer<uint32_t> sort[2];
  PinnedBuffer<double> staging;
  DeviceBuffer<uint32_t> cells;
};
constexpr int kGroupAllocations = 5;

cudaError_t allocate_group(Group* target, size_t n) {
  Group g;
  if (const cudaError_t e = g.keys.allocate(2 * n)) return e;
  if (const cudaError_t e = g.sort[0].allocate(n)) return e;
  if (const cudaError_t e = g.sort[1].allocate(n)) return e;
  if (const cudaError_t e = g.staging.allocate(n)) return e;
  if (const cudaError_t e = g.cells.allocate(n + 1)) return e;
  *target = std::move(g);
  return cudaSuccess;
}

void test_group_all_or_nothing(bool filled) {
  {
    Group target;
    if (filled) EXPECT(allocate_group(&target, 16) == cudaSuccess);
    const void* before[kGroupAllocations] = {target.keys.get(), target.sort[0].get(), target.sort[1].get(), target.staging.get(), target.cells.get()};
    const size_t baseline = live_count();
    EXPECT(baseline == (filled ? kGroupAllocations : 0u));
    for (int k = 0; k < kGroupAllocations; ++k) {
      fail_call = alloc_calls + k;
      EXPECT(allocate_group(&target, 32) == cudaErrorMemoryAllocation);
      const void* after[kGroupAllocations] = {target.keys.get(), target.sort[0].get(), target.sort[1].get(), target.staging.get(), target.cells.get()};
      for (int b = 0; b < kGroupAllocations; ++b) EXPECT(after[b] == before[b]);  // the owner kept what it had
      EXPECT(target.sort[0].size() == (filled ? 16u : 0u));
      EXPECT(live_count() == baseline);  // and the attempt freed what it allocated
    }
    fail_call = -1;
    EXPECT(allocate_group(&target, 32) == cudaSuccess);
    EXPECT(target.keys.size() == 64 && target.sort[0].size() == 32 && target.sort[1].size() == 32 && target.staging.size() == 32 &&
           target.cells.size() == 33);
    EXPECT(live_count() == static_cast<size_t>(kGroupAllocations));  // the old group (if any) went
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

void test_mirrored_grow() {
  {
    MirroredBuffer<double> m;
    EXPECT(m.size() == 0 && m.grow(0) == cudaSuccess && live_count() == 0);
    EXPECT(m.grow(10, 16) == cudaSuccess && m.device.size() == 16 && m.host.size() == 16 && m.size() == 16);
    EXPECT(device_live.size() == 1 && pinned_live.size() == 1);
    double* d = m.device.get();
    const int calls = alloc_calls;
    EXPECT(m.grow(16, 100) == cudaSuccess && m.device.get() == d && alloc_calls == calls);  // room enough in both halves

    fail_call = alloc_calls + 1;  // the pinned half fails
    EXPECT(m.grow(20) == cudaErrorMemoryAllocation);
    EXPECT(m.device.size() == 20 && m.host.get() == nullptr && m.size() == 0 && device_live.size() == 1 && pinned_live.empty());
    fail_call = -1;
    d = m.device.get();
    const int before_retry = alloc_calls;
    EXPECT(m.grow(20) == cudaSuccess && m.size() == 20);  // the short half alone grows again
    EXPECT(m.device.get() == d && alloc_calls == before_retry + 1 && pinned_live.size() == 1);

    fail_call = alloc_calls;  // the device half fails: the pinned half is left as it was
    EXPECT(m.grow(40) == cudaErrorMemoryAllocation);
    EXPECT(m.device.get() == nullptr && m.host.size() == 20 && m.size() == 0 && device_live.empty() && pinned_live.size() == 1);
    fail_call = -1;
    EXPECT(m.grow(40) == cudaSuccess && m.device.size() == 40 && m.host.size() == 40 && m.size() == 40 && live_count() == 2);
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

void test_mirrored_move() {
  {
    MirroredBuffer<uint32_t> a;
    EXPECT(a.grow(8) == cudaSuccess);
    uint32_t* d = a.device.get();
    uint32_t* h = a.host.get();
    MirroredBuffer<uint32_t> b(std::move(a));
    EXPECT(a.device.get() == nullptr && a.host.get() == nullptr && a.size() == 0);
    EXPECT(b.device.get() == d && b.host.get() == h && b.size() == 8 && live_count() == 2);
    MirroredBuffer<uint32_t> c;
    EXPECT(c.grow(4) == cudaSuccess && live_count() == 4);
    c = std::move(b);  // c's own halves are freed, b's move over
    EXPECT(b.size() == 0 && c.device.get() == d && c.host.get() == h && live_count() == 2);
    c = {};  // as a relayout drops a table sized by the old slot count
    EXPECT(c.size() == 0 && live_count() == 0);
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

void test_mirrored_copies() {
  {
    MirroredBuffer<uint64_t> m;
    EXPECT(m.grow(16) == cudaSuccess);
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(static_cast<uintptr_t>(0x5a));
    copies.clear();
    EXPECT(m.to_device(2, 3, stream) == cudaSuccess);
    EXPECT(m.to_host(5, 4, stream) == cudaSuccess);
    EXPECT(copies.size() == 2);
    if (copies.size() == 2) {
      const Copy& up = copies[0];
      EXPECT(up.dst == m.device.get() + 2 && up.src == m.host.get() + 2 && up.bytes == 3 * sizeof(uint64_t));
      EXPECT(up.kind == cudaMemcpyHostToDevice && up.stream == stream);
      const Copy& down = copies[1];
      EXPECT(down.dst == m.host.get() + 5 && down.src == m.device.get() + 5 && down.bytes == 4 * sizeof(uint64_t));
      EXPECT(down.kind == cudaMemcpyDeviceToHost && down.stream == stream);
    }
    copy_result = cudaErrorInvalidValue;  // the copy's error reaches the caller
    EXPECT(m.to_device(0, 1, stream) == cudaErrorInvalidValue && m.to_host(0, 1, stream) == cudaErrorInvalidValue);
    copy_result = cudaSuccess;
  }
  EXPECT(live_count() == 0 && bad_frees == 0);
}

}  // namespace

int main() {
  test_kinds_and_sizes();
  test_move();
  alloc_calls = 0;
  test_grow();
  test_failure_leaves_empty();
  test_group_all_or_nothing(false);
  test_group_all_or_nothing(true);
  test_mirrored_grow();
  test_mirrored_move();
  test_mirrored_copies();
  if (failures == 0) std::printf("all device buffer checks passed\n");
  return failures == 0 ? 0 : 1;
}
