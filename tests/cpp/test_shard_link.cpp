// csrc/shard_link.cpp without a GPU: the CUDA functions the link calls are defined here.  cudaIpcOpenMemHandle and
// cudaIpcCloseMemHandle count the live mappings and fail the k-th open on request; a handle carries the rank and buffer
// it was exported for.  Prints one line per failed check; exit status 0 when all checks pass.
#include "../../beluga_b200/csrc/shard_link.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <set>
#include <vector>

namespace {

std::set<void*> device_live, pinned_live;
std::set<void*> mapped;            // live IPC mappings
std::vector<uint64_t> opened_tags;  // tag of every successful open, in order
int open_calls = 0;
int fail_open = -1;                 // index of the open call that fails (-1: none)
int closes = 0, bad_closes = 0, empty_opens = 0;
int failures = 0;
bb200::ShardExchangeArgs last_exchange{};

// A peer's exported handle: its tag 1 + 4 * rank + buffer in the first 8 bytes, or all zero (no KLD hash array).
cudaIpcMemHandle_t handle_for(int rank, int buffer) {
  cudaIpcMemHandle_t h{};
  const uint64_t tag = 1 + 4 * static_cast<uint64_t>(rank) + static_cast<uint64_t>(buffer);
  std::memcpy(&h, &tag, sizeof(tag));
  return h;
}

#define EXPECT(cond)                                                       \
  do {                                                                     \
    if (!(cond)) {                                                         \
      std::printf("%s:%d: check failed: %s\n", __FILE__, __LINE__, #cond); \
      ++failures;                                                          \
    }                                                                      \
  } while (0)

}  // namespace

cudaError_t cudaMalloc(void** p, size_t bytes) {
  *p = std::malloc(bytes);
  device_live.insert(*p);
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) { return device_live.erase(p) == 1 ? (std::free(p), cudaSuccess) : cudaErrorInvalidValue; }
cudaError_t cudaMallocHost(void** p, size_t bytes) {
  *p = std::malloc(bytes);
  pinned_live.insert(*p);
  return cudaSuccess;
}
cudaError_t cudaFreeHost(void* p) { return pinned_live.erase(p) == 1 ? (std::free(p), cudaSuccess) : cudaErrorInvalidValue; }
cudaError_t cudaMemsetAsync(void* p, int value, size_t bytes, cudaStream_t) {
  std::memset(p, value, bytes);
  return cudaSuccess;
}
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaGetLastError() { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t) { return "stub error"; }
cudaError_t cudaDeviceCanAccessPeer(int* can, int, int) {
  *can = 1;
  return cudaSuccess;
}
cudaError_t cudaDeviceEnablePeerAccess(int, unsigned int) { return cudaSuccess; }
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) {
  std::memset(h, 0, sizeof(*h));
  std::memcpy(h, &p, sizeof(p));
  return cudaSuccess;
}
cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned int) {
  uint64_t tag = 0;
  std::memcpy(&tag, &h, sizeof(tag));
  if (tag == 0) ++empty_opens;
  if (open_calls++ == fail_open) return cudaErrorInvalidResourceHandle;
  *p = std::malloc(1);
  mapped.insert(*p);
  opened_tags.push_back(tag);
  return cudaSuccess;
}
cudaError_t cudaIpcCloseMemHandle(void* p) {
  if (mapped.erase(p) != 1) {
    ++bad_closes;
    return cudaErrorInvalidValue;
  }
  std::free(p);
  ++closes;
  return cudaSuccess;
}

namespace bb200 {
void launch_shard_exchange(const ShardExchangeArgs& args, cudaStream_t) { last_exchange = args; }
int ceil_log2_count(uint64_t n) {
  int b = 0;
  while ((uint64_t{1} << b) < n) ++b;
  return b;
}
}  // namespace bb200

using bb200::ShardLink;

namespace {

constexpr uint64_t kCapacity = 64;
bb200::Pose2 own_states[bb200::kMaxShards][2][1];  // stand-ins for each rank's state buffers (only their addresses are used)

void reset_counts() {
  opened_tags.clear();
  open_calls = closes = bad_closes = empty_opens = 0;
  fail_open = -1;
}

/// Rank `rank` of `world` with its mail block and totals, and its KLD hash array when `kld`.
std::unique_ptr<ShardLink> make_link(std::string* error, int world, int rank, bool kld) {
  auto link = std::make_unique<ShardLink>(error);
  const bb200_filter_config config{0, kCapacity, 7, rank * kCapacity, world * kCapacity, 0};
  EXPECT(link->create(config, own_states[rank][0], own_states[rank][1], nullptr) == cudaSuccess);
  if (kld) EXPECT(link->enable_kld() == BB200_OK);
  return link;
}

/// The handle blobs of a world: every rank's four handles, the KLD handle empty unless `peers_kld`.
std::vector<cudaIpcMemHandle_t> handles_for(int world, bool peers_kld) {
  std::vector<cudaIpcMemHandle_t> h(4 * static_cast<size_t>(world));
  for (int r = 0; r < world; ++r)
    for (int b = 0; b < 4; ++b) h[4 * r + b] = (b < 3 || peers_kld) ? handle_for(r, b) : cudaIpcMemHandle_t{};
  return h;
}

void test_ipc_join_opens_the_peers_handles() {
  for (const int world : {2, 3, 8})
    for (const int rank : {0, world / 2, world - 1})
      for (const int mode : {0, 1, 2}) {  // 0: no KLD, 1: KLD on every rank, 2: KLD here but not on the peers
        const bool own_kld = mode != 0, peers_kld = mode == 1;
        std::string error;
        reset_counts();
        {
          auto link = make_link(&error, world, rank, own_kld);
          const auto h = handles_for(world, peers_kld);
          EXPECT(link->join_ipc(world, rank, h.data()) == BB200_OK);
          EXPECT(link->world() == world && link->rank() == rank && !link->split_posts());
          EXPECT(link->kld() == (mode == 1));
          const int per_peer = mode == 1 ? 4 : 3;
          EXPECT(static_cast<int>(opened_tags.size()) == (world - 1) * per_peer && mapped.size() == opened_tags.size());
          EXPECT(empty_opens == 0);
          std::set<uint64_t> expected;
          for (int r = 0; r < world; ++r)
            for (int b = 0; b < per_peer; ++b)
              if (r != rank) expected.insert(1 + 4 * static_cast<uint64_t>(r) + static_cast<uint64_t>(b));
          EXPECT(std::set<uint64_t>(opened_tags.begin(), opened_tags.end()) == expected);  // each peer handle once, never this rank's own

          // The views: this rank's own buffers at [rank], the mappings elsewhere.
          bb200::ResampleArgs a{};
          link->target_states(&a, 1);
          EXPECT(a.peer_count == world && a.world == world && a.rank == rank && a.rank_totals != nullptr);
          for (int r = 0; r < world; ++r) EXPECT(r == rank ? a.peer_out[r] == own_states[rank][1] : mapped.count(a.peer_out[r]) == 1);
          link->target_hashes(&a);
          EXPECT(a.peer_hash_count == world);
          for (int r = 0; r < world; ++r)
            EXPECT(r == rank ? a.peer_hashes[r] == link->kld_hashes() : (a.peer_hashes[r] == nullptr) == (mode != 1));
          link->exchange(bb200::kExchangeTotal, true, true, nullptr, nullptr, nullptr, nullptr, 0, nullptr);
          EXPECT(last_exchange.world == world && last_exchange.rank == rank && last_exchange.rank_totals == a.rank_totals);
          for (int r = 0; r < world; ++r) EXPECT(r == rank ? device_live.count(last_exchange.peers[r]) == 1 : mapped.count(last_exchange.peers[r]) == 1);
        }
        EXPECT(mapped.empty() && closes == static_cast<int>(opened_tags.size()) && bad_closes == 0);  // destruction closes each once
      }
}

void test_ipc_join_is_all_or_nothing() {
  for (const int world : {2, 3, 8}) {
    const int opens = (world - 1) * 4;
    for (int k = 0; k < opens; ++k) {
      std::string error;
      reset_counts();
      auto link = make_link(&error, world, 1, true);
      const auto h = handles_for(world, true);
      fail_open = k;
      EXPECT(link->join_ipc(world, 1, h.data()) == BB200_ERR_CUDA);
      EXPECT(error.rfind("cudaIpcOpenMemHandle", 0) == 0);
      EXPECT(link->world() == 0 && !link->kld());
      EXPECT(mapped.empty() && closes == k && bad_closes == 0);  // the k mappings opened before the failure were closed
      bb200::ResampleArgs a{};
      link->target_states(&a, 0);
      EXPECT(a.peer_count == 0);
      fail_open = -1;
      EXPECT(link->join_ipc(world, 1, h.data()) == BB200_OK && link->world() == world && link->kld());  // nothing half-joined is left
      EXPECT(static_cast<int>(mapped.size()) == opens);
    }
  }
  EXPECT(mapped.empty() && bad_closes == 0);
}

void test_leave_closes_once() {
  std::string error;
  reset_counts();
  auto link = make_link(&error, 3, 2, true);
  const auto h = handles_for(3, true);
  EXPECT(link->join_ipc(3, 2, h.data()) == BB200_OK && mapped.size() == 8);
  EXPECT(link->join_ipc(3, 2, h.data()) == BB200_ERR_STATE && mapped.size() == 8);  // joined already: nothing opened
  EXPECT(link->leave(nullptr) == BB200_OK);
  EXPECT(link->world() == 0 && mapped.empty() && closes == 8 && bad_closes == 0);
  EXPECT(link->leave(nullptr) == BB200_OK && closes == 8);  // a second leave closes nothing
  EXPECT(link->join_ipc(3, 2, h.data()) == BB200_OK && mapped.size() == 8);  // and the link joins again
  link.reset();
  EXPECT(mapped.empty() && closes == 16 && bad_closes == 0);
}

void test_local_join_closes_nothing() {
  for (const int world : {1, 2, 8}) {
    reset_counts();
    std::vector<std::string> errors(static_cast<size_t>(world));
    std::vector<std::unique_ptr<ShardLink>> links;
    std::vector<ShardLink*> raw;
    for (int r = 0; r < world; ++r) {
      links.push_back(make_link(&errors[static_cast<size_t>(r)], world, r, true));
      raw.push_back(links.back().get());
    }
    EXPECT(ShardLink::join_local(raw.data(), world) == BB200_OK);
    EXPECT(ShardLink::join_local(raw.data(), world) == BB200_ERR_STATE && errors[0] == "the peers' buffers are already mapped");
    for (int r = 0; r < world; ++r) {
      EXPECT(links[r]->world() == world && links[r]->rank() == r && links[r]->split_posts() && links[r]->kld());
      bb200::ResampleArgs a{};
      links[r]->target_states(&a, 0);
      links[r]->target_hashes(&a);
      for (int b = 0; b < world; ++b) EXPECT(a.peer_out[b] == own_states[b][0] && a.peer_hashes[b] == links[b]->kld_hashes());  // borrowed
    }
    EXPECT(links[0]->leave(nullptr) == BB200_OK && links[0]->world() == 0);
    links.clear();
    EXPECT(open_calls == 0 && closes == 0 && bad_closes == 0);
  }
  EXPECT(device_live.empty() && pinned_live.empty());
}

}  // namespace

int main() {
  test_ipc_join_opens_the_peers_handles();
  test_ipc_join_is_all_or_nothing();
  test_leave_closes_once();
  test_local_join_closes_nothing();
  EXPECT(device_live.empty() && pinned_live.empty());
  if (failures == 0) std::printf("all shard link checks passed\n");
  return failures == 0 ? 0 : 1;
}
