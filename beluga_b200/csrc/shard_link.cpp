#include "shard_link.hpp"

#include <cstring>
#include <utility>

namespace bb200 {

cudaError_t ShardLink::create(const bb200_filter_config& config, Pose2* state0, Pose2* state1, cudaStream_t stream) {
  config_ = config;
  own_states_[0] = state0;
  own_states_[1] = state1;
  if (const cudaError_t e = mail_.allocate(1)) return e;  // its own allocation: exported to peer processes through CUDA IPC
  if (const cudaError_t e = totals_.allocate(kMaxShards)) return e;
  return cudaMemsetAsync(mail_.get(), 0, sizeof(ShardMail), stream);
}

int ShardLink::enable_kld() {
  if (kld_hashes_.get() != nullptr) return BB200_OK;
  if (world_ != 0) return reject(BB200_ERR_STATE, "KLD on shards must be enabled before the shards are joined", error_);
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(kld_hashes_.allocate(config_.global_count));  // one spatial hash per candidate slot of the WHOLE filter
  return BB200_OK;
}

int ShardLink::export_handles(void* out256) const {
  BB_CHECK(cudaSetDevice(config_.device));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "four IPC handles are exported as 256 bytes");
  cudaIpcMemHandle_t h[4];
  std::memset(h, 0, sizeof(h));
  BB_CHECK(cudaIpcGetMemHandle(&h[0], own_states_[0]));
  BB_CHECK(cudaIpcGetMemHandle(&h[1], own_states_[1]));
  BB_CHECK(cudaIpcGetMemHandle(&h[2], mail_.get()));
  if (kld_hashes_.get() != nullptr) BB_CHECK(cudaIpcGetMemHandle(&h[3], kld_hashes_.get()));
  std::memcpy(out256, h, sizeof(h));
  return BB200_OK;
}

int ShardLink::join_ipc(int world, int rank, const void* handles) {
  if (world < 1 || world > kMaxShards || rank < 0 || rank >= world) return reject(BB200_ERR_INVALID_ARGUMENT, "shard groups hold 1..8 ranks", error_);
  if (world_ != 0) return reject(BB200_ERR_STATE, "the peers' buffers are already mapped", error_);
  if (config_.first_index != static_cast<uint64_t>(rank) * config_.capacity || config_.global_count != static_cast<uint64_t>(world) * config_.capacity)
    return reject(BB200_ERR_INVALID_ARGUMENT, "shard r of R holds the global indices [r * capacity, (r + 1) * capacity) of R * capacity particles", error_);
  BB_CHECK(cudaSetDevice(config_.device));
  const auto* all = static_cast<const cudaIpcMemHandle_t*>(handles);
  static const cudaIpcMemHandle_t kNoHandle{};
  IpcMapping opened[kMaxShards][4];  // closed on return unless every open succeeds
  for (int r = 0; r < world; ++r) {
    if (r == rank) continue;
    for (int b = 0; b < 4; ++b) {
      if (b == 3 && (kld_hashes_.get() == nullptr || std::memcmp(&all[4 * r + 3], &kNoHandle, sizeof(kNoHandle)) == 0)) continue;  // no KLD on this filter
      void* p = nullptr;
      if (const int st = check(cudaIpcOpenMemHandle(&p, all[4 * r + b], cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle")) return st;
      opened[r][b].reset(p);
    }
  }
  for (int r = 0; r < world; ++r) {
    for (int b = 0; b < 4; ++b) mappings_[r][b] = std::move(opened[r][b]);
    const bool own = r == rank;
    states_[0][r] = own ? own_states_[0] : static_cast<Pose2*>(mappings_[r][0].get());
    states_[1][r] = own ? own_states_[1] : static_cast<Pose2*>(mappings_[r][1].get());
    mail_views_[r] = own ? mail_.get() : static_cast<ShardMail*>(mappings_[r][2].get());
    kld_views_[r] = own ? kld_hashes_.get() : static_cast<unsigned long long*>(mappings_[r][3].get());
  }
  world_ = world;
  rank_ = rank;
  kld_ = true;
  for (int r = 0; r < world; ++r) kld_ = kld_ && kld_views_[r] != nullptr;
  split_posts_ = false;  // every rank has its own host thread: post and wait travel in one launch
  return BB200_OK;
}

int ShardLink::join_local(ShardLink* const* links, int world) {
  if (links == nullptr || world < 1 || world > kMaxShards) return BB200_ERR_INVALID_ARGUMENT;
  for (int r = 0; r < world; ++r) {
    const ShardLink* l = links[r];
    if (l == nullptr || l->mail_.get() == nullptr) return BB200_ERR_INVALID_ARGUMENT;
    const bb200_filter_config& c = l->config_;
    if (l->world_ != 0) return reject(BB200_ERR_STATE, "the peers' buffers are already mapped", l->error_);
    if (c.capacity != links[0]->config_.capacity || c.first_index != static_cast<uint64_t>(r) * c.capacity ||
        c.global_count != static_cast<uint64_t>(world) * c.capacity || c.seed != links[0]->config_.seed)
      return reject(BB200_ERR_INVALID_ARGUMENT, "shard r of R holds the global indices [r * capacity, (r + 1) * capacity) of R * capacity particles, same seed",
                    l->error_);
  }
  for (int a = 0; a < world; ++a) {
    ShardLink* la = links[a];
    for (int b = 0; b < world; ++b) {
      const ShardLink* lb = links[b];
      if (la->config_.device != lb->config_.device) {
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, la->config_.device, lb->config_.device) != cudaSuccess || !can)
          return reject(BB200_ERR_CUDA, "no peer access between the devices of two shards", la->error_);
        if (la->check(cudaSetDevice(la->config_.device), "cudaSetDevice") != BB200_OK) return BB200_ERR_CUDA;
        const cudaError_t e = cudaDeviceEnablePeerAccess(lb->config_.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return la->check(e, "cudaDeviceEnablePeerAccess");
        (void)cudaGetLastError();
      }
      la->states_[0][b] = lb->own_states_[0];
      la->states_[1][b] = lb->own_states_[1];
      la->mail_views_[b] = lb->mail_.get();
      la->kld_views_[b] = lb->kld_hashes_.get();
    }
    la->kld_ = true;
    for (int b = 0; b < world; ++b) la->kld_ = la->kld_ && links[b]->kld_hashes_.get() != nullptr;
    la->world_ = world;
    la->rank_ = a;
    la->split_posts_ = true;  // one thread enqueues all shards: every post must be enqueued before any wait that needs it
  }
  return BB200_OK;
}

int ShardLink::leave(cudaStream_t stream) {
  BB_CHECK(cudaSetDevice(config_.device));
  BB_CHECK(cudaStreamSynchronize(stream));
  for (int r = 0; r < kMaxShards; ++r) {
    for (int b = 0; b < 4; ++b) mappings_[r][b].reset();
    states_[0][r] = states_[1][r] = nullptr;
    mail_views_[r] = nullptr;
    kld_views_[r] = nullptr;
  }
  world_ = 0;
  return BB200_OK;
}

void ShardLink::exchange(int kind, bool post, bool wait, Scalars* scalars, double* results, StepSummary* summary, unsigned long long* tile_state,
                         uint32_t n_tiles, cudaStream_t stream) const {
  ShardExchangeArgs a{};
  a.kind = kind;
  a.post = post ? 1 : 0;
  a.wait = wait ? 1 : 0;
  a.rank = rank_;
  a.world = world_;
  a.epoch = epoch_;
  for (int r = 0; r < world_; ++r) a.peers[r] = mail_views_[r];
  a.scalars = scalars;
  a.results = results;
  a.summary = summary;
  a.rank_totals = totals_.get();
  a.ceil_log2_count = ceil_log2_count(config_.global_count);
  a.tile_state = tile_state;
  a.n_tiles = n_tiles;
  launch_shard_exchange(a, stream);
}

void ShardLink::set_ranks(ResampleArgs* a) const {
  a->rank_totals = totals_.get();
  a->rank = rank_;
  a->world = world_;
}

void ShardLink::target_states(ResampleArgs* a, int buffer) const {
  set_ranks(a);
  a->peer_count = world_;
  for (int r = 0; r < world_; ++r) a->peer_out[r] = states_[buffer][r];
}

void ShardLink::target_hashes(ResampleArgs* a) const {
  set_ranks(a);
  a->peer_hash_count = world_;
  for (int r = 0; r < world_; ++r) a->peer_hashes[r] = kld_views_[r];
}

}  // namespace bb200
