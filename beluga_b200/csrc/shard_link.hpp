// The link between the shards of one filter (DESIGN.md section 5): this rank's mail block, the ranks' totals and the
// whole filter's KLD hash array, the views of every rank's buffers that the exchange and resample kernels write to, and
// the CUDA IPC mappings behind the views of peers in other processes.  Host code only.
#pragma once

#include <cuda_runtime_api.h>

#include <memory>
#include <string>

#include "device_buffer.hpp"
#include "kernels.cuh"

namespace bb200 {

/// One buffer of a peer process mapped into this one (cudaIpcOpenMemHandle), closed exactly once by its owner.
struct IpcClose {
  void operator()(void* p) const { cudaIpcCloseMemHandle(p); }
};
using IpcMapping = std::unique_ptr<void, IpcClose>;

/// The methods returning int return a bb200_status and record its message in the owner's error string.
class ShardLink {
 public:
  explicit ShardLink(std::string* error) : error_(error) {}

  /// This rank's mail block (zeroed on `stream`) and totals.  state0 and state1 are the filter's two state buffers: they
  /// are exported and joined as they are, so the filter never reallocates them.
  cudaError_t create(const bb200_filter_config& config, Pose2* state0, Pose2* state1, cudaStream_t stream);
  /// KLD-adaptive resampling on shards needs one hash array of the WHOLE filter's slot count on every rank, exported
  /// with the other buffers: call before export_handles / join_local.
  int enable_kld();
  /// CUDA IPC handles of the two state buffers, the mail block and the KLD hash array (4 x 64 bytes, the last one zero
  /// without KLD) for peers in OTHER processes.
  int export_handles(void* out256) const;
  /// Maps the peers' buffers from their exported handles (world x 256 bytes, rank order); one process per GPU.  All or
  /// nothing: when an open fails, the link stays unjoined with nothing mapped.
  int join_ipc(int world, int rank, const void* handles);
  /// Shards living in THIS process (one per device, or several on one device): direct pointers, peer access enabled
  /// between distinct devices.  links[r] becomes rank r.
  static int join_local(ShardLink* const* links, int world);
  /// Waits for `stream` (nothing in flight may still use a peer's buffer), then unmaps the peers' buffers.  Every rank
  /// leaves before any frees its own: CUDA IPC requires importers to close first.
  int leave(cudaStream_t stream);

  int world() const { return world_; }
  int rank() const { return rank_; }
  /// Post and wait as separate launches (several shards enqueued by one thread).
  bool split_posts() const { return split_posts_; }
  /// The last join linked every rank's KLD hash array.
  bool kld() const { return kld_; }
  unsigned long long* kld_hashes() const { return kld_hashes_.get(); }

  /// Starts a new batch of exchanges (all ranks count alike).
  void begin_batch() { ++epoch_; }
  /// One post and/or wait of `kind` (launch_shard_exchange) between the filter's buffers and the peers'.
  void exchange(int kind, bool post, bool wait, Scalars* scalars, double* results, StepSummary* summary, unsigned long long* tile_state,
                uint32_t n_tiles, cudaStream_t stream) const;
  /// The link's part of a sharded resample launch: rank, world, the ranks' totals, and every rank's state buffer `buffer`
  /// as the target of its slots.
  void target_states(ResampleArgs* a, int buffer) const;
  /// The same for the KLD counting pass: every rank's hash array as the target of each candidate's hash.
  void target_hashes(ResampleArgs* a) const;

 private:
  int check(cudaError_t e, const char* what) const { return cuda_check(e, what, error_); }
  void set_ranks(ResampleArgs* a) const;

  std::string* error_;
  bb200_filter_config config_{};
  Pose2* own_states_[2]{};
  DeviceBuffer<ShardMail> mail_;                  // this rank's mail block
  DeviceBuffer<unsigned long long> totals_;       // the ranks' fixed-point totals of this step
  DeviceBuffer<unsigned long long> kld_hashes_;   // KLD on shards: spatial hash of every candidate slot (all ranks hold all)

  int world_{0}, rank_{0};
  bool split_posts_{false};
  bool kld_{false};
  unsigned long long epoch_{0};  // sequence number of the next exchange
  // [rank]: every rank's buffers as seen from here ([rank_] are this rank's own).  Views of local peers are borrowed
  // from their filters; those of peers in other processes are the mappings below.
  Pose2* states_[2][kMaxShards]{};
  ShardMail* mail_views_[kMaxShards]{};
  unsigned long long* kld_views_[kMaxShards]{};
  IpcMapping mappings_[kMaxShards][4];  // [rank][states 0, states 1, mail, KLD hashes]
};

}  // namespace bb200
