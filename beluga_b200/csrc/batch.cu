#include "batch.hpp"
#include "measurement_host.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <utility>

namespace bb200 {

namespace {

constexpr uint64_t kSliceAlign = 32;  // particles
static_assert(kBatchMaxParticles <= kBatchClusterMaxParticles, "the batch cluster estimate packs a member's particle index into 15 bits");

/// Moment-partial rows a member of `capacity` particles can need in the finish launch (whichever form it takes).
uint64_t finish_rows(uint64_t capacity) {
  return std::max<uint64_t>({resample_scatter_block_count(capacity), resample_block_count(capacity), moments_block_count(capacity)});
}

/// The CTA ranges of Rows launches over n members, through which their kernels find a CTA's member: ctas(j, c) writes
/// member j's CTA count in row l to c[l].  Row l (first + l * (n + 1)) receives the exclusive prefix of its counts and
/// then their total, which totals[l] receives too.
template <int Rows, class Ctas>
void write_cta_rows(uint32_t* first, uint32_t n, uint32_t* totals, Ctas ctas) {
  for (int l = 0; l < Rows; ++l) totals[l] = 0;
  for (uint32_t j = 0; j < n; ++j) {
    uint32_t c[Rows];
    ctas(j, c);
    for (int l = 0; l < Rows; ++l) {
      first[static_cast<size_t>(l) * (n + 1) + j] = totals[l];
      totals[l] += c[l];
    }
  }
  for (int l = 0; l < Rows; ++l) first[static_cast<size_t>(l) * (n + 1) + n] = totals[l];
}

}  // namespace

int Batch::validate_member(const bb200_amcl_param& p, const bb200_motion_param& motion, int k, int device, uint32_t flags, std::string* error) {
  auto reject = [&](const std::string& m) {
    if (error != nullptr) *error = m;
    return static_cast<int>(BB200_ERR_INVALID_ARGUMENT);
  };
  const bool adaptive = (flags & BB200_BATCH_ADAPTIVE) != 0, selective = (flags & BB200_BATCH_SELECTIVE) != 0;
  const std::string who = "member " + std::to_string(k) + ": ";
  if (p.device != device) return reject(who + "all members of a batch share one device");
  if (p.max_particles == 0 || p.max_particles > kBatchMaxParticles) return reject(who + "max_particles must lie in [1, 32768]");
  if (!adaptive && p.min_particles != p.max_particles)
    return reject(who + "a batch member keeps a fixed particle count (min_particles == max_particles)");
  if (p.min_particles > p.max_particles) return reject(who + "need 0 < min_particles <= max_particles");  // bb200_amcl_create's check
  if (p.selective_resampling && !selective) return reject(who + "selective resampling is not supported in a batch");
  if (p.shard_first_index != 0 || p.shard_capacity != 0) return reject(who + "a batch member is not sharded");
  if (!(p.alpha_slow >= 0.0) || !(p.alpha_slow <= p.alpha_fast)) return reject(who + "need 0 <= alpha_slow <= alpha_fast");
  if (motion.model < BB200_MOTION_DIFFERENTIAL || motion.model > BB200_MOTION_STATIONARY) return reject(who + "unknown motion model");
  return BB200_OK;
}

int Batch::validate(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags, std::string* error) {
  auto reject = [&](const std::string& m) {
    if (error != nullptr) *error = m;
    return static_cast<int>(BB200_ERR_INVALID_ARGUMENT);
  };
  if ((flags & ~static_cast<uint32_t>(BB200_BATCH_ADAPTIVE | BB200_BATCH_SELECTIVE)) != 0) return reject("unknown batch flags");
  if (params == nullptr || motions == nullptr) return reject("null argument");
  if (n_members < 1) return reject("a batch needs at least one member");
  for (int k = 0; k < n_members; ++k)
    if (const int st = validate_member(params[k], motions[k], k, params[0].device, flags, error)) return st;
  return BB200_OK;
}

Batch::Layout Batch::lay_out(const std::vector<const bb200_amcl_param*>& slots) {
  Layout l;
  l.offset.assign(slots.size(), 0);
  l.table_offset.assign(slots.size(), 0);
  l.table_slots.assign(slots.size(), 0);
  for (size_t k = 0; k < slots.size(); ++k) {
    if (slots[k] == nullptr) continue;
    const uint64_t capacity = slots[k]->max_particles;
    // The CDF build reads weights and writes the CDF 16 bytes at a time from the slice's start: slices begin on whole
    // 256-byte lines.
    l.total = (l.total + kSliceAlign - 1) / kSliceAlign * kSliceAlign;
    l.offset[k] = l.total;
    l.total += capacity;
    l.table_offset[k] = l.table_total;
    uint32_t table_slots = 2;
    while (table_slots < 2 * capacity) table_slots <<= 1;
    l.table_slots[k] = table_slots;
    l.table_total += table_slots;
    l.tiles += batch_scan_tiles(capacity);
    l.rows += finish_rows(capacity);
    l.record_ancestors = l.record_ancestors || slots[k]->record_ancestors != 0;
  }
  return l;
}

void Batch::place(const Layout& l) {
  for (size_t k = 0; k < members_.size(); ++k) {
    Member& m = members_[k];
    if (!m.active) continue;
    m.offset = l.offset[k];
    m.table_offset = l.table_offset[k];
    m.table_slots = l.table_slots[k];
  }
  total_ = l.total;
  table_total_ = l.table_total;
  record_ancestors_ = l.record_ancestors;
}

int Batch::allocate(const Layout& l, size_t slots, Storage* s) {
  const size_t k1 = slots + 1;
  BB_CHECK(s->states[0].allocate(l.total));
  BB_CHECK(s->states[1].allocate(l.total));
  BB_CHECK(s->weights.allocate(l.total));
  BB_CHECK(s->cdf.allocate(l.total));
  if (l.record_ancestors) BB_CHECK(s->ancestors.allocate(l.total));
  BB_CHECK(s->scalars.allocate(slots));
  BB_CHECK(s->tile_state.allocate(l.tiles));
  BB_CHECK(s->partials.allocate(l.rows * kMomentCount));
  BB_CHECK(s->table.grow(slots));
  BB_CHECK(s->first.grow(kBatchRows * k1));
  BB_CHECK(s->summary_host.allocate(slots));
  BB_CHECK(cudaMemsetAsync(s->scalars.get(), 0, slots * sizeof(Scalars), stream_));
  return BB200_OK;
}

void Batch::adopt(Storage&& s) {
  states_[0] = std::move(s.states[0]);
  states_[1] = std::move(s.states[1]);
  weights_ = std::move(s.weights);
  cdf_ = std::move(s.cdf);
  ancestors_ = std::move(s.ancestors);
  scalars_ = std::move(s.scalars);
  tile_state_ = std::move(s.tile_state);
  partials_ = std::move(s.partials);
  table_ = std::move(s.table);
  first_ = std::move(s.first);
  summary_host_ = std::move(s.summary_host);
}

Batch::Batch(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags) {
  create_status_ = validate(params, motions, n_members, flags, &error_);
  if (create_status_ != BB200_OK) return;
  flags_ = flags;
  members_.reserve(static_cast<size_t>(n_members));
  std::vector<const bb200_amcl_param*> slots;
  for (int k = 0; k < n_members; ++k) {
    members_.push_back(Member{AmclPolicy(params[k], motions[k])});
    members_.back().capacity = params[k].max_particles;
    slots.push_back(&params[k]);
  }
  const Layout layout = lay_out(slots);
  place(layout);
  device_ = params[0].device;
  create_status_ = check_device(device_, &error_);
  if (create_status_ != BB200_OK) return;
  BB_TRY(cudaSetDevice(device_));
  BB_TRY(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  Storage s;
  create_status_ = allocate(layout, members_.size(), &s);
  if (create_status_ != BB200_OK) return;
  adopt(std::move(s));
  BB_TRY(ticket_host_.allocate(1));
  BB_TRY(members_done_.allocate(1));
  *ticket_host_.get() = 0;  // pinned allocations are recycled with their old contents
  BB_TRY(cudaMemsetAsync(members_done_.get(), 0, sizeof(unsigned int), stream_));
  BB_TRY(cudaStreamSynchronize(stream_));
  created_ = true;
}

int Batch::relayout(const std::vector<const bb200_amcl_param*>& slots, Layout* layout, const Arrival* arrival) {
  BB_CHECK(cudaSetDevice(device_));
  *layout = lay_out(slots);
  // Every allocation before anything moves: a failure frees the attempt and leaves the batch as it was.
  Storage s;
  if (const int st = allocate(*layout, slots.size(), &s)) return st;
  std::vector<BatchRelayoutMember> moves;
  for (size_t k = 0; k < members_.size(); ++k) {
    const Member& m = members_[k];
    if (!m.active || slots[k] == nullptr) continue;
    BatchRelayoutMember r{};
    r.from = m.offset;
    r.to = layout->offset[k];
    r.n = m.n;
    r.cdf_n = m.cdf_total != 0 ? m.n : 0;
    r.ancestors_n = m.policy.params().record_ancestors && ancestors_.get() != nullptr ? m.ancestors_n : 0;
    r.cur = m.cur;
    if (batch_relayout_ctas(r) > 0) moves.push_back(r);
  }
  if (!moves.empty()) {
    BatchRelayoutArgs a{};
    a.states_from[0] = states_[0].get();
    a.states_from[1] = states_[1].get();
    a.weights_from = weights_.get();
    a.cdf_from = cdf_.get();
    a.ancestors_from = ancestors_.get();
    a.states_to = s.states[0].get();
    a.weights_to = s.weights.get();
    a.cdf_to = s.cdf.get();
    a.ancestors_to = s.ancestors.get();
    if (const int st = launch_moves(moves, a)) return st;
  }
  // The arrival is one move: it fits the transfer tables the survivors' launch may have grown, so none is freed in flight.
  if (arrival != nullptr)
    if (const int st = unpack({arrival->state}, {layout->offset[arrival->slot]}, s.states[0].get(), s.weights.get(), s.cdf.get(), s.ancestors.get()))
      return st;
  BB_CHECK(cudaStreamSynchronize(stream_));  // the moves have landed; nothing in flight reads the old buffers

  // Nothing can fail from here on.
  adopt(std::move(s));
  for (size_t k = 0; k < members_.size(); ++k)
    if (members_[k].active && slots[k] != nullptr) members_[k].cur = 0;  // the kernel wrote every survivor's states to buffer 0
  // Scratch allocated on first use and sized by the layout or the slot count: re-created on next use.
  cl_ = ClusterBuffers{};
  kld_ = {};
  sel_ = SelectBuffers{};
  sm_table_ = {};
  inputs_ = {};
  return BB200_OK;
}

int Batch::join(const bb200_amcl_param& params, const bb200_motion_param& motion, const FilterState* state, int map, int* member) {
  size_t slot = 0;
  while (slot < members_.size() && members_[slot].active) ++slot;
  if (const int st = validate_member(params, motion, static_cast<int>(slot), device_, flags_, &error_)) return st;
  if (map != -1 && find_map(map) == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  Member joiner{AmclPolicy(params, motion)};
  joiner.capacity = params.max_particles;
  if (state != nullptr) adopt_state(joiner, *state);
  joiner.map = map;
  members_.reserve(members_.size() + 1);  // the host allocations that could fail come before the device work
  std::vector<const bb200_amcl_param*> slots(std::max(members_.size(), slot + 1), nullptr);
  for (size_t k = 0; k < members_.size(); ++k)
    if (members_[k].active) slots[k] = &members_[k].policy.params();
  slots[slot] = &params;
  Layout layout;
  const Arrival arrival{slot, state};
  if (const int st = relayout(slots, &layout, state != nullptr ? &arrival : nullptr)) return st;
  if (slot == members_.size()) {
    members_.push_back(std::move(joiner));
  } else {
    members_[slot] = std::move(joiner);
  }
  place(layout);
  *member = static_cast<int>(slot);
  return BB200_OK;
}

int Batch::add_member(const bb200_amcl_param& params, const bb200_motion_param& motion, int* member) {
  error_.clear();
  return join(params, motion, nullptr, -1, member);
}

namespace {

/// Where a transfer's staging buffer holds the moved members' arrays: one region per array, each indexed by the members'
/// staging offsets (a member takes max(n, ancestors) entries), so that one batch_relayout_kernel launch fills or empties it.
struct StageLayout {
  uint64_t states{0}, weights{0}, cdf{0}, ancestors{0}, bytes{0};  // byte offsets of the regions, and the total
};

StageLayout stage_layout(uint64_t entries, bool cdf, bool ancestors) {
  StageLayout l;
  l.weights = entries * sizeof(Pose2);
  l.cdf = l.weights + entries * sizeof(double);
  l.ancestors = l.cdf + (cdf ? entries * sizeof(unsigned long long) : 0);
  l.bytes = l.ancestors + (ancestors ? entries * sizeof(long long) : 0);
  return l;
}

}  // namespace

ParticleSetState Batch::particle_set(const Member& m) {
  ParticleSetState s{};
  s.n = m.n;
  s.ancestors_n = m.policy.params().record_ancestors ? m.ancestors_n : 0;
  s.pivot[0] = m.pivot[0];
  s.pivot[1] = m.pivot[1];
  s.cdf_current = m.cdf_total != 0 ? 1 : 0;
  s.cdf_total = m.cdf_total;
  return s;
}

void Batch::adopt_state(Member& m, const FilterState& s) {
  m.policy.restore(s.policy);
  m.capacity = s.params.max_particles;
  m.n = s.set.n;
  m.cur = 0;
  m.pivot[0] = s.set.pivot[0];
  m.pivot[1] = s.set.pivot[1];
  m.ancestors_n = s.set.ancestors_n;
  m.cdf_total = s.set.cdf_current != 0 ? s.set.cdf_total : 0;
}

int Batch::launch_moves(const std::vector<BatchRelayoutMember>& moves, BatchRelayoutArgs a) {
  const uint32_t n = static_cast<uint32_t>(moves.size());
  std::vector<uint32_t> first(n + 1);
  write_cta_rows<1>(first.data(), n, &a.ctas, [&](uint32_t j, uint32_t* c) { *c = batch_relayout_ctas(moves[j]); });
  BB_CHECK(xfer_.table.grow(n));  // every batch call ends synchronised: nothing in flight reads the old tables
  BB_CHECK(xfer_.first.grow(n + 1));
  // Pageable sources: staged before the calls return.
  BB_CHECK(cudaMemcpyAsync(xfer_.table.get(), moves.data(), n * sizeof(BatchRelayoutMember), cudaMemcpyHostToDevice, stream_));
  BB_CHECK(cudaMemcpyAsync(xfer_.first.get(), first.data(), (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, stream_));
  a.members = xfer_.table.get();
  a.first = xfer_.first.get();
  a.n_members = n;
  launches_ += static_cast<uint64_t>(launch_batch_relayout(a, stream_));
  BB_CHECK(cudaGetLastError());
  return BB200_OK;
}

int Batch::unpack(const std::vector<const FilterState*>& states, const std::vector<uint64_t>& to, Pose2* states_to, double* weights_to,
                  unsigned long long* cdf_to, long long* ancestors_to) {
  std::vector<BatchRelayoutMember> moves;
  std::vector<const FilterState*> moved;
  uint64_t entries = 0;
  bool cdf = false, ancestors = false;
  for (size_t j = 0; j < states.size(); ++j) {
    const ParticleSetState& set = states[j]->set;
    BatchRelayoutMember r{};
    r.from = entries;
    r.to = to[j];
    r.n = set.n;
    r.cdf_n = set.cdf_current != 0 ? set.n : 0;
    r.ancestors_n = ancestors_to != nullptr ? set.ancestors_n : 0;
    if (batch_relayout_ctas(r) == 0) continue;
    entries += std::max(r.n, r.ancestors_n);
    cdf = cdf || r.cdf_n > 0;
    ancestors = ancestors || r.ancestors_n > 0;
    moves.push_back(r);
    moved.push_back(states[j]);
  }
  if (moves.empty()) return BB200_OK;
  const StageLayout l = stage_layout(entries, cdf, ancestors);
  BB_CHECK(xfer_.stage.grow(l.bytes));  // every batch call ends synchronised: the staging buffers are free
  unsigned char* host = xfer_.stage.host.get();
  for (size_t j = 0; j < moves.size(); ++j) {
    const BatchRelayoutMember& r = moves[j];
    const FilterState& s = *moved[j];
    if (r.n > 0) std::memcpy(host + l.states + r.from * sizeof(Pose2), s.states, r.n * sizeof(Pose2));
    if (r.n > 0) std::memcpy(host + l.weights + r.from * sizeof(double), s.weights, r.n * sizeof(double));
    if (r.cdf_n > 0) std::memcpy(host + l.cdf + r.from * sizeof(unsigned long long), s.cdf, r.cdf_n * sizeof(unsigned long long));
    if (r.ancestors_n > 0) std::memcpy(host + l.ancestors + r.from * sizeof(long long), s.ancestors, r.ancestors_n * sizeof(long long));
  }
  unsigned char* stage = xfer_.stage.device.get();
  BB_CHECK(xfer_.stage.to_device(0, l.bytes, stream_));
  BatchRelayoutArgs a{};
  a.states_from[0] = a.states_from[1] = reinterpret_cast<const Pose2*>(stage + l.states);
  a.weights_from = reinterpret_cast<const double*>(stage + l.weights);
  a.cdf_from = reinterpret_cast<const unsigned long long*>(stage + l.cdf);
  a.ancestors_from = reinterpret_cast<const long long*>(stage + l.ancestors);
  a.states_to = states_to;
  a.weights_to = weights_to;
  a.cdf_to = cdf_to;
  a.ancestors_to = ancestors_to;
  return launch_moves(moves, a);
}

int Batch::export_members(const uint8_t* present, void* const* out, const uint64_t* capacity, uint64_t* size) {
  error_.clear();
  if (out != nullptr && capacity == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "capacity is null");
  if (const int st = check_present(present)) return st;
  std::vector<uint32_t> written;  // selected members whose blobs are written, in member order
  bool short_buffer = false;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k)) continue;
    const Member& m = members_[k];
    size[k] = state_blob_size(particle_set(m), m.policy.params().record_ancestors != 0);
    if (out == nullptr || out[k] == nullptr) continue;
    if (capacity[k] < size[k]) {
      short_buffer = true;
    } else {
      written.push_back(static_cast<uint32_t>(k));
    }
  }
  if (short_buffer) return fail(BB200_ERR_CAPACITY, "state blob buffer too small for some member (size has the sizes)");
  if (written.empty()) return BB200_OK;

  // The written members' live slices, gathered into the staging buffer by one launch and brought back by one copy.
  std::vector<BatchRelayoutMember> moves;
  std::vector<uint64_t> staged(written.size(), 0);
  uint64_t entries = 0;
  bool cdf = false, ancestors = false;
  for (size_t j = 0; j < written.size(); ++j) {
    const Member& m = members_[written[j]];
    const ParticleSetState set = particle_set(m);
    BatchRelayoutMember r{};
    r.from = m.offset;
    r.to = entries;
    r.n = set.n;
    r.cdf_n = set.cdf_current != 0 ? set.n : 0;
    r.ancestors_n = set.ancestors_n;
    r.cur = m.cur;
    staged[j] = entries;
    if (batch_relayout_ctas(r) == 0) continue;
    entries += std::max(r.n, r.ancestors_n);
    cdf = cdf || r.cdf_n > 0;
    ancestors = ancestors || r.ancestors_n > 0;
    moves.push_back(r);
  }
  const StageLayout l = stage_layout(entries, cdf, ancestors);
  if (!moves.empty()) {
    BB_CHECK(cudaSetDevice(device_));
    BB_CHECK(xfer_.stage.grow(l.bytes));  // every batch call ends synchronised: the staging buffers are free
    unsigned char* stage = xfer_.stage.device.get();
    BatchRelayoutArgs a{};
    a.states_from[0] = states_[0].get();
    a.states_from[1] = states_[1].get();
    a.weights_from = weights_.get();
    a.cdf_from = cdf_.get();
    a.ancestors_from = ancestors_.get();
    a.states_to = reinterpret_cast<Pose2*>(stage + l.states);
    a.weights_to = reinterpret_cast<double*>(stage + l.weights);
    a.cdf_to = reinterpret_cast<unsigned long long*>(stage + l.cdf);
    a.ancestors_to = reinterpret_cast<long long*>(stage + l.ancestors);
    if (const int st = launch_moves(moves, a)) return st;
    BB_CHECK(xfer_.stage.to_host(0, l.bytes, stream_));
    BB_CHECK(cudaStreamSynchronize(stream_));
  }

  // The blobs, written from pinned memory.
  const unsigned char* host = xfer_.stage.host.get();
  for (size_t j = 0; j < written.size(); ++j) {
    const uint32_t k = written[j];
    const Member& m = members_[k];
    FilterState s{};
    s.params = m.policy.params();
    s.motion = m.policy.motion();
    s.policy = m.policy.save();
    s.set = particle_set(m);
    s.states = host + l.states + staged[j] * sizeof(Pose2);
    s.weights = host + l.weights + staged[j] * sizeof(double);
    s.cdf = host + l.cdf + staged[j] * sizeof(unsigned long long);
    s.ancestors = host + l.ancestors + staged[j] * sizeof(long long);
    write_state_blob(s, out[k]);
  }
  return BB200_OK;
}

int Batch::export_member(int member, void* out, uint64_t capacity, uint64_t* size) {
  error_.clear();
  if (const int st = member_ok(member)) return st;
  const size_t k = static_cast<size_t>(member);
  std::vector<uint8_t> present(members_.size(), 0);
  std::vector<void*> outs(members_.size(), nullptr);
  std::vector<uint64_t> capacities(members_.size(), 0), sizes(members_.size(), 0);
  present[k] = 1;
  outs[k] = out;
  capacities[k] = capacity;
  const int st = export_members(present.data(), outs.data(), capacities.data(), sizes.data());
  *size = sizes[k];
  return st;
}

int Batch::import_member(const void* blob, uint64_t size, int map, int* member) {
  error_.clear();
  FilterState s;
  if (const int st = read_state_blob(blob, size, &s, &error_)) return st;
  s.params.device = device_;  // the receiver's device
  return join(s.params, s.motion, &s, map, member);
}

int Batch::restore_members(const std::vector<FilterState>& states) {
  error_.clear();
  BB_CHECK(cudaSetDevice(device_));
  std::vector<const FilterState*> from;
  std::vector<uint64_t> to;
  for (size_t k = 0; k < members_.size(); ++k) {
    adopt_state(members_[k], states[k]);
    from.push_back(&states[k]);
    to.push_back(members_[k].offset);
  }
  if (const int st = unpack(from, to, states_[0].get(), weights_.get(), cdf_.get(), ancestors_.get())) return st;
  BB_CHECK(cudaStreamSynchronize(stream_));
  return BB200_OK;
}

int Batch::remove_member(int member) {
  error_.clear();
  if (const int st = member_ok(member)) return st;
  const size_t slot = static_cast<size_t>(member);
  std::vector<const bb200_amcl_param*> slots(members_.size(), nullptr);
  size_t occupied = 0;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!members_[k].active || k == slot) continue;
    slots[k] = &members_[k].policy.params();
    ++occupied;
  }
  if (occupied == 0) return fail(BB200_ERR_STATE, "a batch keeps at least one member: member " + std::to_string(member) + " is the last");
  Layout layout;
  if (const int st = relayout(slots, &layout)) return st;
  Member vacant{members_[slot].policy};  // its scan table's device buffer goes with the old member
  vacant.active = false;
  members_[slot] = std::move(vacant);
  place(layout);
  return BB200_OK;
}

int Batch::member_active(int member, int* active) const {
  error_.clear();
  if (member < 0 || member >= members()) {
    error_ = "member index out of range";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  *active = members_[static_cast<size_t>(member)].active ? 1 : 0;
  return BB200_OK;
}

int Batch::check_present(const uint8_t* present) {
  if (present == nullptr) return BB200_OK;
  for (size_t k = 0; k < members_.size(); ++k)
    if (present[k] != 0 && !members_[k].active) return fail(BB200_ERR_INVALID_ARGUMENT, "member " + std::to_string(k) + " is a vacant slot");
  return BB200_OK;
}

Batch::~Batch() {
  if (stream_ == nullptr) return;
  cudaStreamSynchronize(stream_);  // nothing in flight reads the buffers the members free
  cudaStreamDestroy(stream_);
}

int Batch::member_ok(int member) const {
  if (member < 0 || member >= members()) {
    error_ = "member index out of range";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  if (!members_[static_cast<size_t>(member)].active) {
    error_ = "member " + std::to_string(member) + " is a vacant slot";
    return BB200_ERR_INVALID_ARGUMENT;
  }
  return BB200_OK;
}

#define BB_MEMBER(member) do { error_.clear(); if (const int st_ = member_ok(member)) return st_; } while (0)

const Batch::MapEntry* Batch::find_map(int id) const {
  const auto it = maps_.find(id);
  if (it != maps_.end()) return &it->second;
  error_ = "unknown map id " + std::to_string(id);
  return nullptr;
}

int Batch::set_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob) {
  error_.clear();
  MapTables tables;
  const int st = prepare_likelihood_field_map(p, grid, prob, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Batch::set_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid) {
  error_.clear();
  MapTables tables;
  const int st = prepare_beam_map(p, grid, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Batch::add_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob, int* id) {
  error_.clear();
  MapTables tables;
  const int st = prepare_likelihood_field_map(p, grid, prob, &tables, &error_);
  return st != BB200_OK ? st : add_map(tables, id);
}

int Batch::add_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid, int* id) {
  error_.clear();
  MapTables tables;
  const int st = prepare_beam_map(p, grid, &tables, &error_);
  return st != BB200_OK ? st : add_map(tables, id);
}

int Batch::set_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map) {
  error_.clear();
  MapTables tables;
  const int st = prepare_landmark_map(lp, bp, map, &tables, &error_);
  return st != BB200_OK ? st : set_map(tables);
}

int Batch::add_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map, int* id) {
  error_.clear();
  MapTables tables;
  const int st = prepare_landmark_map(lp, bp, map, &tables, &error_);
  return st != BB200_OK ? st : add_map(tables, id);
}

int Batch::set_map(const MapTables& tables) {
  // The old maps go before the new one is uploaded, so that the device never holds both; a failed upload leaves the
  // batch without a map.
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  maps_.clear();
  map_table_current_ = false;
  for (Member& m : members_) m.map = -1;
  int id = -1;
  const int st = add_map(tables, &id);
  if (st != BB200_OK) return st;
  for (Member& m : members_)
    if (m.active) m.map = id;
  return BB200_OK;
}

int Batch::add_map(const MapTables& tables, int* id) {
  BB_CHECK(cudaSetDevice(device_));
  const int new_id = next_map_id_;
  MapEntry& e = maps_[new_id];
  const int st = e.map.upload(tables, stream_, &error_);
  launches_ += e.map.launches();
  if (st != BB200_OK) {
    maps_.erase(new_id);
    return st;
  }
  map_table_current_ = false;
  ++next_map_id_;
  *id = new_id;
  return BB200_OK;
}

int Batch::update_map(int member, int id) {
  BB_MEMBER(member);
  if (find_map(id) == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  members_[static_cast<size_t>(member)].map = id;
  return BB200_OK;
}

int Batch::member_map(int member, int* id) const {
  error_.clear();
  if (const int st = member_ok(member)) return st;
  *id = members_[static_cast<size_t>(member)].map;
  return BB200_OK;
}

int Batch::remove_map(int id) {
  error_.clear();
  if (find_map(id) == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  for (size_t k = 0; k < members_.size(); ++k)
    if (members_[k].active && members_[k].map == id) return fail(BB200_ERR_STATE, "member " + std::to_string(k) + " reads map " + std::to_string(id));
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));  // nothing in flight reads its tables
  maps_.erase(id);
  map_table_current_ = false;
  return BB200_OK;
}

int Batch::get_likelihood_field(int id, float* out, uint64_t capacity) const {
  error_.clear();
  const MapEntry* e = find_map(id);
  if (e == nullptr) return BB200_ERR_INVALID_ARGUMENT;
  const std::vector<float>& field = e->map.field_host;
  if (field.empty()) {
    error_ = "map " + std::to_string(id) + " is not a likelihood-field map";
    return BB200_ERR_STATE;
  }
  if (capacity < field.size()) {
    error_ = "capacity below the field's cells";
    return BB200_ERR_CAPACITY;
  }
  std::memcpy(out, field.data(), field.size() * sizeof(float));
  return BB200_OK;
}

int Batch::ensure_map_table() {
  if (map_table_current_) return BB200_OK;
  std::vector<BatchMap> host;
  host.reserve(maps_.size());
  for (auto& [id, e] : maps_) {
    const DeviceMap& d = e.map;
    e.slot = static_cast<int>(host.size());
    host.push_back(BatchMap{d.field, d.occupancy, d.beam, d.free_cells, d.n_free, d.grid_width, d.grid_resolution, d.grid_origin, d.landmark,
                            d.landmarks, d.n_landmarks, {d.box[0], d.box[1], d.box[2], d.box[3]}});
  }
  BB_CHECK(map_table_.grow(host.size()));  // every batch call ends synchronised: no step reads the old table
  // On the batch's stream, so that the step's launches follow the copy in order; the pageable source is staged before the
  // call returns.
  BB_CHECK(cudaMemcpyAsync(map_table_.get(), host.data(), host.size() * sizeof(BatchMap), cudaMemcpyHostToDevice, stream_));
  map_table_current_ = true;
  return BB200_OK;
}

int Batch::initialize(int member, const double mean[3], const double cov[9]) {
  BB_MEMBER(member);
  Member& m = members_[static_cast<size_t>(member)];
  double transform[9];
  std::string message;
  if (!normal_transform(cov, transform, &message)) return fail(BB200_ERR_INVALID_ARGUMENT, message);
  BB_CHECK(cudaSetDevice(device_));
  m.cdf_total = 0;
  launch_initialize_normal(states_[m.cur].get() + m.offset, weights_.get() + m.offset, m.capacity, mean, transform, m.policy.params().seed, 0, stream_);
  ++launches_;
  BB_CHECK(cudaGetLastError());
  BB_CHECK(cudaStreamSynchronize(stream_));
  m.n = m.capacity;
  m.pivot[0] = mean[0];
  m.pivot[1] = mean[1];
  m.policy.force_update();  // amcl_core.hpp:136
  return BB200_OK;
}

int Batch::initialize_from_map(int member) {
  BB_MEMBER(member);
  Member& m = members_[static_cast<size_t>(member)];
  if (m.map < 0) return fail(BB200_ERR_STATE, "initialize_from_map needs a map (set_*_map or update_map first)");
  const DeviceMap& map = maps_.at(m.map).map;
  if (!map.can_draw_states())
    return fail(BB200_ERR_STATE, map.landmark_map() ? "the landmark map's box is empty or not finite" : "the map has no free cell to sample from");
  BB_CHECK(cudaSetDevice(device_));
  m.cdf_total = 0;
  if (map.landmark_map()) {
    launch_initialize_box(states_[m.cur].get() + m.offset, weights_.get() + m.offset, m.capacity, map.box, m.policy.params().seed, 0, stream_);
  } else {
    launch_initialize_uniform(states_[m.cur].get() + m.offset, weights_.get() + m.offset, m.capacity, map.free_cells, map.n_free, map.grid_width,
                              map.grid_resolution, map.grid_origin, m.policy.params().seed, 0, stream_);
  }
  ++launches_;
  BB_CHECK(cudaGetLastError());
  BB_CHECK(cudaStreamSynchronize(stream_));
  m.n = m.capacity;
  map.centre(m.pivot);
  m.policy.force_update();
  return BB200_OK;
}

int Batch::initialize_states(int member, const double* states, const double* weights, uint64_t n) {
  BB_MEMBER(member);
  Member& m = members_[static_cast<size_t>(member)];
  if (n > m.capacity) return fail(BB200_ERR_CAPACITY, "more particles than the member's max_particles");
  if (n > 0 && states == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "states is null");
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  m.cdf_total = 0;
  if (n > 0) {
    BB_CHECK(cudaMemcpy(states_[m.cur].get() + m.offset, states, n * sizeof(Pose2), cudaMemcpyHostToDevice));
    const std::vector<double> ones(weights == nullptr ? n : 0, 1.0);
    BB_CHECK(cudaMemcpy(weights_.get() + m.offset, weights != nullptr ? weights : ones.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    m.pivot[0] = states[2];
    m.pivot[1] = states[3];
  }
  m.n = n;
  m.policy.force_update();
  return BB200_OK;
}

int Batch::force_update(int member) {
  BB_MEMBER(member);
  members_[static_cast<size_t>(member)].policy.force_update();
  return BB200_OK;
}

int Batch::get_particles(int member, double* states, double* weights, uint64_t capacity) {
  BB_MEMBER(member);
  const Member& m = members_[static_cast<size_t>(member)];
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, m.n);
  if (states != nullptr && n > 0) BB_CHECK(cudaMemcpy(states, states_[m.cur].get() + m.offset, n * sizeof(Pose2), cudaMemcpyDeviceToHost));
  if (weights != nullptr && n > 0) BB_CHECK(cudaMemcpy(weights, weights_.get() + m.offset, n * sizeof(double), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

int Batch::member_size(int member, uint64_t* n) const {
  BB_MEMBER(member);
  *n = members_[static_cast<size_t>(member)].n;
  return BB200_OK;
}

int Batch::ancestors(int member, int64_t* out, uint64_t capacity) {
  BB_MEMBER(member);
  const Member& m = members_[static_cast<size_t>(member)];
  if (!m.policy.params().record_ancestors) return fail(BB200_ERR_STATE, "the member was created without record_ancestors");
  BB_CHECK(cudaSetDevice(device_));
  BB_CHECK(cudaStreamSynchronize(stream_));
  const uint64_t n = std::min(capacity, m.ancestors_n);
  if (out != nullptr && n > 0) BB_CHECK(cudaMemcpy(out, ancestors_.get() + m.offset, n * sizeof(int64_t), cudaMemcpyDeviceToHost));
  return BB200_OK;
}

int Batch::cluster_estimate(int member, const bb200_cluster_param& p, bb200_estimate* out) {
  BB_MEMBER(member);
  std::vector<uint8_t> present(members_.size(), 0);
  present[static_cast<size_t>(member)] = 1;
  std::vector<bb200_estimate> all(members_.size());  // indexed by member
  const int st = cluster_estimates(p, present.data(), all.data(), nullptr, nullptr);
  if (st == BB200_OK) *out = all[static_cast<size_t>(member)];
  return st;
}

int Batch::ensure_cluster_scratch() {
  if (cl_.hashes.get() != nullptr) return BB200_OK;
  const size_t k = members_.size();
  ClusterBuffers c;
  BB_CHECK(c.hashes.allocate(total_));
  BB_CHECK(c.keys.allocate(table_total_));
  BB_CHECK(c.first.allocate(table_total_));
  BB_CHECK(c.ids.allocate(table_total_));
  BB_CHECK(c.cell_of.allocate(total_));
  BB_CHECK(c.sort[0].allocate(total_));
  BB_CHECK(c.sort[1].allocate(total_));
  BB_CHECK(c.starts.allocate(total_ + k));
  BB_CHECK(c.records.allocate(total_));
  BB_CHECK(c.table.grow(k));
  BB_CHECK(c.cells.grow(k));
  cl_ = std::move(c);
  return BB200_OK;
}

int Batch::ensure_kld_scratch() {
  if (const int st = ensure_cluster_scratch()) return st;
  BB_CHECK(kld_.grow(members_.size()));
  return BB200_OK;
}

int Batch::ensure_select_scratch() {
  if (const int st = ensure_cluster_scratch()) return st;
  if (sel_.results.get() != nullptr) return BB200_OK;
  const RehashTable& table = rehash_table();
  const size_t k = members_.size();
  SelectBuffers s;
  s.offsets.resize(k);
  uint64_t bytes = 0;
  for (size_t m = 0; m < k; ++m) {
    s.offsets[m] = bytes;
    if (members_[m].active) bytes += (select_scratch_bytes(members_[m].capacity) + 255) / 256 * 256;
  }
  BB_CHECK(s.schedule_start.allocate(table.start.size()));
  BB_CHECK(s.schedule.allocate(table.steps.size()));
  BB_CHECK(s.scratch.allocate(bytes));
  BB_CHECK(s.post.grow(k));
  BB_CHECK(s.results.allocate(k));
  BB_CHECK(cudaMemcpy(s.schedule_start.get(), table.start.data(), table.start.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  BB_CHECK(cudaMemcpy(s.schedule.get(), table.steps.data(), table.steps.size() * sizeof(RehashStep), cudaMemcpyHostToDevice));
  sel_ = std::move(s);
  return BB200_OK;
}

int Batch::ensure_cluster_records(uint64_t cells) {
  BB_CHECK(cl_records_host_.grow(cells, std::min<uint64_t>(total_, std::max<uint64_t>(4096, 2 * cells))));
  return BB200_OK;
}

int Batch::cluster_estimates(const bb200_cluster_param& p, const uint8_t* present, bb200_estimate* out, uint32_t* n_cells, uint32_t* n_clusters) {
  error_.clear();
  if (const char* why = cluster_param_error(p)) return fail(BB200_ERR_INVALID_ARGUMENT, why);
  std::vector<uint32_t> selected;
  if (const int st = select_members(present, &selected)) return st;
  if (selected.empty()) return BB200_OK;
  if (const int st = cell_records(p.linear_hash_resolution, p.angular_hash_resolution, selected)) return st;

  // Host pass per member (Clusterizer::estimate's): the flood over the cells, then the estimate about the member's pivot.
  const HostCell* cells = reinterpret_cast<const HostCell*>(cl_records_host_.get());
  for (size_t j = 0; j < selected.size(); ++j) {
    const uint32_t k = selected[j];
    const Member& m = members_[k];
    const uint32_t count = cl_.cells.host.get()[j];
    const ClusterSelection sel = select_cluster(cells, count, m.n, p.linear_hash_resolution, p.angular_hash_resolution, p.weight_cap_percentile);
    if (out != nullptr) estimate_from_moments(sel.moments, m.pivot, &out[k]);
    if (n_cells != nullptr) n_cells[k] = count;
    if (n_clusters != nullptr) n_clusters[k] = sel.clusters;
    cells += count;
  }
  return BB200_OK;
}

int Batch::select_members(const uint8_t* present, std::vector<uint32_t>* selected) {
  if (const int st = check_present(present)) return st;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k)) continue;
    if (members_[k].n == 0) return fail(BB200_ERR_STATE, "member " + std::to_string(k) + ": no particles");
    selected->push_back(static_cast<uint32_t>(k));
  }
  return BB200_OK;
}

int Batch::cell_records(double linear, double angular, const std::vector<uint32_t>& selected) {
  BB_CHECK(cudaSetDevice(device_));
  if (const int st = ensure_cluster_scratch()) return st;  // every batch call ends synchronised: the pinned buffers are free

  const uint32_t n_sel = static_cast<uint32_t>(selected.size());
  for (uint32_t j = 0; j < n_sel; ++j) cl_.table.host.get()[j] = cluster_member(selected[j]);
  cudaStream_t stream = stream_;
  BB_CHECK(cl_.table.to_device(0, n_sel, stream));
  launch_batch_cluster_cells(cluster_args(linear, angular), n_sel, stream);
  BB_LAUNCHED("batch_cluster_cells");
  BB_CHECK(cl_.cells.to_host(0, n_sel, stream));
  BB_CHECK(cudaStreamSynchronize(stream));  // 1: the cell counts size the records' read-back
  uint64_t total_cells = 0;
  for (uint32_t j = 0; j < n_sel; ++j) total_cells += cl_.cells.host.get()[j];
  if (const int st = ensure_cluster_records(total_cells)) return st;
  launch_batch_cluster_compact(cl_.table.device.get(), cl_.cells.device.get(), cl_.records.get(), n_sel, cl_records_host_.get(), stream);
  BB_LAUNCHED("batch_cluster_compact");
  BB_CHECK(cudaStreamSynchronize(stream));  // 2: every record is in pinned memory
  static_assert(sizeof(HostCell) == sizeof(CellRecord), "record layouts must agree");
  return BB200_OK;
}

BatchClusterMember Batch::cluster_member(uint32_t k) const {
  const Member& m = members_[k];
  BatchClusterMember c{};
  c.offset = m.offset;
  c.table_offset = m.table_offset;
  c.starts_offset = m.offset + k;  // a member's cells + 1 starts end before the next member's slice begins
  c.n = static_cast<uint32_t>(m.n);
  c.table_mask = m.table_slots - 1;
  c.cur = static_cast<uint32_t>(m.cur);
  c.pivot_x = m.pivot[0];
  c.pivot_y = m.pivot[1];
  return c;
}

BatchClusterArgs Batch::cluster_args(double linear, double angular) const {
  BatchClusterArgs a{};
  a.members = cl_.table.device.get();
  a.states[0] = states_[0].get();
  a.states[1] = states_[1].get();
  a.weights = weights_.get();
  a.linear = linear;
  a.angular = angular;
  a.hashes = cl_.hashes.get();
  a.keys = cl_.keys.get();
  a.first = cl_.first.get();
  a.ids = cl_.ids.get();
  a.cell_of = cl_.cell_of.get();
  a.sort_a = cl_.sort[0].get();
  a.sort_b = cl_.sort[1].get();
  a.starts = cl_.starts.get();
  a.records = cl_.records.get();
  a.cells = cl_.cells.device.get();
  return a;
}

int Batch::particle_histograms(double linear, double angular, const uint8_t* present, bb200_cluster_cell* const* bins, const uint64_t* capacity,
                               uint64_t* n_bins, double* max_bin_weight) {
  error_.clear();
  if (!(linear > 0.0) || !(angular > 0.0)) return fail(BB200_ERR_INVALID_ARGUMENT, "histogram resolutions must be positive");
  if (bins != nullptr && capacity == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, "capacity is null");
  std::vector<uint32_t> selected;
  if (const int st = select_members(present, &selected)) return st;
  if (selected.empty()) return BB200_OK;
  if (const int st = cell_records(linear, angular, selected)) return st;

  // Filter::particle_histogram's host half per member.
  static_assert(sizeof(bb200_cluster_cell) == sizeof(CellRecord), "public and internal cell records must agree");
  const CellRecord* cells = cl_records_host_.get();
  bool short_buffer = false;
  for (size_t j = 0; j < selected.size(); ++j) {
    const uint32_t k = selected[j];
    const uint32_t count = cl_.cells.host.get()[j];
    double top = 1e-3;  // beluga_ros/particle_cloud.hpp:197
    for (uint32_t c = 0; c < count; ++c) top = cells[c].weight > top ? cells[c].weight : top;
    if (n_bins != nullptr) n_bins[k] = count;
    if (max_bin_weight != nullptr) max_bin_weight[k] = top;
    if (bins != nullptr && bins[k] != nullptr) {
      if (capacity[k] < count) {
        short_buffer = true;
      } else {
        std::memcpy(bins[k], cells, count * sizeof(CellRecord));
      }
    }
    cells += count;
  }
  if (short_buffer) return fail(BB200_ERR_CAPACITY, "histogram bin buffer too small for some member (n_bins has the counts)");
  return BB200_OK;
}

int Batch::sample_states(const uint64_t* counts, uint32_t step, const uint8_t* present, double* const* states_out) {
  error_.clear();
  // Filter::sample_states's checks per member, all before anything reaches the device.
  std::vector<uint32_t> drawn;  // selected members with something to draw, in member order
  uint64_t draws = 0;
  if (const int st = check_present(present)) return st;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k)) continue;
    const Member& m = members_[k];
    const std::string who = "member " + std::to_string(k) + ": ";
    if (m.n == 0) return fail(BB200_ERR_STATE, who + "no particles");
    if (counts[k] > m.capacity) return fail(BB200_ERR_CAPACITY, who + "more samples than its max_particles");
    if (counts[k] > 0 && states_out[k] == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, who + "states_out is null");
    if (counts[k] == 0) continue;
    drawn.push_back(static_cast<uint32_t>(k));
    draws += counts[k];
  }
  if (drawn.empty()) return BB200_OK;
  BB_CHECK(cudaSetDevice(device_));
  // Every batch call ends synchronised: the pinned buffers are free.  The draws follow one CDF total per member.
  const uint64_t header = (members_.size() * sizeof(unsigned long long) + sizeof(Pose2) - 1) / sizeof(Pose2);
  const uint64_t want = std::min<uint64_t>(total_, std::max<uint64_t>(4096, 2 * draws));  // draws <= total_
  BB_CHECK(sm_table_.grow(members_.size()));
  BB_CHECK(samples_.grow(header + draws, header + want));

  const uint32_t n_sel = static_cast<uint32_t>(drawn.size());
  BatchSampleArgs a{};
  a.n_members = n_sel;
  uint64_t out_offset = 0;
  for (uint32_t j = 0; j < n_sel; ++j) {
    const uint32_t k = drawn[j];
    const Member& m = members_[k];
    BatchSampleMember& s = sm_table_.host.get()[j];
    s = BatchSampleMember{};
    s.offset = m.offset;
    s.n = m.n;
    s.count = counts[k];
    s.out_offset = out_offset;
    s.seed = m.policy.params().seed;
    s.total = m.cdf_total;
    s.cur = m.cur;
    s.ceil_log2_count = ceil_log2_count(m.capacity);
    out_offset += s.count;
  }
  // The step's range buffers are free between calls.
  write_cta_rows<kSampleLaunches>(first_.host.get(), n_sel, a.ctas, [&](uint32_t j, uint32_t* c) {
    const BatchSampleMember& s = sm_table_.host.get()[j];
    batch_sample_ctas(s, s.total == 0, c);
  });
  cudaStream_t stream = stream_;
  BB_CHECK(sm_table_.to_device(0, n_sel, stream));
  BB_CHECK(first_.to_device(0, kSampleLaunches * (n_sel + 1), stream));
  a.members = sm_table_.device.get();
  a.first = first_.device.get();
  a.step = step;
  a.states[0] = states_[0].get();
  a.states[1] = states_[1].get();
  a.weights = weights_.get();
  a.cdf = cdf_.get();
  a.scalars = scalars_.get();
  a.tile_state = tile_state_.get();
  a.partials = partials_.get();  // the step's moment rows are free between calls
  a.totals = reinterpret_cast<unsigned long long*>(samples_.device.get());
  a.out = samples_.device.get() + header;
  launches_ += static_cast<uint64_t>(launch_batch_sample(a, stream));
  BB_CHECK(cudaGetLastError());
  BB_CHECK(samples_.to_host(0, header + draws, stream));
  BB_CHECK(cudaStreamSynchronize(stream));

  const unsigned long long* totals = reinterpret_cast<const unsigned long long*>(samples_.host.get());
  const Pose2* out = samples_.host.get() + header;
  for (uint32_t j = 0; j < n_sel; ++j) {
    const BatchSampleMember& s = sm_table_.host.get()[j];
    members_[drawn[j]].cdf_total = totals[j];  // a rebuilt CDF is current until the member's particles or weights change
    std::memcpy(states_out[drawn[j]], out + s.out_offset, s.count * sizeof(Pose2));
  }
  return BB200_OK;
}

int Batch::cast_rays(const uint8_t* present, const int* map_ids, const double* const* poses, const uint64_t* n_poses, const double* const* bearings,
                     const uint64_t* n_bearings, const double* max_range, double* const* ranges) {
  error_.clear();
  // Filter::cast_rays's checks per member, all before anything reaches the device.
  if (const int st = check_present(present)) return st;
  struct Cast {
    size_t k;
    DeviceMap* map;
    uint64_t n_rays;
  };
  std::vector<Cast> casts;  // selected members with rays to cast, in member order
  uint64_t pose_doubles = 0, bearing_doubles = 0, total_rays = 0, ctas = 0;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k)) continue;
    const std::string who = "member " + std::to_string(k) + ": ";
    const bool override_map = map_ids != nullptr && map_ids[k] != -1;
    const int id = override_map ? map_ids[k] : members_[k].map;
    if (override_map && find_map(id) == nullptr) return fail(BB200_ERR_INVALID_ARGUMENT, who + error_);
    if (id < 0) return fail(BB200_ERR_STATE, who + "no map");
    if (maps_.at(id).map.landmark_map()) return fail(BB200_ERR_STATE, who + "a landmark map has no grid to cast rays on");
    uint64_t n_rays = 0;
    if (!cast_ray_count(n_poses[k], n_bearings[k], &n_rays)) return fail(BB200_ERR_INVALID_ARGUMENT, who + "n_poses * n_bearings overflows");
    if ((poses[k] == nullptr && n_poses[k] > 0) || (bearings[k] == nullptr && n_bearings[k] > 0) || (ranges[k] == nullptr && n_rays > 0))
      return fail(BB200_ERR_INVALID_ARGUMENT, who + "null array with a non-zero count");
    if (n_rays == 0) continue;
    if (n_rays > kMaxCastRays) return fail(BB200_ERR_CAPACITY, who + "too many rays for one launch");
    ctas += cast_rays_ctas(n_rays);
    if (ctas > kMaxCastRays / 256) return fail(BB200_ERR_CAPACITY, "too many rays for one launch");
    // n_poses and n_bearings are at most n_rays here, and the CTA bound keeps every sum far from overflowing
    pose_doubles += 4 * n_poses[k];
    bearing_doubles += 2 * n_bearings[k];
    total_rays += n_rays;
    casts.push_back(Cast{k, &maps_.at(id).map, n_rays});
  }
  if (casts.empty()) return BB200_OK;
  BB_CHECK(cudaSetDevice(device_));
  const uint32_t n_sel = static_cast<uint32_t>(casts.size());
  // Every batch call ends synchronised: nothing in flight reads the old buffers.
  const uint64_t doubles = pose_doubles + bearing_doubles + total_rays;
  BB_CHECK(rays_.table.grow(n_sel, members_.size()));
  BB_CHECK(rays_.data.grow(doubles, std::max<uint64_t>(doubles + doubles / 2, 4096)));
  double* staged = rays_.data.host.get();
  uint64_t pose_offset = 0, bearing_offset = 0, ray_offset = 0;
  BatchRayArgs a{};
  a.n_members = n_sel;
  for (uint32_t j = 0; j < n_sel; ++j) {
    const size_t k = casts[j].k;
    BatchRayMember& r = rays_.table.host.get()[j];
    r = BatchRayMember{};
    if (const int st = casts[j].map->ray_view(stream_, &r.grid, &error_)) return st;  // a likelihood-field map's first cast uploads its table
    r.pose_offset = pose_offset;
    r.bearing_offset = bearing_offset;
    r.ray_offset = ray_offset;
    r.n_bearings = n_bearings[k];
    r.n_rays = casts[j].n_rays;
    r.max_range = max_range[k];
    std::memcpy(staged + 4 * pose_offset, poses[k], 4 * n_poses[k] * sizeof(double));
    std::memcpy(staged + pose_doubles + 2 * bearing_offset, bearings[k], 2 * n_bearings[k] * sizeof(double));
    pose_offset += n_poses[k];
    bearing_offset += n_bearings[k];
    ray_offset += r.n_rays;
  }
  // The step's range buffers are free between calls.
  write_cta_rows<1>(first_.host.get(), n_sel, &a.ctas, [&](uint32_t j, uint32_t* c) { *c = cast_rays_ctas(rays_.table.host.get()[j].n_rays); });
  cudaStream_t stream = stream_;
  double* d = rays_.data.device.get();
  BB_CHECK(rays_.data.to_device(0, pose_doubles + bearing_doubles, stream));
  BB_CHECK(rays_.table.to_device(0, n_sel, stream));
  BB_CHECK(first_.to_device(0, n_sel + 1, stream));
  a.members = rays_.table.device.get();
  a.first = first_.device.get();
  a.poses = reinterpret_cast<const Pose2*>(d);
  a.bearings = reinterpret_cast<const double2*>(d + pose_doubles);
  a.ranges = d + pose_doubles + bearing_doubles;
  launches_ += static_cast<uint64_t>(launch_batch_cast_rays(a, stream));
  BB_CHECK(cudaGetLastError());
  BB_CHECK(rays_.data.to_host(pose_doubles + bearing_doubles, total_rays, stream));
  BB_CHECK(cudaStreamSynchronize(stream));
  const double* out = staged + pose_doubles + bearing_doubles;
  for (uint32_t j = 0; j < n_sel; ++j) {
    const BatchRayMember& r = rays_.table.host.get()[j];
    std::memcpy(ranges[casts[j].k], out + r.ray_offset, r.n_rays * sizeof(double));
  }
  return BB200_OK;
}

int Batch::set_detections(const bb200_landmark_detection* const* detections, const uint64_t* n, const uint8_t* present) {
  error_.clear();
  if (const int st = check_present(present)) return st;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k)) continue;
    const std::string who = "member " + std::to_string(k) + ": ";
    if (n[k] > 0 && (detections == nullptr || detections[k] == nullptr)) return fail(BB200_ERR_INVALID_ARGUMENT, who + "detections is null");
    if (n[k] >= 0xffffffffull) return fail(BB200_ERR_INVALID_ARGUMENT, who + "too many detections");
  }
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k)) continue;
    Member& m = members_[k];
    m.detections.assign(detections != nullptr && n[k] > 0 ? detections[k] : nullptr, detections != nullptr && n[k] > 0 ? detections[k] + n[k] : nullptr);
    m.detections_staged = true;
  }
  return BB200_OK;
}

bool Batch::ensure_hits(uint64_t words) {
  // Every batch call ends synchronised: nothing in flight reads the old buffer.
  // words is at most one pass's worth (the caller checks), so the slack never takes the buffer past that
  const uint64_t room = std::min<uint64_t>(std::max<uint64_t>(words + words / 2, 4096), kBeamHitPassBytes / sizeof(uint32_t));
  if (hits_.grow(words, room) != cudaSuccess) {
    (void)cudaGetLastError();  // no room for the hit words: the fused kernel needs none
    return false;
  }
  return true;
}

int Batch::ensure_scan_table(Member& m, const bb200_laser_scan& scan) {
  uint32_t angle_min_bits, angle_increment_bits;
  std::memcpy(&angle_min_bits, &scan.angle_min, sizeof(float));
  std::memcpy(&angle_increment_bits, &scan.angle_increment, sizeof(float));
  Member::ScanTable& t = m.scan;
  if (t.valid && t.n_ranges == scan.n_ranges && t.max_beams == scan.max_beams && t.angle_min_bits == angle_min_bits &&
      t.angle_increment_bits == angle_increment_bits)
    return BB200_OK;
  const uint64_t kept = scan_beam_count(scan);
  std::vector<uint64_t> indices(kept);
  std::vector<double2> directions(kept);
  for (uint64_t pos = 0; pos < kept; ++pos) {
    const ScanBeam beam = scan_beam(scan, pos);
    indices[pos] = beam.index;
    directions[pos] = double2{beam.c, beam.s};
  }
  t.valid = false;  // until the new table is on the device
  BB_CHECK(t.directions.grow(kept));  // every batch call ends synchronised: no step reads the old table
  // Pageable source: staged before the call returns, and ordered before the step's launches on the batch's stream.
  if (kept > 0) BB_CHECK(cudaMemcpyAsync(t.directions.get(), directions.data(), kept * sizeof(double2), cudaMemcpyHostToDevice, stream_));
  t.indices = std::move(indices);
  t.n_ranges = scan.n_ranges;
  t.max_beams = scan.max_beams;
  t.angle_min_bits = angle_min_bits;
  t.angle_increment_bits = angle_increment_bits;
  t.valid = true;
  return BB200_OK;
}

namespace {

/// Why the single filter would refuse member k's measurement (bb200_amcl_update / _update_scan / _update_point_cloud), or
/// an empty string.
std::string measurement_error(const bb200_measurement& in) {
  switch (in.kind) {
    case BB200_MEASUREMENT_POINTS:
      return in.points_xy == nullptr && in.n_points > 0 ? "points_xy is null" : "";
    case BB200_MEASUREMENT_SCAN:
      if (in.scan == nullptr) return "scan is null";
      return in.scan->ranges == nullptr && in.scan->n_ranges > 0 ? "scan ranges are null" : "";
    case BB200_MEASUREMENT_CLOUD:
      if (in.cloud == nullptr) return "cloud is null";
      return cloud_valid(*in.cloud) ? ""
                                    : "point cloud: datatype must be 7 (FLOAT32) or 8 (FLOAT64), x, y and z must fit in point_step, data must be set";
    case BB200_MEASUREMENT_LANDMARKS:
      return "";  // the member's staged detections (set_detections), checked against its map by the step
    default:
      return "unknown measurement kind";
  }
}

/// The points a member's measurement can yield: the exact count for points and clouds, the kept beams for a scan.
uint64_t measurement_bound(const bb200_measurement& in) {
  if (in.kind == BB200_MEASUREMENT_WEIGHTS || in.kind == BB200_MEASUREMENT_LANDMARKS) return 0;
  return in.kind == BB200_MEASUREMENT_SCAN ? scan_beam_count(*in.scan) : in.kind == BB200_MEASUREMENT_CLOUD ? in.cloud->n_points : in.n_points;
}

/// A sensor origin's rows 0 and 1 in a BatchPointsMember (none: has_origin stays 0).
void set_origin(BatchPointsMember& d, const double* origin) {
  d.has_origin = origin != nullptr;
  if (origin != nullptr) std::memcpy(d.origin, origin, sizeof(d.origin));
}

/// Packs the x, y, z of every point of a valid cloud as floats, read as bb200_point_cloud_to_points reads them.
template <class Scalar>
void pack_cloud(const bb200_point_cloud& c, float* out) {
  for (uint64_t i = 0; i < c.n_points; ++i) cloud_point<Scalar>(c, i, out + 3 * i);
}

}  // namespace

int Batch::check_measurements(const bb200_measurement* in, const uint8_t* present, bool weighed_by_caller) {
  if (const int st = check_present(present)) return st;
  for (size_t k = 0; k < members_.size(); ++k) {
    if (!selected_member(present, k) || (weighed_by_caller && in[k].kind == BB200_MEASUREMENT_WEIGHTS)) continue;
    const std::string why = measurement_error(in[k]);
    if (!why.empty()) return fail(BB200_ERR_INVALID_ARGUMENT, "member " + std::to_string(k) + ": " + why);
  }
  return BB200_OK;
}

int Batch::update(const double* control_poses, const double* const* points_xy, const uint64_t* n_points, const uint8_t* present,
                  bb200_update_result* out) {
  std::vector<bb200_measurement> in(members_.size());
  for (size_t k = 0; k < members_.size(); ++k)
    if (members_[k].active) in[k] = bb200_measurement{BB200_MEASUREMENT_POINTS, points_xy[k], n_points[k], nullptr, nullptr};
  return step(control_poses, in.data(), present, out);
}

int Batch::update_measurements(const double* control_poses, const bb200_measurement* measurements, const uint8_t* present,
                               bb200_update_result* out) {
  error_.clear();
  for (size_t k = 0; k < members_.size(); ++k) out[k] = bb200_update_result{};
  if (const int st = check_measurements(measurements, present, false)) return st;
  return step(control_poses, measurements, present, out);
}

int Batch::update_clustered(const double* control_poses, const bb200_measurement* measurements, const uint8_t* present, const bb200_cluster_param& p,
                            bb200_update_result* out, bb200_estimate* clustered, uint32_t* n_cells, uint32_t* n_clusters) {
  error_.clear();
  for (size_t k = 0; k < members_.size(); ++k) out[k] = bb200_update_result{};
  if (const char* why = cluster_param_error(p)) return fail(BB200_ERR_INVALID_ARGUMENT, why);
  if (const int st = check_measurements(measurements, present, false)) return st;
  const ClusteredOut co{&p, clustered, n_cells, n_clusters};
  return step(control_poses, measurements, present, out, &co);
}

int Batch::step(const double* control_poses, const bb200_measurement* in, const uint8_t* present, bb200_update_result* out,
                const ClusteredOut* clustered) {
  for (size_t k = 0; k < members_.size(); ++k) out[k] = bb200_update_result{};
  if (const int st = step_begin(control_poses, in, present, nullptr)) return st;
  return step_end(clustered, out);
}

int Batch::update_begin(const double* control_poses, const bb200_measurement* measurements, const uint8_t* present, bb200_weigh_view* views) {
  error_.clear();
  if (open_.open) return fail(BB200_ERR_STATE, "a weighed step is already open (bb200_amcl_batch_update_end closes it)");
  if (const int st = check_measurements(measurements, present, true)) return st;
  return step_begin(control_poses, measurements, present, views);
}

int Batch::update_end(const bb200_cluster_param* cluster, bb200_update_result* out, bb200_estimate* clustered, uint32_t* n_cells, uint32_t* n_clusters) {
  error_.clear();
  for (size_t k = 0; k < members_.size(); ++k) out[k] = bb200_update_result{};
  if (!open_.open) return fail(BB200_ERR_STATE, "no weighed step is open (bb200_amcl_batch_update_begin)");
  if (cluster != nullptr)
    if (const char* why = cluster_param_error(*cluster)) return fail(BB200_ERR_INVALID_ARGUMENT, why);
  const ClusteredOut co{cluster, clustered, n_cells, n_clusters};
  return step_end(cluster != nullptr ? &co : nullptr, out);
}

int Batch::step_begin(const double* control_poses, const bb200_measurement* in, const uint8_t* present, bb200_weigh_view* views) {
  error_.clear();
  const size_t count = members_.size();
  if (views != nullptr)
    for (size_t k = 0; k < count; ++k) views[k] = bb200_weigh_view{};
  if (const int st = check_present(present)) return st;
  // A landmark map weighs detections and a grid map points, scans or clouds, as Filter::check_measurement decides.
  for (size_t k = 0; k < count; ++k) {
    if (!selected_member(present, k) || in[k].kind == BB200_MEASUREMENT_WEIGHTS) continue;
    const Member& m = members_[k];
    const bool detections = in[k].kind == BB200_MEASUREMENT_LANDMARKS;
    const bool landmark_map = m.map >= 0 && maps_.at(m.map).map.landmark_map();
    const std::string who = "member " + std::to_string(k) + ": ";
    if (detections && m.map >= 0 && !landmark_map) return fail(BB200_ERR_STATE, who + "detections need a landmark map");
    if (!detections && landmark_map) return fail(BB200_ERR_STATE, who + "a landmark map weighs detections, not points");
    if (detections && !m.detections_staged) return fail(BB200_ERR_STATE, who + "no detections staged (bb200_amcl_batch_set_detections)");
  }
  std::vector<AmclPolicy> before;
  before.reserve(count);
  for (const Member& m : members_) before.push_back(m.policy);
  auto rollback = [&](int st) {
    for (size_t k = 0; k < count; ++k) members_[k].policy = before[k];
    if (views != nullptr)
      for (size_t k = 0; k < count; ++k) views[k] = bb200_weigh_view{};
    return st;
  };

  // Host half of every present member's Amcl::update (amcl_core.hpp:165-190).
  std::vector<bb200_step_plan> plans(count);
  std::vector<uint32_t> active;  // members that update in this step, in member order
  for (size_t k = 0; k < count; ++k) {
    if (!selected_member(present, k)) continue;
    members_[k].policy.plan_update(control_poses + 4 * k, members_[k].n, &plans[k]);
    if (plans[k].update) active.push_back(static_cast<uint32_t>(k));
  }
  auto weighed = [&](uint32_t k) { return in[k].kind == BB200_MEASUREMENT_WEIGHTS; };
  const bool any_weighed = std::any_of(active.begin(), active.end(), weighed);
  if (active.empty()) {
    open_ = OpenStep{};
    open_.open = true;
    open_.before = std::move(before);
    return BB200_OK;
  }

  // Points sent by the host come first in the point buffer, in member order; the points of scans and clouds, written by
  // batch_points_kernel, follow them.  Scans and clouds are sized by their bounds (measurement_bound).
  uint64_t points_total = 0, host_points = 0, input_floats = 0, detections_total = 0;
  bool landmark_maps = false;
  uint32_t max_points = 0;
  // The map every updating member with a map reads, -1 when they read several, -2 when none has one (every updating
  // member is weighed by the caller and none may inject).
  int step_map = -2;
  std::vector<int> forms(count, kBatchField);
  for (const uint32_t k : active)
    if (members_[k].map < 0 && !weighed(k))
      return rollback(fail(BB200_ERR_STATE, maps_.empty() ? "no map set" : "member " + std::to_string(k) + " has no map"));
  for (const uint32_t k : active) {
    const uint64_t bound = measurement_bound(in[k]);
    if (bound > 0xffffffffull) return rollback(fail(BB200_ERR_INVALID_ARGUMENT, "too many points"));
    if (in[k].kind == BB200_MEASUREMENT_POINTS && in[k].n_points > 0 && in[k].points_xy == nullptr)
      return rollback(fail(BB200_ERR_INVALID_ARGUMENT, "points_xy is null"));
    const int id = members_[k].map;
    const bool injects = plans[k].resample && plans[k].random_state_probability > 0.0;
    if (injects && (id < 0 || !maps_.at(id).map.can_draw_states()))
      return rollback(fail(BB200_ERR_STATE, id >= 0 && maps_.at(id).map.landmark_map() ? "recovery injection needs a non-empty, finite landmark box"
                                                                                       : "recovery injection needs a map with free cells"));
    if (weighed(k)) forms[k] = kBatchWeighed;
    if (id < 0) continue;
    const DeviceMap& map = maps_.at(id).map;
    // The beam model walks a member's rays in two passes when its map allows it (the rule of the single filter).
    if (map.sensor == BB200_SENSOR_BEAM && !weighed(k)) forms[k] = beam_two_pass_map(map) ? kBatchBeamTwoPass : kBatchBeamFused;
    if (in[k].kind == BB200_MEASUREMENT_LANDMARKS) {
      forms[k] = kBatchLandmark;
      detections_total += members_[k].detections.size();
    }
    landmark_maps = landmark_maps || map.landmark_map();
    step_map = step_map == -2 || step_map == id ? id : -1;
    points_total += bound;
    if (in[k].kind == BB200_MEASUREMENT_POINTS) host_points += bound;
    input_floats += in[k].kind == BB200_MEASUREMENT_CLOUD ? 3 * bound : in[k].kind == BB200_MEASUREMENT_SCAN ? bound : 0;
    max_points = std::max(max_points, static_cast<uint32_t>(bound));
  }
  const bool convert = std::any_of(active.begin(), active.end(),
                                   [&](uint32_t k) { return in[k].kind == BB200_MEASUREMENT_SCAN || in[k].kind == BB200_MEASUREMENT_CLOUD; });
  // Amcl::update_device's KLD path: a resampling member with min_particles < max_particles sizes its new set with
  // take_while_kld (Filter::resample_kld).
  auto resamples_kld = [&](uint32_t k) { return plans[k].resample != 0 && plans[k].opts.min_particles < plans[k].opts.max_particles; };
  const bool kld = std::any_of(active.begin(), active.end(), resamples_kld);
  // on_effective_size_drop: a selective member whose every_n fired resamples only when its effective sample size drops
  // below n / 2, decided on the device (batch_ess_kernel).
  const bool ess = std::any_of(active.begin(), active.end(), [&](uint32_t k) { return plans[k].needs_ess != 0; });
  // The staging buffers grow with room to spare, points and detections once the stream has drained.
  const uint64_t point_room = 2 * std::max<uint64_t>(points_total + points_total / 2, 4096);
  const uint64_t detection_room = std::max<uint64_t>(detections_total + detections_total / 2, 256);
  const uint64_t input_room = std::max<uint64_t>(input_floats + input_floats / 2, 4096);
  int st = check(cudaSetDevice(device_), "cudaSetDevice");
  if (st == BB200_OK && 2 * points_total > points_.size()) st = check(cudaStreamSynchronize(stream_), "cudaStreamSynchronize");
  if (st == BB200_OK) st = check(points_.grow(2 * points_total, point_room), "point staging");
  if (st == BB200_OK && detections_total > detections_.size()) st = check(cudaStreamSynchronize(stream_), "cudaStreamSynchronize");
  if (st == BB200_OK) st = check(detections_.grow(detections_total, detection_room), "detection staging");
  if (st == BB200_OK && step_map == -1) st = ensure_map_table();
  if (st == BB200_OK && convert) st = check(inputs_.grow(count), "measurement table");
  if (st == BB200_OK && convert) st = check(input_.grow(input_floats, input_room), "measurement staging");
  if (st == BB200_OK && kld) st = ensure_kld_scratch();
  if (st == BB200_OK && any_weighed) st = check(factors_.grow(weights_.size()), "factor buffer");  // laid out like the weights
  for (auto k = active.begin(); st == BB200_OK && k != active.end(); ++k)
    if (in[*k].kind == BB200_MEASUREMENT_SCAN) st = ensure_scan_table(members_[*k], *in[*k].scan);
  if (st != BB200_OK) return rollback(st);

  // The step's member table and the concatenated scans.
  const uint32_t n_active = static_cast<uint32_t>(active.size());
  BatchStepArgs a{};
  a.n_members = n_active;
  uint64_t point_offset = 0, device_offset = host_points, input_offset = 0, hit_words = 0, detection_offset = 0;
  std::vector<LandmarkDetection> prepared;
  for (uint32_t j = 0; j < n_active; ++j) {
    const uint32_t k = active[j];
    const Member& m = members_[k];
    const bb200_step_plan& plan = plans[k];
    const bb200_measurement& meas = in[k];
    const uint64_t bound = measurement_bound(meas);
    BatchMember& b = table_.host.get()[j];
    b = BatchMember{};
    b.offset = m.offset;
    b.n = m.n;
    b.slots = m.capacity;
    b.seed = m.policy.params().seed;
    b.step = plan.step;
    b.resample = plan.needs_ess ? kBatchResampleEss : plan.resample;
    b.scheme = plan.opts.scheme;
    b.cur = m.cur;
    b.ceil_log2_count = ceil_log2_count(m.capacity);
    b.map = step_map == -1 && m.map >= 0 ? maps_.at(m.map).slot : 0;
    b.random_state_probability = plan.random_state_probability;
    b.pivot_x = m.pivot[0];
    b.pivot_y = m.pivot[1];
    b.sampling = to_kernel_sampling(plan.sampling);
    b.kld = resamples_kld(k) ? 1 : 0;
    if (b.kld) {
      BatchKldMember& q = kld_.host.get()[j];
      q = BatchKldMember{};
      q.min_particles = plan.opts.min_particles;
      q.two_epsilon = 2 * plan.opts.kld_epsilon;
      q.z = plan.opts.kld_z;
      for (int d = 0; d < 3; ++d) q.hash_resolution[d] = plan.opts.spatial_resolution[d];
      q.table_offset = m.table_offset;
      q.table_mask = m.table_slots - 1;
    }
    if (meas.kind == BB200_MEASUREMENT_WEIGHTS) {
      b.point_offset = 0;  // no points: the caller's factors stand for the sensor model
      b.n_points = 0;
      b.points_radius = 0.0;
    } else if (meas.kind == BB200_MEASUREMENT_LANDMARKS) {
      // No points: point_offset and n_points index the step's prepared detections instead.
      prepare_detections(maps_.at(m.map).map.landmark_slices, m.detections.data(), m.detections.size(), &prepared);
      if (!prepared.empty()) std::memcpy(detections_.host.get() + detection_offset, prepared.data(), prepared.size() * sizeof(LandmarkDetection));
      b.point_offset = detection_offset;
      b.n_points = static_cast<uint32_t>(prepared.size());
      b.points_radius = 0.0;
      detection_offset += prepared.size();
    } else if (meas.kind == BB200_MEASUREMENT_POINTS) {
      b.point_offset = point_offset;
      b.n_points = static_cast<uint32_t>(meas.n_points);
      b.points_radius = scan_radius(meas.points_xy, meas.n_points);
      if (meas.n_points > 0) std::memcpy(points_.host.get() + 2 * point_offset, meas.points_xy, 2 * meas.n_points * sizeof(double));
      point_offset += meas.n_points;
    } else {
      b.point_offset = device_offset;
      b.n_points = static_cast<uint32_t>(bound);  // a scan's survivors replace it on the device
      b.points_radius = 0.0;                      // raised to the points' largest |x| + |y| on the device
      device_offset += bound;
    }
    if (convert) {
      BatchPointsMember& d = inputs_.host.get()[j];
      d = BatchPointsMember{};
      d.kind = meas.kind;  // points and weighed members have no CTA there
      d.input_offset = input_offset;
      d.count = static_cast<uint32_t>(bound);
      float* raw = input_.host.get() + input_offset;
      if (meas.kind == BB200_MEASUREMENT_SCAN) {
        const bb200_laser_scan& scan = *meas.scan;
        const std::vector<uint64_t>& indices = m.scan.indices;
        for (uint64_t pos = 0; pos < bound; ++pos) raw[pos] = scan.ranges[indices[pos]];
        d.min_range = scan.min_range;
        d.max_range = scan.max_range;
        d.directions = m.scan.directions.get();
        set_origin(d, scan.laser_origin);
        input_offset += bound;
      } else if (meas.kind == BB200_MEASUREMENT_CLOUD) {
        const bb200_point_cloud& cloud = *meas.cloud;
        if (cloud.datatype == BB200_POINT_FLOAT32) {
          pack_cloud<float>(cloud, raw);
        } else {
          pack_cloud<double>(cloud, raw);
        }
        set_origin(d, cloud.origin);
        input_offset += 3 * bound;
      }
    }
    b.hit_stride = (m.n + 31) / 32 * 32;
    if (forms[k] == kBatchBeamTwoPass) {
      b.hit_offset = hit_words;
      hit_words += b.hit_stride * bound;
    }
  }
  // The two-pass members keep that form when their hit words fit under the single filter's bound for one pass and in
  // device memory; otherwise they take the fused kernel.
  if (hit_words > 0 && !(hit_words <= kBeamHitPassBytes / sizeof(uint32_t) && ensure_hits(hit_words)))
    for (const uint32_t k : active)
      if (forms[k] == kBatchBeamTwoPass) forms[k] = kBatchBeamFused;
  // The CTA ranges of every row: each member in the reweight row of its form.
  auto row = [&](int l) { return first_.host.get() + static_cast<size_t>(l) * (n_active + 1); };
  for (const uint32_t k : active) a.forms |= 1 << forms[k];
  write_cta_rows<kBatchLaunches>(row(0), n_active, a.ctas,
                                 [&](uint32_t j, uint32_t* c) { batch_member_ctas(table_.host.get()[j], forms[active[j]], c); });
  BatchPointsArgs pa{};
  if (convert) write_cta_rows<1>(row(kBatchPointsRow), n_active, &pa.ctas, [&](uint32_t j, uint32_t* c) { *c = batch_points_ctas(inputs_.host.get()[j]); });
  if (kld || ess) {
    static_assert(kBatchMomentsRow == kBatchKldRow + 1 && kBatchEssRow == kBatchKldRow + 2, "batch_post_ctas fills three adjacent rows");
    uint32_t totals[3];
    write_cta_rows<3>(row(kBatchKldRow), n_active, totals, [&](uint32_t j, uint32_t* c) { batch_post_ctas(table_.host.get()[j], c); });
    a.post_ctas[0] = totals[0];
    a.post_ctas[1] = totals[1];
    a.ess_ctas = totals[2];
  }
  const bool any_landmark = std::any_of(active.begin(), active.end(), [&](uint32_t k) { return forms[k] == kBatchLandmark; });
  if (any_landmark)
    write_cta_rows<1>(row(kBatchLandmarkRow), n_active, &a.landmark_ctas, [&](uint32_t j, uint32_t* c) {
      *c = forms[active[j]] == kBatchLandmark ? batch_landmark_ctas(table_.host.get()[j]) : 0;
    });
  if (any_weighed)
    write_cta_rows<1>(row(kBatchWeighRow), n_active, &a.weigh_ctas,
                      [&](uint32_t j, uint32_t* c) { *c = weighed(active[j]) ? batch_weigh_ctas(table_.host.get()[j]) : 0; });
  const int rows = any_landmark ? kBatchRows : kld || ess || any_weighed ? kBatchLandmarkRow : convert ? kBatchLaunches + 1 : kBatchLaunches;

  cudaStream_t stream = stream_;
  for (const uint32_t k : active) members_[k].cdf_total = 0;  // from here on the step may have rewritten their CDFs
  seq_ = seq_ == 0x7fffffff ? 1 : seq_ + 1;
  *ticket_host_.get() = 0;
  st = check(table_.to_device(0, n_active, stream), "upload member table");
  if (st == BB200_OK) st = check(first_.to_device(0, rows * (n_active + 1), stream), "upload ranges");
  if (st == BB200_OK && host_points > 0) st = check(points_.to_device(0, 2 * host_points, stream), "upload points");
  if (st == BB200_OK && convert) st = check(inputs_.to_device(0, n_active, stream), "upload measurement table");
  if (st == BB200_OK && detection_offset > 0) st = check(detections_.to_device(0, detection_offset, stream), "upload detections");
  if (st == BB200_OK && input_floats > 0) st = check(input_.to_device(0, input_floats, stream), "upload measurements");
  if (st == BB200_OK && kld) st = check(kld_.to_device(0, n_active, stream), "upload KLD table");
  if (st != BB200_OK) return rollback(st);
  if (convert) {
    pa.members = table_.device.get();
    pa.first = first_.device.get() + static_cast<size_t>(kBatchPointsRow) * (n_active + 1);
    pa.n_members = n_active;
    pa.inputs = inputs_.device.get();
    pa.input = input_.device.get();
    pa.points = points_.device.get();
    launches_ += static_cast<uint64_t>(launch_batch_points(pa, stream));
  }
  a.members = table_.device.get();
  a.first = first_.device.get();
  a.max_points = max_points;
  a.states[0] = states_[0].get();
  a.states[1] = states_[1].get();
  a.weights = weights_.get();
  a.cdf = cdf_.get();
  a.ancestors = ancestors_.get();
  a.tile_state = tile_state_.get();
  a.scalars = scalars_.get();
  a.partials = partials_.get();
  a.points = points_.device.get();
  if (step_map >= 0) {
    const DeviceMap& map = maps_.at(step_map).map;
    a.field = map.field;
    a.free_cells = map.free_cells;
    a.n_free = map.n_free;
    a.grid_width = map.grid_width;
    a.grid_resolution = map.grid_resolution;
    a.grid_origin = map.grid_origin;
    a.occupancy = map.occupancy;
    a.beam = map.beam;
    a.landmark = map.landmark;
    a.landmarks = map.landmarks;
    a.n_landmarks = map.n_landmarks;
    for (int c = 0; c < 4; ++c) a.box[c] = map.box[c];
  } else if (step_map == -1) {
    a.maps = map_table_.get();
  }
  a.hits = hits_.get();
  if (kld) {
    a.kld = kld_.device.get();
    a.hashes = cl_.hashes.get();
    a.keys = cl_.keys.get();
    a.vals = cl_.first.get();
  }
  a.summary = summary_host_.get();
  a.members_done = members_done_.get();
  a.ticket = ticket_host_.get();
  a.seq = seq_;
  a.factors = factors_.get();
  a.detections = detections_.device.get();
  a.landmark_maps = landmark_maps ? 1 : 0;
  launches_ += static_cast<uint64_t>(launch_batch_step_head(a, stream));
  st = check(cudaGetLastError(), "batch step launch");
  if (st != BB200_OK) return rollback(st);
  if (views != nullptr)
    for (const uint32_t k : active) {
      const Member& m = members_[k];
      bb200_weigh_view& v = views[k];
      v.updated = 1;
      if (!weighed(k)) continue;
      v.n = m.n;
      v.states = reinterpret_cast<const double*>(states_[m.cur].get() + m.offset);
      v.factors = factors_.get() + m.offset;
      v.stream = stream;
    }
  open_ = OpenStep{};
  open_.open = true;
  open_.before = std::move(before);
  open_.plans = std::move(plans);
  open_.active = std::move(active);
  open_.kld = kld;
  open_.args = a;
  return BB200_OK;
}

int Batch::step_end(const ClusteredOut* clustered, bb200_update_result* out) {
  OpenStep step = std::move(open_);
  open_ = OpenStep{};
  const size_t count = members_.size();
  auto rollback = [&](int st) {
    for (size_t k = 0; k < count; ++k) members_[k].policy = step.before[k];
    return st;
  };
  const std::vector<bb200_step_plan>& plans = step.plans;
  const std::vector<uint32_t>& active = step.active;
  if (active.empty()) return BB200_OK;
  const uint32_t n_active = static_cast<uint32_t>(active.size());
  auto resamples_kld = [&](uint32_t k) { return plans[k].resample != 0 && plans[k].opts.min_particles < plans[k].opts.max_particles; };
  BatchStepArgs& a = step.args;
  cudaStream_t stream = stream_;
  int st = BB200_OK;
  if (clustered != nullptr) st = ensure_select_scratch();
  if (st != BB200_OK) return rollback(st);
  // update_clustered: the pre-step cluster table and how the step may change each member (batch_cluster_table_kernel).
  if (clustered != nullptr) {
    for (uint32_t j = 0; j < n_active; ++j) {
      const uint32_t k = active[j];
      const Member& m = members_[k];
      const bb200_step_plan& plan = plans[k];
      cl_.table.host.get()[j] = cluster_member(k);
      BatchClusterPost& q = sel_.post.host.get()[j];
      q = BatchClusterPost{};
      q.scratch_offset = sel_.offsets[k];
      q.capacity = static_cast<uint32_t>(m.capacity);
      q.mode = plan.needs_ess ? 2 : plan.resample ? 1 : 0;
      q.kld = resamples_kld(k) ? 1 : 0;
    }
  }

  if (st == BB200_OK && clustered != nullptr) st = check(cl_.table.to_device(0, n_active, stream), "upload cluster table");
  if (st == BB200_OK && clustered != nullptr) st = check(sel_.post.to_device(0, n_active, stream), "upload cluster steps");
  if (st != BB200_OK) return rollback(st);
  launches_ += static_cast<uint64_t>(launch_batch_step_tail(a, stream));
  st = check(cudaGetLastError(), "batch step launch");
  if (st != BB200_OK) return rollback(st);
  const bb200_cluster_param* cp = clustered != nullptr ? clustered->p : nullptr;
  if (cp != nullptr) {
    // After the step's last kernel: the post-step cluster table, the cells of every updated member, their selection.
    BatchSelectArgs sa{};
    sa.members = cl_.table.device.get();
    sa.post = sel_.post.device.get();
    sa.summary = summary_host_.get();
    sa.n_members = n_active;
    sa.records = cl_.records.get();
    sa.cells = cl_.cells.device.get();
    sa.keys = cl_.keys.get();
    sa.ids = cl_.ids.get();
    sa.schedule_start = sel_.schedule_start.get();
    sa.schedule = sel_.schedule.get();
    sa.scratch = sel_.scratch.get();
    sa.linear = cp->linear_hash_resolution;
    sa.angular = cp->angular_hash_resolution;
    sa.percentile = cp->weight_cap_percentile;
    const Rot2 zero = rot_exp(0.0), plus = rot_exp(+sa.angular), minus = rot_exp(-sa.angular);  // glibc, as select_cluster
    const double lin = sa.linear;
    const Pose2 adjacent[6] = {Pose2{zero.c, zero.s, +lin, 0.0}, Pose2{zero.c, zero.s, -lin, 0.0}, Pose2{zero.c, zero.s, 0.0, +lin},
                               Pose2{zero.c, zero.s, 0.0, -lin}, Pose2{plus.c, plus.s, 0.0, 0.0},  Pose2{minus.c, minus.s, 0.0, 0.0}};
    for (int s = 0; s < 6; ++s) sa.adjacent[s] = adjacent[s];
    sa.results = sel_.results.get();
    launch_batch_cluster_table(sa, stream);
    launch_batch_cluster_cells(cluster_args(sa.linear, sa.angular), n_active, stream);
    launch_batch_cluster_select(sa, stream);
    launches_ += 3;
    st = check(cudaGetLastError(), "batch cluster selection launch");
    if (st != BB200_OK) return rollback(st);
  }

  // The last member to finish stores the ticket into pinned memory; the cluster selection runs after it, so a step with
  // one waits for the whole stream instead.
  const bool done = cp == nullptr && wait_for_ticket(ticket_host_.get(), seq_, stream);
  if (!done) st = check(cudaStreamSynchronize(stream), "batch step");
  if (st == BB200_OK && !done && *static_cast<volatile int*>(ticket_host_.get()) != seq_) st = fail(BB200_ERR_CUDA, "the batch step ended without its completion ticket");
  if (st != BB200_OK) return rollback(st);

  // What the step did to each member, committed once nothing can fail any more.
  struct Outcome {
    int cur;
    uint64_t n;
    double pivot[2];
    bb200_update_result r;
  };
  std::vector<Outcome> outcome(n_active);
  for (uint32_t j = 0; j < n_active; ++j) {
    const uint32_t k = active[j];
    const Member& m = members_[k];
    const StepSummary& s = summary_host_.get()[j];
    const bb200_step_plan& plan = plans[k];
    Outcome& o = outcome[j];
    bb200_update_result& r = o.r;
    r = bb200_update_result{};
    estimate_from_moments(s.moments, m.pivot, &r.estimate);
    o.pivot[0] = m.pivot[0];
    o.pivot[1] = m.pivot[1];
    pivot_to_estimate(r.estimate, o.pivot);
    const bool resampled = plan.needs_ess ? s.resampled != 0 : plan.resample != 0;  // the device's decision for a selective member
    o.cur = resampled ? m.cur ^ 1 : m.cur;
    o.n = resampled ? (table_.host.get()[j].kld ? s.accepted : m.capacity) : m.n;
    r.updated = 1;
    r.resampled = resampled ? 1 : 0;
    r.n_particles = o.n;
    r.random_state_probability = plan.random_state_probability;
    r.weight_sum = std::ldexp(static_cast<double>(s.total), -s.exponent);
    r.weights_degenerate = s.valid != 0 ? 0 : 1;
  }

  if (cp != nullptr) {
    // Members the device could not promise the host's bits for: their records back to back (batch_cluster_compact_kernel
    // over those members alone), then select_cluster on the host.
    const BatchClusterResult* res = sel_.results.get();
    std::vector<uint32_t> flagged;
    uint64_t flagged_cells = 0;
    for (uint32_t j = 0; j < n_active; ++j) {
      if (!res[j].fallback) continue;
      BatchClusterMember& c = cl_.table.host.get()[flagged.size()];
      c = BatchClusterMember{};
      c.offset = members_[active[j]].offset;
      cl_.cells.host.get()[flagged.size()] = res[j].cells;
      flagged_cells += res[j].cells;
      flagged.push_back(j);
    }
    std::vector<ClusterSelection> host_sel(flagged.size());
    if (!flagged.empty()) {
      const uint32_t n_flagged = static_cast<uint32_t>(flagged.size());
      st = ensure_cluster_records(flagged_cells);
      if (st == BB200_OK) st = check(cl_.table.to_device(0, n_flagged, stream), "upload fallback table");
      if (st == BB200_OK) st = check(cl_.cells.to_device(0, n_flagged, stream), "upload fallback cells");
      if (st == BB200_OK) {
        launch_batch_cluster_compact(cl_.table.device.get(), cl_.cells.device.get(), cl_.records.get(), n_flagged, cl_records_host_.get(), stream);
        ++launches_;
        st = check(cudaGetLastError(), "batch_cluster_compact");
      }
      if (st == BB200_OK) st = check(cudaStreamSynchronize(stream), "batch cluster fallback");
      if (st != BB200_OK) return rollback(st);
      const HostCell* cells = reinterpret_cast<const HostCell*>(cl_records_host_.get());
      for (size_t f = 0; f < flagged.size(); ++f) {
        const uint32_t count = res[flagged[f]].cells;
        host_sel[f] = select_cluster(cells, count, outcome[flagged[f]].n, cp->linear_hash_resolution, cp->angular_hash_resolution,
                                     cp->weight_cap_percentile);
        cells += count;
      }
    }
    size_t f = 0;
    for (uint32_t j = 0; j < n_active; ++j) {
      const uint32_t k = active[j];
      const double* moments = res[j].moments;
      uint32_t clusters = res[j].clusters;
      if (f < flagged.size() && flagged[f] == j) {
        moments = host_sel[f].moments;
        clusters = host_sel[f].clusters;
        ++f;
      }
      if (clustered->estimates != nullptr) estimate_from_moments(moments, outcome[j].pivot, &clustered->estimates[k]);
      if (clustered->n_cells != nullptr) clustered->n_cells[k] = res[j].cells;
      if (clustered->n_clusters != nullptr) clustered->n_clusters[k] = clusters;
    }
  }

  for (uint32_t j = 0; j < n_active; ++j) {
    const uint32_t k = active[j];
    Member& m = members_[k];
    const Outcome& o = outcome[j];
    if (o.r.resampled) {
      m.ancestors_n = o.n;
    } else {
      m.cdf_total = summary_host_.get()[j].total;  // the step's scan, over the weights before normalisation
    }
    m.cur = o.cur;
    m.n = o.n;
    m.pivot[0] = o.pivot[0];
    m.pivot[1] = o.pivot[1];
    out[k] = o.r;
    m.policy.commit_update(o.r.resampled, plans[k].random_state_probability);
  }
  return BB200_OK;
}

}  // namespace bb200
