#include "state_blob.hpp"

#include <cstring>

namespace bb200 {

namespace {

static_assert(sizeof(StateBlobHeader) == 88, "the header has no padding");
static_assert(sizeof(PolicyState) == 136 && sizeof(ParticleSetState) == 48, "the scalar sections have no padding");
static_assert(sizeof(bb200_amcl_param) % 8 == 0 && sizeof(bb200_motion_param) % 8 == 0, "sections keep 8-byte lengths");

const char* const kSectionNames[kStateSections] = {"params", "motion", "policy", "set", "states", "weights", "cdf", "ancestors"};

/// The parameter blocks with zeroed padding, so that a blob's bytes depend on the filter alone and carry no stray memory.
bb200_amcl_param canonical(const bb200_amcl_param& p) {
  bb200_amcl_param q;
  std::memset(&q, 0, sizeof(q));
  q.update_min_d = p.update_min_d;
  q.update_min_a = p.update_min_a;
  q.resample_interval = p.resample_interval;
  q.selective_resampling = p.selective_resampling;
  q.min_particles = p.min_particles;
  q.max_particles = p.max_particles;
  q.alpha_slow = p.alpha_slow;
  q.alpha_fast = p.alpha_fast;
  q.kld_epsilon = p.kld_epsilon;
  q.kld_z = p.kld_z;
  for (int k = 0; k < 3; ++k) q.spatial_resolution[k] = p.spatial_resolution[k];
  q.resample_scheme = p.resample_scheme;
  q.seed = p.seed;
  q.device = p.device;
  q.record_ancestors = p.record_ancestors;
  q.shard_first_index = p.shard_first_index;
  q.shard_capacity = p.shard_capacity;
  q.recovery_probability_override = p.recovery_probability_override;
  return q;
}

bb200_motion_param canonical(const bb200_motion_param& m) {
  bb200_motion_param q;
  std::memset(&q, 0, sizeof(q));
  q.model = m.model;
  q.rotation_noise_from_rotation = m.rotation_noise_from_rotation;
  q.rotation_noise_from_translation = m.rotation_noise_from_translation;
  q.translation_noise_from_translation = m.translation_noise_from_translation;
  q.translation_noise_from_rotation = m.translation_noise_from_rotation;
  q.strafe_noise_from_translation = m.strafe_noise_from_translation;
  q.distance_threshold = m.distance_threshold;
  return q;
}

int reject(const std::string& message, std::string* error) {
  if (error != nullptr) *error = "state blob: " + message;
  return BB200_ERR_INVALID_ARGUMENT;
}

}  // namespace

void state_blob_sections(const ParticleSetState& set, bool record_ancestors, uint64_t bytes[kStateSections]) {
  bytes[kSectionParams] = sizeof(bb200_amcl_param);
  bytes[kSectionMotion] = sizeof(bb200_motion_param);
  bytes[kSectionPolicy] = sizeof(PolicyState);
  bytes[kSectionSet] = sizeof(ParticleSetState);
  bytes[kSectionStates] = set.n * 32;
  bytes[kSectionWeights] = set.n * 8;
  bytes[kSectionCdf] = set.cdf_current != 0 ? set.n * 8 : 0;
  bytes[kSectionAncestors] = record_ancestors ? set.ancestors_n * 8 : 0;
}

uint64_t state_blob_size(const ParticleSetState& set, bool record_ancestors) {
  uint64_t bytes[kStateSections];
  state_blob_sections(set, record_ancestors, bytes);
  uint64_t total = sizeof(StateBlobHeader);
  for (const uint64_t b : bytes) total += b;
  return total;
}

void write_state_blob(const FilterState& s, void* out) {
  const bool record = s.params.record_ancestors != 0;
  StateBlobHeader h{};
  std::memcpy(h.magic, kStateBlobMagic, sizeof(h.magic));
  h.blob_version = kStateBlobVersion;
  h.abi_version = BB200_ABI_VERSION;
  h.total_size = state_blob_size(s.set, record);
  state_blob_sections(s.set, record, h.section_bytes);
  const bb200_amcl_param params = canonical(s.params);
  const bb200_motion_param motion = canonical(s.motion);
  const void* sources[kStateSections] = {&params, &motion, &s.policy, &s.set, s.states, s.weights, s.cdf, s.ancestors};
  unsigned char* p = static_cast<unsigned char*>(out);
  std::memcpy(p, &h, sizeof(h));
  p += sizeof(h);
  for (int k = 0; k < kStateSections; ++k) {
    if (h.section_bytes[k] > 0) std::memcpy(p, sources[k], h.section_bytes[k]);
    p += h.section_bytes[k];
  }
}

int read_state_blob(const void* blob, uint64_t size, FilterState* out, std::string* error) {
  if (blob == nullptr) return reject("null blob", error);
  StateBlobHeader h;
  if (size < sizeof(h)) return reject("truncated: " + std::to_string(size) + " bytes, the header alone takes " + std::to_string(sizeof(h)), error);
  const unsigned char* p = static_cast<const unsigned char*>(blob);
  std::memcpy(&h, p, sizeof(h));
  if (std::memcmp(h.magic, kStateBlobMagic, sizeof(h.magic)) != 0) return reject("wrong magic (not a beluga_b200 filter state)", error);
  if (h.blob_version != kStateBlobVersion)
    return reject("blob version " + std::to_string(h.blob_version) + " (this library reads version " + std::to_string(kStateBlobVersion) + ")", error);
  if (h.abi_version != BB200_ABI_VERSION)
    return reject("written for C ABI version " + std::to_string(h.abi_version) + " (this library has " + std::to_string(BB200_ABI_VERSION) + ")", error);
  if (h.total_size != size) return reject("the header gives " + std::to_string(h.total_size) + " bytes, the blob has " + std::to_string(size), error);

  FilterState s{};
  const uint64_t fixed[4] = {sizeof(s.params), sizeof(s.motion), sizeof(s.policy), sizeof(s.set)};
  for (int k = 0; k < 4; ++k)
    if (h.section_bytes[k] != fixed[k])
      return reject("section " + std::string(kSectionNames[k]) + " has " + std::to_string(h.section_bytes[k]) + " bytes, expected " + std::to_string(fixed[k]), error);
  if (size < sizeof(h) + fixed[0] + fixed[1] + fixed[2] + fixed[3]) return reject("truncated inside the scalar sections", error);
  p += sizeof(h);
  std::memcpy(&s.params, p, sizeof(s.params));
  p += sizeof(s.params);
  std::memcpy(&s.motion, p, sizeof(s.motion));
  p += sizeof(s.motion);
  std::memcpy(&s.policy, p, sizeof(s.policy));
  p += sizeof(s.policy);
  std::memcpy(&s.set, p, sizeof(s.set));
  p += sizeof(s.set);

  // Scalars no unsharded filter holds: bb200_amcl_create_with_motion's checks, then the set's own.
  const bb200_amcl_param& q = s.params;
  if (q.shard_first_index != 0 || q.shard_capacity != 0) return reject("the state of a shard (sharded filters have no state blob)", error);
  if (q.max_particles == 0 || q.min_particles > q.max_particles) return reject("need 0 < min_particles <= max_particles", error);
  if (s.motion.model < BB200_MOTION_DIFFERENTIAL || s.motion.model > BB200_MOTION_STATIONARY) return reject("unknown motion model", error);
  if (s.set.n > q.max_particles) return reject("more particles than max_particles", error);
  if (s.set.ancestors_n > q.max_particles) return reject("more ancestors than max_particles", error);
  if (q.record_ancestors == 0 && s.set.ancestors_n != 0) return reject("ancestors of a filter that does not record them", error);
  if (s.set.cdf_current > 1 || s.set.reserved != 0) return reject("unknown flags in the particle set section", error);
  if ((s.set.cdf_current != 0) != (s.set.cdf_total != 0) || (s.set.cdf_current != 0 && s.set.n == 0))
    return reject("a current CDF needs particles and a positive total", error);
  if (s.policy.window_size < 0 || s.policy.window_size > 2 || s.policy.has_latest_pose > 1 || s.policy.force_update > 1)
    return reject("policy section out of range", error);

  uint64_t want[kStateSections];
  state_blob_sections(s.set, q.record_ancestors != 0, want);
  for (int k = kSectionStates; k < kStateSections; ++k)
    if (h.section_bytes[k] != want[k])
      return reject("section " + std::string(kSectionNames[k]) + " has " + std::to_string(h.section_bytes[k]) + " bytes, the particle set needs " +
                        std::to_string(want[k]),
                    error);
  if (state_blob_size(s.set, q.record_ancestors != 0) != size) return reject("the sections do not add up to the blob's size", error);
  const void** arrays[4] = {&s.states, &s.weights, &s.cdf, &s.ancestors};
  for (int k = kSectionStates; k < kStateSections; ++k) {
    *arrays[k - kSectionStates] = want[k] > 0 ? p : nullptr;
    p += want[k];
  }
  *out = s;
  return BB200_OK;
}

}  // namespace bb200
