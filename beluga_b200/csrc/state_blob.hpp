// The state blob: everything that decides a filter's future, as one versioned, self-describing byte string.  The standalone
// filter (bb200_amcl_export_state / bb200_amcl_create_from_state) and the batch (bb200_amcl_batch_export_members,
// _import_member, _create_from_states) write and read it through this one codec, so a blob moves a robot between any two of
// them.  The codec touches no device.
//
// Layout (every integer and double in the byte order of the machine that wrote it: a blob is read back on a machine of the
// same endianness):
//
//   StateBlobHeader    magic, blob version, BB200_ABI_VERSION, total size, the byte length of each section below
//   params             bb200_amcl_param, verbatim with its padding zeroed (its device is not honoured on import: the
//                      receiver's device wins)
//   motion             bb200_motion_param, the same
//   policy             PolicyState: AmclPolicy's on_motion pose, every_n phase, recovery filters, control window, flags, step
//   set                ParticleSetState: particle count, ancestors count, pivot, whether the CDF is current and its total
//   states             n x {cos, sin, x, y} doubles
//   weights            n doubles
//   cdf                n uint64 when the CDF is current, else empty
//   ancestors          ancestors_n int64 when params.record_ancestors, else empty
//
// Every section has a length that is a multiple of 8 bytes.  Maps are not part of a filter's state: the receiver attaches one.
#pragma once

#include <cstdint>
#include <string>

#include "../../include/beluga_b200.h"

namespace bb200 {

constexpr uint32_t kStateBlobVersion = 1;
constexpr char kStateBlobMagic[8] = {'B', 'B', '2', '0', '0', 'S', 'T', 'A'};

/// The host half of a filter that is not its parameters (AmclPolicy's private fields, amcl.hpp).
struct PolicyState {
  double latest_pose[4];    // on_motion's last accepted pose {cos, sin, x, y}, when has_latest_pose
  double window[2][4];      // the rolling control window, newest first
  uint64_t every_n_current;
  double slow_output, fast_output;  // the recovery estimator's exponential filters
  uint32_t step;
  int32_t window_size;
  uint32_t has_latest_pose;
  uint32_t force_update;
};

/// The particle set's scalars.
struct ParticleSetState {
  uint64_t n;            // particles
  uint64_t ancestors_n;  // entries of the ancestors section (0 when the filter does not record them)
  double pivot[2];       // of the raw moments (the last estimate)
  uint64_t cdf_total;    // fixed-point total of the current CDF (0 when cdf_current is 0)
  uint32_t cdf_current;  // 1: the cdf section holds the CDF the next pose draw samples from
  uint32_t reserved;     // 0
};

enum StateSection : int {
  kSectionParams = 0,
  kSectionMotion,
  kSectionPolicy,
  kSectionSet,
  kSectionStates,
  kSectionWeights,
  kSectionCdf,
  kSectionAncestors,
  kStateSections
};

struct StateBlobHeader {
  char magic[8];
  uint32_t blob_version;
  uint32_t abi_version;
  uint64_t total_size;
  uint64_t section_bytes[kStateSections];
};

/// A filter's state.  The arrays point to host memory (the blob itself after read_state_blob) and need no alignment.
struct FilterState {
  bb200_amcl_param params;
  bb200_motion_param motion;
  PolicyState policy;
  ParticleSetState set;
  const void* states;     // set.n x 32 bytes
  const void* weights;    // set.n x 8 bytes
  const void* cdf;        // set.n x 8 bytes when set.cdf_current
  const void* ancestors;  // set.ancestors_n x 8 bytes when params.record_ancestors
};

/// The byte length of each section of the blob of a filter with these scalars.
void state_blob_sections(const ParticleSetState& set, bool record_ancestors, uint64_t bytes[kStateSections]);
/// The size of that blob, header included.
uint64_t state_blob_size(const ParticleSetState& set, bool record_ancestors);
/// Writes the blob of `s` (state_blob_size bytes) to `out`.
void write_state_blob(const FilterState& s, void* out);
/// Checks a blob of `size` bytes and decodes it into *out, whose arrays then point into the blob.  BB200_OK, or
/// BB200_ERR_INVALID_ARGUMENT with the reason in *error: a truncated or padded blob, a wrong magic, a blob version this
/// library does not read, another ABI version, section lengths that do not match the scalars, or scalars no filter holds.
int read_state_blob(const void* blob, uint64_t size, FilterState* out, std::string* error);

}  // namespace bb200
