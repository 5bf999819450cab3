// The state blob codec (beluga_b200/csrc/state_blob.cpp) on the host: a round trip restores every scalar and array bit
// for bit, the header's section lengths follow the particle set, and every malformed blob is refused with its reason.
// Writes one valid blob to argv[1] and prints STATE_BLOB_PROBE_OK when every check passes.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "state_blob.hpp"

using namespace bb200;

namespace {

int failures = 0;

void expect(bool ok, const std::string& what) {
  if (!ok) {
    std::printf("FAIL %s\n", what.c_str());
    ++failures;
  }
}

struct Sample {
  FilterState state{};
  std::vector<double> states, weights;
  std::vector<uint64_t> cdf;
  std::vector<int64_t> ancestors;
};

Sample sample(uint64_t n, bool cdf_current, bool record, uint64_t ancestors_n) {
  Sample s;
  FilterState& f = s.state;
  f.params.max_particles = 4096;
  f.params.min_particles = 1000;
  f.params.resample_interval = 3;
  f.params.seed = 77;
  f.params.record_ancestors = record ? 1 : 0;
  f.params.spatial_resolution[2] = 0.1745;
  f.motion.model = BB200_MOTION_OMNIDIRECTIONAL;
  f.motion.strafe_noise_from_translation = 0.25;
  f.policy.has_latest_pose = 1;
  f.policy.latest_pose[0] = 1.0;
  f.policy.latest_pose[2] = -3.5;
  f.policy.window[1][3] = 2.25;
  f.policy.window_size = 2;
  f.policy.every_n_current = 2;
  f.policy.slow_output = 1e-3;
  f.policy.fast_output = 2e-3;
  f.policy.step = 41;
  f.set.n = n;
  f.set.ancestors_n = ancestors_n;
  f.set.pivot[0] = 1.5;
  f.set.pivot[1] = -0.5;
  f.set.cdf_current = cdf_current ? 1 : 0;
  f.set.cdf_total = cdf_current ? 123456789 : 0;
  for (uint64_t i = 0; i < 4 * n; ++i) s.states.push_back(0.001 * static_cast<double>(i) - 1.0);
  for (uint64_t i = 0; i < n; ++i) s.weights.push_back(1.0 / static_cast<double>(i + 1));
  if (cdf_current)
    for (uint64_t i = 0; i < n; ++i) s.cdf.push_back(1000 * (i + 1));
  for (uint64_t i = 0; i < ancestors_n; ++i) s.ancestors.push_back(static_cast<int64_t>(i) - 1);
  f.states = s.states.data();
  f.weights = s.weights.data();
  f.cdf = s.cdf.data();
  f.ancestors = s.ancestors.data();
  return s;
}

std::vector<unsigned char> write(const FilterState& f) {
  std::vector<unsigned char> blob(state_blob_size(f.set, f.params.record_ancestors != 0));
  write_state_blob(f, blob.data());
  return blob;
}

std::string refusal(const std::vector<unsigned char>& blob) {
  FilterState out;
  std::string error;
  const int st = read_state_blob(blob.data(), blob.size(), &out, &error);
  return st == BB200_ERR_INVALID_ARGUMENT ? error : "accepted (" + std::to_string(st) + ")";
}

void expect_refused(const std::vector<unsigned char>& blob, const std::string& reason, const std::string& what) {
  const std::string got = refusal(blob);
  expect(got.find(reason) != std::string::npos && got.rfind("state blob: ", 0) == 0, what + ": " + got);
}

template <class T>
void poke(std::vector<unsigned char>& blob, size_t offset, T value) {
  std::memcpy(blob.data() + offset, &value, sizeof(value));
}

}  // namespace

int main(int argc, char** argv) {
  // Round trips: current and stale CDFs, with and without ancestors, an empty set.
  const struct {
    uint64_t n;
    bool cdf, record;
    uint64_t ancestors;
  } cases[] = {{1000, true, true, 1000}, {1000, false, false, 0}, {0, false, true, 0}, {10, false, true, 700}, {1, true, false, 0}};
  for (const auto& c : cases) {
    const Sample s = sample(c.n, c.cdf, c.record, c.ancestors);
    const std::vector<unsigned char> blob = write(s.state);
    const std::string name = "n=" + std::to_string(c.n) + " cdf=" + std::to_string(c.cdf) + " ancestors=" + std::to_string(c.ancestors);
    StateBlobHeader h;
    std::memcpy(&h, blob.data(), sizeof(h));
    expect(std::memcmp(h.magic, "BB200STA", 8) == 0 && h.blob_version == 1 && h.abi_version == BB200_ABI_VERSION && h.total_size == blob.size(),
           name + ": header");
    const uint64_t want[kStateSections] = {sizeof(bb200_amcl_param), sizeof(bb200_motion_param), 136, 48, 32 * c.n, 8 * c.n, c.cdf ? 8 * c.n : 0,
                                           c.record ? 8 * c.ancestors : 0};
    uint64_t total = sizeof(StateBlobHeader);
    for (int k = 0; k < kStateSections; ++k) {
      expect(h.section_bytes[k] == want[k], name + ": section " + std::to_string(k));
      total += want[k];
    }
    expect(total == blob.size(), name + ": size");
    FilterState out;
    std::string error;
    expect(read_state_blob(blob.data(), blob.size(), &out, &error) == BB200_OK, name + ": read " + error);
    expect(std::memcmp(&out.params, &s.state.params, sizeof(out.params)) == 0 && std::memcmp(&out.motion, &s.state.motion, sizeof(out.motion)) == 0 &&
               std::memcmp(&out.policy, &s.state.policy, sizeof(out.policy)) == 0 && std::memcmp(&out.set, &s.state.set, sizeof(out.set)) == 0,
           name + ": scalars");
    expect(c.n == 0 || (std::memcmp(out.states, s.states.data(), 32 * c.n) == 0 && std::memcmp(out.weights, s.weights.data(), 8 * c.n) == 0),
           name + ": particles");
    expect(c.cdf ? std::memcmp(out.cdf, s.cdf.data(), 8 * c.n) == 0 : out.cdf == nullptr, name + ": cdf");
    expect(want[kSectionAncestors] > 0 ? std::memcmp(out.ancestors, s.ancestors.data(), want[kSectionAncestors]) == 0 : out.ancestors == nullptr,
           name + ": ancestors");
    expect(write(out) == blob, name + ": rewrite");
  }

  // Refusals.
  const Sample s = sample(100, true, true, 100);
  const std::vector<unsigned char> good = write(s.state);
  const size_t set_at = sizeof(StateBlobHeader) + sizeof(bb200_amcl_param) + sizeof(bb200_motion_param) + sizeof(PolicyState);
  expect_refused({good.begin(), good.begin() + 87}, "truncated", "short header");
  expect_refused({good.begin(), good.end() - 1}, "the header gives", "truncated");
  std::vector<unsigned char> b = good;
  b.push_back(0);
  expect_refused(b, "the header gives", "padded");
  b = good;
  b[0] = 'X';
  expect_refused(b, "wrong magic", "magic");
  b = good;
  poke<uint32_t>(b, 8, 2);
  expect_refused(b, "blob version 2 (this library reads version 1)", "future version");
  b = good;
  poke<uint32_t>(b, 12, 1);
  expect_refused(b, "C ABI version 1", "abi");
  b = good;
  poke<uint64_t>(b, 24 + 8 * kSectionPolicy, 128);
  expect_refused(b, "section policy has 128 bytes, expected 136", "policy length");
  b = good;
  poke<uint64_t>(b, 24 + 8 * kSectionCdf, 0);
  expect_refused(b, "section cdf has 0 bytes, the particle set needs 800", "cdf length");
  b = good;
  poke<uint64_t>(b, set_at, 101);  // n: the sections no longer match
  expect_refused(b, "section states has 3200 bytes, the particle set needs 3232", "count");
  b = good;
  poke<uint64_t>(b, set_at, 5000);
  expect_refused(b, "more particles than max_particles", "too many");
  b = good;
  poke<uint32_t>(b, set_at + 40, 3);
  expect_refused(b, "unknown flags", "flags");
  b = good;
  poke<uint64_t>(b, set_at + 32, 0);
  expect_refused(b, "a current CDF needs particles and a positive total", "zero total");
  b = good;
  poke<int32_t>(b, set_at - 12, 3);  // the policy's window_size
  expect_refused(b, "policy section out of range", "window");
  Sample q = sample(10, false, false, 0);
  q.state.params.shard_capacity = 5;
  expect_refused(write(q.state), "shard", "sharded");
  q = sample(10, false, false, 0);
  q.state.params.min_particles = 5000;
  expect_refused(write(q.state), "need 0 < min_particles <= max_particles", "params");
  q = sample(10, false, false, 0);
  q.state.motion.model = 7;
  expect_refused(write(q.state), "unknown motion model", "motion");
  q = sample(10, false, false, 0);
  q.state.set.ancestors_n = 4;
  expect_refused(write(q.state), "ancestors of a filter that does not record them", "ancestors");
  FilterState out;
  std::string error;
  expect(read_state_blob(nullptr, 0, &out, &error) == BB200_ERR_INVALID_ARGUMENT, "null");

  if (argc > 1) {
    FILE* f = std::fopen(argv[1], "wb");
    expect(f != nullptr && std::fwrite(good.data(), 1, good.size(), f) == good.size(), "write the blob file");
    if (f != nullptr) std::fclose(f);
  }
  if (failures == 0) std::printf("STATE_BLOB_PROBE_OK\n");
  return failures == 0 ? 0 : 1;
}
