#include "cluster_host.hpp"

#include <algorithm>
#include <cmath>
#include <limits>
#include <queue>
#include <unordered_map>

#include "se2_math.cuh"

namespace bb200 {

namespace {

struct Node {
  double weight;      // cell weight after normalisation and capping
  uint32_t cell;      // index into the record array
  int64_t cluster;    // -1 while unassigned (std::optional in the reference)
};

struct Queued {  // KeyWithPriority, cluster_based_estimation.hpp:75-82
  double priority;
  std::size_t key;
  bool operator<(const Queued& other) const { return priority < other.priority; }
};

}  // namespace

ClusterSelection select_cluster(const HostCell* cells, std::size_t n_cells, std::uint64_t n_particles, double linear, double angular,
                                double percentile) {
  ClusterSelection out;
  out.cluster_of_cell.assign(n_cells, 0);
  if (n_cells == 0) return out;

  // The same container, reserve and insertion sequence as make_cluster_map (:143-158): with
  // libstdc++ the iteration order of the map -- which seeds the heap below and therefore decides
  // between equally heavy cells -- is a function of exactly that sequence.
  // The map is kept between calls (per thread) and emptied key by key at the end: an emptied map with the same
  // bucket count is indistinguishable from a freshly reserved one, and neither the allocation nor the zeroing of
  // n/5 buckets (1.6 MB at 1M particles) has to be paid again.
  thread_local std::unordered_map<std::size_t, Node> map;
  thread_local std::size_t reserved_for = static_cast<std::size_t>(-1);
  thread_local std::size_t fresh_buckets = 0;
  const std::size_t want = static_cast<std::size_t>(n_particles / 5);
  // ... as long as its bucket count is still the freshly reserved one: more cells than n/5 make the map rehash while it
  // fills (as the reference's does), and a map that has grown would iterate in a different order next time.
  if (reserved_for != want || !map.empty() || map.bucket_count() != fresh_buckets) {
    std::unordered_map<std::size_t, Node>().swap(map);
    map.reserve(want);
    reserved_for = want;
    fresh_buckets = map.bucket_count();
  }
  for (std::size_t k = 0; k < n_cells; ++k) {
    // normalize_and_cap_weights, first loop (:181-184)
    map.try_emplace(static_cast<std::size_t>(cells[k].hash), Node{cells[k].weight / static_cast<double>(cells[k].count), static_cast<uint32_t>(k), -1});
  }
  {  // calculate_percentile_threshold (:107-112) and the cap (:189-191)
    std::vector<double> values;
    values.reserve(map.size());
    for (const auto& kv : map) values.push_back(kv.second.weight);
    const auto nth = static_cast<std::ptrdiff_t>(static_cast<double>(values.size()) * percentile);
    std::nth_element(values.begin(), values.begin() + nth, values.end());
    const double cap = values[static_cast<std::size_t>(nth)];
    for (auto& kv : map) kv.second.weight = std::min(kv.second.weight, cap);
  }

  // assign_clusters (:205-253)
  std::vector<Queued> seed;
  seed.reserve(map.size());
  for (const auto& kv : map) seed.push_back(Queued{kv.second.weight, kv.first});
  std::priority_queue<Queued> queue(seed.begin(), seed.end());
  const double max_priority = queue.top().priority;

  // ParticleClusterizer::adjacent_grid_cells_ (:330-337)
  const Rot2 zero = rot_exp(0.0), plus = rot_exp(+angular), minus = rot_exp(-angular);
  const Pose2 adjacent[6] = {Pose2{zero.c, zero.s, +linear, 0.0}, Pose2{zero.c, zero.s, -linear, 0.0}, Pose2{zero.c, zero.s, 0.0, +linear},
                             Pose2{zero.c, zero.s, 0.0, -linear}, Pose2{plus.c, plus.s, 0.0, 0.0},     Pose2{minus.c, minus.s, 0.0, 0.0}};

  int64_t next_cluster = 0;
  while (!queue.empty()) {
    const std::size_t hash = queue.top().key;
    queue.pop();
    Node& cell = map.find(hash)->second;
    if (cell.cluster < 0) cell.cluster = next_cluster++;
    const double* r = cells[cell.cell].representative;
    const Pose2 pose{r[0], r[1], r[2], r[3]};
    for (const Pose2& step : adjacent) {
      const std::size_t neighbor_hash = static_cast<std::size_t>(spatial_hash(pose_mul(pose, step), linear, linear, angular));  // :289-293
      const auto it = map.find(neighbor_hash);
      if (it == map.end() || it->second.cluster >= 0 || !(it->second.weight <= cell.weight)) continue;  // :232-238
      it->second.cluster = cell.cluster;
      queue.push(Queued{max_priority + it->second.weight, neighbor_hash});  // :247
    }
  }
  out.clusters = static_cast<uint32_t>(next_cluster);
  for (const auto& kv : map) out.cluster_of_cell[kv.second.cell] = static_cast<uint32_t>(kv.second.cluster);

  // estimate_clusters (:351-398): per-cluster particle counts and moments, cells added in cell order.
  std::vector<std::uint64_t> count(out.clusters, 0);
  std::vector<double> moments(static_cast<std::size_t>(out.clusters) * 9, 0.0);
  for (std::size_t k = 0; k < n_cells; ++k) {
    const uint32_t c = out.cluster_of_cell[k];
    count[c] += cells[k].count;
    for (int j = 0; j < 9; ++j) moments[static_cast<std::size_t>(c) * 9 + j] += cells[k].moments[j];
  }
  // cluster_based_estimate (:420-431): heaviest cluster among those with more than one particle
  // (ranges::max_element keeps the first of equals; clusters are visited in ascending id).
  for (uint32_t c = 0; c < out.clusters; ++c) {
    if (count[c] <= 1) continue;
    if (!out.found || moments[static_cast<std::size_t>(out.best) * 9] < moments[static_cast<std::size_t>(c) * 9]) {
      out.best = c;
      out.found = true;
    }
  }
  for (std::size_t k = 0; k < n_cells; ++k) map.erase(static_cast<std::size_t>(cells[k].hash));  // leave it empty for the next call
  if (out.found) {
    for (int j = 0; j < 9; ++j) out.moments[j] = moments[static_cast<std::size_t>(out.best) * 9 + j];
  } else {  // "maybe the particles are too fragmented": the overall estimate (:422-425)
    for (std::size_t k = 0; k < n_cells; ++k)
      for (int j = 0; j < 9; ++j) out.moments[j] += cells[k].moments[j];
  }
  return out;
}

void estimate_from_moments(const double m[9], const double pivot[2], bb200_estimate* out) {
  // Normalised weights w/S: mean of (cos, sin, x, y); cov = (E[d d^T] - E[d] E[d]^T) / (1 - sum (w/S)^2).
  const double sum = m[0];
  const double mc = m[2] / sum, ms = m[3] / sum, mdx = m[4] / sum, mdy = m[5] / sum;
  const double correction = 1.0 - m[1] / (sum * sum);
  for (double& c : out->cov) c = 0.0;
  out->cov[0] = (m[6] / sum - mdx * mdx) / correction;
  out->cov[1] = (m[7] / sum - mdx * mdy) / correction;
  out->cov[3] = out->cov[1];
  out->cov[4] = (m[8] / sum - mdy * mdy) / correction;
  out->mean[2] = pivot[0] + mdx;
  out->mean[3] = pivot[1] + mdy;
  const double norm = std::sqrt(mc * mc + ms * ms);
  if (norm < std::numeric_limits<double>::epsilon()) {
    out->cov[8] = std::numeric_limits<double>::infinity();
    out->mean[0] = 1.0;
    out->mean[1] = 0.0;
  } else {
    out->cov[8] = -2.0 * std::log(norm);
    const double len = std::hypot(mc, ms);
    out->mean[0] = mc / len;
    out->mean[1] = ms / len;
  }
}

void pivot_to_estimate(const bb200_estimate& e, double pivot[2]) {
  if (!std::isfinite(e.mean[2]) || !std::isfinite(e.mean[3])) return;
  pivot[0] = e.mean[2];
  pivot[1] = e.mean[3];
}

}  // namespace bb200
