// Host-only probe of csrc/cluster_select.cuh, the order-defining half of the device cluster selection, against the real
// containers it restates (tests/test_cluster_select_cpu.py).  Built with g++ against libbeluga_b200 (select_cluster and the
// probed rehash schedules) and the oracle's clusterizer; needs no GPU.  Prints one summary line per check:
//   reserve <wants> <mismatches>                    every want's bucket count after reserve against its schedule's first entry
//   map <cases> <thresholds crossed> <mismatches>    iteration order against std::unordered_map<std::size_t, T>
//   select <cases> <tied cases> <mismatches> <oracle mismatches>
//   edge <headings> <flagged> <violations>          headings the fallback predicate lets through keep their bucket
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <unordered_map>
#include <vector>

#include "cluster_host.hpp"
#include "cluster_oracle.hpp"

using namespace bb200;

namespace {

std::vector<uint32_t> real_order(const std::vector<uint64_t>& hashes, uint32_t want) {
  std::unordered_map<std::size_t, uint32_t> map;
  map.reserve(want);
  for (uint32_t k = 0; k < hashes.size(); ++k) map.try_emplace(static_cast<std::size_t>(hashes[k]), k);
  std::vector<uint32_t> out;
  for (const auto& kv : map) out.push_back(kv.second);
  return out;
}

std::vector<uint32_t> emulated_order(const std::vector<uint64_t>& hashes, uint32_t want) {
  const RehashTable& t = rehash_table();
  const RehashStep* schedule = t.steps.data() + t.start[want];
  const uint32_t c = static_cast<uint32_t>(hashes.size());
  uint32_t max_buckets = 0;
  const int phases = rehash_phases(schedule, c, &max_buckets);
  std::vector<uint32_t> bkt(static_cast<size_t>(phases) * c), next(c + 1), before(max_buckets), order(c);
  for (int ph = 0; ph < phases; ++ph)
    for (uint32_t i = 0; i < c; ++i) bkt[static_cast<size_t>(ph) * c + i] = static_cast<uint32_t>(hashes[i] % schedule[ph].buckets);
  map_order(schedule, bkt.data(), c, next.data(), before.data(), order.data());
  return order;
}

struct Emulated {
  std::vector<uint32_t> cluster;
  SelectOutcome outcome;
};

/// select_cluster's inputs through the device path's stages, on the host.
Emulated emulate(const std::vector<HostCell>& cells, uint64_t n_particles, double linear, double angular, double percentile) {
  const uint32_t c = static_cast<uint32_t>(cells.size());
  std::vector<double> capped(c);
  for (uint32_t i = 0; i < c; ++i) capped[i] = cells[i].weight / static_cast<double>(cells[i].count);
  if (c > 0) {
    std::vector<double> values = capped;
    const auto nth = static_cast<std::ptrdiff_t>(static_cast<double>(c) * percentile);
    std::nth_element(values.begin(), values.begin() + nth, values.end());
    const double cap = values[static_cast<size_t>(nth)];
    for (double& w : capped) w = cap < w ? cap : w;
  }
  std::unordered_map<uint64_t, uint32_t> index;
  for (uint32_t i = 0; i < c; ++i) index[cells[i].hash] = i;
  const Rot2 zero = rot_exp(0.0), plus = rot_exp(+angular), minus = rot_exp(-angular);
  const Pose2 adjacent[6] = {Pose2{zero.c, zero.s, +linear, 0.0}, Pose2{zero.c, zero.s, -linear, 0.0}, Pose2{zero.c, zero.s, 0.0, +linear},
                             Pose2{zero.c, zero.s, 0.0, -linear}, Pose2{plus.c, plus.s, 0.0, 0.0},     Pose2{minus.c, minus.s, 0.0, 0.0}};
  std::vector<uint32_t> neighbors(6ull * c);
  for (uint32_t i = 0; i < c; ++i) {
    const double* r = cells[i].representative;
    for (int s = 0; s < 6; ++s) {
      const auto it = index.find(spatial_hash(pose_mul(Pose2{r[0], r[1], r[2], r[3]}, adjacent[s]), linear, linear, angular));
      neighbors[6ull * i + s] = it == index.end() ? kSelectNone : it->second;
    }
  }
  std::vector<uint64_t> hashes(c);
  for (uint32_t i = 0; i < c; ++i) hashes[i] = cells[i].hash;
  const std::vector<uint32_t> order = emulated_order(hashes, static_cast<uint32_t>(n_particles / 5));
  std::vector<SelectQueued> heap(2ull * c + 1);
  Emulated e;
  e.cluster.resize(c);
  e.outcome = select_in_order(cells.data(), c, order.data(), capped.data(), neighbors.data(), heap.data(), e.cluster.data());
  return e;
}

/// make_cluster_map's cells in first-occurrence order with raw moments about the origin; cell_of per particle.
std::vector<HostCell> cell_records(const std::vector<Pose2>& states, const std::vector<double>& weights, double linear, double angular,
                                   std::vector<uint32_t>* cell_of) {
  std::unordered_map<uint64_t, uint32_t> index;
  std::vector<HostCell> cells;
  cell_of->resize(states.size());
  for (size_t i = 0; i < states.size(); ++i) {
    const Pose2& s = states[i];
    const uint64_t h = spatial_hash(s, linear, linear, angular);
    auto [it, inserted] = index.try_emplace(h, static_cast<uint32_t>(cells.size()));
    if (inserted) {
      HostCell c{};
      c.representative[0] = s.c, c.representative[1] = s.s, c.representative[2] = s.x, c.representative[3] = s.y;
      c.hash = h;
      c.first_index = static_cast<unsigned>(i);
      cells.push_back(c);
    }
    HostCell& c = cells[it->second];
    const double w = weights[i];
    c.count += 1;
    c.weight += w;
    const double m[9] = {w, w * w, w * s.c, w * s.s, w * s.x, w * s.y, w * s.x * s.x, w * s.x * s.y, w * s.y * s.y};
    for (int j = 0; j < 9; ++j) c.moments[j] += m[j];
    (*cell_of)[i] = it->second;
  }
  return cells;
}

}  // namespace

int main() {
  std::mt19937_64 rng(20261016);
  const RehashTable& table = rehash_table();

  // reserve: every want's initial bucket count is its schedule's.
  {
    int mismatches = 0;
    for (uint32_t w = 0; w < table.start.size(); ++w) {
      std::unordered_map<std::size_t, double> map;
      map.reserve(w);
      if (map.bucket_count() != table.steps[table.start[w]].buckets) ++mismatches;
    }
    std::printf("reserve %zu %d\n", table.start.size(), mismatches);
  }

  // map: every distinct schedule, at its smallest and largest want, with cell counts on both sides of every threshold.
  {
    int cases = 0, crossed = 0, mismatches = 0;
    std::vector<uint32_t> lo(table.steps.size(), kSelectNone), hi(table.steps.size(), 0);
    for (uint32_t w = 0; w < table.start.size(); ++w) {
      lo[table.start[w]] = std::min(lo[table.start[w]], w);
      hi[table.start[w]] = std::max(hi[table.start[w]], w);
    }
    for (size_t s = 0; s < table.steps.size(); ++s) {
      if (lo[s] == kSelectNone) continue;
      for (const uint32_t want : {lo[s], hi[s]}) {
        const uint32_t most = static_cast<uint32_t>(std::min<uint64_t>(5ull * want + 4, kSelectMaxCells));
        std::vector<uint32_t> counts = {0, 1, most};
        for (size_t e = s + 1; table.steps[e].count != kSelectNone; ++e) {
          if (table.steps[e].count + 1 > most) continue;
          counts.push_back(table.steps[e].count);
          counts.push_back(table.steps[e].count + 1);
          ++crossed;
        }
        for (const uint32_t c : counts) {
          std::vector<uint64_t> hashes(c);
          for (uint64_t& h : hashes) h = rng();
          if (c > 2) hashes[2] = hashes[0] + (1 + rng() % 7) * table.steps[s].buckets;  // share a bucket with cell 0
          if (real_order(hashes, want) != emulated_order(hashes, want)) ++mismatches;
          ++cases;
        }
      }
    }
    std::printf("map %d %d %d\n", cases, crossed, mismatches);
  }

  // select: random particle sets whose capped cells tie, against select_cluster and the oracle's clusterizer.
  {
    int cases = 0, tied = 0, mismatches = 0, oracle_mismatches = 0;
    std::uniform_real_distribution<double> uni(0.0, 1.0);
    std::normal_distribution<double> normal(0.0, 1.0);
    const double resolutions[][2] = {{0.2, 0.524}, {0.05, 0.1}, {0.5, 1.0}, {1.0, 1.5707963267948966}, {0.1, 0.3}};
    const double percentiles[] = {0.9, 0.0, 0.5, 0.99, 0.75};
    for (int round = 0; round < 3000; ++round) {
      const uint64_t n = round % 500 == 499 ? 32768 : 1 + rng() % (round % 10 == 0 ? 6000 : 1500);
      const double* res = resolutions[rng() % 5];
      const double percentile = percentiles[rng() % 5];
      const int hypotheses = 1 + static_cast<int>(rng() % 4);
      const double spread = 0.05 + 2.0 * uni(rng), heading = 3.0 * uni(rng);
      std::vector<Pose2> states(n);
      std::vector<double> weights(n, 1.0);
      const int kind = static_cast<int>(rng() % 4);  // 0, 1: unit weights (every cell ties); 2: few distinct; 3: continuous
      double centre[4][2];
      for (auto& ctr : centre) ctr[0] = 10.0 * uni(rng), ctr[1] = 10.0 * uni(rng);
      for (uint64_t i = 0; i < n; ++i) {
        const int h = static_cast<int>(rng() % hypotheses);
        const double th = heading + (h + 1) * 0.7 + 0.3 * spread * normal(rng);
        const Rot2 r = rot_exp(th);
        states[i] = Pose2{r.c, r.s, centre[h][0] + spread * normal(rng), centre[h][1] + spread * normal(rng)};
        if (kind == 2) weights[i] = 0.25 * static_cast<double>(1 + rng() % 3);
        if (kind == 3) weights[i] = 0.1 + uni(rng);
      }
      std::vector<uint32_t> cell_of;
      const std::vector<HostCell> cells = cell_records(states, weights, res[0], res[1], &cell_of);
      const ClusterSelection want = select_cluster(cells.data(), cells.size(), n, res[0], res[1], percentile);
      const Emulated got = emulate(cells, n, res[0], res[1], percentile);
      bool same = want.clusters == got.outcome.clusters && want.found == (got.outcome.found != 0) &&
                  (!want.found || want.best == got.outcome.best) && std::memcmp(want.moments, got.outcome.moments, sizeof(want.moments)) == 0;
      for (size_t k = 0; k < cells.size() && same; ++k) same = want.cluster_of_cell[k] == got.cluster[k];
      mismatches += same ? 0 : 1;
      tied += kind < 3 && cells.size() > 2 ? 1 : 0;
      if (n <= 6000) {
        std::vector<oracle::SE2> os(n);
        for (uint64_t i = 0; i < n; ++i) os[i] = oracle::SE2(oracle::SO2::raw(states[i].c, states[i].s), states[i].x, states[i].y);
        const std::vector<std::size_t> ids = oracle::ParticleClusterizer{{res[0], res[1], percentile}}(os, weights);
        bool agree = true;
        for (uint64_t i = 0; i < n && agree; ++i) agree = ids[i] == got.cluster[cell_of[i]];
        oracle_mismatches += agree ? 0 : 1;
      }
      ++cases;
    }
    std::printf("select %d %d %d %d\n", cases, tied, mismatches, oracle_mismatches);
  }

  // edge: headings the predicate lets through keep their bucket when moved by the error it assumes.
  {
    int checked = 0, flagged = 0, violations = 0;
    std::uniform_real_distribution<double> uni(-3.141592653589793, 3.141592653589793);
    const double angulars[] = {0.524, 0.1, 1.5707963267948966, 0.01, 0.7853981633974483};
    for (int i = 0; i < 200000; ++i) {
      const double angular = angulars[i % 5];
      double th = uni(rng);
      if (i % 4 == 0) th = std::round(th / angular) * angular * (1.0 + (static_cast<double>(rng() % 65) - 32.0) * 0x1p-52);  // at an edge
      const Rot2 r = rot_exp(th);
      if (heading_near_bucket_edge(r.s, r.c, angular)) {
        ++flagged;
        continue;
      }
      const double t = std::atan2(r.s, r.c);
      const double b = std::floor(t / angular);
      for (const double e : {-kHeadingRelativeError, kHeadingRelativeError})
        if (std::floor((t * (1.0 + e)) / angular) != b) ++violations;
      ++checked;
    }
    std::printf("edge %d %d %d\n", checked, flagged, violations);
  }
  return 0;
}
