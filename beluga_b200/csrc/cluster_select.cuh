// The order-defining half of select_cluster (cluster_host.cpp), restated so that one thread of a CTA can run it on the
// device (batch_cluster_select_kernel) and the host can run the same code against the real containers (the CPU tests).
//
// select_cluster seeds a std::priority_queue from a std::unordered_map's iteration order, and after the percentile cap
// many cells weigh the same: which of them is popped first is decided by libstdc++'s containers alone.  So this restates
//  - the iteration order of std::unordered_map<std::size_t, T> (identity hash, bucket = key % buckets) after reserve and
//    one insertion per cell, rehashes included: a node goes to the front of its bucket, and a bucket that becomes
//    non-empty goes to the front of the list; a rehash relinks the nodes, in iteration order, by the same rule.  The
//    bucket counts come from the running libstdc++ (rehash_schedule(), probed on the host), never from a copied table;
//  - std::make_heap / push_heap / pop_heap (bits/stl_heap.h: hole descent, then sift-up) under operator< on the priority;
//  - the flood (cluster ids in pop order), the per-cluster sums in ascending cell order, the first strictly heaviest
//    cluster with more than one particle and its moments (or those of every cell).
#pragma once

#include <cstdint>

#include "se2_math.cuh"

namespace bb200 {

constexpr uint32_t kSelectNone = 0xffffffffu;

/// One entry of a map's bucket-count schedule: inserting a cell while `count` cells are in the map first rehashes it to
/// `buckets` buckets.  A schedule starts with {0, buckets after reserve} and ends with {kSelectNone, 0}.
struct RehashStep {
  uint32_t count;
  uint32_t buckets;
};
/// Largest cell count the schedules cover (a batch member's largest particle count).
constexpr uint32_t kSelectMaxCells = 32768;

/// KeyWithPriority of cluster_based_estimation.hpp:75-82, with the cell index standing for its key.
struct SelectQueued {
  double priority;
  uint32_t cell;
  uint32_t pad;
};

// ---- std::priority_queue<Queued> (libstdc++ bits/stl_heap.h) ---------------------------------------------------------

/// std::__push_heap
BB_HD void heap_sift_up(SelectQueued* first, int64_t hole, int64_t top, const SelectQueued value) {
  int64_t parent = (hole - 1) / 2;
  while (hole > top && first[parent].priority < value.priority) {
    first[hole] = first[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  first[hole] = value;
}
/// std::__adjust_heap
BB_HD void heap_adjust(SelectQueued* first, int64_t hole, int64_t len, const SelectQueued value) {
  const int64_t top = hole;
  int64_t child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (first[child].priority < first[child - 1].priority) child--;
    first[hole] = first[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    first[hole] = first[child - 1];
    hole = child - 1;
  }
  heap_sift_up(first, hole, top, value);
}
/// std::make_heap
BB_HD void heap_make(SelectQueued* first, int64_t len) {
  if (len < 2) return;
  for (int64_t parent = (len - 2) / 2;; --parent) {
    heap_adjust(first, parent, len, first[parent]);
    if (parent == 0) return;
  }
}
/// std::push_heap over [first, first + len) (the new element is the last)
BB_HD void heap_push(SelectQueued* first, int64_t len) { heap_sift_up(first, len - 1, 0, first[len - 1]); }
/// std::pop_heap over [first, first + len)
BB_HD void heap_pop(SelectQueued* first, int64_t len) {
  if (len < 2) return;
  const SelectQueued value = first[len - 1];
  first[len - 1] = first[0];
  heap_adjust(first, 0, len - 1, value);
}

// ---- std::unordered_map<std::size_t, T> iteration order ---------------------------------------------------------------

/// The phases a map of `cells` cells passes through under `schedule`: 1 + the rehashes on the way; *max_buckets receives the
/// largest bucket count among them.
BB_HD int rehash_phases(const RehashStep* schedule, uint32_t cells, uint32_t* max_buckets) {
  int phases = 1;
  uint32_t top = schedule[0].buckets;
  while (schedule[phases].count != kSelectNone && schedule[phases].count < cells) {
    top = schedule[phases].buckets > top ? schedule[phases].buckets : top;
    ++phases;
  }
  *max_buckets = top;
  return phases;
}

/// _M_insert_bucket_begin, and the relinking of _M_rehash_aux: node `p` goes to the front of its bucket `bkt[p]`, or, when
/// that bucket is empty, to the front of the list.  next[c] is the list head (_M_before_begin); before[b] is the node
/// before bucket b's first node (or the head), kSelectNone while b is empty.
BB_HD void map_link(uint32_t p, uint32_t head, const uint32_t* bkt, uint32_t* next, uint32_t* before) {
  const uint32_t b = bkt[p];
  if (before[b] != kSelectNone) {
    next[p] = next[before[b]];
    next[before[b]] = p;
  } else {
    next[p] = next[head];
    next[head] = p;
    if (next[p] != kSelectNone) before[bkt[next[p]]] = p;
    before[b] = head;
  }
}

/// The iteration order of the map after reserve and the insertion of cells 0 .. c-1 (keyed by their hashes) into order[].
/// bkt holds one row of c bucket indices per phase (hash % buckets of that phase); next has c + 1 entries, before as many
/// as the largest bucket count of the phases.
BB_HD void map_order(const RehashStep* schedule, const uint32_t* bkt, uint32_t c, uint32_t* next, uint32_t* before, uint32_t* order) {
  const uint32_t head = c;
  next[head] = kSelectNone;
  for (uint32_t b = 0; b < schedule[0].buckets; ++b) before[b] = kSelectNone;
  int phase = 0;
  for (uint32_t k = 0; k < c; ++k) {
    if (schedule[phase + 1].count == k) {  // _M_need_rehash before this insertion
      ++phase;
      bkt += c;
      for (uint32_t b = 0; b < schedule[phase].buckets; ++b) before[b] = kSelectNone;
      uint32_t p = next[head];
      next[head] = kSelectNone;
      while (p != kSelectNone) {
        const uint32_t after = next[p];
        map_link(p, head, bkt, next, before);
        p = after;
      }
    }
    map_link(k, head, bkt, next, before);
  }
  uint32_t i = 0;
  for (uint32_t p = next[head]; p != kSelectNone; p = next[p]) order[i++] = p;
}

// ---- one member's scratch -------------------------------------------------------------------------------------------

/// Byte offsets of the arrays of one member's selection over c cells (16-byte aligned), and their total.
struct SelectLayout {
  uint64_t heap, capped, neighbors, bkt, next, before, order, cluster, bytes;
};
BB_HD SelectLayout select_layout(uint32_t c, int phases, uint32_t max_buckets) {
  SelectLayout l{};
  uint64_t at = 0;
  auto take = [&at](uint64_t bytes) {
    const uint64_t p = at;
    at += (bytes + 15) / 16 * 16;
    return p;
  };
  l.heap = take(2ull * c * sizeof(SelectQueued));
  l.capped = take(8ull * c);
  l.neighbors = take(24ull * c);
  l.bkt = take(4ull * c * static_cast<uint64_t>(phases));
  l.next = take(4ull * (c + 1ull));
  l.before = take(4ull * max_buckets);
  l.order = take(4ull * c);
  l.cluster = take(4ull * c);
  l.bytes = at;
  return l;
}

// ---- the flood and the selection ------------------------------------------------------------------------------------

struct SelectOutcome {
  uint32_t clusters;
  uint32_t found;
  uint32_t best;
  double moments[9];
};

/// assign_clusters (:205-253) and cluster_based_estimate's selection (:351-432) over c cells: order is the map's iteration
/// order, capped the normalised and capped cell weights, neighbors six cell indices per cell (kSelectNone: no such cell).
/// heap holds 2 c entries; cluster receives the cluster id of every cell.  Cell is HostCell or CellRecord.
template <class Cell>
BB_HD SelectOutcome select_in_order(const Cell* cells, uint32_t c, const uint32_t* order, const double* capped, const uint32_t* neighbors,
                                    SelectQueued* heap, uint32_t* cluster) {
  SelectOutcome out{};
  for (uint32_t i = 0; i < c; ++i) {
    heap[i] = SelectQueued{capped[order[i]], order[i], 0};
    cluster[i] = kSelectNone;
  }
  heap_make(heap, c);
  int64_t len = c;
  const double max_priority = c > 0 ? heap[0].priority : 0.0;
  uint32_t next_cluster = 0;
  while (len > 0) {
    const uint32_t cell = heap[0].cell;
    heap_pop(heap, len);
    --len;
    if (cluster[cell] == kSelectNone) cluster[cell] = next_cluster++;
    const double weight = capped[cell];
    for (int s = 0; s < 6; ++s) {
      const uint32_t nb = neighbors[6 * static_cast<uint64_t>(cell) + s];
      if (nb == kSelectNone || cluster[nb] != kSelectNone || !(capped[nb] <= weight)) continue;
      cluster[nb] = cluster[cell];
      heap[len] = SelectQueued{max_priority + capped[nb], nb, 0};
      ++len;
      heap_push(heap, len);
    }
  }
  out.clusters = next_cluster;
  // Per-cluster particle counts and weight sums, cells in ascending order (the heap's room is free again).
  uint64_t* count = reinterpret_cast<uint64_t*>(heap);
  double* sum = reinterpret_cast<double*>(heap) + c;
  for (uint32_t k = 0; k < next_cluster; ++k) {
    count[k] = 0;
    sum[k] = 0.0;
  }
  for (uint32_t k = 0; k < c; ++k) {
    count[cluster[k]] += cells[k].count;
    sum[cluster[k]] += cells[k].moments[0];
  }
  for (uint32_t k = 0; k < next_cluster; ++k) {
    if (count[k] <= 1) continue;
    if (!out.found || sum[out.best] < sum[k]) {
      out.best = k;
      out.found = 1;
    }
  }
  for (int j = 0; j < 9; ++j) out.moments[j] = 0.0;
  for (uint32_t k = 0; k < c; ++k) {
    if (out.found && cluster[k] != out.best) continue;
    for (int j = 0; j < 9; ++j) out.moments[j] += cells[k].moments[j];
  }
  return out;
}

// ---- where the device's heading may differ from glibc's ---------------------------------------------------------------

/// Relative error of a neighbour's heading atan2(s, c) on the device against glibc's that the check below allows for.  The
/// CUDA math library documents 2 ulp for hypot and for atan2 (double); the neighbour's (c, s) are divided by the hypot and
/// then enter atan2, which with glibc's own sub-ulp rounding stays below 16 ulp = 2^-48.  The predicate keeps a margin of
/// 2^8 on top of that.
constexpr double kHeadingRelativeError = 0x1p-48;
constexpr double kHeadingMargin = 0x1p-40;

/// Whether the angular bucket floor(atan2(s, c) / angular) of a heading could change under that error: the quotient lies
/// within kHeadingMargin (relative) of an integer.  A heading with s == 0 is exact on both sides and never flagged.
BB_HD bool heading_near_bucket_edge(double s, double c, double angular) {
  if (s == 0.0) return false;
  const double t = atan2(s, c) / angular;
  const double f = floor(t);
  const double gap = fmin(t - f, (f + 1.0) - t);
  return !(gap > kHeadingMargin * fabs(t));
}

}  // namespace bb200
