// Prints the offset of every field of BatchStepArgs and BatchMap that the batch kernels read, and both sizes: the batch
// kernels take BatchStepArgs as their parameter block and index BatchMap tables, so a field that moves changes their code.
#include <cstddef>
#include <cstdio>

#include "kernels.cuh"

#define FIELD(T, f) std::printf("%s.%s %zu\n", #T, #f, offsetof(bb200::T, f))

int main() {
  FIELD(BatchStepArgs, members);
  FIELD(BatchStepArgs, first);
  FIELD(BatchStepArgs, n_members);
  FIELD(BatchStepArgs, ctas);
  FIELD(BatchStepArgs, max_points);
  FIELD(BatchStepArgs, states);
  FIELD(BatchStepArgs, weights);
  FIELD(BatchStepArgs, cdf);
  FIELD(BatchStepArgs, ancestors);
  FIELD(BatchStepArgs, tile_state);
  FIELD(BatchStepArgs, scalars);
  FIELD(BatchStepArgs, partials);
  FIELD(BatchStepArgs, points);
  FIELD(BatchStepArgs, field);
  FIELD(BatchStepArgs, free_cells);
  FIELD(BatchStepArgs, n_free);
  FIELD(BatchStepArgs, grid_width);
  FIELD(BatchStepArgs, grid_resolution);
  FIELD(BatchStepArgs, grid_origin);
  FIELD(BatchStepArgs, summary);
  FIELD(BatchStepArgs, members_done);
  FIELD(BatchStepArgs, ticket);
  FIELD(BatchStepArgs, seq);
  FIELD(BatchStepArgs, forms);
  FIELD(BatchStepArgs, occupancy);
  FIELD(BatchStepArgs, beam);
  FIELD(BatchStepArgs, hits);
  FIELD(BatchStepArgs, maps);
  FIELD(BatchStepArgs, kld);
  FIELD(BatchStepArgs, hashes);
  FIELD(BatchStepArgs, keys);
  FIELD(BatchStepArgs, vals);
  FIELD(BatchStepArgs, post_ctas);
  FIELD(BatchStepArgs, ess_ctas);
  FIELD(BatchStepArgs, weigh_ctas);
  FIELD(BatchStepArgs, factors);
  FIELD(BatchMap, field);
  FIELD(BatchMap, occupancy);
  FIELD(BatchMap, beam);
  FIELD(BatchMap, free_cells);
  FIELD(BatchMap, n_free);
  FIELD(BatchMap, grid_width);
  FIELD(BatchMap, grid_resolution);
  FIELD(BatchMap, grid_origin);
  FIELD(BatchMember, hit_stride);
  std::printf("sizeof.BatchStepArgs %zu\nsizeof.BatchMap %zu\nsizeof.BatchMember %zu\n", sizeof(bb200::BatchStepArgs), sizeof(bb200::BatchMap),
              sizeof(bb200::BatchMember));
  return 0;
}
