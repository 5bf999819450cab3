#include "device_map.hpp"

#include <cmath>
#include <cstring>

#include "map_host.hpp"

namespace bb200 {

namespace {

Pose2 pose_from_array(const double* d) { return Pose2{d[0], d[1], d[2], d[3]}; }

/// Checks the grid and fills in what every sensor model has: the geometry and the free cells.
int prepare_grid(const bb200_occupancy_grid& g, MapTables* t, std::string* error) {
  if (g.cells == nullptr || g.width <= 0 || g.height <= 0 || !(g.resolution > 0.0)) return reject(BB200_ERR_INVALID_ARGUMENT, "invalid occupancy grid", error);
  *t = MapTables{};
  t->free_cells = make_free_cells(g);
  t->n_free = t->free_cells.size();
  t->grid_width = g.width;
  t->grid_height = g.height;
  t->grid_resolution = g.resolution;
  t->grid_origin = pose_from_array(g.origin);
  return BB200_OK;
}

}  // namespace

int prepare_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& g, bool prob, MapTables* t, std::string* error) {
  const int st = prepare_grid(g, t, error);
  if (st != BB200_OK) return st;
  if (!(p.sigma_hit > 0.0) || !(p.max_laser_distance > 0.0)) return reject(BB200_ERR_INVALID_ARGUMENT, "invalid likelihood field parameters", error);
  const char* too_large = "map too large for 32-bit cell indices";
  t->field_host = make_likelihood_field(p, g);
  t->ray_grid.assign(g.cells, g.cells + static_cast<size_t>(g.width) * static_cast<size_t>(g.height));
  const size_t count = t->field_host.size();
  if (count + 64 >= (1ull << 32)) return reject(BB200_ERR_CAPACITY, too_large, error);
  // The lookup table the reweight kernel gathers from: f(pz) per cell as double, f = pz^3 (LikelihoodFieldModel) or
  // log pz (LikelihoodFieldProbModel).  f is a pure function of the float cell value, so tabulating it is bit-identical to
  // evaluating it per beam as likelihood_field_model.hpp:84-89 / likelihood_field_prob_model.hpp:84-86 do.
  std::vector<double> table(count);  // row-major: the source of the layout the map's kernel reads
  auto f = [prob](float pzf) {
    const double pz = static_cast<double>(pzf);
    return prob ? std::log(pz) : pz * pz * pz;
  };
  for (size_t i = 0; i < count; ++i) table[i] = f(t->field_host[i]);
  const double unknown = f(static_cast<float>(1. / p.max_laser_distance));  // what out-of-grid end points read
  FieldView& v = t->field;
  if (g.width + 2 <= kFixedMaxSide && g.height + 2 <= kFixedMaxSide) {
    // Bordered tile layout for the fixed-point kernel.
    int kx = 0;
    while ((1 << kx) < (g.width + 2 + 3) / 4) ++kx;
    const size_t tile_rows = static_cast<size_t>((g.height + 2 + 3) / 4);
    t->bordered.assign(tile_rows << (kx + 4), unknown);
    for (int yi = 0; yi < g.height; ++yi)
      for (int xi = 0; xi < g.width; ++xi)
        t->bordered[bordered_index(static_cast<uint32_t>(xi + 1), static_cast<uint32_t>(yi + 1), kx)] = table[static_cast<size_t>(yi) * g.width + xi];
    v.border_kx = kx;
    v.border_pitch = 1u << kx;
    v.border_x_max = static_cast<uint32_t>(4 * (g.width + 1) + 3);
    v.border_y_max = static_cast<uint32_t>(g.height + 1);
    v.use_fixed = 1;
    t->bordered_bytes = t->bordered.size() * sizeof(double);
  } else {
    // Tiled layout (4x4-cell tiles, no border, spare cell at the end) for the general kernel.
    const int tiles_x = (g.width + 3) / 4, tiles_y = (g.height + 3) / 4;
    if (static_cast<size_t>(tiles_x) * tiles_y * 16 + 64 >= (1ull << 32)) return reject(BB200_ERR_CAPACITY, too_large, error);
    t->tiled.assign(static_cast<size_t>(tiles_x) * tiles_y * 16 + 1, unknown);
    for (int yi = 0; yi < g.height; ++yi)
      for (int xi = 0; xi < g.width; ++xi) t->tiled[tiled_index(xi, yi, tiles_x)] = table[static_cast<size_t>(yi) * g.width + xi];
    v.tiles_x = tiles_x;
    v.spare_index = static_cast<uint32_t>(t->tiled.size() - 1);
  }
  v.width = g.width;
  v.height = g.height;
  v.inv_resolution = 1. / g.resolution;
  v.unknown_value = unknown;
  v.init = prob ? 0.0 : 1.0;
  v.exp_epilogue = prob ? 1 : 0;
  v.world_to_field = pose_inverse(pose_from_array(g.origin));
  t->sensor = prob ? BB200_SENSOR_LIKELIHOOD_FIELD_PROB : BB200_SENSOR_LIKELIHOOD_FIELD;
  return BB200_OK;
}

int prepare_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& g, MapTables* t, std::string* error) {
  const int st = prepare_grid(g, t, error);
  if (st != BB200_OK) return st;
  t->cells.assign(g.cells, g.cells + static_cast<size_t>(g.width) * static_cast<size_t>(g.height));
  t->free_distance = make_free_distance(g);
  OccupancyView& v = t->occupancy;
  // padded copy for the two-pass walk: a border of zeros, power-of-two pitch
  int shift = 1;
  while ((1 << shift) < g.width + 2) ++shift;
  if (shift <= 16 && g.height <= 65535) {
    t->free_padded.assign((static_cast<size_t>(g.height) + 2) << shift, 0);
    for (int y = 0; y < g.height; ++y)
      std::memcpy(t->free_padded.data() + ((static_cast<size_t>(y) + 1) << shift) + 1, t->free_distance.data() + static_cast<size_t>(y) * g.width,
                  static_cast<size_t>(g.width));
    v.pad_shift = shift;
  }
  v.width = g.width;
  v.height = g.height;
  v.resolution = g.resolution;
  v.inv_resolution = 1. / g.resolution;
  v.world_to_grid = pose_inverse(pose_from_array(g.origin));
  t->beam = BeamParams{p.z_hit, p.z_short, p.z_max, p.z_rand, p.sigma_hit, p.lambda_short, p.beam_max_range, nullptr, 0};
  t->sensor = BB200_SENSOR_BEAM;
  return BB200_OK;
}

bool beam_two_pass_map(const MapLayout& map) {
  // spans of the walk's 32-bit arithmetic: far ends lie within beam_max_range of the source, sources inside the grid
  const double reach_cells = map.beam.beam_max_range * map.occupancy.inv_resolution + 4.0;
  return map.occupancy.free_padded != nullptr && reach_cells < static_cast<double>(1 << 21);
}

// ---------------------------------------------------------------------------------------------------

void DeviceMap::release() {
  tables_ = Tables{};
  ray_ = RayTables{};
  static_cast<MapLayout&>(*this) = MapLayout{};
  field_host.clear();
  free_cells = nullptr;
  landmark_slices.clear();
}

template <class T>
cudaError_t DeviceMap::copy(const std::vector<T>& v, DeviceBuffer<T>* table, const T** view, cudaStream_t stream) {
  *view = nullptr;
  if (v.empty()) return cudaSuccess;
  if (const cudaError_t e = table->allocate(v.size())) return e;
  *view = table->get();
  return cudaMemcpyAsync(table->get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, stream);
}

int DeviceMap::upload(const MapTables& t, cudaStream_t stream, std::string* error) {
  auto check = [error](cudaError_t e, const char* what) { return cuda_check(e, what, error); };
  BB_CHECK(cudaStreamSynchronize(stream));  // nothing in flight reads the old tables any more
  release();
  static_cast<MapLayout&>(*this) = t;
  sensor = -1;  // until every table is in place
  BB_CHECK(copy(t.bordered, &tables_.bordered, &field.bordered, stream));
  if (field.bordered != nullptr) {
    // The biased index of element e is e + bias modulo 2^32; it equals e + bias, and the moved-back base then finds the
    // element, only if no element's biased index passes 2^32.
    const uint32_t bias = fixed_index_bias(field.border_pitch);
    if (static_cast<uint64_t>(bias) + t.bordered.size() <= (1ull << 32))
      field.bordered_biased = reinterpret_cast<const double*>(reinterpret_cast<uintptr_t>(field.bordered) - uintptr_t{bias} * sizeof(double));
  }
  BB_CHECK(copy(t.tiled, &tables_.tiled, &field.tiled, stream));
  BB_CHECK(copy(t.cells, &tables_.cells, &occupancy.cells, stream));
  BB_CHECK(copy(t.free_distance, &tables_.free_distance, &occupancy.free_distance, stream));
  BB_CHECK(copy(t.free_padded, &tables_.free_padded, &occupancy.free_padded, stream));
  BB_CHECK(copy(t.free_cells, &tables_.free_cells, &free_cells, stream));
  BB_CHECK(copy(t.landmark_points, &tables_.landmarks, &landmarks, stream));
  if (t.sensor == BB200_SENSOR_BEAM) {
    if (const uint32_t entries = beam_eta_entries(beam.beam_max_range, grid_resolution)) {
      BB_CHECK(tables_.eta.allocate(entries));
      launch_beam_eta_table(beam, grid_resolution, tables_.eta.get(), entries, stream);
      BB_LAUNCHED("beam_eta_table");
      beam.eta = tables_.eta.get();
      beam.eta_entries = entries;
    }
  }
  BB_CHECK(cudaStreamSynchronize(stream));  // the host tables may go once this returns
  field_host = t.field_host;
  landmark_slices = t.landmark_slices;
  ray_.grid = t.ray_grid;
  sensor = t.sensor;
  return BB200_OK;
}

int DeviceMap::ray_view(cudaStream_t stream, OccupancyView* view, std::string* error) {
  auto check = [error](cudaError_t e, const char* what) { return cuda_check(e, what, error); };
  if (sensor < 0) return reject(BB200_ERR_STATE, "no map", error);
  if (landmark_map()) return reject(BB200_ERR_STATE, "a landmark map has no grid to cast rays on", error);
  if (sensor == BB200_SENSOR_BEAM) {
    *view = occupancy;
    return BB200_OK;
  }
  if (ray_.free_distance.get() == nullptr) {
    const bb200_occupancy_grid g{ray_.grid.data(), grid_width, grid_height, grid_resolution, {grid_origin.c, grid_origin.s, grid_origin.x, grid_origin.y}};
    const std::vector<uint8_t> free_distance = make_free_distance(g);
    DeviceBuffer<uint8_t> table;
    BB_CHECK(table.allocate(free_distance.size()));
    // pageable source: staged before the call returns, and the launch that reads the table follows the copy on `stream`
    BB_CHECK(cudaMemcpyAsync(table.get(), free_distance.data(), free_distance.size(), cudaMemcpyHostToDevice, stream));
    OccupancyView& v = ray_.view;
    v = OccupancyView{};
    v.free_distance = table.get();
    v.width = grid_width;
    v.height = grid_height;
    v.resolution = grid_resolution;
    v.inv_resolution = 1. / grid_resolution;
    v.world_to_grid = pose_inverse(grid_origin);
    ray_.free_distance = std::move(table);
    ray_.grid = std::vector<int8_t>{};  // the table is made from it once
  }
  *view = ray_.view;
  return BB200_OK;
}

void DeviceMap::centre(double pivot[2]) const {
  if (landmark_map()) {
    pivot[0] = 0.5 * (box[0] + box[1]);
    pivot[1] = 0.5 * (box[2] + box[3]);
    return;
  }
  const double cx = 0.5 * grid_width * grid_resolution, cy = 0.5 * grid_height * grid_resolution;
  pivot[0] = (grid_origin.c * cx - grid_origin.s * cy) + grid_origin.x;
  pivot[1] = (grid_origin.s * cx + grid_origin.c * cy) + grid_origin.y;
}

}  // namespace bb200
