// The map a sensor model reads, in two halves: MapTables, prepared on the host once per map without touching a device,
// and DeviceMap, one device's copy of those tables.  A filter holds one DeviceMap, a batch holds one for all its members,
// and a sharded filter prepares the tables once and uploads them to every shard.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "device_buffer.hpp"
#include "kernels.cuh"
#include "reweight_landmark.cuh"

namespace bb200 {

/// What the kernels are handed: the sensor model, its views and the grid geometry.  The views' device pointers are null
/// in MapTables and set in DeviceMap.
struct MapLayout {
  int sensor{-1};  // -1: no map yet
  FieldView field{};
  OccupancyView occupancy{};
  BeamParams beam{};
  int grid_width{0}, grid_height{0};
  double grid_resolution{1.0};
  Pose2 grid_origin{1.0, 0.0, 0.0, 0.0};
  uint64_t n_free{0};          // free cells
  uint64_t bordered_bytes{0};  // size of the bordered table
  LandmarkParams landmark{};   // landmark and bearing models: the model constants ...
  const LandmarkPoint* landmarks{nullptr};  // ... and the landmarks sorted by category (no grid)
  uint32_t n_landmarks{0};
  double box[4]{0.0, 0.0, 0.0, 0.0};  // landmark maps: the bounds' {min_x, max_x, min_y, max_y}, the random states' box ...
  bool box_valid{false};              // ... when it is finite and not empty
  /// Whether initialize_from_map and recovery injection can draw states: free cells, or a landmark map's box.
  bool can_draw_states() const { return (sensor == BB200_SENSOR_LANDMARK || sensor == BB200_SENSOR_BEARING) ? box_valid : n_free > 0; }
};

/// The landmarks of one category: [begin, end) of the category-sorted map.
struct LandmarkSlice {
  uint32_t category, begin, end;
};

/// Everything the device copy of a map is made from.
struct MapTables : MapLayout {
  std::vector<float> field_host;  // likelihood field (get_likelihood_field); empty for the beam model
  std::vector<double> bordered;   // f(pz) in the bordered layout of the fixed-point kernel (maps up to kFixedMaxSide) ...
  std::vector<double> tiled;      // ... or in the tiled layout of the general kernel
  std::vector<int8_t> cells;      // beam model: the grid, its free distance and the padded copy of that
  std::vector<uint8_t> free_distance;
  std::vector<uint8_t> free_padded;
  std::vector<uint32_t> free_cells;  // recovery injection and initialize_from_map
  std::vector<int8_t> ray_grid;      // likelihood-field models: the grid, kept for ray casts (DeviceMap::ray_view)
  std::vector<LandmarkPoint> landmark_points;  // landmark maps: the landmarks stably sorted by category ...
  std::vector<LandmarkSlice> landmark_slices;  // ... and one slice per category, by category
};

/// Host preparation of a likelihood-field map (LikelihoodFieldModel, or LikelihoodFieldProbModel when prob).  Returns a
/// bb200_status; on failure *error holds the message.
int prepare_likelihood_field_map(const bb200_likelihood_field_param& p, const bb200_occupancy_grid& grid, bool prob, MapTables* out,
                                 std::string* error);
/// Host preparation of a beam-model map.
int prepare_beam_map(const bb200_beam_param& p, const bb200_occupancy_grid& grid, MapTables* out, std::string* error);
/// Host preparation of a landmark map for LandmarkSensorModel2d (lp) or, with lp null, BearingSensorModel2d (bp).
int prepare_landmark_map(const bb200_landmark_param* lp, const bb200_bearing_param* bp, const bb200_landmark_map& map, MapTables* out,
                         std::string* error);
/// The particle-independent part of a step's detections: range, unit vector and the candidate slice of each.
void prepare_detections(const std::vector<LandmarkSlice>& slices, const bb200_landmark_detection* in, uint64_t n, std::vector<LandmarkDetection>* out);
/// w *= the landmark or bearing model's likelihood (params.model) over n_detections prepared detections; the largest
/// weight into the device scalars.
void launch_reweight_landmark(const Pose2* states, double* weights, uint64_t n, const LandmarkParams& params, const LandmarkPoint* landmarks,
                              const LandmarkDetection* detections, uint32_t n_detections, Scalars* scalars, cudaStream_t stream);
/// Whether the beam model's two-pass walk can take this map: it has the padded free-distance copy (grids up to 65534
/// cells wide and 65535 high) and its rays stay short enough for the walk's 32-bit span arithmetic.  Filter and Batch both decide by it.
bool beam_two_pass_map(const MapLayout& map);

/// One device's copy of the current map.
struct DeviceMap : MapLayout {
  DeviceMap() = default;
  DeviceMap(const DeviceMap&) = delete;
  DeviceMap& operator=(const DeviceMap&) = delete;

  /// Replaces the map with `t` on the current device: waits for `stream`, copies the tables and, for the beam model,
  /// builds the normaliser table there.  Returns a bb200_status; on failure *error holds the message.
  int upload(const MapTables& t, cudaStream_t stream, std::string* error);
  /// The middle of the map in the global frame: the pivot of the raw moments after initialize_from_map.
  void centre(double pivot[2]) const;
  uint64_t launches() const { return launches_; }  // the beam model's normaliser tables
  /// The occupancy view ray casts walk (raycast.cuh): the beam model's own, or, for a likelihood-field map, one made the
  /// first time it is asked for: the free-distance map is built on the host from the grid kept at upload and copied on
  /// `stream`, with no launch.  BB200_ERR_STATE without a map.
  int ray_view(cudaStream_t stream, OccupancyView* view, std::string* error);

  bool landmark_map() const { return sensor == BB200_SENSOR_LANDMARK || sensor == BB200_SENSOR_BEARING; }

  std::vector<float> field_host;
  const uint32_t* free_cells{nullptr};
  std::vector<LandmarkSlice> landmark_slices;

 private:
  void release();
  template <class T>
  cudaError_t copy(const std::vector<T>& v, DeviceBuffer<T>* table, const T** view, cudaStream_t stream);

  struct Tables {  // the device tables of the current map, one per view (an empty host table leaves both null)
    DeviceBuffer<double> bordered, tiled;
    DeviceBuffer<int8_t> cells;
    DeviceBuffer<uint8_t> free_distance, free_padded;
    DeviceBuffer<uint32_t> free_cells;
    DeviceBuffer<double2> eta;  // beam model: normaliser table
    DeviceBuffer<LandmarkPoint> landmarks;
  };
  Tables tables_;
  // Ray casts on a likelihood-field map, apart from tables_ so that upload copies exactly what the sensor model reads: the
  // grid until the first cast, then the free-distance map on the device and its view.
  struct RayTables {
    std::vector<int8_t> grid;
    DeviceBuffer<uint8_t> free_distance;
    OccupancyView view{};
  };
  RayTables ray_;
  uint64_t launches_{0};
};

}  // namespace bb200
