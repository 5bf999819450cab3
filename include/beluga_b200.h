/*
 * beluga_b200 -- C ABI of the CUDA-native (H100, sm_90a) MCL particle-filter update.
 *
 * This is the drop-in boundary for ONE path of Ekumen-OS/beluga: the per-step
 * particle-filter update `beluga::Amcl::update`
 * (beluga/include/beluga/algorithm/amcl_core.hpp:165-201) and the models, actions, views and
 * reductions it composes.  The reference is a header-only C++17 template library without any
 * FFI; the C++ adaptors in include/beluga_b200/ give these entry points the reference's own
 * MotionModel / SensorModel / Amcl shapes (see INTEGRATION.md).  Each entry point cites the
 * reference interface it replaces (paths relative to /root/reference/beluga/include/beluga).
 *
 * Conventions
 *   - Poses are `double[4]` in Sophus::SE2d::data() order {cos, sin, x, y}
 *     (what estimation.hpp:448-452 relies on); particle states are arrays of such quadruples.
 *   - Every function returns BB200_OK (0) or a negative bb200_status; bb200_last_error() gives
 *     the message of the last failure on that context.  Nothing throws across this boundary.
 *   - All pointers are HOST pointers unless the name says `_device`.  A context owns its
 *     device buffers and one CUDA stream; calls on one context must come from one thread at a
 *     time (same contract as the reference: no internal locking, amcl_node.cpp:581-603).
 *   - There is NO CPU fallback: creating a context without a usable CUDA device fails.
 */
#ifndef BELUGA_B200_H_
#define BELUGA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BB200_ABI_VERSION 2

typedef enum bb200_status {
  BB200_OK = 0,
  BB200_ERR_INVALID_ARGUMENT = -1,
  BB200_ERR_CUDA = -2,
  BB200_ERR_NO_DEVICE = -3,
  BB200_ERR_STATE = -4, /* call sequence error: no map, no particles, ... */
  BB200_ERR_CAPACITY = -5
} bb200_status;

typedef struct bb200_filter bb200_filter; /* device-resident particle set + kernels        */
typedef struct bb200_amcl bb200_amcl;     /* beluga::Amcl control flow on top of a filter   */

/* ---------------------------------------------------------------------------------------------
 * Parameter blocks (plain doubles/ints; same members and defaults as the reference structs)
 * ------------------------------------------------------------------------------------------- */

/* beluga::DifferentialDriveModelParam -- motion/differential_drive_model.hpp:40-68 */
typedef struct bb200_diff_drive_param {
  double rotation_noise_from_rotation;       /* alpha1 */
  double rotation_noise_from_translation;    /* alpha2 */
  double translation_noise_from_translation; /* alpha3 */
  double translation_noise_from_rotation;    /* alpha4 */
  double distance_threshold;                 /* default 0.01 */
} bb200_diff_drive_param;

/* The three std::normal_distribution parameter sets that sampling_fn_2d derives from a control
 * action -- motion/differential_drive_model.hpp:141-154. */
typedef struct bb200_diff_drive_sampling {
  double rot1_mean, rot1_std;
  double trans_mean, trans_std;
  double rot2_mean, rot2_std;
} bb200_diff_drive_sampling;

/* The motion models of beluga_ros::Amcl::motion_model_variant (beluga_ros/include/beluga_ros/amcl.hpp:108-111). */
typedef enum bb200_motion_model {
  BB200_MOTION_DIFFERENTIAL = 0,    /* motion/differential_drive_model.hpp */
  BB200_MOTION_OMNIDIRECTIONAL = 1, /* motion/omnidirectional_drive_model.hpp */
  BB200_MOTION_STATIONARY = 2       /* motion/stationary_model.hpp */
} bb200_motion_model;

/* DifferentialDriveModelParam / OmnidirectionalDriveModelParam (omnidirectional_drive_model.hpp:36-68)
 * in one block; strafe_noise_from_translation is only read by the omnidirectional model. */
typedef struct bb200_motion_param {
  int model; /* bb200_motion_model */
  double rotation_noise_from_rotation;
  double rotation_noise_from_translation;
  double translation_noise_from_translation;
  double translation_noise_from_rotation;
  double strafe_noise_from_translation;
  double distance_threshold; /* default 0.01 */
} bb200_motion_param;

/* What a motion model derives from one control action: three normal distributions, drawn per
 * particle in this order, and (omnidirectional only) the deterministic first rotation.
 *   differential:     (rot1, trans, rot2)            state * SE2(rot1, 0) * SE2(rot2, (trans, 0))
 *   omnidirectional:  (rotation, translation, strafe) state * SE2(first, 0) * SE2(SO2(rotation) * first^-1, (translation, -strafe))
 *   stationary:       (theta, x, y) ~ N(0, 0.02)      state * SE2(theta, (x, y)) */
typedef struct bb200_motion_sampling {
  int model;
  double mean[3];
  double stddev[3];
  double first_rotation[2]; /* {cos, sin} */
} bb200_motion_sampling;

/* beluga::LikelihoodFieldModelBaseParam -- sensor/likelihood_field_model_base.hpp:42-64 */
typedef struct bb200_likelihood_field_param {
  double max_obstacle_distance; /* default 100.0 */
  double max_laser_distance;    /* default 2.0 */
  double z_hit;                 /* default 0.5 */
  double z_random;              /* default 0.5 */
  double sigma_hit;             /* default 0.2 */
  int model_unknown_space;      /* default 0 */
  int only_obstacle_boundaries; /* default 0 */
} bb200_likelihood_field_param;

/* beluga::BeamModelParam -- sensor/beam_model.hpp:43-58 */
typedef struct bb200_beam_param {
  double z_hit, z_short, z_max, z_rand, sigma_hit, lambda_short, beam_max_range;
} bb200_beam_param;

/* Occupancy grid view -- the OccupancyGrid2 named requirement (sensor/data/occupancy_grid.hpp)
 * with the ROS trinary value traits (beluga_ros/include/beluga_ros/occupancy_grid.hpp:48-64):
 * 0 free, 100 occupied, -1 unknown; row-major, index = yi*width + xi (linear_grid.hpp:73-75). */
typedef struct bb200_occupancy_grid {
  const int8_t* cells;
  int32_t width, height;
  double resolution;
  double origin[4]; /* grid.origin() as {cos, sin, x, y} */
} bb200_occupancy_grid;

typedef enum bb200_sensor_model {
  BB200_SENSOR_LIKELIHOOD_FIELD = 0,      /* sensor/likelihood_field_model.hpp:69-90: 1 + sum pz^3 */
  BB200_SENSOR_LIKELIHOOD_FIELD_PROB = 1, /* sensor/likelihood_field_prob_model.hpp:69-90: exp(sum log pz) */
  BB200_SENSOR_BEAM = 2,                  /* sensor/beam_model.hpp:104-150 */
  BB200_SENSOR_LANDMARK = 3,              /* sensor/landmark_sensor_model.hpp:96-156: range and bearing to the nearest landmark */
  BB200_SENSOR_BEARING = 4                /* sensor/bearing_sensor_model.hpp:92-140: bearing to the best-aligned landmark */
} bb200_sensor_model;

/* One landmark of a beluga::LandmarkMap (sensor/data/landmark_map.hpp:40-166): its position in the world frame and its
 * category (LandmarkPositionDetection, types/landmark_detection_types.hpp:39-42). */
typedef struct bb200_landmark {
  double x, y, z;
  uint32_t category;
} bb200_landmark;

/* LandmarkMap{boundaries, landmarks} (landmark_map.hpp:49-51), or LandmarkMap{landmarks} with null bounds: the implicit
 * bounds are the landmarks' componentwise minimum and maximum (:61-71).  Only x and y of the bounds are used: they are
 * the box of MultivariateUniformDistribution<SE2d, AlignedBox2d> (random/multivariate_uniform_distribution.hpp:43-73). */
typedef struct bb200_landmark_map {
  const bb200_landmark* landmarks;
  uint64_t n;
  const double* bounds_min3; /* {x, y, z}, or NULL with bounds_max3 NULL */
  const double* bounds_max3;
} bb200_landmark_map;

/* beluga::LandmarkModelParam -- sensor/landmark_sensor_model.hpp:44-48 */
typedef struct bb200_landmark_param {
  double sigma_range;   /* > 0 */
  double sigma_bearing; /* > 0 */
  double random_prob;   /* in [0, 1]; also the factor of a detection with no landmark of its category */
} bb200_landmark_param;

/* beluga::BearingModelParam -- sensor/bearing_sensor_model.hpp:42-45 */
typedef struct bb200_bearing_param {
  double sigma_bearing;             /* > 0 */
  double sensor_pose_in_robot[12];  /* 3x4 row-major [R | t]; R a rotation (within 1e-9) */
} bb200_bearing_param;

/* One detection: LandmarkPositionDetection (a position in the robot frame) for BB200_SENSOR_LANDMARK, or
 * LandmarkBearingDetection (a bearing vector in the sensor frame, any length) for BB200_SENSOR_BEARING
 * (types/landmark_detection_types.hpp:39-48). */
typedef struct bb200_landmark_detection {
  double x, y, z;
  uint32_t category;
} bb200_landmark_detection;

typedef enum bb200_resample_scheme {
  BB200_RESAMPLE_MULTINOMIAL = 0, /* views/sample.hpp:128-135 in counter-RNG form */
  BB200_RESAMPLE_SYSTEMATIC = 1   /* not in the reference; low-variance comb over the same CDF */
} bb200_resample_scheme;

/* Pose estimate -- std::pair<Sophus::SE2d, Sophus::Matrix3d> of algorithm/estimation.hpp:436-475 */
typedef struct bb200_estimate {
  double mean[4]; /* {cos, sin, x, y}, rotation renormalised */
  double cov[9];  /* row-major 3x3 over (x, y, theta) */
} bb200_estimate;

/* ---------------------------------------------------------------------------------------------
 * Library
 * ------------------------------------------------------------------------------------------- */

int bb200_abi_version(void);
/* Number of CUDA devices visible; 0 when there is none (then every create call fails). */
int bb200_device_count(void);
/* Message of the last failure of a create call on this thread. */
const char* bb200_create_error(void);

/* ---------------------------------------------------------------------------------------------
 * bb200_filter -- the particle set on the device and the per-step kernels.
 * Replaces beluga::TupleVector<std::tuple<SE2d, Weight>> (containers/tuple_vector.hpp:50-223)
 * plus the range adaptors that iterate it.
 * ------------------------------------------------------------------------------------------- */

typedef struct bb200_filter_config {
  int device;             /* CUDA device ordinal */
  uint64_t capacity;      /* maximum number of LOCAL particles (max_particles, or the shard size) */
  uint64_t seed;          /* counter-RNG key (Philox4x32-10) */
  /* Sharding (single GPU: rank 0 of 1).  Global particle index = first_index + local index. */
  uint64_t first_index;   /* global index of local particle 0 */
  uint64_t global_count;  /* total particles over all ranks (0: same as local) */
  int record_ancestors;   /* keep the resample indices for bb200_filter_ancestors (parity hook) */
} bb200_filter_config;

int bb200_filter_create(const bb200_filter_config* config, bb200_filter** out);
void bb200_filter_destroy(bb200_filter* f);
const char* bb200_last_error(const bb200_filter* f);

/* Sensor models.  LikelihoodFieldModel{params, grid} (likelihood_field_model.hpp:58-59): builds
 * the likelihood field on the host exactly as make_likelihood_field
 * (likelihood_field_model_base.hpp:130-185, distance_map.hpp:55-98) and uploads it.
 * `prob` selects LikelihoodFieldProbModel.  Also the target of update_map() (:113-116). */
int bb200_filter_set_likelihood_field_map(bb200_filter* f, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid, int prob);
/* BeamSensorModel{params, grid} (beam_model.hpp:96) / update_map (:156). */
int bb200_filter_set_beam_map(bb200_filter* f, const bb200_beam_param* p, const bb200_occupancy_grid* grid);
/* LandmarkSensorModel2d<LandmarkMap>{params, map} (landmark_sensor_model.hpp:83-84) / update_map (:160) and
 * BearingSensorModel2d<LandmarkMap>{params, map} (bearing_sensor_model.hpp:80-81) / update_map (:144).  A landmark map has
 * no grid: ray casts, bb200_filter_get_likelihood_field and point steps return BB200_ERR_STATE on it, and a detections
 * step on a grid map returns BB200_ERR_STATE.  initialize_from_map and recovery injection draw from
 * MultivariateUniformDistribution<SE2d, AlignedBox2d> over the map's x-y bounds (multivariate_uniform_distribution.hpp:
 * 43-73; counter streams 6 and 7, DESIGN.md §1); on an empty or non-finite box they return BB200_ERR_STATE.  The landmarks are kept stably sorted by category on the device, so every detection scans its
 * category's landmarks in the map's order. */
int bb200_filter_set_landmark_map(bb200_filter* f, const bb200_landmark_param* p, const bb200_landmark_map* map);
int bb200_filter_set_bearing_map(bb200_filter* f, const bb200_bearing_param* p, const bb200_landmark_map* map);
/* actions::reweight(sensor_model(detections)) (actions/reweight.hpp:54-60) on a landmark map: w *= L(state), with L the
 * std::transform_reduce product over the detections (landmark_sensor_model.hpp:155, bearing_sensor_model.hpp:139). */
int bb200_filter_reweight_landmarks(bb200_filter* f, const bb200_landmark_detection* detections, uint64_t n);
/* likelihood_field() accessor (likelihood_field_model_base.hpp:102): width*height floats. */
int bb200_filter_get_likelihood_field(const bb200_filter* f, float* out, uint64_t capacity);

/* Particle set access.  weights == NULL means 1.0 (make_from_state, particle_traits.hpp:105). */
int bb200_filter_set_particles(bb200_filter* f, const double* states, const double* weights, uint64_t n);
int bb200_filter_size(const bb200_filter* f, uint64_t* n);
/* particles() (amcl_core.hpp:128): copies min(n, capacity) particles out; either may be NULL. */
int bb200_filter_get_particles(bb200_filter* f, double* states, double* weights, uint64_t capacity);
/* Amcl::initialize(pose, covariance) (amcl_core.hpp:145-147) with
 * MultivariateNormalDistribution<SE2d> (random/multivariate_normal_distribution.hpp:96-126):
 * n particles ~ N(mean {x, y, theta}, cov 3x3), weights 1. */
int bb200_filter_initialize_normal(bb200_filter* f, const double mean_xytheta[3], const double cov[9], uint64_t n);
/* Global localisation: n particles from MultivariateUniformDistribution<SE2d, OccupancyGrid>
 * (random/multivariate_uniform_distribution.hpp:127-161) over the map set by bb200_filter_set_*_map: a free cell drawn
 * uniformly, its centroid in the global frame, yaw ~ U[-pi, pi); weights 1.  Counter RNG stream 6 at step 0,
 * keyed by the global particle index (same generator as the recovery injection of bb200_filter_resample). */
int bb200_filter_initialize_uniform(bb200_filter* f, uint64_t n);

/* actions::propagate(model(control)) (actions/propagate.hpp:57-79) for DifferentialDriveModel:
 * per particle 3 normals (counter RNG keyed by seed / global index / step) and the SE2 compose of
 * differential_drive_model.hpp:156-163. */
int bb200_filter_propagate(bb200_filter* f, const bb200_motion_sampling* s, uint32_t step);
/* actions::reweight(sensor_model(points)) (actions/reweight.hpp:54-60): w *= L(state). */
int bb200_filter_reweight(bb200_filter* f, const double* points_xy, uint64_t n_points);
/* Fused propagate | reweight (one pass over the particle set). */
int bb200_filter_propagate_reweight(bb200_filter* f, const bb200_motion_sampling* s, uint32_t step, const double* points_xy, uint64_t n_points);

/* Weight statistics of the local shard after reweight: the largest weight and, once an exponent
 * is fixed, the fixed-point total.  Single GPU: bb200_filter_normalize does all of it. */
int bb200_filter_max_weight(bb200_filter* f, double* wmax);
/* Fixes the quantisation exponent from the GLOBAL largest weight (all ranks pass the same value),
 * builds the local inclusive fixed-point CDF and returns the local total. */
int bb200_filter_build_cdf(bb200_filter* f, double global_wmax, uint64_t* local_total, int* exponent);
/* actions::normalize (actions/normalize.hpp:54-85): w /= S with S = global_total * 2^-exponent.
 * Also returns sum((w/S)^2) over the local shard (effective_sample_size.hpp:46-59). */
int bb200_filter_normalize_by(bb200_filter* f, uint64_t global_total, double* local_sum_sq);
/* Single-GPU convenience: max -> cdf -> normalize.  Returns the factor S and sum of squares. */
int bb200_filter_normalize(bb200_filter* f, double* factor, double* sum_sq);

/* views::sample | random_intersperse | take_while_kld | actions::assign
 * (views/sample.hpp:128-153, views/random_intersperse.hpp:93-100, views/take_while_kld.hpp:72-137,
 *  actions/assign.hpp:56-63) in counter-RNG form. */
typedef struct bb200_resample_opts {
  int scheme;                       /* bb200_resample_scheme */
  uint32_t step;
  uint64_t min_particles;           /* KLD lower bound (== max_particles disables KLD) */
  uint64_t max_particles;           /* number of output slots */
  double kld_epsilon, kld_z;
  double spatial_resolution[3];     /* spatial_hash<SE2d>{x, y, theta} (spatial_hash.hpp:160-197) */
  double random_state_probability;  /* recovery injection probability */
} bb200_resample_opts;
int bb200_filter_resample(bb200_filter* f, const bb200_resample_opts* o, uint64_t* new_size);
/* Sharded filter (one rank per GPU, contiguous global index ranges; see INTEGRATION.md):
 * produce the output slots [slot_begin, slot_end) -- those whose systematic-comb position lies in this
 * rank's span [cdf_offset, cdf_offset + local_total) of the global fixed-point CDF -- in slot order
 * into the staging state buffer (bb200_filter_device_pointer(f, 3)).  The caller moves them to the
 * ranks that own the slots (all-to-all) and then calls bb200_filter_adopt on the receivers. */
int bb200_filter_resample_range(bb200_filter* f, const bb200_resample_opts* o, uint64_t global_total, uint64_t cdf_offset,
                                uint64_t slot_begin, uint64_t slot_end);
/* Declare that n particle states have been written into the current (from_staging = 0) or staging
 * (from_staging = 1) state buffer: they become the particle set with weights 1. */
int bb200_filter_adopt(bb200_filter* f, uint64_t n, int from_staging);
/* Host helpers of the sharded step: the systematic comb (stride = total / slots, offset in [0, stride)
 * from the counter RNG) and beluga::estimate from globally summed raw moments (bb200_filter_moments). */
int bb200_systematic_comb(uint64_t seed, uint32_t step, uint64_t global_total, uint64_t total_slots, uint64_t* stride, uint64_t* offset);
int bb200_estimate_from_moments(const double moments[9], const double pivot_xy[2], bb200_estimate* out);
/* Stream-ordered variants for sharded callers that put collectives on the same CUDA stream
 * (bb200_filter_set_stream, e.g. torch's current stream): they only enqueue work -- no host
 * synchronisation, no read-back; intermediate scalars stay on the device (device pointers 4 and 5).
 *   enqueue_propagate_reweight: begin_step | propagate | schedule | reweight; the shard's largest weight is left in scalars.wmax_bits
 *   enqueue_build_cdf:          exponent from scalars.wmax_bits (all-reduce it with MAX first), fixed-point scan; total in scalars.total
 *   enqueue_resample_range / enqueue_adopt / enqueue_moments: as the synchronous calls above. */
int bb200_filter_set_stream(bb200_filter* f, void* cuda_stream);
int bb200_filter_enqueue_propagate_reweight(bb200_filter* f, const bb200_motion_sampling* s, uint32_t step, const double* points_xy, uint64_t n_points);
int bb200_filter_enqueue_build_cdf(bb200_filter* f);
int bb200_filter_enqueue_resample_range(bb200_filter* f, const bb200_resample_opts* o, uint64_t global_total, uint64_t cdf_offset,
                                        uint64_t slot_begin, uint64_t slot_end);
int bb200_filter_enqueue_adopt(bb200_filter* f, uint64_t n);
int bb200_filter_enqueue_moments(bb200_filter* f, const double pivot_xy[2]);
/* Ancestor index of every particle produced by the last resample (-1: injected random state). */
int bb200_filter_ancestors(bb200_filter* f, int64_t* out, uint64_t capacity);
/* The local fixed-point CDF built by the last build_cdf / normalize (parity hook). */
int bb200_filter_cdf(bb200_filter* f, uint64_t* out, uint64_t capacity);

/* beluga::estimate(states, weights) (algorithm/estimation.hpp:436-475). */
int bb200_filter_estimate(bb200_filter* f, bb200_estimate* out);
/* beluga::ParticleClusterizerParam (algorithm/cluster_based_estimation.hpp:259-276), same defaults
 * when filled by bb200_cluster_param_default. */
typedef struct bb200_cluster_param {
  double linear_hash_resolution;  /* 0.20 */
  double angular_hash_resolution; /* 0.524 */
  double weight_cap_percentile;   /* 0.90 */
} bb200_cluster_param;
void bb200_cluster_param_default(bb200_cluster_param* p);
/* beluga::cluster_based_estimate(states, weights, parameters) (cluster_based_estimation.hpp:415-432),
 * what beluga_ros::Amcl::update returns (beluga_ros/src/amcl.cpp:125): mean and covariance of the
 * heaviest cluster with more than one particle, or of the whole set when there is none.
 * Optional outputs (may be NULL): cluster_ids[i] = ParticleClusterizer::operator() (:304-316) for
 * particle i (ids_capacity >= particle count), the number of occupied cells and of clusters. */
int bb200_filter_cluster_estimate(bb200_filter* f, const bb200_cluster_param* p, bb200_estimate* out, uint32_t* cluster_ids,
                                  uint64_t ids_capacity, uint32_t* n_cells, uint32_t* n_clusters);
/* The per-CELL half of the cluster-based estimate, host only (no device needed): what
 * bb200_filter_cluster_estimate runs on the cell records its kernels produce.  cells[] lists the occupied
 * spatial-hash cells in the order in which the particle sequence first touches them
 * (clusterizer_detail::make_cluster_map, cluster_based_estimation.hpp:141-161).  Outputs: the cluster id of
 * every cell (assign_clusters, :205-253), the number of clusters, whether a cluster with more than one
 * particle exists and, if so, the id of the heaviest (cluster_based_estimate, :420-431), and the raw moments
 * to estimate from (that cluster's, else the whole set's). */
typedef struct bb200_cluster_cell {
  double representative[4]; /* state of the first particle in the cell {cos, sin, x, y} */
  uint64_t hash;            /* spatial_hash<SE2d>{linear, linear, angular}(representative) */
  uint32_t first_index;     /* index of that first particle */
  uint32_t count;           /* particles in the cell */
  double weight;            /* sum of their weights, in particle order */
  double moments[9];        /* raw moments of the cell's particles (layout of bb200_filter_moments) */
} bb200_cluster_cell;
int bb200_cluster_select_host(const bb200_cluster_cell* cells, uint64_t n_cells, uint64_t n_particles, const bb200_cluster_param* p,
                              uint32_t* cluster_of_cell, uint32_t* n_clusters, int* found, uint32_t* best, double moments_out[9]);
/* ---- output side (SURVEY 8f rank 4): what beluga_ros publishes after a step, without moving N x 40 bytes to the host ----
 * Device-side histogram of the particle cloud over spatial_hash<SE2d>{linear, linear, angular} buckets -- the
 * unordered_map pass of assign_particle_cloud(particles, linear_resolution, angular_resolution, MarkerArray)
 * (beluga_ros/include/beluga_ros/particle_cloud.hpp:197-210): one bin per occupied bucket, in the order in which the
 * particle sequence first touches them; representative = the first particle of the bucket, weight = the bucket's weights
 * added in particle order.  After a resample the million particles are copies of a few thousand candidates: the
 * publish costs a few-KB read-back.  (The reference's map additionally splits a bucket when two of its states are
 * not detail::almost_equal_to; with its 1 mm / 1 mrad defaults a bucket holds exact copies, and that refinement is not
 * reproduced.)  bins may be NULL to query the count.  max_bin_weight: max(1e-3, heaviest bin) (:197,205-207). */
int bb200_filter_particle_histogram(bb200_filter* f, double linear_resolution, double angular_resolution, bb200_cluster_cell* bins, uint64_t capacity,
                                    uint64_t* n_bins, double* max_bin_weight);
/* assign_particle_cloud(particles, size, PoseArray) (particle_cloud.hpp:129-147): `count` states drawn by weight
 * (views::sample | take_exactly) -- multinomial counter-RNG draws of `step` -- into states_out (count x {cos, sin, x, y});
 * the particle set is not modified. */
int bb200_filter_sample_states(bb200_filter* f, uint64_t count, uint32_t step, double* states_out);
/* Ray2d::cast (algorithm/raycasting.hpp:79-107, standard Bresenham) on the filter's current map, whichever sensor model it
 * is for: n_poses sensor poses {cos, sin, x, y} in the map frame times n_bearings bearings {cos, sin}, taken as given
 * (SO2::raw: not normalised; the library computes no trigonometry).  ranges receives n_poses x n_bearings doubles, pose
 * major (ray i * n_bearings + j is pose i, bearing j): min(distance, max_range) where the ray hits a non-free cell, +inf
 * where Ray2d::cast returns std::nullopt.  max_range is any double, as Ray2d takes it; a NaN makes every ray a miss.  One
 * kernel launch and one host synchronisation (none when there are no rays); the particle set is not touched.  A
 * likelihood-field map's first cast also builds the map's free-distance table on the host and uploads it (no launch); a
 * map that is never cast keeps only its likelihood field on the device.  BB200_ERR_STATE without a map,
 * BB200_ERR_INVALID_ARGUMENT for a null array with a non-zero count or when n_poses * n_bearings overflows. */
int bb200_filter_cast_rays(bb200_filter* f, const double* poses, uint64_t n_poses, const double* bearings_cs, uint64_t n_bearings, double max_range,
                           double* ranges);
/* Host only.  The marker geometry of assign_particle_cloud(..., MarkerArray) (particle_cloud.hpp:212-294) from the
 * histogram bins: 2 vertices per bin for the LINE_LIST "bodies" marker, 3 per bin for the TRIANGLE_LIST "heads"
 * marker, each with its RGBA colour (detail::alphaHueToRGBA, :56-70), and arrow_bodies.scale.x. */
typedef struct bb200_marker_vertex {
  double x, y, z;
  float r, g, b, a;
} bb200_marker_vertex;
int bb200_particle_cloud_markers(const bb200_cluster_cell* bins, uint64_t n_bins, bb200_marker_vertex* bodies, bb200_marker_vertex* heads,
                                 double* body_scale_x);
/* Host only.  assign_likelihood_field (beluga_ros/include/beluga_ros/likelihood_field.hpp:44-79): the likelihood field
 * (bb200_filter_get_likelihood_field) normalised to the [0, 100] int8 cells of a nav_msgs/OccupancyGrid. */
int bb200_likelihood_field_to_occupancy(const float* field, uint64_t n, int8_t* out);
/* Raw weighted moments of the local shard for a multi-rank estimate:
 * {sum w, sum w^2, sum w*cos, sum w*sin, sum w*dx, sum w*dy, sum w*dx^2, sum w*dx*dy, sum w*dy^2}
 * with (dx, dy) = (x, y) - pivot. */
int bb200_filter_moments(bb200_filter* f, const double pivot_xy[2], double out[9]);

/* Device-side timing (milliseconds, CUDA events on the filter's stream) of the kernels launched
 * since bb200_filter_clear_timings; names[i] are static strings.  Returns the count. */
int bb200_filter_set_timing(bb200_filter* f, int enabled);
int bb200_filter_clear_timings(bb200_filter* f);
int bb200_filter_last_timings(const bb200_filter* f, const char** names, float* ms, int capacity);
/* Total number of kernel launches issued by this filter since creation. */
uint64_t bb200_filter_launch_count(const bb200_filter* f);
/* Block until everything enqueued on the filter's stream has finished. */
int bb200_filter_synchronize(bb200_filter* f);
/* Raw device pointers (for torch.distributed / peer access plumbing): which = 0 states (double4),
 * 1 weights (double), 2 cdf (uint64), 3 staging states buffer (double4), 4 the scalar block
 * {u64 wmax_bits, u64 ticket, u64 total, i32 exponent, i32 valid, ...}, 5 the result block (9 raw moments). */
int bb200_filter_device_pointer(bb200_filter* f, int which, void** ptr, uint64_t* bytes);

/* ---------------------------------------------------------------------------------------------
 * bb200_amcl -- beluga::Amcl (algorithm/amcl_core.hpp:81-233) on top of a filter: update /
 * resample policies, rolling control window, recovery estimator, estimate.
 * ------------------------------------------------------------------------------------------- */

/* beluga::AmclParams (amcl_core.hpp:34-55) + spatial hasher resolutions + backend knobs. */
typedef struct bb200_amcl_param {
  double update_min_d;         /* 0.25 */
  double update_min_a;         /* 0.2 */
  uint64_t resample_interval;  /* 1 */
  int selective_resampling;    /* 0 */
  uint64_t min_particles;      /* 500 */
  uint64_t max_particles;      /* 2000 */
  double alpha_slow;           /* 0.001 */
  double alpha_fast;           /* 0.1 */
  double kld_epsilon;          /* 0.05 */
  double kld_z;                /* 3.0 */
  double spatial_resolution[3];/* spatial_hash<SE2d>: x, y, theta */
  int resample_scheme;         /* bb200_resample_scheme */
  uint64_t seed;
  int device;
  int record_ancestors;
  /* Sharding (both 0: single GPU).  max_particles is then the GLOBAL count; this rank holds
   * shard_capacity particles starting at global index shard_first_index. */
  uint64_t shard_first_index;
  uint64_t shard_capacity;
  /* > 0: views::random_intersperse runs with this probability on every resample instead of the recovery
   * estimator's output (which is identically 0 while the particle count is constant, see DESIGN.md); 0: the estimator. */
  double recovery_probability_override;
} bb200_amcl_param;

/* What Amcl::update decided on the host for this step (policies, control window, recovery
 * estimator; amcl_core.hpp:166-190) -- lets a sharded caller run the device part with collectives
 * in between (see beluga_b200/distributed.py). */
typedef struct bb200_step_plan {
  int update;                         /* 0: std::nullopt, nothing to do */
  int resample;                       /* every_n fired */
  int needs_ess;                      /* selective resampling: resample only if ESS < N/2 */
  uint32_t step;
  double random_state_probability;
  bb200_motion_sampling sampling;
  bb200_resample_opts opts;
} bb200_step_plan;

typedef struct bb200_update_result {
  int updated;                 /* 0: std::nullopt (no motion / no particles) */
  int resampled;
  uint64_t n_particles;
  bb200_estimate estimate;
  double random_state_probability;
  double weight_sum;           /* normalisation factor S of this step */
  int weights_degenerate;      /* 1: no particle had a positive finite weight after the reweight (the reference would
                                  divide by zero in normalize.hpp:82); a uniform CDF was substituted, weights left as they were */
} bb200_update_result;

int bb200_amcl_create(const bb200_amcl_param* p, const bb200_diff_drive_param* motion, bb200_amcl** out);
void bb200_amcl_destroy(bb200_amcl* a);
const char* bb200_amcl_last_error(const bb200_amcl* a);
/* The filter owned by the driver (for set_*_map, get_particles, timings ...). */
bb200_filter* bb200_amcl_filter(bb200_amcl* a);
/* Amcl::initialize(pose, covariance) -- amcl_core.hpp:145-147 (max_particles samples). */
int bb200_amcl_initialize(bb200_amcl* a, const double mean_xytheta[3], const double cov[9]);
/* beluga_ros::Amcl::initialize_from_map() (beluga_ros/include/beluga_ros/amcl.hpp:192-209): max_particles samples of the
 * map distribution (uniform over the free cells), weights 1, next update forced. */
int bb200_amcl_initialize_from_map(bb200_amcl* a);
/* Amcl::initialize from explicit states (tests / custom distributions, amcl_core.hpp:131-137). */
int bb200_amcl_initialize_states(bb200_amcl* a, const double* states, const double* weights, uint64_t n);
/* Amcl::force_update -- amcl_core.hpp:204 */
void bb200_amcl_force_update(bb200_amcl* a);
/* Amcl::update(control_action, measurement) -- amcl_core.hpp:165-201.  `points_xy` is the
 * measurement_type std::vector<std::pair<double,double>> flattened (x0, y0, x1, y1, ...). */
int bb200_amcl_update(bb200_amcl* a, const double control_pose[4], const double* points_xy, uint64_t n_points, bb200_update_result* out);
/* Amcl::update(control, detections) (amcl_core.hpp:165-200) with a landmark or bearing sensor model: the same step as
 * bb200_amcl_update, with the map's model weighing the detections.  BB200_ERR_STATE on a grid map, on a filter joined
 * to shards, and for bb200_amcl_update on a landmark map. */
int bb200_amcl_update_landmarks(bb200_amcl* a, const double control_pose[4], const bb200_landmark_detection* detections, uint64_t n,
                                bb200_update_result* out);
/* Scan preprocessing in front of the path (SURVEY 8f): what beluga_ros does between the sensor message
 * and Amcl::update -- beluga_ros::LaserScan (beluga_ros/include/beluga_ros/laser_scan.hpp:69-80:
 * take_evenly(max_beams) over ranges and angles, angle = float(angle_min + float(i) * angle_increment)),
 * BaseLaserScan::points_in_polar/cartesian_coordinates (beluga/sensor/data/laser_scan.hpp:64-91: drop
 * NaN and out-of-[min_range, max_range] readings, x = r cos a, y = r sin a) and the laser-to-base
 * transform of beluga_ros/src/amcl.cpp:57-62.  `laser_origin` is the 3x4 row-major [R | t] of the
 * laser frame in the base frame (NULL: identity); only x and y of the transformed point are kept. */
typedef struct bb200_laser_scan {
  const float* ranges;
  uint64_t n_ranges;
  float angle_min, angle_increment;
  double min_range, max_range; /* already combined with the message's range_min / range_max */
  uint64_t max_beams;          /* take_evenly count; 0 or >= n_ranges keeps every reading */
  const double* laser_origin;  /* 12 doubles or NULL */
} bb200_laser_scan;
/* Writes at most `capacity` points (x, y pairs) and their count. */
int bb200_scan_to_points(const bb200_laser_scan* scan, double* points_xy, uint64_t capacity, uint64_t* n_points);
/* Host only.  The directions {cos, sin} of the beams a bb200_laser_scan with these fields keeps (take_evenly(max_beams)),
 * computed exactly as bb200_scan_to_points computes them, without dropping any reading by its range: the bearings of a
 * scan geometry's expected scan (bb200_filter_cast_rays).  *n receives the count; BB200_ERR_CAPACITY, with nothing
 * written, when it exceeds capacity (bearings_cs may be NULL with capacity 0 to query it). */
int bb200_scan_bearings(float angle_min, float angle_increment, uint64_t n_ranges, uint64_t max_beams, double* bearings_cs, uint64_t capacity,
                        uint64_t* n);
/* take_evenly (beluga/views/take_evenly.hpp:118-145): the indices kept out of `size` elements. */
int bb200_take_evenly_indices(uint64_t size, uint64_t count, uint64_t* indices, uint64_t capacity, uint64_t* n_indices);
/* Amcl::update(base_pose_in_odom, laser_scan) -- beluga_ros/src/amcl.cpp:54-64. */
int bb200_amcl_update_scan(bb200_amcl* a, const double control_pose[4], const bb200_laser_scan* scan, bb200_update_result* out);
/* The point-cloud input of the same step: a sensor_msgs/PointCloud2 read the way beluga_ros::SparsePointCloud3f reads it
 * (beluga_ros/include/beluga_ros/sparse_point_cloud.hpp:102-125) and moved into the base frame by beluga_ros/src/amcl.cpp:67-81.
 * Point i is the three consecutive scalars (x, y, z) at data + i * point_step + x_offset (no alignment required); float64
 * coordinates are narrowed to float first (the alias is the non-strict float one), then every coordinate is widened to double
 * and (x, y) = rows 0 and 1 of R * (x, y, z) + t, summed left to right.  `origin` is the 3x4 row-major [R | t] of the cloud's
 * frame in the base frame (NULL: identity, coordinates pass unchanged), the convention of bb200_laser_scan::laser_origin; Sophus
 * applies the rotation through its unit quaternion, so the two agree to rounding.  No point is dropped or reordered: NaN
 * points go on to the sensor model, which treats them as out of the grid.  Checking the message's field names (x, y, z
 * first, all of one type) is the caller's part. */
typedef enum bb200_point_datatype {
  BB200_POINT_FLOAT32 = 7, /* sensor_msgs/PointField FLOAT32 */
  BB200_POINT_FLOAT64 = 8  /* sensor_msgs/PointField FLOAT64 */
} bb200_point_datatype;
typedef struct bb200_point_cloud {
  const void* data;
  uint64_t n_points;      /* width * height */
  uint32_t point_step;    /* bytes from one point to the next */
  uint32_t x_offset;      /* byte offset of x inside a point; y and z follow it */
  int datatype;           /* bb200_point_datatype */
  const double* origin;   /* 12 doubles or NULL */
} bb200_point_cloud;
/* Writes the n_points (x, y) pairs and their count.  BB200_ERR_INVALID_ARGUMENT for a datatype other than 7 or 8,
 * x_offset + 3 * sizeof(scalar) > point_step, or data == NULL with n_points > 0 (the std::invalid_argument cases of the
 * reference that reach this layer); BB200_ERR_CAPACITY when n_points > capacity.  On failure nothing is written. */
int bb200_point_cloud_to_points(const bb200_point_cloud* cloud, double* points_xy, uint64_t capacity, uint64_t* n_points);
/* Amcl::update(base_pose_in_odom, point_cloud) -- beluga_ros/src/amcl.cpp:67-81.  A sharded filter takes it through
 * bb200_sharded_amcl_update_point_cloud. */
int bb200_amcl_update_point_cloud(bb200_amcl* a, const double control_pose[4], const bb200_point_cloud* cloud, bb200_update_result* out);

/* A step weighed by the caller's own sensor model (the SensorModel template parameter of beluga::Amcl, amcl_core.hpp:74-81),
 * in two calls.  bb200_amcl_update_begin makes the host decisions of bb200_amcl_update (update policy, every_n, control
 * window, recovery probability, motion sampling), checks the step and enqueues the motion update on the filter's stream; it
 * does not synchronise.  When the policies skip the step (updated = 0) nothing reaches the device.  Otherwise the caller
 * writes factors[i] = L(states_i) for every particle, on `stream` or synchronised with it, and bb200_amcl_update_end then
 * runs w_i *= factors_i (the built-in reweight's multiply) and everything bb200_amcl_update runs after its sensor model:
 * normalize, the recovery estimator, every_n / selective / KLD resampling, injection and the estimate.  Factors that are
 * 0, negative, NaN or +-inf follow the rules of a built-in weight of that value (weights_degenerate when none is left).
 * With factors bit-equal to a stock model's likelihoods the step is byte-identical to bb200_amcl_update with that model.
 *
 * While a step is open every other call on the handle, and on its bb200_amcl_filter view, returns BB200_ERR_STATE;
 * bb200_amcl_destroy is allowed.  bb200_amcl_update_end must follow every successful begin, skipped steps included, and
 * returns BB200_ERR_STATE without one.  Both calls are atomic as bb200_amcl_update: on failure the policies, the control
 * window and the recovery estimator are as before the begin, and the step is closed.  No map is needed, except for a step
 * that may inject random states (BB200_ERR_STATE before any device work).  Shards refuse begin and end with
 * BB200_ERR_STATE: a sharded filter takes weighed steps through bb200_sharded_amcl_update_begin / _end.  The factor buffer
 * belongs to the filter and is allocated by the first begin. */
typedef struct bb200_weigh_view {
  int updated;           /* 0: the policies skip this step; end returns updated = 0 */
  uint64_t n;            /* particles to weigh */
  const double* states;  /* device: n x {cos, sin, x, y}, the propagated states */
  double* factors;       /* device: n doubles the caller writes, L(state_i) */
  void* stream;          /* cudaStream_t: order the weighing on it */
} bb200_weigh_view;
int bb200_amcl_update_begin(bb200_amcl* a, const double control_pose[4], bb200_weigh_view* view);
int bb200_amcl_update_end(bb200_amcl* a, bb200_update_result* out);

/* ---------------------------------------------------------------------------------------------
 * One filter over several GPUs (SURVEY 8e).  Particles are split into equal contiguous global index
 * ranges ("shards"); map and scan are replicated; the counter RNG is keyed by the GLOBAL particle /
 * slot index and the CDF is an integer prefix sum, so the particle set does not depend on the number
 * of shards.  The three exchanges of a step (largest weight, fixed-point totals, raw moments) and the
 * post-resample redistribution all go through peer memory from inside the library's own kernels:
 * no NCCL, no host round trip, one host synchronisation per step.
 *
 * (1) One process, several devices (or several shards on one device): bb200_sharded_amcl -- the shape
 *     of beluga_ros::Amcl (one node, one thread calling update; beluga_ros/src/amcl.cpp:83-126).
 * (2) One process per GPU (torchrun, MPI): every rank creates a bb200_amcl with shard_first_index /
 *     shard_capacity set, exports 256 bytes of CUDA IPC handles (bb200_amcl_export_shard), gathers
 *     the handles of all ranks by whatever transport it has, maps them (bb200_amcl_join_shards) and
 *     from then on calls bb200_amcl_update in lock step with its peers.
 * Policies: every_n resampling and selective resampling (on_effective_size_drop), systematic or
 * multinomial, recovery injection, KLD-adaptive particle counts (min_particles < max_particles: every rank
 * sees the spatial hash of every candidate slot and counts distinct buckets over the same ordered stream, so
 * all ranks stop at the reference's count; the new set is re-split into equal contiguous shards).
 * ------------------------------------------------------------------------------------------- */
typedef struct bb200_sharded_amcl bb200_sharded_amcl;
/* p->max_particles is the GLOBAL particle count (a multiple of n_shards); devices[r] is the CUDA ordinal of
 * shard r (ordinals may repeat: several shards on one device). */
int bb200_sharded_amcl_create(const bb200_amcl_param* p, const bb200_motion_param* motion, int n_shards, const int* devices,
                              bb200_sharded_amcl** out);
void bb200_sharded_amcl_destroy(bb200_sharded_amcl* g);
const char* bb200_sharded_amcl_last_error(const bb200_sharded_amcl* g);
int bb200_sharded_amcl_shards(const bb200_sharded_amcl* g);
/* Shard r as a bb200_amcl (not owned by the caller): timings, per-shard particles, bb200_amcl_filter. */
bb200_amcl* bb200_sharded_amcl_shard(bb200_sharded_amcl* g, int rank);
int bb200_sharded_amcl_set_likelihood_field_map(bb200_sharded_amcl* g, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid, int prob);
int bb200_sharded_amcl_set_beam_map(bb200_sharded_amcl* g, const bb200_beam_param* p, const bb200_occupancy_grid* grid);
/* bb200_filter_set_landmark_map / _set_bearing_map on every shard: the map is prepared once and uploaded to each.  A map
 * or parameters the filter calls refuse get the same status and message, and every shard keeps its map.  On a sharded
 * landmark map, bb200_sharded_amcl_update, _update_scan, _update_point_cloud and _cast_rays return BB200_ERR_STATE;
 * initialize_from_map and recovery injection draw from the map's box, as on one filter. */
int bb200_sharded_amcl_set_landmark_map(bb200_sharded_amcl* g, const bb200_landmark_param* p, const bb200_landmark_map* map);
int bb200_sharded_amcl_set_bearing_map(bb200_sharded_amcl* g, const bb200_bearing_param* p, const bb200_landmark_map* map);
int bb200_sharded_amcl_initialize(bb200_sharded_amcl* g, const double mean_xytheta[3], const double cov[9]);
int bb200_sharded_amcl_initialize_from_map(bb200_sharded_amcl* g);
void bb200_sharded_amcl_force_update(bb200_sharded_amcl* g);
/* Amcl::update (amcl_core.hpp:165-201) over all shards. */
int bb200_sharded_amcl_update(bb200_sharded_amcl* g, const double control_pose[4], const double* points_xy, uint64_t n_points,
                              bb200_update_result* out);
/* bb200_amcl_update_landmarks over all shards: the detections are prepared once on the host and copied to every shard
 * (no kernel launch), then every shard weighs its particles with the map's model and the step continues as
 * bb200_sharded_amcl_update does.  Particles, weights and the result's decisions, counts and weight_sum equal those of
 * one filter with the same parameters and seed, whatever the shard count.  BB200_ERR_INVALID_ARGUMENT for a NULL
 * detections with n > 0 and for n >= 2^32 - 1, BB200_ERR_STATE on a grid map, all before any device work; atomic as
 * bb200_sharded_amcl_update.  A shard joined by bb200_amcl_join_shards (one process per GPU) takes no detections. */
int bb200_sharded_amcl_update_landmarks(bb200_sharded_amcl* g, const double control_pose[4], const bb200_landmark_detection* detections, uint64_t n,
                                        bb200_update_result* out);
/* bb200_amcl_update_begin / _end over all shards: a step weighed by the caller's own sensor model.  views has
 * bb200_sharded_amcl_shards(g) entries; view r is shard r's contiguous slice of the global particle order, on devices[r] as
 * passed to bb200_sharded_amcl_create, with that shard's stream (a KLD-sized shard may hold n = 0: nothing to weigh).  The
 * caller writes every shard's factors on its stream or synchronised with it; end then runs w_i *= factors_i on every
 * shard and everything bb200_sharded_amcl_update runs after its sensor model.  No shard's exchanges start before every
 * shard's factors are applied: end makes each shard's stream wait for the others' (no host synchronisation), so a sensor
 * model may take as long as it needs.  With factors bit-equal to a stock model's likelihoods the step is byte-identical to
 * bb200_sharded_amcl_update with that model.  The rules are those of bb200_amcl_update_begin / _end: while a step is open
 * every other bb200_sharded_amcl_* call, and every call on the shards' bb200_amcl handles and their bb200_amcl_filter
 * views (bb200_amcl_update_end included), returns BB200_ERR_STATE; bb200_sharded_amcl_force_update is ignored and
 * bb200_sharded_amcl_destroy is allowed.  A step the policies skip launches nothing, and end still closes it.  Both calls
 * are atomic: on failure every shard's policies are as before the begin and the step is closed.  Factors that are 0,
 * negative, NaN or +-inf follow the built-in rules, weights_degenerate included. */
int bb200_sharded_amcl_update_begin(bb200_sharded_amcl* g, const double control_pose[4], bb200_weigh_view* views);
int bb200_sharded_amcl_update_end(bb200_sharded_amcl* g, bb200_update_result* out);
/* beluga::cluster_based_estimate over all shards: every shard builds its cell records on its device
 * (bb200_filter_particle_histogram with the clusterizer's resolutions), the records are merged on the host in rank
 * order (bb200_cluster_merge_host) and flooded like the single-GPU estimate.  Counts, weights and moments of a cell
 * that spans shards are added shard by shard: exact for unit weights (the state after a resample), otherwise equal to
 * the reference's single sequential sum up to the grouping of the additions. */
int bb200_sharded_amcl_cluster_estimate(bb200_sharded_amcl* g, const bb200_cluster_param* p, bb200_estimate* out, uint32_t* n_cells,
                                        uint32_t* n_clusters);
/* Host only: merges per-shard cell records (each list in its shard's first-occurrence order, shards in rank order) into
 * the global first-occurrence order; shard_first_index (may be NULL) turns local particle indices into global ones.
 * One process per GPU: gather the lists of bb200_filter_particle_histogram with the application's transport, then
 * bb200_cluster_merge_host + bb200_cluster_select_host + bb200_estimate_from_moments. */
int bb200_cluster_merge_host(const bb200_cluster_cell* const* shard_cells, const uint64_t* shard_counts, const uint64_t* shard_first_index, int shards,
                             bb200_cluster_cell* merged, uint64_t capacity, uint64_t* n_merged);
/* particles() in global index order (rank 0's shard first). */
int bb200_sharded_amcl_get_particles(bb200_sharded_amcl* g, double* states, double* weights, uint64_t capacity);
/* bb200_amcl_update_scan and bb200_amcl_update_point_cloud on a sharded filter: the scan or cloud is converted on the host
 * exactly as the standalone calls convert it (bb200_scan_to_points, bb200_point_cloud_to_points), then
 * bb200_sharded_amcl_update runs.  A scan or cloud the standalone calls refuse is refused with the same status before any
 * device work, and the filter is left unchanged. */
int bb200_sharded_amcl_update_scan(bb200_sharded_amcl* g, const double control_pose[4], const bb200_laser_scan* scan, bb200_update_result* out);
int bb200_sharded_amcl_update_point_cloud(bb200_sharded_amcl* g, const double control_pose[4], const bb200_point_cloud* cloud,
                                          bb200_update_result* out);
/* bb200_filter_particle_histogram over the whole filter: every shard that holds particles builds its cell records on its
 * device (the launches of bb200_filter_particle_histogram, once per call), and the records are merged on the host in rank order
 * (bb200_cluster_merge_host), as bb200_sharded_amcl_cluster_estimate merges them.  Same contract as the filter call: bins
 * may be NULL to query the count, BB200_ERR_CAPACITY leaves n_bins filled, max_bin_weight is max(1e-3, heaviest bin).
 * Hashes, first indices, representatives and counts are those of one filter holding the same particles.  A cell that spans
 * shards has its weight and raw moments added shard by shard: the weight is exact for unit weights (the state after a
 * resample), otherwise it equals the single sequential sum up to the grouping of the additions; the moments always
 * follow the grouping. */
int bb200_sharded_amcl_particle_histogram(bb200_sharded_amcl* g, double linear_resolution, double angular_resolution, bb200_cluster_cell* bins,
                                          uint64_t capacity, uint64_t* n_bins, double* max_bin_weight);
/* bb200_filter_sample_states over the GLOBAL particle set: `count` multinomial draws of `step`, byte-identical to what one
 * filter holding the same particles and weights returns, whatever the shard count; no shard's particles or weights change.
 * The global CDF is the one the last step left when it kept its particles; otherwise every shard builds its CDF with the
 * exponent of the largest weight of all shards (bb200_filter_max_weight, bb200_filter_build_cdf: 2 + 2 launches and 2
 * synchronisations per shard); current CDFs that were quantised with different exponents (built shard by shard) are
 * rebuilt the same way.  Then every shard with particles draws the slots of [0, count) whose position lands in its
 * span of the global CDF (1 launch) and stores each into the staging buffer of the shard that owns the slot; one
 * synchronisation per shard, and the host reads the staging buffers back in slot order.  BB200_ERR_STATE without
 * particles, BB200_ERR_CAPACITY for count > max_particles, BB200_ERR_INVALID_ARGUMENT for a NULL states_out with count > 0. */
int bb200_sharded_amcl_sample_states(bb200_sharded_amcl* g, uint64_t count, uint32_t step, double* states_out);
/* bb200_filter_cast_rays on the shards' copies of the map: every ray equals the filter call's on the same map.  The poses
 * are cut into contiguous ranges, one per shard in rank order; every shard with poses casts its range (1 launch) before
 * any reads back, then the host reads each range back with one synchronisation per such shard.  ranges is pose major.
 * Refusals are those of bb200_filter_cast_rays, before any device work. */
int bb200_sharded_amcl_cast_rays(bb200_sharded_amcl* g, const double* poses, uint64_t n_poses, const double* bearings_cs, uint64_t n_bearings,
                                 double max_range, double* ranges);
#define BB200_SHARD_HANDLE_BYTES 256
/* One process per GPU: CUDA IPC handles of this shard's two state buffers, mail block and (KLD) hash array (256 bytes) ... */
int bb200_amcl_export_shard(bb200_amcl* a, void* out256);
/* ... and the mapping of all ranks' handles (world x 256 bytes, rank order).  shard_capacity * world must equal
 * max_particles and shard_first_index must be rank * shard_capacity. */
int bb200_amcl_join_shards(bb200_amcl* a, int world, int rank, const void* handles);
/* Unmap the peers' buffers again.  CUDA IPC wants every importer to close before the exporter frees: call this on all
 * ranks, synchronise the ranks (barrier), then destroy. */
int bb200_amcl_leave_shards(bb200_amcl* a);

/* ---------------------------------------------------------------------------------------------
 * Many independent filters on one GPU: a batch of K beluga::Amcl members that share one device -- a
 * fleet server localising many robots on one or several site maps, a simulator with many agents.
 * bb200_amcl_batch_update steps every member that has a new scan with a fixed number of kernel launches
 * and one host synchronisation, whatever K is; each member's result and particles are bit-identical to
 * what a standalone bb200_amcl with the same parameters returns for the same inputs.
 *
 * Every member has its own parameter block (seed, policies, resampling scheme, recovery override) and
 * motion model.  Members of a batch made by bb200_amcl_batch_create keep a fixed particle count: it rejects, before
 * touching a device, with BB200_ERR_INVALID_ARGUMENT: n_members < 1, min_particles != max_particles (KLD), selective
 * resampling, non-zero shard fields, max_particles of 0 or above 32768, and members on different devices.
 * bb200_amcl_batch_create_adaptive accepts min_particles <= max_particles as bb200_amcl_create does: a member with
 * min_particles < max_particles resizes its particle set on every resampling step with KLD (take_while_kld), exactly
 * as a standalone bb200_amcl; bb200_amcl_batch_member_size returns its current count.
 * bb200_amcl_batch_create_with_flags takes the same checks as a set of flags: 0 is bb200_amcl_batch_create,
 * BB200_BATCH_ADAPTIVE is bb200_amcl_batch_create_adaptive, and BB200_BATCH_SELECTIVE (alone or with
 * BB200_BATCH_ADAPTIVE) accepts members with selective_resampling: when such a member's resample_interval fires, it
 * normalises its weights and resamples only when the effective sample size 1 / sum w^2 drops below n / 2 (beluga's
 * on_effective_size_drop), exactly as a standalone bb200_amcl, and bb200_update_result::resampled reports the decision.
 * The decision is made on the device, so the step keeps its one host synchronisation.
 *
 * A step takes 4 launches, plus those of the reweight forms (below), plus:
 *  - 1 when some updating member passes a laser scan or a point cloud (bb200_amcl_batch_update_measurements);
 *  - 2 when some updating member resamples under KLD (the members' KLD counts and the moments of the particles they
 *    keep) and no updating member runs the effective-sample-size test;
 *  - 2 when some updating member runs that test and none resamples under KLD (the test, and the moments of the new
 *    sets of those that resample);
 *  - 3 when both happen (the test, the KLD counts, the moments).
 * These counts are fixed before the step runs: they depend on neither K, nor the particle counts, nor the
 * members' decisions.
 *
 * A batch holds a set of maps, each a grid with its sensor model (likelihood-field model or the beam model) or a
 * landmark map with the landmark or bearing model.  Each member reads one of them or none.  bb200_amcl_batch_set_likelihood_field_map and _set_beam_map give every
 * member one map; bb200_amcl_batch_add_*_map and bb200_amcl_batch_update_map let members read different maps and
 * move between them, as a node's Amcl::update_map does.  Each reweight form that some updating member takes costs
 * launches: the likelihood field 1, the beam model 2 on maps where a standalone filter walks its rays in two
 * passes, 1 otherwise, and the landmark and bearing models 1 together.  A step takes 4 launches plus those, so 5 to 9,
 * whatever K and the number of maps are;
 * a step whose updating members read one map takes 5, or 6 for the two-pass beam form.  The two-pass members of a
 * step take the fused beam kernel instead when their hit words (sum of round_up(n, 32) x scan points x 4 bytes)
 * exceed 3 GiB or cannot be allocated.  Either way every member's results stay bit-identical to its standalone twin's.
 *
 * The fleet loop of a beluga_ros node per member is bb200_amcl_batch_update, then
 * bb200_amcl_batch_cluster_estimates for the members that updated: the estimate every node publishes, for all of them
 * with two kernel launches and two host synchronisations, whatever K and the members' cell counts are.  On the publish
 * timer a node also publishes its particle cloud, as markers and as a pose array: bb200_amcl_batch_particle_histograms
 * (2 launches, 2 synchronisations) and bb200_amcl_batch_sample_states (1 launch, or 4 when some member's CDF has to
 * be rebuilt; 1 synchronisation) do that for every selected member at once.
 * ------------------------------------------------------------------------------------------- */
typedef struct bb200_amcl_batch bb200_amcl_batch;
/* params[m] and motions[m] configure member m (params[m].device must be the same for all). */
int bb200_amcl_batch_create(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, bb200_amcl_batch** out);
/* bb200_amcl_batch_create whose members may have min_particles < max_particles (KLD-adaptive particle counts); it
 * rejects min_particles > max_particles and keeps the other refusals.  A member with min_particles == max_particles
 * keeps a fixed count, and a batch whose members all do computes what a bb200_amcl_batch_create batch computes. */
int bb200_amcl_batch_create_adaptive(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, bb200_amcl_batch** out);
/* Flags of bb200_amcl_batch_create_with_flags; any other bit is BB200_ERR_INVALID_ARGUMENT. */
typedef enum bb200_batch_flags {
  BB200_BATCH_ADAPTIVE = 1,  /* members may have min_particles < max_particles (KLD) */
  BB200_BATCH_SELECTIVE = 2  /* members may have selective_resampling */
} bb200_batch_flags;
/* bb200_amcl_batch_create with the refusals that `flags` lifts: 0 and BB200_BATCH_ADAPTIVE check exactly what
 * bb200_amcl_batch_create and bb200_amcl_batch_create_adaptive check.  A BB200_BATCH_SELECTIVE batch whose members
 * have no selective_resampling computes what a batch without the flag computes, with the same launches. */
int bb200_amcl_batch_create_with_flags(const bb200_amcl_param* params, const bb200_motion_param* motions, int n_members, uint32_t flags,
                                       bb200_amcl_batch** out);
/* Member m's current particle count in *n (any batch): max_particles after a fixed-size resample, the count KLD kept
 * after an adaptive one, n after bb200_amcl_batch_initialize_states. */
int bb200_amcl_batch_member_size(const bb200_amcl_batch* b, int member, uint64_t* n);
void bb200_amcl_batch_destroy(bb200_amcl_batch* b);
const char* bb200_amcl_batch_last_error(const bb200_amcl_batch* b);
int bb200_amcl_batch_members(const bb200_amcl_batch* b);
/* One likelihood field (prob != 0: the prob model) for every member, built and uploaded once.  Replaces any earlier
 * map, whichever sensor model it was for: removes every map, adds this one (it takes the next map id) and assigns
 * every member to it. */
int bb200_amcl_batch_set_likelihood_field_map(bb200_amcl_batch* b, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid,
                                              int prob);
/* One beam-model map (BeamSensorModel) for every member, built and uploaded once; replaces any earlier map the same way.
 * BB200_ERR_INVALID_ARGUMENT for a null handle or argument. */
int bb200_amcl_batch_set_beam_map(bb200_amcl_batch* b, const bb200_beam_param* p, const bb200_occupancy_grid* grid);
/* Build and upload a map without assigning it to any member (LikelihoodFieldModel / LikelihoodFieldProbModel, or
 * BeamSensorModel); *map_id receives its id.  Ids start at 0 over the batch's life, increase, and are never reused. */
int bb200_amcl_batch_add_likelihood_field_map(bb200_amcl_batch* b, const bb200_likelihood_field_param* p, const bb200_occupancy_grid* grid,
                                              int prob, int* map_id);
int bb200_amcl_batch_add_beam_map(bb200_amcl_batch* b, const bb200_beam_param* p, const bb200_occupancy_grid* grid, int* map_id);
/* Landmark maps: LandmarkSensorModel2d<LandmarkMap> / BearingSensorModel2d<LandmarkMap> on `map`, prepared and checked
 * exactly as bb200_filter_set_landmark_map / _set_bearing_map prepare them (the same statuses and messages).  _set_*
 * replaces every map as bb200_amcl_batch_set_beam_map does; _add_* adds one without assigning it.  A member on a landmark
 * map steps with BB200_MEASUREMENT_LANDMARKS (bb200_amcl_batch_set_detections); its initialize_from_map and recovery
 * injection draw from the map's box.  bb200_amcl_batch_get_likelihood_field and bb200_amcl_batch_cast_rays refuse a
 * landmark map with BB200_ERR_STATE. */
int bb200_amcl_batch_set_landmark_map(bb200_amcl_batch* b, const bb200_landmark_param* p, const bb200_landmark_map* map);
int bb200_amcl_batch_set_bearing_map(bb200_amcl_batch* b, const bb200_bearing_param* p, const bb200_landmark_map* map);
int bb200_amcl_batch_add_landmark_map(bb200_amcl_batch* b, const bb200_landmark_param* p, const bb200_landmark_map* map, int* map_id);
int bb200_amcl_batch_add_bearing_map(bb200_amcl_batch* b, const bb200_bearing_param* p, const bb200_landmark_map* map, int* map_id);
/* Amcl::update_map (amcl_core.hpp:150) / beluga_ros::Amcl::update_map (beluga_ros/src/amcl.cpp:48-51) for one member:
 * its particles and policies are kept; its next reweight, recovery injection and initialize_from_map use map_id. */
int bb200_amcl_batch_update_map(bb200_amcl_batch* b, int member, int map_id);
/* The map of a member (-1: none). */
int bb200_amcl_batch_member_map(const bb200_amcl_batch* b, int member, int* map_id);
/* Free a map; BB200_ERR_STATE while a member uses it. */
int bb200_amcl_batch_remove_map(bb200_amcl_batch* b, int map_id);
/* likelihood_field() of a likelihood-field map, height x width row-major (what a node publishes after a map update,
 * amcl_node.cpp:473-476).  BB200_ERR_STATE for a beam-model map, BB200_ERR_CAPACITY when capacity is too small.
 * Every call above returns BB200_ERR_INVALID_ARGUMENT for a null handle or argument, a bad member index or an unknown
 * or removed map id, and then leaves the batch unchanged. */
int bb200_amcl_batch_get_likelihood_field(const bb200_amcl_batch* b, int map_id, float* out, uint64_t capacity);
/* bb200_amcl_initialize / _initialize_from_map / _initialize_states / _force_update for member `member`.
 * _initialize_from_map samples the member's own map (BB200_ERR_STATE when it has none). */
int bb200_amcl_batch_initialize(bb200_amcl_batch* b, int member, const double mean_xytheta[3], const double cov[9]);
int bb200_amcl_batch_initialize_from_map(bb200_amcl_batch* b, int member);
int bb200_amcl_batch_initialize_states(bb200_amcl_batch* b, int member, const double* states, const double* weights, uint64_t n);
int bb200_amcl_batch_force_update(bb200_amcl_batch* b, int member);
/* Member m's particles (at most `capacity`; either output may be NULL). */
int bb200_amcl_batch_get_particles(bb200_amcl_batch* b, int member, double* states, double* weights, uint64_t capacity);
/* Resample indices of member m's last resample (params[m].record_ancestors must be set). */
int bb200_amcl_batch_ancestors(bb200_amcl_batch* b, int member, int64_t* out, uint64_t capacity);
/* beluga::cluster_based_estimate of member m's particles (bb200_amcl_batch_cluster_estimates with member m alone). */
int bb200_amcl_batch_cluster_estimate(bb200_amcl_batch* b, int member, const bb200_cluster_param* p, bb200_estimate* out);
/* beluga::cluster_based_estimate of every member m with present[m] != 0 (present NULL: all members), with one set of
 * clusterizer parameters for all of them.  out[m] receives member m's estimate.  n_cells and n_clusters may be NULL;
 * when they are not, entry m receives member m's occupied cells and clusters.  Entries of members not selected are not
 * written.  The number of kernel launches does not depend on K or on the members' cell counts.  Every selected member's
 * result is bit-identical to bb200_amcl_batch_cluster_estimate(b, m, p, ...) and to a standalone filter's
 * bb200_filter_cluster_estimate over the same particles.  Fails before any launch with BB200_ERR_INVALID_ARGUMENT for
 * bad parameters and with BB200_ERR_STATE when a selected member holds no particles. */
int bb200_amcl_batch_cluster_estimates(bb200_amcl_batch* b, const bb200_cluster_param* p, const uint8_t* present,
                                       bb200_estimate* out, uint32_t* n_cells, uint32_t* n_clusters);
/* bb200_filter_particle_histogram for every member m with present[m] != 0 (present NULL: all members), with two kernel
 * launches and two host synchronisations whatever K and the bin counts are.  bins[m] receives member m's bins in
 * first-occurrence order when capacity[m] holds them; bins or bins[m] may be NULL to query the counts only (capacity may
 * then be NULL too).  n_bins[m] and max_bin_weight[m] (max(1e-3, heaviest bin)) are written for selected members; either
 * array may be NULL.  Entries of members not selected are not written.  Every selected member's output is bit-identical
 * to a standalone filter's bb200_filter_particle_histogram over the same particles.  BB200_ERR_CAPACITY when some
 * selected member's buffer is too small (n_bins is still filled, and the members whose buffers fit get their bins).
 * Fails before any launch with BB200_ERR_INVALID_ARGUMENT for non-positive resolutions or a null handle, or bins without
 * capacity, and with BB200_ERR_STATE when a selected member holds no particles. */
int bb200_amcl_batch_particle_histograms(bb200_amcl_batch* b, double linear_resolution, double angular_resolution, const uint8_t* present,
                                         bb200_cluster_cell* const* bins, const uint64_t* capacity, uint64_t* n_bins, double* max_bin_weight);
/* bb200_filter_sample_states(counts[m], step) for every member m with present[m] != 0 (present NULL: all members):
 * counts[m] states drawn by weight into states_out[m] (counts[m] x {cos, sin, x, y}), bit-identical to what a standalone
 * filter draws; no member's particle set is modified.  A member samples from the CDF a standalone filter would use: the
 * one its last step built when that step normalised instead of resampling, otherwise one rebuilt from its weights in
 * this call (and kept for later calls until its particles or weights change).  One kernel launch when no CDF has to be
 * rebuilt, four otherwise, and one host synchronisation, whatever K and the counts are.  counts[m] == 0 draws nothing.
 * Fails before any launch with BB200_ERR_STATE when a selected member holds no particles, BB200_ERR_CAPACITY when
 * counts[m] exceeds its max_particles, and BB200_ERR_INVALID_ARGUMENT for a null handle, counts or states_out, or a null
 * states_out[m] with counts[m] > 0. */
int bb200_amcl_batch_sample_states(bb200_amcl_batch* b, const uint64_t* counts, uint32_t step, const uint8_t* present, double* const* states_out);
/* bb200_filter_cast_rays for every member m with present[m] != 0 (present NULL: every occupied slot): n_poses[m] x
 * n_bearings[m] rays from poses[m] along bearings_cs[m] up to max_range[m] into ranges[m], on member m's own map, or on
 * map map_ids[m] of the batch when map_ids is not NULL and map_ids[m] != -1 (e.g. a simulator's world map).  Every
 * member's ranges are bit-identical to bb200_filter_cast_rays on the same map.  One kernel launch and one host
 * synchronisation whatever K, the maps and the ray counts are (none when no selected member has a ray).  Refused before
 * anything reaches the device, with the batch unchanged: a vacant selected slot, an unknown or removed map id, a null
 * array with a non-zero count or an overflowing n_poses[m] * n_bearings[m] (BB200_ERR_INVALID_ARGUMENT), and a selected
 * member without a map and no map id (BB200_ERR_STATE).  No member is modified. */
int bb200_amcl_batch_cast_rays(bb200_amcl_batch* b, const uint8_t* present, const int* map_ids, const double* const* poses, const uint64_t* n_poses,
                               const double* const* bearings_cs, const uint64_t* n_bearings, const double* max_range, double* const* ranges);
/* Amcl::update for every member m with present[m] != 0 (present NULL: all members).  control_poses holds K poses of 4
 * doubles, points_xy[m] member m's n_points[m] (x, y) pairs (NULL when n_points[m] == 0), out[m] its result.  An absent
 * member is left untouched -- no policy is evaluated -- and gets out[m].updated = 0.  Present members go through their
 * own on_motion / every_n / recovery-estimator logic exactly as in bb200_amcl_update.  The call is atomic: when it fails,
 * every member's host state is as if it had not been made. */
int bb200_amcl_batch_update(bb200_amcl_batch* b, const double* control_poses, const double* const* points_xy, const uint64_t* n_points,
                            const uint8_t* present, bb200_update_result* out);
/* One member's measurement in a step: base-frame points, a laser scan or a point cloud, each as the single filter's
 * bb200_amcl_update, bb200_amcl_update_scan and bb200_amcl_update_point_cloud take it.  Only the fields of `kind` are read. */
/* BB200_MEASUREMENT_WEIGHTS: this member is weighed by the caller (bb200_amcl_batch_update_begin / _end only; the other
 * update calls refuse it); no field of the measurement is read. */
/* BB200_MEASUREMENT_LANDMARKS: this member, on a landmark map, weighs the detections staged for it by
 * bb200_amcl_batch_set_detections, as bb200_amcl_update_landmarks weighs them; no field of the measurement is read.  The
 * update calls refuse with BB200_ERR_STATE, before anything reaches the device, a present LANDMARKS member on a grid map
 * or without staged detections, and a present points, scan or cloud member on a landmark map. */
typedef enum bb200_measurement_kind {
  BB200_MEASUREMENT_POINTS = 0,
  BB200_MEASUREMENT_SCAN = 1,
  BB200_MEASUREMENT_CLOUD = 2,
  BB200_MEASUREMENT_WEIGHTS = 3,
  BB200_MEASUREMENT_LANDMARKS = 4
} bb200_measurement_kind;
typedef struct bb200_measurement {
  int kind;                        /* bb200_measurement_kind */
  const double* points_xy;         /* POINTS: n_points (x, y) pairs (NULL when n_points == 0) */
  uint64_t n_points;
  const bb200_laser_scan* scan;    /* SCAN */
  const bb200_point_cloud* cloud;  /* CLOUD */
} bb200_measurement;
/* bb200_amcl_batch_update with measurements[m] as member m's input, so that members with 2-D lidars, 3-D lidars and
 * points step in one call.  Scans and clouds are converted on the device: the host sends 4 bytes per kept beam (the
 * range) or 12 bytes per cloud point (x, y, z as floats), and the beam directions, computed on the host as
 * bb200_scan_to_points computes them, are uploaded once per scan geometry (n_ranges, max_beams, angle_min,
 * angle_increment) and member.  A step in which some updating member passes a scan or a cloud takes one kernel launch
 * more than bb200_amcl_batch_update's count; a step whose updating members all pass points takes the same launches.
 *
 * Bit-identity: every present member's out[m], particles, ancestors and later steps are bit-identical to a standalone
 * bb200_amcl with the same parameters fed bb200_amcl_update_scan / bb200_amcl_update_point_cloud / bb200_amcl_update,
 * and to bb200_amcl_batch_update given the points bb200_scan_to_points / bb200_point_cloud_to_points return.
 * Validation: BB200_ERR_INVALID_ARGUMENT, before anything reaches the device, for a null handle, control_poses,
 * measurements or out, and for a present member whose measurement the single filter refuses: an unknown kind, a null
 * scan or cloud, null ranges or points with a non-zero count, a cloud datatype other than 7 or 8, or
 * x_offset + 3 * sizeof(scalar) > point_step.  Every present member is checked, whether it updates in this step or not.
 * Atomicity: as bb200_amcl_batch_update -- on failure every member's host state is as if the call had not been made. */
int bb200_amcl_batch_update_measurements(bb200_amcl_batch* b, const double* control_poses, const bb200_measurement* measurements,
                                         const uint8_t* present, bb200_update_result* out);
/* bb200_amcl_batch_update_measurements, then beluga::cluster_based_estimate (cluster_based_estimation.hpp:415-432) of
 * every member that updated: what beluga_ros::Amcl::update returns (beluga_ros/src/amcl.cpp:125), for the whole batch in
 * one call.  out[m] is exactly what bb200_amcl_batch_update_measurements writes.  clustered[m], n_cells[m] and
 * n_clusters[m] (n_cells and n_clusters may be NULL) are written for the members with out[m].updated, and they are
 * byte-identical to bb200_amcl_batch_cluster_estimates(b, p, mask of updated members, ...) called right after the update.
 *
 * The per-cell flood of the estimate runs on the device, one CTA per member: the call takes the update's launches plus 3
 * and one host synchronisation, whatever K and the cell counts are.  A member for which the device cannot promise the
 * host's result -- a NaN cell weight, or a neighbour heading within a few ulps of an angular bucket edge -- gets the host
 * pass instead; a call in which that happens takes 1 launch and 1 synchronisation more.  The cluster parameters are
 * checked as bb200_amcl_batch_cluster_estimates checks them, before anything reaches the device (BB200_ERR_INVALID_ARGUMENT),
 * and the call is atomic as bb200_amcl_batch_update_measurements is. */
int bb200_amcl_batch_update_clustered(bb200_amcl_batch* b, const double* control_poses, const bb200_measurement* measurements,
                                      const uint8_t* present, const bb200_cluster_param* p, bb200_update_result* out,
                                      bb200_estimate* clustered, uint32_t* n_cells, uint32_t* n_clusters);
/* bb200_amcl_batch_update_measurements / _update_clustered in two calls, for a step in which some members are weighed by
 * the caller's own sensor model (measurements[m].kind == BB200_MEASUREMENT_WEIGHTS): the semantics of
 * bb200_amcl_update_begin / _end, per member.  begin makes every present member's host decisions, checks the step and
 * enqueues the conversion of scans and clouds, the propagate and the built-in reweight of the members that pass points,
 * scans or clouds, so that their sensor work overlaps the caller's; it does not synchronise.  views[m] (one per slot) is
 * written for every slot: updated = 1 for a present member that updates in this step, and for a weighed one n, its current
 * state slice and its slice of one batch-owned factor buffer laid out like the particle buffers, and the batch's stream.
 * The caller writes factors[i] = L(state_i) for every particle of every weighed updating member, on that stream or
 * synchronised with it.  end enqueues w *= factor for the weighed members (one launch, a CTA range per member), then the
 * rest of the step and, with `cluster` (NULL: none), the cluster estimates of bb200_amcl_batch_update_clustered, and
 * synchronises once.  A step without weighed members launches exactly what bb200_amcl_batch_update_measurements (or
 * _update_clustered) launches.  Weighed members need no map unless their step may inject random states.  While a step is
 * open every other call on the batch returns BB200_ERR_STATE, except bb200_amcl_batch_update_end and destroy; end without
 * an open step returns BB200_ERR_STATE.  Both calls are atomic as bb200_amcl_batch_update_measurements; a failed end closes
 * the step. */
int bb200_amcl_batch_update_begin(bb200_amcl_batch* b, const double* control_poses, const bb200_measurement* measurements, const uint8_t* present,
                                  bb200_weigh_view* views);
/* Stages detections[m][0, n[m]) for every member m with present[m] != 0 (present NULL: every occupied slot), replacing
 * what was staged for it; they stay staged, and every BB200_MEASUREMENT_LANDMARKS step of the member weighs them, until
 * they are replaced or the member is removed.  A host copy: nothing reaches the device.  Each detection's category is
 * resolved against the member's map when a step weighs it.  BB200_ERR_INVALID_ARGUMENT, with nothing staged, for a
 * null handle or n, a vacant selected slot, a null detections or detections[m] with n[m] > 0, or n[m] >= 2^32 - 1. */
int bb200_amcl_batch_set_detections(bb200_amcl_batch* b, const bb200_landmark_detection* const* detections, const uint64_t* n, const uint8_t* present);
int bb200_amcl_batch_update_end(bb200_amcl_batch* b, const bb200_cluster_param* cluster, bb200_update_result* out, bb200_estimate* clustered,
                                uint32_t* n_cells, uint32_t* n_clusters);
/* Kernel launches issued by this batch so far (steps, initialisations, cluster estimates, particle-cloud histograms and
 * pose samples, ray casts, membership changes, and the beam model's map uploads). */
uint64_t bb200_amcl_batch_launch_count(const bb200_amcl_batch* b);

/* Members that join and leave a running batch (a fleet server whose robots connect, disconnect and reconnect with new
 * parameters).  Member indices are slots: a slot is occupied or vacant, and an index keeps its meaning while its member
 * lives.  bb200_amcl_batch_members returns the number of slots, occupied and vacant; slots are never removed, so every
 * per-member array a call takes (control_poses, measurements, present, out, counts, ...) keeps that length.
 *  - present == NULL selects every occupied slot.  present[m] != 0 on a vacant slot is BB200_ERR_INVALID_ARGUMENT before
 *    anything reaches the device, and the batch is unchanged (bb200_amcl_batch_update, _update_measurements,
 *    _update_clustered, _cluster_estimates, _particle_histograms, _sample_states).  A vacant slot's inputs are not read,
 *    and its out[m] is written as an absent member's (updated = 0).
 *  - Every per-member call (_initialize*, _force_update, _get_particles, _ancestors, _member_size, _update_map,
 *    _member_map, _cluster_estimate, _remove_member) refuses a vacant slot with BB200_ERR_INVALID_ARGUMENT, as it refuses
 *    an unknown index.
 *  - _set_*_map assigns the map to every occupied slot; a vacant slot reads no map and never blocks _remove_map.
 * Each call below is atomic -- when it fails, for validation or allocation, the batch is exactly as before -- and ends
 * synchronised.  Every member's results stay byte-identical to those of a standalone bb200_amcl created when it joined
 * (or when the batch was created) and fed the same inputs; after any sequence of joins and leaves, a step, cluster
 * estimate, histogram or pose draw launches exactly what it launches on a freshly created batch of the same members. */

/* Adds a member configured by params and motion, validated exactly as bb200_amcl_batch_create_with_flags validates a
 * member under this batch's flags and device (the same messages, naming the slot it would take).  It takes the lowest
 * vacant slot, or appends a new one; *member receives the slot.  The new member inherits nothing from the slot's earlier
 * occupant: it reads no map and holds no particles, ancestors or CDF, and its policies start fresh, as those of a member
 * of a freshly created batch.  Every other member's particles, weights, valid CDF, ancestors, policies and map are kept.
 * The particle buffers are laid out again as create lays them out for the members now present: one kernel launch moves
 * the other members' live data (none when no other member holds particles). */
int bb200_amcl_batch_add_member(bb200_amcl_batch* b, const bb200_amcl_param* params, const bb200_motion_param* motion, int* member);
/* Makes slot `member` vacant and frees its share of the device buffers (one kernel launch moves the other members' live
 * data, none when none of them holds particles).  BB200_ERR_STATE when it is the last occupied slot: a batch always
 * holds at least one member, as create requires. */
int bb200_amcl_batch_remove_member(bb200_amcl_batch* b, int member);
/* *active = 1 for an occupied slot, 0 for a vacant one (BB200_ERR_INVALID_ARGUMENT for an index out of range). */
int bb200_amcl_batch_member_active(const bb200_amcl_batch* b, int member, int* active);

/* A filter's complete state as a byte string (a "state blob"): checkpoint a fleet before a restart, move a robot between
 * batches, processes, devices and standalone filters, or capture one robot's filter to replay its logged scans offline.
 * A blob holds the filter's parameters and motion model, its policies' state (on_motion pose, every_n phase, recovery
 * filters, control window, forced update, step counter), its particles, weights, pivot, its CDF while that is current,
 * and its ancestors when it records them.  It does not hold a map: the receiver attaches one.  A filter restored from a
 * blob computes, step for step, exactly what the filter that wrote it would have computed (counter RNG keyed by seed,
 * step and particle index).  The layout is versioned and described in DESIGN.md; it is in the byte order of the machine
 * that wrote it, so blobs move between machines of the same endianness only.  params.device is not read on import: the
 * receiver's device wins.  A blob that is truncated, padded, of another magic, blob version or ABI version, whose section
 * lengths do not match its scalars, or whose scalars no filter holds is refused with BB200_ERR_INVALID_ARGUMENT.
 *
 * Size query: with out == NULL, *size receives the blob's size; BB200_ERR_CAPACITY (and *size) when capacity is below it.
 * Sharded filters have no state blob: a shard (inside bb200_sharded_amcl, or with shard fields set) is BB200_ERR_STATE. */
int bb200_amcl_export_state(bb200_amcl* a, void* out, uint64_t capacity, uint64_t* size);
/* A standalone filter on `device` with the blob's parameters and state.  It has no map: an update before
 * bb200_filter_set_*_map fails as on a newly created filter.  Failures are reported by bb200_create_error. */
int bb200_amcl_create_from_state(const void* blob, uint64_t size, int device, bb200_amcl** out);
/* Host only: checks a blob and returns its parameters and motion model (BB200_ERR_INVALID_ARGUMENT with the reason in
 * bb200_create_error for a blob the calls here refuse). */
int bb200_amcl_state_params(const void* blob, uint64_t size, bb200_amcl_param* params, bb200_motion_param* motion);
/* The fleet checkpoint: the blob of every member m with present[m] != 0 (present NULL: every occupied slot).  size[m]
 * receives member m's blob size; out[m] receives the blob when out and out[m] are not NULL and capacity[m] holds it.
 * BB200_ERR_CAPACITY, before anything reaches the device, when some selected member's buffer is too small (size is still
 * filled).  One kernel launch gathers the members' particle data, one copy brings it to the host and one synchronisation
 * ends the call, whatever K is.  A vacant selected slot is BB200_ERR_INVALID_ARGUMENT. */
int bb200_amcl_batch_export_members(bb200_amcl_batch* b, const uint8_t* present, void* const* out, const uint64_t* capacity, uint64_t* size);
/* bb200_amcl_batch_export_members with member `member` alone selected. */
int bb200_amcl_batch_export_member(bb200_amcl_batch* b, int member, void* out, uint64_t capacity, uint64_t* size);
/* bb200_amcl_batch_add_member with a history: the blob's member joins in the lowest vacant slot or a new one (*member),
 * validated exactly as bb200_amcl_batch_add_member validates its params under this batch's flags and device, and reads
 * map map_id (-1: none, then it behaves as a joined member without a map).  The other members are kept as add_member keeps
 * them.  One kernel launch more than add_member puts the blob's particle data in place.  Atomic: on failure the batch is
 * unchanged. */
int bb200_amcl_batch_import_member(bb200_amcl_batch* b, const void* blob, uint64_t size, int map_id, int* member);
/* A batch whose member m is blobs[m]'s filter (sizes[m] bytes), on `device`, validated as bb200_amcl_batch_create_with_flags
 * validates the blobs' parameters with `flags`.  One copy and one kernel launch restore every member's particle data,
 * whatever K is.  The batch has no map: add them and assign them with bb200_amcl_batch_update_map. */
int bb200_amcl_batch_create_from_states(const void* const* blobs, const uint64_t* sizes, int n_members, uint32_t flags, int device,
                                        bb200_amcl_batch** out);

/* The two host halves of bb200_amcl_update for callers that drive the filter themselves. */
int bb200_amcl_plan_update(bb200_amcl* a, const double control_pose[4], bb200_step_plan* plan);
void bb200_amcl_commit_update(bb200_amcl* a, int resampled, double random_state_probability);
/* Amcl with any of the three motion models (bb200_amcl_create is the differential-drive shorthand). */
int bb200_amcl_create_with_motion(const bb200_amcl_param* p, const bb200_motion_param* motion, bb200_amcl** out);
/* MotionModel::operator()(control) host part for any model (differential_drive_model.hpp:129-154,
 * omnidirectional_drive_model.hpp:101-129, stationary_model.hpp:52). */
int bb200_motion_sampling_from_control(const bb200_motion_param* p, const double pose[4], const double previous_pose[4], bb200_motion_sampling* out);
/* DifferentialDriveModel::operator()(control) host part -- differential_drive_model.hpp:129-154. */
int bb200_diff_drive_sampling_from_control(const bb200_diff_drive_param* p, const double pose[4], const double previous_pose[4], bb200_diff_drive_sampling* out);

#ifdef __cplusplus
}
#endif
#endif /* BELUGA_B200_H_ */
