"""ctypes declarations for libbeluga_b200.so -- one entry per function of include/beluga_b200.h.

The library is the product; this module only loads it.  There is no Python or CPU fallback: if the
shared object is missing, `load()` raises, and on a box without a CUDA device every
`bb200_*_create` call returns BB200_ERR_NO_DEVICE.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libbeluga_b200.so")

OK, ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_NO_DEVICE, ERR_STATE, ERR_CAPACITY = 0, -1, -2, -3, -4, -5
BATCH_ADAPTIVE, BATCH_SELECTIVE = 1, 2  # bb200_batch_flags

SENSOR_LIKELIHOOD_FIELD, SENSOR_LIKELIHOOD_FIELD_PROB, SENSOR_BEAM, SENSOR_LANDMARK, SENSOR_BEARING = 0, 1, 2, 3, 4
RESAMPLE_MULTINOMIAL, RESAMPLE_SYSTEMATIC = 0, 1


class DiffDriveParam(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "rotation_noise_from_rotation", "rotation_noise_from_translation", "translation_noise_from_translation",
        "translation_noise_from_rotation", "distance_threshold")]


class DiffDriveSampling(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("rot1_mean", "rot1_std", "trans_mean", "trans_std", "rot2_mean", "rot2_std")]


MOTION_DIFFERENTIAL, MOTION_OMNIDIRECTIONAL, MOTION_STATIONARY = 0, 1, 2


class MotionParam(C.Structure):
    _fields_ = [("model", C.c_int)] + [(n, C.c_double) for n in (
        "rotation_noise_from_rotation", "rotation_noise_from_translation", "translation_noise_from_translation",
        "translation_noise_from_rotation", "strafe_noise_from_translation", "distance_threshold")]


class MotionSampling(C.Structure):
    _fields_ = [("model", C.c_int), ("mean", C.c_double * 3), ("stddev", C.c_double * 3), ("first_rotation", C.c_double * 2)]


class LikelihoodFieldParam(C.Structure):
    _fields_ = [("max_obstacle_distance", C.c_double), ("max_laser_distance", C.c_double), ("z_hit", C.c_double),
                ("z_random", C.c_double), ("sigma_hit", C.c_double), ("model_unknown_space", C.c_int),
                ("only_obstacle_boundaries", C.c_int)]


class BeamParam(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("z_hit", "z_short", "z_max", "z_rand", "sigma_hit", "lambda_short", "beam_max_range")]


class Landmark(C.Structure):  # also bb200_landmark_detection: the same layout
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("z", C.c_double), ("category", C.c_uint32)]


class LandmarkMap(C.Structure):
    _fields_ = [("landmarks", C.POINTER(Landmark)), ("n", C.c_uint64), ("bounds_min3", C.POINTER(C.c_double)), ("bounds_max3", C.POINTER(C.c_double))]


class LandmarkParam(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("sigma_range", "sigma_bearing", "random_prob")]


class BearingParam(C.Structure):
    _fields_ = [("sigma_bearing", C.c_double), ("sensor_pose_in_robot", C.c_double * 12)]


class OccupancyGrid(C.Structure):
    _fields_ = [("cells", C.POINTER(C.c_int8)), ("width", C.c_int32), ("height", C.c_int32), ("resolution", C.c_double),
                ("origin", C.c_double * 4)]


class Estimate(C.Structure):
    _fields_ = [("mean", C.c_double * 4), ("cov", C.c_double * 9)]


class ClusterParam(C.Structure):
    _fields_ = [("linear_hash_resolution", C.c_double), ("angular_hash_resolution", C.c_double), ("weight_cap_percentile", C.c_double)]


class ClusterCell(C.Structure):
    _fields_ = [("representative", C.c_double * 4), ("hash", C.c_uint64), ("first_index", C.c_uint32), ("count", C.c_uint32),
                ("weight", C.c_double), ("moments", C.c_double * 9)]


class FilterConfig(C.Structure):
    _fields_ = [("device", C.c_int), ("capacity", C.c_uint64), ("seed", C.c_uint64), ("first_index", C.c_uint64),
                ("global_count", C.c_uint64), ("record_ancestors", C.c_int)]


class ResampleOpts(C.Structure):
    _fields_ = [("scheme", C.c_int), ("step", C.c_uint32), ("min_particles", C.c_uint64), ("max_particles", C.c_uint64),
                ("kld_epsilon", C.c_double), ("kld_z", C.c_double), ("spatial_resolution", C.c_double * 3),
                ("random_state_probability", C.c_double)]


class AmclParam(C.Structure):
    _fields_ = [("update_min_d", C.c_double), ("update_min_a", C.c_double), ("resample_interval", C.c_uint64),
                ("selective_resampling", C.c_int), ("min_particles", C.c_uint64), ("max_particles", C.c_uint64),
                ("alpha_slow", C.c_double), ("alpha_fast", C.c_double), ("kld_epsilon", C.c_double), ("kld_z", C.c_double),
                ("spatial_resolution", C.c_double * 3), ("resample_scheme", C.c_int), ("seed", C.c_uint64), ("device", C.c_int),
                ("record_ancestors", C.c_int), ("shard_first_index", C.c_uint64), ("shard_capacity", C.c_uint64),
                ("recovery_probability_override", C.c_double)]


class StepPlan(C.Structure):
    _fields_ = [("update", C.c_int), ("resample", C.c_int), ("needs_ess", C.c_int), ("step", C.c_uint32),
                ("random_state_probability", C.c_double), ("sampling", MotionSampling), ("opts", ResampleOpts)]


class LaserScan(C.Structure):
    _fields_ = [("ranges", C.POINTER(C.c_float)), ("n_ranges", C.c_uint64), ("angle_min", C.c_float), ("angle_increment", C.c_float),
                ("min_range", C.c_double), ("max_range", C.c_double), ("max_beams", C.c_uint64), ("laser_origin", C.POINTER(C.c_double))]


POINT_FLOAT32, POINT_FLOAT64 = 7, 8  # sensor_msgs/PointField datatypes


class PointCloud(C.Structure):
    _fields_ = [("data", C.c_void_p), ("n_points", C.c_uint64), ("point_step", C.c_uint32), ("x_offset", C.c_uint32), ("datatype", C.c_int),
                ("origin", C.POINTER(C.c_double))]


class MarkerVertex(C.Structure):
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("z", C.c_double), ("r", C.c_float), ("g", C.c_float), ("b", C.c_float), ("a", C.c_float)]


MEASUREMENT_POINTS, MEASUREMENT_SCAN, MEASUREMENT_CLOUD, MEASUREMENT_WEIGHTS, MEASUREMENT_LANDMARKS = 0, 1, 2, 3, 4


class Measurement(C.Structure):
    _fields_ = [("kind", C.c_int), ("points_xy", C.POINTER(C.c_double)), ("n_points", C.c_uint64), ("scan", C.POINTER(LaserScan)),
                ("cloud", C.POINTER(PointCloud))]


class UpdateResult(C.Structure):
    _fields_ = [("updated", C.c_int), ("resampled", C.c_int), ("n_particles", C.c_uint64), ("estimate", Estimate),
                ("random_state_probability", C.c_double), ("weight_sum", C.c_double), ("weights_degenerate", C.c_int)]


class WeighView(C.Structure):
    _fields_ = [("updated", C.c_int), ("n", C.c_uint64), ("states", C.c_void_p), ("factors", C.c_void_p), ("stream", C.c_void_p)]


_P = C.POINTER
_dbl = _P(C.c_double)
_vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/beluga_b200.h declaration by declaration.
SIGNATURES = {
    "bb200_abi_version": (C.c_int, []),
    "bb200_device_count": (C.c_int, []),
    "bb200_create_error": (C.c_char_p, []),
    "bb200_filter_create": (C.c_int, [_P(FilterConfig), _P(_vp)]),
    "bb200_filter_destroy": (None, [_vp]),
    "bb200_last_error": (C.c_char_p, [_vp]),
    "bb200_filter_set_likelihood_field_map": (C.c_int, [_vp, _P(LikelihoodFieldParam), _P(OccupancyGrid), C.c_int]),
    "bb200_filter_set_beam_map": (C.c_int, [_vp, _P(BeamParam), _P(OccupancyGrid)]),
    "bb200_filter_set_landmark_map": (C.c_int, [_vp, _P(LandmarkParam), _P(LandmarkMap)]),
    "bb200_filter_set_bearing_map": (C.c_int, [_vp, _P(BearingParam), _P(LandmarkMap)]),
    "bb200_filter_reweight_landmarks": (C.c_int, [_vp, _P(Landmark), C.c_uint64]),
    "bb200_filter_get_likelihood_field": (C.c_int, [_vp, _P(C.c_float), C.c_uint64]),
    "bb200_filter_set_particles": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64]),
    "bb200_filter_size": (C.c_int, [_vp, _P(C.c_uint64)]),
    "bb200_filter_get_particles": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64]),
    "bb200_filter_initialize_normal": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64]),
    "bb200_filter_initialize_uniform": (C.c_int, [_vp, C.c_uint64]),
    "bb200_filter_propagate": (C.c_int, [_vp, _P(MotionSampling), C.c_uint32]),
    "bb200_filter_reweight": (C.c_int, [_vp, _dbl, C.c_uint64]),
    "bb200_filter_propagate_reweight": (C.c_int, [_vp, _P(MotionSampling), C.c_uint32, _dbl, C.c_uint64]),
    "bb200_filter_max_weight": (C.c_int, [_vp, _dbl]),
    "bb200_filter_build_cdf": (C.c_int, [_vp, C.c_double, _P(C.c_uint64), _P(C.c_int)]),
    "bb200_filter_normalize_by": (C.c_int, [_vp, C.c_uint64, _dbl]),
    "bb200_filter_normalize": (C.c_int, [_vp, _dbl, _dbl]),
    "bb200_filter_resample": (C.c_int, [_vp, _P(ResampleOpts), _P(C.c_uint64)]),
    "bb200_filter_resample_range": (C.c_int, [_vp, _P(ResampleOpts), C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64]),
    "bb200_filter_adopt": (C.c_int, [_vp, C.c_uint64, C.c_int]),
    "bb200_systematic_comb": (C.c_int, [C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, _P(C.c_uint64), _P(C.c_uint64)]),
    "bb200_estimate_from_moments": (C.c_int, [_dbl, _dbl, _P(Estimate)]),
    "bb200_filter_set_stream": (C.c_int, [_vp, _vp]),
    "bb200_filter_enqueue_propagate_reweight": (C.c_int, [_vp, _P(MotionSampling), C.c_uint32, _dbl, C.c_uint64]),
    "bb200_filter_enqueue_build_cdf": (C.c_int, [_vp]),
    "bb200_filter_enqueue_resample_range": (C.c_int, [_vp, _P(ResampleOpts), C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64]),
    "bb200_filter_enqueue_adopt": (C.c_int, [_vp, C.c_uint64]),
    "bb200_filter_enqueue_moments": (C.c_int, [_vp, _dbl]),
    "bb200_filter_ancestors": (C.c_int, [_vp, _P(C.c_int64), C.c_uint64]),
    "bb200_filter_cdf": (C.c_int, [_vp, _P(C.c_uint64), C.c_uint64]),
    "bb200_filter_estimate": (C.c_int, [_vp, _P(Estimate)]),
    "bb200_cluster_param_default": (None, [_P(ClusterParam)]),
    "bb200_cluster_select_host": (C.c_int, [_P(ClusterCell), C.c_uint64, C.c_uint64, _P(ClusterParam), _P(C.c_uint32), _P(C.c_uint32), _P(C.c_int),
                                            _P(C.c_uint32), _dbl]),
    "bb200_filter_cluster_estimate": (C.c_int, [_vp, _P(ClusterParam), _P(Estimate), _P(C.c_uint32), C.c_uint64, _P(C.c_uint32), _P(C.c_uint32)]),
    "bb200_filter_particle_histogram": (C.c_int, [_vp, C.c_double, C.c_double, _P(ClusterCell), C.c_uint64, _P(C.c_uint64), _dbl]),
    "bb200_filter_sample_states": (C.c_int, [_vp, C.c_uint64, C.c_uint32, _dbl]),
    "bb200_filter_cast_rays": (C.c_int, [_vp, _dbl, C.c_uint64, _dbl, C.c_uint64, C.c_double, _dbl]),
    "bb200_particle_cloud_markers": (C.c_int, [_P(ClusterCell), C.c_uint64, _P(MarkerVertex), _P(MarkerVertex), _dbl]),
    "bb200_likelihood_field_to_occupancy": (C.c_int, [_P(C.c_float), C.c_uint64, _P(C.c_int8)]),
    "bb200_filter_moments": (C.c_int, [_vp, _dbl, _dbl]),
    "bb200_filter_set_timing": (C.c_int, [_vp, C.c_int]),
    "bb200_filter_clear_timings": (C.c_int, [_vp]),
    "bb200_filter_last_timings": (C.c_int, [_vp, _P(C.c_char_p), _P(C.c_float), C.c_int]),
    "bb200_filter_launch_count": (C.c_uint64, [_vp]),
    "bb200_filter_synchronize": (C.c_int, [_vp]),
    "bb200_filter_device_pointer": (C.c_int, [_vp, C.c_int, _P(_vp), _P(C.c_uint64)]),
    "bb200_amcl_create": (C.c_int, [_P(AmclParam), _P(DiffDriveParam), _P(_vp)]),
    "bb200_amcl_destroy": (None, [_vp]),
    "bb200_amcl_last_error": (C.c_char_p, [_vp]),
    "bb200_amcl_filter": (_vp, [_vp]),
    "bb200_amcl_initialize": (C.c_int, [_vp, _dbl, _dbl]),
    "bb200_amcl_initialize_states": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64]),
    "bb200_amcl_initialize_from_map": (C.c_int, [_vp]),
    "bb200_amcl_force_update": (None, [_vp]),
    "bb200_amcl_update": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64, _P(UpdateResult)]),
    "bb200_amcl_update_landmarks": (C.c_int, [_vp, _dbl, _P(Landmark), C.c_uint64, _P(UpdateResult)]),
    "bb200_scan_to_points": (C.c_int, [_P(LaserScan), _dbl, C.c_uint64, _P(C.c_uint64)]),
    "bb200_scan_bearings": (C.c_int, [C.c_float, C.c_float, C.c_uint64, C.c_uint64, _dbl, C.c_uint64, _P(C.c_uint64)]),
    "bb200_take_evenly_indices": (C.c_int, [C.c_uint64, C.c_uint64, _P(C.c_uint64), C.c_uint64, _P(C.c_uint64)]),
    "bb200_amcl_update_scan": (C.c_int, [_vp, _dbl, _P(LaserScan), _P(UpdateResult)]),
    "bb200_point_cloud_to_points": (C.c_int, [_P(PointCloud), _dbl, C.c_uint64, _P(C.c_uint64)]),
    "bb200_amcl_update_point_cloud": (C.c_int, [_vp, _dbl, _P(PointCloud), _P(UpdateResult)]),
    "bb200_amcl_update_begin": (C.c_int, [_vp, _dbl, _P(WeighView)]),
    "bb200_amcl_batch_update_begin": (C.c_int, [_vp, _dbl, _P(Measurement), _P(C.c_uint8), _P(WeighView)]),
    "bb200_amcl_batch_update_end": (C.c_int, [_vp, _P(ClusterParam), _P(UpdateResult), _P(Estimate), _P(C.c_uint32), _P(C.c_uint32)]),
    "bb200_amcl_update_end": (C.c_int, [_vp, _P(UpdateResult)]),
    "bb200_sharded_amcl_create": (C.c_int, [_P(AmclParam), _P(MotionParam), C.c_int, _P(C.c_int), _P(_vp)]),
    "bb200_sharded_amcl_destroy": (None, [_vp]),
    "bb200_sharded_amcl_last_error": (C.c_char_p, [_vp]),
    "bb200_sharded_amcl_shards": (C.c_int, [_vp]),
    "bb200_sharded_amcl_shard": (_vp, [_vp, C.c_int]),
    "bb200_sharded_amcl_set_likelihood_field_map": (C.c_int, [_vp, _P(LikelihoodFieldParam), _P(OccupancyGrid), C.c_int]),
    "bb200_sharded_amcl_set_beam_map": (C.c_int, [_vp, _P(BeamParam), _P(OccupancyGrid)]),
    "bb200_sharded_amcl_set_landmark_map": (C.c_int, [_vp, _P(LandmarkParam), _P(LandmarkMap)]),
    "bb200_sharded_amcl_set_bearing_map": (C.c_int, [_vp, _P(BearingParam), _P(LandmarkMap)]),
    "bb200_sharded_amcl_initialize": (C.c_int, [_vp, _dbl, _dbl]),
    "bb200_sharded_amcl_initialize_from_map": (C.c_int, [_vp]),
    "bb200_sharded_amcl_force_update": (None, [_vp]),
    "bb200_sharded_amcl_update": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64, _P(UpdateResult)]),
    "bb200_sharded_amcl_update_landmarks": (C.c_int, [_vp, _dbl, _P(Landmark), C.c_uint64, _P(UpdateResult)]),
    "bb200_sharded_amcl_update_begin": (C.c_int, [_vp, _dbl, _P(WeighView)]),
    "bb200_sharded_amcl_update_end": (C.c_int, [_vp, _P(UpdateResult)]),
    "bb200_sharded_amcl_get_particles": (C.c_int, [_vp, _dbl, _dbl, C.c_uint64]),
    "bb200_sharded_amcl_cluster_estimate": (C.c_int, [_vp, _P(ClusterParam), _P(Estimate), _P(C.c_uint32), _P(C.c_uint32)]),
    "bb200_sharded_amcl_update_scan": (C.c_int, [_vp, _dbl, _P(LaserScan), _P(UpdateResult)]),
    "bb200_sharded_amcl_update_point_cloud": (C.c_int, [_vp, _dbl, _P(PointCloud), _P(UpdateResult)]),
    "bb200_sharded_amcl_particle_histogram": (C.c_int, [_vp, C.c_double, C.c_double, _P(ClusterCell), C.c_uint64, _P(C.c_uint64), _dbl]),
    "bb200_sharded_amcl_sample_states": (C.c_int, [_vp, C.c_uint64, C.c_uint32, _dbl]),
    "bb200_sharded_amcl_cast_rays": (C.c_int, [_vp, _dbl, C.c_uint64, _dbl, C.c_uint64, C.c_double, _dbl]),
    "bb200_cluster_merge_host": (C.c_int, [_P(_P(ClusterCell)), _P(C.c_uint64), _P(C.c_uint64), C.c_int, _P(ClusterCell), C.c_uint64, _P(C.c_uint64)]),
    "bb200_amcl_export_shard": (C.c_int, [_vp, _vp]),
    "bb200_amcl_join_shards": (C.c_int, [_vp, C.c_int, C.c_int, _vp]),
    "bb200_amcl_leave_shards": (C.c_int, [_vp]),
    "bb200_amcl_batch_create": (C.c_int, [_P(AmclParam), _P(MotionParam), C.c_int, _P(_vp)]),
    "bb200_amcl_batch_create_adaptive": (C.c_int, [_P(AmclParam), _P(MotionParam), C.c_int, _P(_vp)]),
    "bb200_amcl_batch_create_with_flags": (C.c_int, [_P(AmclParam), _P(MotionParam), C.c_int, C.c_uint32, _P(_vp)]),
    "bb200_amcl_batch_member_size": (C.c_int, [_vp, C.c_int, _P(C.c_uint64)]),
    "bb200_amcl_batch_destroy": (None, [_vp]),
    "bb200_amcl_batch_last_error": (C.c_char_p, [_vp]),
    "bb200_amcl_batch_members": (C.c_int, [_vp]),
    "bb200_amcl_batch_set_likelihood_field_map": (C.c_int, [_vp, _P(LikelihoodFieldParam), _P(OccupancyGrid), C.c_int]),
    "bb200_amcl_batch_set_beam_map": (C.c_int, [_vp, _P(BeamParam), _P(OccupancyGrid)]),
    "bb200_amcl_batch_add_likelihood_field_map": (C.c_int, [_vp, _P(LikelihoodFieldParam), _P(OccupancyGrid), C.c_int, _P(C.c_int)]),
    "bb200_amcl_batch_add_beam_map": (C.c_int, [_vp, _P(BeamParam), _P(OccupancyGrid), _P(C.c_int)]),
    "bb200_amcl_batch_set_landmark_map": (C.c_int, [_vp, _P(LandmarkParam), _P(LandmarkMap)]),
    "bb200_amcl_batch_set_bearing_map": (C.c_int, [_vp, _P(BearingParam), _P(LandmarkMap)]),
    "bb200_amcl_batch_add_landmark_map": (C.c_int, [_vp, _P(LandmarkParam), _P(LandmarkMap), _P(C.c_int)]),
    "bb200_amcl_batch_add_bearing_map": (C.c_int, [_vp, _P(BearingParam), _P(LandmarkMap), _P(C.c_int)]),
    "bb200_amcl_batch_set_detections": (C.c_int, [_vp, _P(_P(Landmark)), _P(C.c_uint64), _P(C.c_uint8)]),
    "bb200_amcl_batch_update_map": (C.c_int, [_vp, C.c_int, C.c_int]),
    "bb200_amcl_batch_member_map": (C.c_int, [_vp, C.c_int, _P(C.c_int)]),
    "bb200_amcl_batch_remove_map": (C.c_int, [_vp, C.c_int]),
    "bb200_amcl_batch_get_likelihood_field": (C.c_int, [_vp, C.c_int, _P(C.c_float), C.c_uint64]),
    "bb200_amcl_batch_initialize": (C.c_int, [_vp, C.c_int, _dbl, _dbl]),
    "bb200_amcl_batch_initialize_from_map": (C.c_int, [_vp, C.c_int]),
    "bb200_amcl_batch_initialize_states": (C.c_int, [_vp, C.c_int, _dbl, _dbl, C.c_uint64]),
    "bb200_amcl_batch_force_update": (C.c_int, [_vp, C.c_int]),
    "bb200_amcl_batch_get_particles": (C.c_int, [_vp, C.c_int, _dbl, _dbl, C.c_uint64]),
    "bb200_amcl_batch_ancestors": (C.c_int, [_vp, C.c_int, _P(C.c_int64), C.c_uint64]),
    "bb200_amcl_batch_cluster_estimate": (C.c_int, [_vp, C.c_int, _P(ClusterParam), _P(Estimate)]),
    "bb200_amcl_batch_cluster_estimates": (C.c_int, [_vp, _P(ClusterParam), _P(C.c_uint8), _P(Estimate), _P(C.c_uint32), _P(C.c_uint32)]),
    "bb200_amcl_batch_particle_histograms": (C.c_int, [_vp, C.c_double, C.c_double, _P(C.c_uint8), _P(_P(ClusterCell)), _P(C.c_uint64),
                                                       _P(C.c_uint64), _dbl]),
    "bb200_amcl_batch_sample_states": (C.c_int, [_vp, _P(C.c_uint64), C.c_uint32, _P(C.c_uint8), _P(_dbl)]),
    "bb200_amcl_batch_cast_rays": (C.c_int, [_vp, _P(C.c_uint8), _P(C.c_int), _P(_dbl), _P(C.c_uint64), _P(_dbl), _P(C.c_uint64), _dbl, _P(_dbl)]),
    "bb200_amcl_batch_update": (C.c_int, [_vp, _dbl, _P(_dbl), _P(C.c_uint64), _P(C.c_uint8), _P(UpdateResult)]),
    "bb200_amcl_batch_update_measurements": (C.c_int, [_vp, _dbl, _P(Measurement), _P(C.c_uint8), _P(UpdateResult)]),
    "bb200_amcl_batch_update_clustered": (C.c_int, [_vp, _dbl, _P(Measurement), _P(C.c_uint8), _P(ClusterParam), _P(UpdateResult), _P(Estimate),
                                                    _P(C.c_uint32), _P(C.c_uint32)]),
    "bb200_amcl_batch_launch_count": (C.c_uint64, [_vp]),
    "bb200_amcl_batch_add_member": (C.c_int, [_vp, _P(AmclParam), _P(MotionParam), _P(C.c_int)]),
    "bb200_amcl_batch_remove_member": (C.c_int, [_vp, C.c_int]),
    "bb200_amcl_batch_member_active": (C.c_int, [_vp, C.c_int, _P(C.c_int)]),
    "bb200_amcl_batch_export_members": (C.c_int, [_vp, _P(C.c_uint8), _P(_vp), _P(C.c_uint64), _P(C.c_uint64)]),
    "bb200_amcl_batch_export_member": (C.c_int, [_vp, C.c_int, _vp, C.c_uint64, _P(C.c_uint64)]),
    "bb200_amcl_batch_import_member": (C.c_int, [_vp, _vp, C.c_uint64, C.c_int, _P(C.c_int)]),
    "bb200_amcl_batch_create_from_states": (C.c_int, [_P(_vp), _P(C.c_uint64), C.c_int, C.c_uint32, C.c_int, _P(_vp)]),
    "bb200_amcl_export_state": (C.c_int, [_vp, _vp, C.c_uint64, _P(C.c_uint64)]),
    "bb200_amcl_create_from_state": (C.c_int, [_vp, C.c_uint64, C.c_int, _P(_vp)]),
    "bb200_amcl_state_params": (C.c_int, [_vp, C.c_uint64, _P(AmclParam), _P(MotionParam)]),
    "bb200_amcl_plan_update": (C.c_int, [_vp, _dbl, _P(StepPlan)]),
    "bb200_amcl_commit_update": (None, [_vp, C.c_int, C.c_double]),
    "bb200_amcl_create_with_motion": (C.c_int, [_P(AmclParam), _P(MotionParam), _P(_vp)]),
    "bb200_motion_sampling_from_control": (C.c_int, [_P(MotionParam), _dbl, _dbl, _P(MotionSampling)]),
    "bb200_diff_drive_sampling_from_control": (C.c_int, [_P(DiffDriveParam), _dbl, _dbl, _P(DiffDriveSampling)]),
}

_lib = None


def load() -> C.CDLL:
    """Loads libbeluga_b200.so.  Raises if it has not been built (python -m beluga_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OSError(f"{LIB_PATH} is missing: build it with `python -m beluga_b200.build` (there is no fallback path)")
        lib = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib
