"""beluga_b200 -- H100-native (sm_90a) backend for the MCL particle-filter update of Ekumen-OS/beluga.

The product is `libbeluga_b200.so` (hand-written sm_90a CUDA kernels behind the C ABI of
`include/beluga_b200.h`) plus the header-only C++ adaptors in `include/beluga_b200/` that give it
beluga's MotionModel / SensorModel / Amcl shapes.  This package is the thin Python view of the same
C ABI used by the tests and by bench.py; names follow the reference:

    reference (C++)                                         here
    ------------------------------------------------------  --------------------------------------
    beluga::Amcl<...> (algorithm/amcl_core.hpp:81)          Amcl
    Amcl::initialize(pose, covariance)  (:145)              Amcl.initialize(mean_xytheta, cov)
    Amcl::update(control, measurement)  (:165)              Amcl.update(control_pose, points)
    beluga_ros::Amcl::update(pose, laser_scan / cloud)      Amcl.update_scan(...) / Amcl.update_point_cloud(...)
    Amcl::update_map(map)               (:150)              Amcl.update_map(...)
    Amcl::particles()                   (:128)              Amcl.particles()
    DifferentialDriveModelParam                             DifferentialDriveModelParam
    LikelihoodFieldModelParam / BeamModelParam              LikelihoodFieldModelParam / BeamModelParam
    AmclParams                                              AmclParams

No computation happens in Python and there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _capi
from ._capi import (RESAMPLE_MULTINOMIAL, RESAMPLE_SYSTEMATIC, SENSOR_BEAM, SENSOR_BEARING, SENSOR_LANDMARK, SENSOR_LIKELIHOOD_FIELD,
                    SENSOR_LIKELIHOOD_FIELD_PROB)

__all__ = [
    "Amcl", "AmclBatch", "AmclParams", "BeamModelParam", "DifferentialDriveModelParam", "OmnidirectionalDriveModelParam", "StationaryModelParam",
    "Filter", "LikelihoodFieldModelParam", "motion_sampling", "scan_to_points", "scan_bearings", "point_cloud_to_points",
    "take_evenly_indices",
    "OccupancyGrid", "BelugaB200Error", "device_count", "se2", "LaserScan", "PointCloud",
    "LandmarkModelParam", "BearingModelParam", "LandmarkMap", "Detections", "RESAMPLE_MULTINOMIAL", "RESAMPLE_SYSTEMATIC", "SENSOR_BEAM", "SENSOR_BEARING", "SENSOR_LANDMARK", "SENSOR_LIKELIHOOD_FIELD", "SENSOR_LIKELIHOOD_FIELD_PROB",
]


class BelugaB200Error(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"[bb200 status {status}] {message}")
        self.status = status


def device_count() -> int:
    return _capi.load().bb200_device_count()


def se2(x: float, y: float, theta: float) -> np.ndarray:
    """Sophus::SE2d{theta, (x, y)} in data() order (cos, sin, x, y), normalised through hypot."""
    c, s = np.cos(theta), np.sin(theta)
    n = np.hypot(c, s)
    return np.array([c / n, s / n, x, y], dtype=np.float64)


def systematic_comb(seed: int, step: int, global_total: int, total_slots: int):
    """(stride, offset) of the systematic resampling comb over a fixed-point CDF with the given total."""
    stride, offset = C.c_uint64(), C.c_uint64()
    st = _capi.load().bb200_systematic_comb(seed, step, global_total, total_slots, C.byref(stride), C.byref(offset))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_systematic_comb")
    return stride.value, offset.value


def cluster_select_host(cells, n_particles: int, linear: float = 0.20, angular: float = 0.524, percentile: float = 0.90):
    """Host half of the cluster-based estimate (bb200_cluster_select_host) on a list of cell records
    (representative[4], hash, first_index, count, weight, moments[9]) in first-occurrence order.
    -> (cluster id per cell, number of clusters, found, best, moments[9])."""
    lib = _capi.load()
    arr = (_capi.ClusterCell * max(len(cells), 1))()
    for k, (rep, h, first, count, weight, moments) in enumerate(cells):
        arr[k].representative[:] = list(rep)
        arr[k].hash, arr[k].first_index, arr[k].count, arr[k].weight = int(h), int(first), int(count), float(weight)
        arr[k].moments[:] = list(moments)
    ids = (C.c_uint32 * max(len(cells), 1))()
    n_clusters, found, best = C.c_uint32(0), C.c_int(0), C.c_uint32(0)
    out = np.zeros(9)
    p = _capi.ClusterParam(linear, angular, percentile)
    st = lib.bb200_cluster_select_host(arr, len(cells), n_particles, C.byref(p), ids, C.byref(n_clusters), C.byref(found), C.byref(best), _dptr(out))
    if st != 0:
        raise RuntimeError(f"bb200_cluster_select_host: status {st}")
    return np.array(ids[: len(cells)], dtype=np.uint32), n_clusters.value, bool(found.value), best.value, out


def particle_cloud_markers(bins):
    """Host half of assign_particle_cloud(..., MarkerArray) (beluga_ros/particle_cloud.hpp:212-294) on histogram bins
    (representative[4], weight): -> (bodies [2n, 7], heads [3n, 7], body_scale_x); columns x, y, z, r, g, b, a."""
    lib = _capi.load()
    n = len(bins)
    arr = (_capi.ClusterCell * max(n, 1))()
    for k, (rep, weight) in enumerate(bins):
        arr[k].representative[:] = list(rep)
        arr[k].weight = float(weight)
    bodies = (_capi.MarkerVertex * max(2 * n, 1))()
    heads = (_capi.MarkerVertex * max(3 * n, 1))()
    scale = C.c_double(0.0)
    st = lib.bb200_particle_cloud_markers(arr, n, bodies, heads, C.byref(scale))
    if st != 0:
        raise RuntimeError(f"bb200_particle_cloud_markers: status {st}")
    unpack = lambda vs, m: np.array([[v.x, v.y, v.z, v.r, v.g, v.b, v.a] for v in vs[:m]]).reshape(m, 7)  # noqa: E731
    return unpack(bodies, 2 * n), unpack(heads, 3 * n), scale.value


def likelihood_field_to_occupancy(field) -> np.ndarray:
    """assign_likelihood_field (beluga_ros/likelihood_field.hpp:44-79): float field -> int8 cells in [0, 100]."""
    lib = _capi.load()
    f = np.ascontiguousarray(field, dtype=np.float32)
    out = np.zeros(f.shape, dtype=np.int8)
    st = lib.bb200_likelihood_field_to_occupancy(f.ctypes.data_as(C.POINTER(C.c_float)), f.size, out.ctypes.data_as(C.POINTER(C.c_int8)))
    if st != 0:
        raise RuntimeError(f"bb200_likelihood_field_to_occupancy: status {st}")
    return out


def estimate_from_moments(moments, pivot):
    """beluga::estimate (algorithm/estimation.hpp:436-475) from globally summed raw moments."""
    e = _capi.Estimate()
    m, p = _f64(moments), _f64(pivot)
    st = _capi.load().bb200_estimate_from_moments(m.ctypes.data_as(C.POINTER(C.c_double)), p.ctypes.data_as(C.POINTER(C.c_double)), C.byref(e))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_estimate_from_moments")
    return np.array(e.mean), np.array(e.cov).reshape(3, 3)


def take_evenly_indices(size: int, count: int) -> np.ndarray:
    """beluga::views::take_evenly (views/take_evenly.hpp): indices kept out of `size` elements."""
    out = np.zeros(max(size, 1), dtype=np.uint64)
    n = C.c_uint64()
    st = _capi.load().bb200_take_evenly_indices(size, count, out.ctypes.data_as(C.POINTER(C.c_uint64)), len(out), C.byref(n))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_take_evenly_indices")
    return out[: n.value].astype(np.int64)


def _laser_scan(ranges, angle_min, angle_increment, min_range, max_range, max_beams, laser_origin):
    r = np.ascontiguousarray(ranges, dtype=np.float32)
    origin = None if laser_origin is None else _f64(laser_origin).reshape(12)
    scan = _capi.LaserScan(r.ctypes.data_as(C.POINTER(C.c_float)), len(r), angle_min, angle_increment, min_range, max_range, max_beams,
                           None if origin is None else origin.ctypes.data_as(C.POINTER(C.c_double)))
    return scan, (r, origin)  # keep the arrays alive


def scan_to_points(ranges, angle_min: float, angle_increment: float, min_range: float = 0.0, max_range: float = float("inf"),
                   max_beams: int = 0, laser_origin=None) -> np.ndarray:
    """beluga_ros::LaserScan + BaseLaserScan::points_in_cartesian_coordinates + laser-to-base transform
    (beluga_ros/laser_scan.hpp:69-80, beluga/sensor/data/laser_scan.hpp:64-91, beluga_ros/src/amcl.cpp:57-62)."""
    scan, keep = _laser_scan(ranges, angle_min, angle_increment, min_range, max_range, max_beams, laser_origin)
    out = np.zeros((len(keep[0]) + 1, 2))
    n = C.c_uint64()
    st = _capi.load().bb200_scan_to_points(C.byref(scan), _dptr(out), len(out), C.byref(n))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_scan_to_points")
    return out[: n.value]


def scan_bearings(angle_min: float, angle_increment: float, n_ranges: int, max_beams: int = 0) -> np.ndarray:
    """The (n, 2) directions [cos, sin] of the beams a laser scan of this geometry keeps (take_evenly(max_beams)), exactly as
    scan_to_points computes them and without dropping readings by range: the bearings of the scan's expected ranges
    (Filter.cast_rays)."""
    lib = _capi.load()
    n = C.c_uint64()
    st = lib.bb200_scan_bearings(angle_min, angle_increment, n_ranges, max_beams, None, 0, C.byref(n))
    if st not in (_capi.OK, _capi.ERR_CAPACITY):
        raise BelugaB200Error(st, "bb200_scan_bearings")
    out = np.zeros((n.value, 2))
    st = lib.bb200_scan_bearings(angle_min, angle_increment, n_ranges, max_beams, _dptr(out) if n.value else None, n.value, C.byref(n))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_scan_bearings")
    return out


def _rays(poses, bearings):
    """Contiguous (n, 4) poses and (m, 2) bearings for a ray cast."""
    return _f64(poses).reshape(-1, 4), _f64(bearings).reshape(-1, 2)


def _point_cloud(data, point_step: int, x_offset: int, dtype, origin, n_points):
    if isinstance(data, np.ndarray):
        raw = np.ascontiguousarray(data).reshape(-1).view(np.uint8)
    else:
        raw = np.frombuffer(data, dtype=np.uint8)
    if n_points is None:
        n_points = len(raw) // point_step if point_step > 0 else 0
    if n_points * point_step > len(raw):
        raise ValueError(f"{n_points} points of {point_step} bytes do not fit in {len(raw)} bytes")
    if isinstance(dtype, (int, np.integer)):
        datatype = int(dtype)
    else:  # any other numpy type is not a coordinate type: 0 makes the library reject it
        datatype = {np.dtype(np.float32): _capi.POINT_FLOAT32, np.dtype(np.float64): _capi.POINT_FLOAT64}.get(np.dtype(dtype), 0)
    o = None if origin is None else _f64(origin).reshape(12)
    cloud = _capi.PointCloud(raw.ctypes.data if len(raw) else None, n_points, point_step, x_offset, datatype,
                             None if o is None else o.ctypes.data_as(C.POINTER(C.c_double)))
    return cloud, (raw, o)  # keep the buffers alive


def point_cloud_to_points(data, point_step: int, x_offset: int, dtype, origin=None, n_points: int | None = None) -> np.ndarray:
    """beluga_ros::SparsePointCloud3f::points() moved into the base frame (beluga_ros/include/beluga_ros/sparse_point_cloud.hpp:102-125,
    beluga_ros/src/amcl.cpp:67-81): the (x, y) of every point of a packed PointCloud2 buffer, in order, NaN points included.

    `data`: the message's bytes (bytes, bytearray, memoryview or any contiguous numpy array, structured ones included);
    `dtype`: the x/y/z field type, a PointField code (7 FLOAT32, 8 FLOAT64) or a numpy type; `origin`: 3x4 [R | t] of the cloud's
    frame in the base frame, None for the identity; `n_points`: width * height, by default as many points as the buffer holds."""
    cloud, keep = _point_cloud(data, point_step, x_offset, dtype, origin, n_points)
    out = np.zeros((max(cloud.n_points, 1), 2))
    n = C.c_uint64()
    st = _capi.load().bb200_point_cloud_to_points(C.byref(cloud), _dptr(out), cloud.n_points, C.byref(n))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_point_cloud_to_points: datatype must be 7 (FLOAT32) or 8 (FLOAT64) and x, y, z must fit in point_step")
    return out[: n.value]


@dataclass
class LaserScan:
    """A laser scan as Amcl.update_scan takes it (sensor_msgs/LaserScan with the node's range limits and max_beams), one member's
    measurement in AmclBatch.update_measurements."""
    ranges: object
    angle_min: float
    angle_increment: float
    min_range: float = 0.0
    max_range: float = float("inf")
    max_beams: int = 0
    laser_origin: object = None


@dataclass
class PointCloud:
    """A packed PointCloud2 buffer as Amcl.update_point_cloud takes it (arguments as point_cloud_to_points), one member's
    measurement in AmclBatch.update_measurements."""
    data: object
    point_step: int
    x_offset: int
    dtype: object
    origin: object = None
    n_points: int | None = None


def _measurement(m):
    """bb200_measurement of a LaserScan, a PointCloud or an (n, 2) array of points, and the objects that must outlive the call."""
    if isinstance(m, LaserScan):
        scan, keep = _laser_scan(m.ranges, m.angle_min, m.angle_increment, m.min_range, m.max_range, m.max_beams, m.laser_origin)
        return _capi.Measurement(_capi.MEASUREMENT_SCAN, None, 0, C.pointer(scan), None), (scan, keep)
    if isinstance(m, PointCloud):
        cloud, keep = _point_cloud(m.data, m.point_step, m.x_offset, m.dtype, m.origin, m.n_points)
        return _capi.Measurement(_capi.MEASUREMENT_CLOUD, None, 0, None, C.pointer(cloud)), (cloud, keep)
    pts = _f64(m).reshape(-1, 2)
    return _capi.Measurement(_capi.MEASUREMENT_POINTS, _dptr(pts) if len(pts) else None, len(pts), None, None), pts


@dataclass
class Detections:
    """One member's landmark detections in AmclBatch.update_measurements, update_clustered and update_weighted, as
    Amcl.update_landmarks takes them: (n, 3) positions in the robot frame (SENSOR_LANDMARK) or bearings in the sensor frame
    (SENSOR_BEARING), and n categories."""
    positions: object
    categories: object


def _dptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _f64(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float64)


@dataclass
class DifferentialDriveModelParam:
    """beluga::DifferentialDriveModelParam (motion/differential_drive_model.hpp:40-68)."""
    rotation_noise_from_rotation: float = 0.0
    rotation_noise_from_translation: float = 0.0
    translation_noise_from_translation: float = 0.0
    translation_noise_from_rotation: float = 0.0
    distance_threshold: float = 0.01

    def c(self) -> _capi.DiffDriveParam:
        return _capi.DiffDriveParam(self.rotation_noise_from_rotation, self.rotation_noise_from_translation,
                                    self.translation_noise_from_translation, self.translation_noise_from_rotation,
                                    self.distance_threshold)


    def c_motion(self) -> _capi.MotionParam:
        return _capi.MotionParam(_capi.MOTION_DIFFERENTIAL, self.rotation_noise_from_rotation, self.rotation_noise_from_translation,
                                 self.translation_noise_from_translation, self.translation_noise_from_rotation, 0.0, self.distance_threshold)


@dataclass
class OmnidirectionalDriveModelParam:
    """beluga::OmnidirectionalDriveModelParam (motion/omnidirectional_drive_model.hpp:36-68)."""
    rotation_noise_from_rotation: float = 0.0
    rotation_noise_from_translation: float = 0.0
    translation_noise_from_translation: float = 0.0
    translation_noise_from_rotation: float = 0.0
    strafe_noise_from_translation: float = 0.0
    distance_threshold: float = 0.01

    def c_motion(self) -> _capi.MotionParam:
        return _capi.MotionParam(_capi.MOTION_OMNIDIRECTIONAL, self.rotation_noise_from_rotation, self.rotation_noise_from_translation,
                                 self.translation_noise_from_translation, self.translation_noise_from_rotation,
                                 self.strafe_noise_from_translation, self.distance_threshold)


@dataclass
class StationaryModelParam:
    """beluga::StationaryModel (motion/stationary_model.hpp:39-62) has no parameters."""

    def c_motion(self) -> _capi.MotionParam:
        return _capi.MotionParam(_capi.MOTION_STATIONARY, 0.0, 0.0, 0.0, 0.0, 0.0, 0.01)


def motion_sampling(motion, pose, previous_pose) -> _capi.MotionSampling:
    """MotionModel::operator()(control): the per-step sampling parameters of any of the three models."""
    out = _capi.MotionSampling()
    p = motion.c_motion()
    st = _capi.load().bb200_motion_sampling_from_control(C.byref(p), _dptr(_f64(pose)), _dptr(_f64(previous_pose)), C.byref(out))
    if st != _capi.OK:
        raise BelugaB200Error(st, "bb200_motion_sampling_from_control")
    return out


@dataclass
class LikelihoodFieldModelParam:
    """beluga::LikelihoodFieldModelParam (sensor/likelihood_field_model_base.hpp:42-64)."""
    max_obstacle_distance: float = 100.0
    max_laser_distance: float = 2.0
    z_hit: float = 0.5
    z_random: float = 0.5
    sigma_hit: float = 0.2
    model_unknown_space: bool = False
    only_obstacle_boundaries: bool = False

    def c(self) -> _capi.LikelihoodFieldParam:
        return _capi.LikelihoodFieldParam(self.max_obstacle_distance, self.max_laser_distance, self.z_hit, self.z_random,
                                          self.sigma_hit, int(self.model_unknown_space), int(self.only_obstacle_boundaries))


@dataclass
class BeamModelParam:
    """beluga::BeamModelParam (sensor/beam_model.hpp:43-58)."""
    z_hit: float = 0.5
    z_short: float = 0.5
    z_max: float = 0.05
    z_rand: float = 0.05
    sigma_hit: float = 0.2
    lambda_short: float = 0.1
    beam_max_range: float = 60.0

    def c(self) -> _capi.BeamParam:
        return _capi.BeamParam(self.z_hit, self.z_short, self.z_max, self.z_rand, self.sigma_hit, self.lambda_short, self.beam_max_range)


@dataclass
class LandmarkModelParam:
    """beluga::LandmarkModelParam (sensor/landmark_sensor_model.hpp:44-48)."""
    sigma_range: float = 1.0
    sigma_bearing: float = 1.0
    random_prob: float = 1e-4

    def c(self) -> _capi.LandmarkParam:
        return _capi.LandmarkParam(self.sigma_range, self.sigma_bearing, self.random_prob)


@dataclass
class BearingModelParam:
    """beluga::BearingModelParam (sensor/bearing_sensor_model.hpp:42-45); sensor_pose_in_robot is a 3x4 [R | t]."""
    sigma_bearing: float = 1.0
    sensor_pose_in_robot: object = None  # None: the identity

    def c(self) -> _capi.BearingParam:
        m = np.eye(3, 4) if self.sensor_pose_in_robot is None else _f64(self.sensor_pose_in_robot).reshape(3, 4)
        return _capi.BearingParam(self.sigma_bearing, (C.c_double * 12)(*m.reshape(12)))


def _landmark_array(positions, categories):
    pos = _f64(positions).reshape(-1, 3)
    cat = np.ascontiguousarray(categories, dtype=np.uint32).reshape(-1)
    if len(cat) != len(pos):
        raise ValueError("one category per position")
    arr = (_capi.Landmark * max(len(pos), 1))()
    for k in range(len(pos)):
        arr[k] = _capi.Landmark(pos[k, 0], pos[k, 1], pos[k, 2], int(cat[k]))
    return arr, len(pos)


class LandmarkMap:
    """beluga::LandmarkMap (sensor/data/landmark_map.hpp:40-166): (n, 3) world positions and n categories, with explicit
    bounds {x, y, z} or, when both are None, the landmarks' own (:61-71)."""

    def __init__(self, positions, categories, bounds_min=None, bounds_max=None):
        self.landmarks, self.n = _landmark_array(positions, categories)
        self.bounds_min = None if bounds_min is None else _f64(bounds_min).reshape(3)
        self.bounds_max = None if bounds_max is None else _f64(bounds_max).reshape(3)

    def c(self) -> _capi.LandmarkMap:
        lo = None if self.bounds_min is None else _dptr(self.bounds_min)
        hi = None if self.bounds_max is None else _dptr(self.bounds_max)
        return _capi.LandmarkMap(self.landmarks, self.n, lo, hi)


@dataclass
class AmclParams:
    """beluga::AmclParams (algorithm/amcl_core.hpp:34-55) + spatial hash resolutions + backend knobs."""
    update_min_d: float = 0.25
    update_min_a: float = 0.2
    resample_interval: int = 1
    selective_resampling: bool = False
    min_particles: int = 500
    max_particles: int = 2000
    alpha_slow: float = 0.001
    alpha_fast: float = 0.1
    kld_epsilon: float = 0.05
    kld_z: float = 3.0
    spatial_resolution: tuple = (0.5, 0.5, float(np.deg2rad(10.0)))  # beluga_ros/amcl.hpp:91-97
    resample_scheme: int = RESAMPLE_MULTINOMIAL
    seed: int = 0
    device: int = 0
    record_ancestors: bool = False
    shard_first_index: int = 0  # sharded filters: global index of this rank's first particle
    shard_capacity: int = 0     # ... and its particle count (0: single GPU); max_particles is then the global count
    recovery_probability_override: float = 0.0  # > 0: random_intersperse with this probability instead of the estimator's

    def c(self) -> _capi.AmclParam:
        return _capi.AmclParam(self.update_min_d, self.update_min_a, self.resample_interval, int(self.selective_resampling),
                               self.min_particles, self.max_particles, self.alpha_slow, self.alpha_fast, self.kld_epsilon,
                               self.kld_z, (C.c_double * 3)(*self.spatial_resolution), self.resample_scheme, self.seed,
                               self.device, int(self.record_ancestors), self.shard_first_index, self.shard_capacity,
                               self.recovery_probability_override)


def state_params(blob: bytes):
    """The parameters of a state blob (bb200_amcl_state_params, no device needed) -> (AmclParams, motion model param)."""
    lib = _capi.load()
    p, m = _capi.AmclParam(), _capi.MotionParam()
    st = lib.bb200_amcl_state_params(blob, len(blob), C.byref(p), C.byref(m))
    if st != _capi.OK:
        raise BelugaB200Error(st, lib.bb200_create_error().decode())
    params = AmclParams(p.update_min_d, p.update_min_a, p.resample_interval, bool(p.selective_resampling), p.min_particles,
                        p.max_particles, p.alpha_slow, p.alpha_fast, p.kld_epsilon, p.kld_z, tuple(p.spatial_resolution),
                        p.resample_scheme, p.seed, p.device, bool(p.record_ancestors), p.shard_first_index, p.shard_capacity,
                        p.recovery_probability_override)
    noise = (m.rotation_noise_from_rotation, m.rotation_noise_from_translation, m.translation_noise_from_translation,
             m.translation_noise_from_rotation)
    if m.model == _capi.MOTION_OMNIDIRECTIONAL:
        motion = OmnidirectionalDriveModelParam(*noise, m.strafe_noise_from_translation, m.distance_threshold)
    elif m.model == _capi.MOTION_STATIONARY:
        motion = StationaryModelParam()
    else:
        motion = DifferentialDriveModelParam(*noise, m.distance_threshold)
    return params, motion


@dataclass
class OccupancyGrid:
    """Occupancy grid with ROS trinary values: int8 [height, width], 0 free / 100 occupied / -1 unknown."""
    cells: np.ndarray
    resolution: float = 1.0
    origin: np.ndarray = field(default_factory=lambda: np.array([1.0, 0.0, 0.0, 0.0]))

    def __post_init__(self):
        c = np.asarray(self.cells)
        if c.dtype == np.bool_:
            c = np.where(c, 100, 0)
        self.cells = np.ascontiguousarray(c, dtype=np.int8)
        self.origin = _f64(self.origin)

    def c(self) -> _capi.OccupancyGrid:
        return _capi.OccupancyGrid(self.cells.ctypes.data_as(C.POINTER(C.c_int8)), self.cells.shape[1], self.cells.shape[0],
                                   float(self.resolution), (C.c_double * 4)(*self.origin))


class Filter:
    """bb200_filter: the device-resident particle set and the per-step kernels."""

    def __init__(self, capacity: int | None = None, seed: int = 0, device: int = 0, first_index: int = 0, global_count: int = 0,
                 record_ancestors: bool = False, _handle=None, _owner=None):
        self._lib = _capi.load()
        self._owner = _owner
        if _handle is not None:
            self._h = C.c_void_p(_handle)
            return
        cfg = _capi.FilterConfig(device, capacity, seed, first_index, global_count, int(record_ancestors))
        h = C.c_void_p()
        st = self._lib.bb200_filter_create(C.byref(cfg), C.byref(h))
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_create_error().decode())
        self._h = h

    def close(self):
        if getattr(self, "_h", None) and self._owner is None:
            self._lib.bb200_filter_destroy(self._h)
        self._h = None

    def __del__(self):
        self.close()

    def _check(self, st: int):
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_last_error(self._h).decode())

    # maps
    def set_likelihood_field_map(self, params: LikelihoodFieldModelParam, grid: OccupancyGrid, prob: bool = False):
        p, g = params.c(), grid.c()
        self._grid_shape = grid.cells.shape
        self._check(self._lib.bb200_filter_set_likelihood_field_map(self._h, C.byref(p), C.byref(g), int(prob)))

    def set_beam_map(self, params: BeamModelParam, grid: OccupancyGrid):
        p, g = params.c(), grid.c()
        self._grid_shape = grid.cells.shape
        self._check(self._lib.bb200_filter_set_beam_map(self._h, C.byref(p), C.byref(g)))

    def set_landmark_map(self, params: LandmarkModelParam, landmark_map: LandmarkMap):
        """LandmarkSensorModel2d on `landmark_map`; replaces the map set before, of any model."""
        p, m = params.c(), landmark_map.c()
        self._check(self._lib.bb200_filter_set_landmark_map(self._h, C.byref(p), C.byref(m)))

    def set_bearing_map(self, params: BearingModelParam, landmark_map: LandmarkMap):
        """BearingSensorModel2d on `landmark_map`; replaces the map set before, of any model."""
        p, m = params.c(), landmark_map.c()
        self._check(self._lib.bb200_filter_set_bearing_map(self._h, C.byref(p), C.byref(m)))

    def reweight_landmarks(self, positions, categories):
        """w *= L(state) of the landmark map's model for the detections: (n, 3) positions in the robot frame (landmark
        model) or bearings in the sensor frame (bearing model), and n categories."""
        arr, n = _landmark_array(positions, categories)
        self._check(self._lib.bb200_filter_reweight_landmarks(self._h, arr, n))

    def likelihood_field(self) -> np.ndarray:
        out = np.zeros(self._grid_shape, dtype=np.float32)
        self._check(self._lib.bb200_filter_get_likelihood_field(self._h, out.ctypes.data_as(C.POINTER(C.c_float)), out.size))
        return out

    # particles
    def set_particles(self, states, weights=None):
        st = _f64(states).reshape(-1, 4)
        w = None if weights is None else _f64(weights)
        self._check(self._lib.bb200_filter_set_particles(self._h, _dptr(st), None if w is None else _dptr(w), len(st)))

    def size(self) -> int:
        n = C.c_uint64()
        self._check(self._lib.bb200_filter_size(self._h, C.byref(n)))
        return n.value

    def particles(self):
        n = self.size()
        st, w = np.zeros((n, 4)), np.zeros(n)
        self._check(self._lib.bb200_filter_get_particles(self._h, _dptr(st), _dptr(w), n))
        return st, w

    def initialize_normal(self, mean_xytheta, cov, n: int):
        self._check(self._lib.bb200_filter_initialize_normal(self._h, _dptr(_f64(mean_xytheta)), _dptr(_f64(cov).reshape(9)), n))

    def initialize_uniform(self, n: int):
        """n particles uniform over the free cells of the current map (MultivariateUniformDistribution<SE2d, OccupancyGrid>)."""
        self._check(self._lib.bb200_filter_initialize_uniform(self._h, n))

    # per-step operations
    @staticmethod
    def _sampling(s) -> _capi.MotionSampling:
        """Accepts a MotionSampling or the six differential-drive scalars (rot1, trans, rot2 mean/std pairs)."""
        if isinstance(s, _capi.MotionSampling):
            return s
        if isinstance(s, _capi.DiffDriveSampling):
            s = [s.rot1_mean, s.rot1_std, s.trans_mean, s.trans_std, s.rot2_mean, s.rot2_std]
        v = [float(x) for x in s]
        return _capi.MotionSampling(_capi.MOTION_DIFFERENTIAL, (C.c_double * 3)(v[0], v[2], v[4]), (C.c_double * 3)(v[1], v[3], v[5]),
                                    (C.c_double * 2)(1.0, 0.0))

    def propagate(self, sampling, step: int):
        s = self._sampling(sampling)
        self._check(self._lib.bb200_filter_propagate(self._h, C.byref(s), step))

    def reweight(self, points):
        pts = _f64(points).reshape(-1, 2)
        self._check(self._lib.bb200_filter_reweight(self._h, _dptr(pts), len(pts)))

    def propagate_reweight(self, sampling, step: int, points):
        s = self._sampling(sampling)
        pts = _f64(points).reshape(-1, 2)
        self._check(self._lib.bb200_filter_propagate_reweight(self._h, C.byref(s), step, _dptr(pts), len(pts)))

    def max_weight(self) -> float:
        v = C.c_double()
        self._check(self._lib.bb200_filter_max_weight(self._h, C.byref(v)))
        return v.value

    def build_cdf(self, global_wmax: float = -1.0):
        total, ex = C.c_uint64(), C.c_int()
        self._check(self._lib.bb200_filter_build_cdf(self._h, global_wmax, C.byref(total), C.byref(ex)))
        return total.value, ex.value

    def normalize_by(self, global_total: int) -> float:
        sq = C.c_double()
        self._check(self._lib.bb200_filter_normalize_by(self._h, global_total, C.byref(sq)))
        return sq.value

    def normalize(self):
        f, sq = C.c_double(), C.c_double()
        self._check(self._lib.bb200_filter_normalize(self._h, C.byref(f), C.byref(sq)))
        return f.value, sq.value

    def resample(self, scheme: int, step: int, max_particles: int, min_particles: int | None = None, kld_epsilon: float = 0.05,
                 kld_z: float = 3.0, spatial_resolution=(0.5, 0.5, float(np.deg2rad(10.0))), random_state_probability: float = 0.0) -> int:
        o = _capi.ResampleOpts(scheme, step, max_particles if min_particles is None else min_particles, max_particles, kld_epsilon,
                               kld_z, (C.c_double * 3)(*spatial_resolution), random_state_probability)
        n = C.c_uint64()
        self._check(self._lib.bb200_filter_resample(self._h, C.byref(o), C.byref(n)))
        return n.value

    def resample_range(self, opts: _capi.ResampleOpts, global_total: int, cdf_offset: int, slot_begin: int, slot_end: int):
        self._check(self._lib.bb200_filter_resample_range(self._h, C.byref(opts), global_total, cdf_offset, slot_begin, slot_end))

    def adopt(self, n: int, from_staging: bool = False):
        self._check(self._lib.bb200_filter_adopt(self._h, n, int(from_staging)))

    # stream-ordered variants (sharded filters; see distributed.py)
    def set_stream(self, cuda_stream: int):
        self._check(self._lib.bb200_filter_set_stream(self._h, C.c_void_p(cuda_stream)))

    def enqueue_propagate_reweight(self, sampling, step: int, points):
        s = self._sampling(sampling)
        pts = _f64(points).reshape(-1, 2)
        self._check(self._lib.bb200_filter_enqueue_propagate_reweight(self._h, C.byref(s), step, _dptr(pts), len(pts)))

    def enqueue_build_cdf(self):
        self._check(self._lib.bb200_filter_enqueue_build_cdf(self._h))

    def enqueue_resample_range(self, opts: _capi.ResampleOpts, global_total: int, cdf_offset: int, slot_begin: int, slot_end: int):
        self._check(self._lib.bb200_filter_enqueue_resample_range(self._h, C.byref(opts), global_total, cdf_offset, slot_begin, slot_end))

    def enqueue_adopt(self, n: int):
        self._check(self._lib.bb200_filter_enqueue_adopt(self._h, n))

    def enqueue_moments(self, pivot):
        self._check(self._lib.bb200_filter_enqueue_moments(self._h, _dptr(_f64(pivot))))

    def ancestors(self) -> np.ndarray:
        out = np.zeros(self.size(), dtype=np.int64)
        self._check(self._lib.bb200_filter_ancestors(self._h, out.ctypes.data_as(C.POINTER(C.c_int64)), len(out)))
        return out

    def cdf(self) -> np.ndarray:
        out = np.zeros(self.size(), dtype=np.uint64)
        self._check(self._lib.bb200_filter_cdf(self._h, out.ctypes.data_as(C.POINTER(C.c_uint64)), len(out)))
        return out

    def estimate(self):
        e = _capi.Estimate()
        self._check(self._lib.bb200_filter_estimate(self._h, C.byref(e)))
        return np.array(e.mean), np.array(e.cov).reshape(3, 3)

    def cluster_estimate(self, linear: float = 0.20, angular: float = 0.524, percentile: float = 0.90, with_ids: bool = False):
        """beluga::cluster_based_estimate (algorithm/cluster_based_estimation.hpp:415-432) -> (mean[4], cov[3,3]);
        with_ids adds (cluster id per particle, number of occupied cells, number of clusters)."""
        e = _capi.Estimate()
        p = _capi.ClusterParam(linear, angular, percentile)
        ids = np.zeros(self.size() if with_ids else 0, dtype=np.uint32)
        cells, clusters = C.c_uint32(0), C.c_uint32(0)
        self._check(self._lib.bb200_filter_cluster_estimate(
            self._h, C.byref(p), C.byref(e), ids.ctypes.data_as(C.POINTER(C.c_uint32)) if with_ids else None, ids.size,
            C.byref(cells), C.byref(clusters)))
        est = (np.array(e.mean), np.array(e.cov).reshape(3, 3))
        return (*est, ids, cells.value, clusters.value) if with_ids else est

    def particle_histogram(self, linear: float = 1e-3, angular: float = 1e-3):
        """Device-side histogram of the cloud over spatial-hash buckets (beluga_ros/particle_cloud.hpp:197-210).
        -> (representatives [m, 4], weights [m], counts [m], first_index [m], max_bin_weight)."""
        n_bins, top = C.c_uint64(0), C.c_double(0.0)
        self._check(self._lib.bb200_filter_particle_histogram(self._h, linear, angular, None, 0, C.byref(n_bins), C.byref(top)))
        m = n_bins.value
        arr = (_capi.ClusterCell * max(m, 1))()
        self._check(self._lib.bb200_filter_particle_histogram(self._h, linear, angular, arr, m, C.byref(n_bins), C.byref(top)))
        raw = np.frombuffer(arr, dtype=np.dtype([("rep", "<f8", 4), ("hash", "<u8"), ("first", "<u4"), ("count", "<u4"), ("weight", "<f8"), ("m", "<f8", 9)]),
                            count=m)
        return raw["rep"].copy(), raw["weight"].copy(), raw["count"].copy(), raw["first"].copy(), top.value

    def sample_states(self, count: int, step: int = 0xFFFFFFFF) -> np.ndarray:
        """`count` states drawn by weight without touching the set (assign_particle_cloud(..., size, PoseArray))."""
        out = np.zeros((count, 4))
        self._check(self._lib.bb200_filter_sample_states(self._h, count, step, _dptr(out) if count else None))
        return out

    def cast_rays(self, poses, bearings, max_range: float) -> np.ndarray:
        """Ray2d::cast on the current map (bb200_filter_cast_rays): sensor poses (n, 4) [cos, sin, x, y] in the map frame
        times bearings (m, 2) [cos, sin] taken as given -> (n, m) ranges, min(distance, max_range) on a hit, inf on a miss."""
        p, b = _rays(poses, bearings)
        out = np.zeros((len(p), len(b)))
        self._check(self._lib.bb200_filter_cast_rays(self._h, _dptr(p) if len(p) else None, len(p), _dptr(b) if len(b) else None, len(b),
                                                     max_range, _dptr(out) if out.size else None))
        return out

    def moments(self, pivot=(0.0, 0.0)) -> np.ndarray:
        out = np.zeros(9)
        self._check(self._lib.bb200_filter_moments(self._h, _dptr(_f64(pivot)), _dptr(out)))
        return out

    def set_timing(self, enabled: bool):
        self._check(self._lib.bb200_filter_set_timing(self._h, int(enabled)))

    def clear_timings(self):
        self._check(self._lib.bb200_filter_clear_timings(self._h))

    def last_timings(self) -> list[tuple[str, float]]:
        """(kernel, ms) pairs recorded since clear_timings()."""
        names = (C.c_char_p * 128)()
        ms = (C.c_float * 128)()
        n = self._lib.bb200_filter_last_timings(self._h, names, ms, 128)
        return [(names[i].decode(), ms[i]) for i in range(min(n, 128))]

    def launch_count(self) -> int:
        return self._lib.bb200_filter_launch_count(self._h)

    def synchronize(self):
        self._check(self._lib.bb200_filter_synchronize(self._h))

    def device_pointer(self, which: int):
        p, b = C.c_void_p(), C.c_uint64()
        self._check(self._lib.bb200_filter_device_pointer(self._h, which, C.byref(p), C.byref(b)))
        return p.value, b.value


class Amcl:
    """bb200_amcl: beluga::Amcl (algorithm/amcl_core.hpp:81-233) with the particle set on the GPU."""

    def __init__(self, motion, params: AmclParams):
        """`motion`: DifferentialDriveModelParam, OmnidirectionalDriveModelParam or StationaryModelParam."""
        self._lib = _capi.load()
        p, m = params.c(), motion.c_motion()
        h = C.c_void_p()
        st = self._lib.bb200_amcl_create_with_motion(C.byref(p), C.byref(m), C.byref(h))
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_create_error().decode())
        self._h = h
        self.params = params
        self.filter = Filter(_handle=self._lib.bb200_amcl_filter(self._h), _owner=self)

    @classmethod
    def from_state(cls, blob: bytes, device: int = 0) -> "Amcl":
        """The filter a state blob holds (bb200_amcl_create_from_state) on `device`, without a map: update_map before updating."""
        self = cls.__new__(cls)
        self._lib = _capi.load()
        h = C.c_void_p()
        st = self._lib.bb200_amcl_create_from_state(blob, len(blob), device, C.byref(h))
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_create_error().decode())
        self._h = h
        self.params = state_params(blob)[0]
        self.params.device = device
        self.filter = Filter(_handle=self._lib.bb200_amcl_filter(self._h), _owner=self)
        return self

    def export_state(self) -> bytes:
        """This filter's state blob (bb200_amcl_export_state): parameters, policies, particles, weights, CDF and ancestors."""
        size = C.c_uint64(0)
        self._check(self._lib.bb200_amcl_export_state(self._h, None, 0, C.byref(size)))
        buf = C.create_string_buffer(size.value)
        self._check(self._lib.bb200_amcl_export_state(self._h, buf, size.value, C.byref(size)))
        return buf.raw

    def close(self):
        if getattr(self, "_h", None):
            self.filter._h = None
            self._lib.bb200_amcl_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def _check(self, st: int):
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_amcl_last_error(self._h).decode())

    def update_map(self, sensor: int, params, grid):
        """Amcl::update_map (amcl_core.hpp:150) / sensor model construction.  `grid` is an OccupancyGrid, or a LandmarkMap
        for SENSOR_LANDMARK and SENSOR_BEARING."""
        if sensor == SENSOR_LANDMARK:
            self.filter.set_landmark_map(params, grid)
        elif sensor == SENSOR_BEARING:
            self.filter.set_bearing_map(params, grid)
        elif sensor == SENSOR_BEAM:
            self.filter.set_beam_map(params, grid)
        else:
            self.filter.set_likelihood_field_map(params, grid, prob=(sensor == SENSOR_LIKELIHOOD_FIELD_PROB))

    def initialize(self, mean_xytheta, cov):
        self._check(self._lib.bb200_amcl_initialize(self._h, _dptr(_f64(mean_xytheta)), _dptr(_f64(cov).reshape(9))))

    def initialize_from_map(self):
        """beluga_ros::Amcl::initialize_from_map (beluga_ros/include/beluga_ros/amcl.hpp:209): global localisation start."""
        self._check(self._lib.bb200_amcl_initialize_from_map(self._h))

    def initialize_states(self, states, weights=None):
        st = _f64(states).reshape(-1, 4)
        w = None if weights is None else _f64(weights)
        self._check(self._lib.bb200_amcl_initialize_states(self._h, _dptr(st), None if w is None else _dptr(w), len(st)))

    def force_update(self):
        self._lib.bb200_amcl_force_update(self._h)

    def particles(self):
        return self.filter.particles()

    def cast_rays(self, poses, bearings, max_range: float) -> np.ndarray:
        """Filter.cast_rays on the map of update_map."""
        return self.filter.cast_rays(poses, bearings, max_range)

    def update_scan(self, control_pose, ranges, angle_min: float, angle_increment: float, min_range: float = 0.0,
                    max_range: float = float("inf"), max_beams: int = 0, laser_origin=None) -> _capi.UpdateResult:
        """Amcl::update(base_pose_in_odom, laser_scan) (beluga_ros/src/amcl.cpp:54-64)."""
        scan, keep = _laser_scan(ranges, angle_min, angle_increment, min_range, max_range, max_beams, laser_origin)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_amcl_update_scan(self._h, _dptr(_f64(control_pose)), C.byref(scan), C.byref(res)))
        return res

    def update_point_cloud(self, control_pose, data, point_step: int, x_offset: int, dtype, origin=None,
                           n_points: int | None = None) -> _capi.UpdateResult:
        """Amcl::update(base_pose_in_odom, point_cloud) (beluga_ros/src/amcl.cpp:67-81); arguments as point_cloud_to_points."""
        cloud, keep = _point_cloud(data, point_step, x_offset, dtype, origin, n_points)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_amcl_update_point_cloud(self._h, _dptr(_f64(control_pose)), C.byref(cloud), C.byref(res)))
        return res

    def export_shard(self) -> bytes:
        """256 bytes of CUDA IPC handles (two state buffers, mail block, KLD hash array) for the peer ranks of a sharded filter."""
        buf = C.create_string_buffer(256)
        self._check(self._lib.bb200_amcl_export_shard(self._h, buf))
        return buf.raw

    def join_shards(self, world: int, rank: int, handles: bytes):
        """Map every rank's exported buffers (world x 256 bytes, rank order); update() then runs in lock step with the peers."""
        assert len(handles) == 256 * world
        self._check(self._lib.bb200_amcl_join_shards(self._h, world, rank, C.create_string_buffer(handles, len(handles))))

    def leave_shards(self):
        self._check(self._lib.bb200_amcl_leave_shards(self._h))

    def plan_update(self, control_pose) -> _capi.StepPlan:
        """Host half of Amcl::update (policies, control window, recovery estimator)."""
        plan = _capi.StepPlan()
        self._check(self._lib.bb200_amcl_plan_update(self._h, _dptr(_f64(control_pose)), C.byref(plan)))
        return plan

    def commit_update(self, resampled: bool, random_state_probability: float):
        self._lib.bb200_amcl_commit_update(self._h, int(resampled), random_state_probability)

    def update(self, control_pose, points) -> _capi.UpdateResult:
        """Amcl::update: returns the result block; `.updated == 0` is the reference's std::nullopt."""
        pts = _f64(points).reshape(-1, 2)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_amcl_update(self._h, _dptr(_f64(control_pose)), _dptr(pts), len(pts), C.byref(res)))
        return res

    def update_landmarks(self, control_pose, positions, categories) -> _capi.UpdateResult:
        """Amcl::update with the landmark map's model: (n, 3) detection positions in the robot frame (SENSOR_LANDMARK) or
        bearings in the sensor frame (SENSOR_BEARING), and n categories."""
        arr, n = _landmark_array(positions, categories)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_amcl_update_landmarks(self._h, _dptr(_f64(control_pose)), arr, n, C.byref(res)))
        return res

    def update_weighted(self, control_pose, weigh) -> _capi.UpdateResult:
        """Amcl::update with the caller's own sensor model (bb200_amcl_update_begin / _end).

        `weigh(states, factors)` receives torch CUDA tensors over the step's device views, without a copy: the propagated
        states, (n, 4) float64 rows {cos, sin, x, y}, and the factors, (n,) float64, which it fills with L(states[i]).  It
        runs inside torch.cuda.stream(torch.cuda.ExternalStream(view.stream)), so torch work it issues is ordered before the
        rest of the step; other work must be synchronised with that stream by `weigh`.  It is not called when the policies
        skip the step.  When `weigh` raises, the step is closed with every factor 1 (a step without a measurement) and the
        exception propagates."""
        view = _capi.WeighView()
        self._check(self._lib.bb200_amcl_update_begin(self._h, _dptr(_f64(control_pose)), C.byref(view)))
        res = _capi.UpdateResult()
        if not view.updated:
            self._check(self._lib.bb200_amcl_update_end(self._h, C.byref(res)))
            return res
        import torch

        device = torch.device("cuda", self.params.device)
        states = torch.as_tensor(_CudaArray(view.states, (view.n, 4)), device=device)
        factors = torch.as_tensor(_CudaArray(view.factors, (view.n,)), device=device)
        with torch.cuda.stream(torch.cuda.ExternalStream(view.stream, device=device)):
            try:
                weigh(states, factors)
            except BaseException:
                factors.fill_(1.0)
                self._lib.bb200_amcl_update_end(self._h, C.byref(res))
                raise
        self._check(self._lib.bb200_amcl_update_end(self._h, C.byref(res)))
        return res


class _CudaArray:
    """A float64 device array in the __cuda_array_interface__ protocol (no stream to wait on: the consumer orders its work)."""

    def __init__(self, ptr: int, shape: tuple):
        self.__cuda_array_interface__ = {"shape": tuple(int(d) for d in shape), "typestr": "<f8", "data": (int(ptr), False), "version": 3,
                                         "strides": None, "stream": None}


class ShardedAmcl:
    """bb200_sharded_amcl: ONE filter over several shards driven by one host thread (include/beluga_b200.h).

    `devices[r]` is the CUDA ordinal of shard r; ordinals may repeat (several shards on one device -- how the
    single-GPU tests exercise the sharded kernels).  params.max_particles is the GLOBAL particle count."""

    def __init__(self, motion, params: AmclParams, devices):
        self._lib = _capi.load()
        p, m = params.c(), motion.c_motion()
        dev = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        st = self._lib.bb200_sharded_amcl_create(C.byref(p), C.byref(m), len(devices), dev, C.byref(h))
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_create_error().decode())
        self._h = h
        self.params = params
        self.devices = list(devices)
        self.shards = [Filter(_handle=self._lib.bb200_amcl_filter(self._lib.bb200_sharded_amcl_shard(self._h, r)), _owner=self)
                       for r in range(len(devices))]

    def close(self):
        if getattr(self, "_h", None):
            for f in self.shards:
                f._h = None
            self._lib.bb200_sharded_amcl_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def _check(self, st: int):
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_sharded_amcl_last_error(self._h).decode())

    def update_map(self, sensor: int, params, grid):
        """Amcl.update_map on every shard: `grid` is an OccupancyGrid, or a LandmarkMap for SENSOR_LANDMARK and SENSOR_BEARING."""
        g = grid.c()
        p = params.c()
        if sensor == SENSOR_LANDMARK:
            self._check(self._lib.bb200_sharded_amcl_set_landmark_map(self._h, C.byref(p), C.byref(g)))
        elif sensor == SENSOR_BEARING:
            self._check(self._lib.bb200_sharded_amcl_set_bearing_map(self._h, C.byref(p), C.byref(g)))
        elif sensor == SENSOR_BEAM:
            self._check(self._lib.bb200_sharded_amcl_set_beam_map(self._h, C.byref(p), C.byref(g)))
        else:
            self._check(self._lib.bb200_sharded_amcl_set_likelihood_field_map(self._h, C.byref(p), C.byref(g), int(sensor == SENSOR_LIKELIHOOD_FIELD_PROB)))

    def initialize(self, mean_xytheta, cov):
        self._check(self._lib.bb200_sharded_amcl_initialize(self._h, _dptr(_f64(mean_xytheta)), _dptr(_f64(cov).reshape(9))))

    def initialize_from_map(self):
        self._check(self._lib.bb200_sharded_amcl_initialize_from_map(self._h))

    def force_update(self):
        self._lib.bb200_sharded_amcl_force_update(self._h)

    def update(self, control_pose, points) -> _capi.UpdateResult:
        pts = _f64(points).reshape(-1, 2)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_sharded_amcl_update(self._h, _dptr(_f64(control_pose)), _dptr(pts) if len(pts) else None, len(pts), C.byref(res)))
        return res

    def update_landmarks(self, control_pose, positions, categories) -> _capi.UpdateResult:
        """Amcl.update_landmarks over all shards (bb200_sharded_amcl_update_landmarks)."""
        arr, n = _landmark_array(positions, categories)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_sharded_amcl_update_landmarks(self._h, _dptr(_f64(control_pose)), arr, n, C.byref(res)))
        return res

    def update_weighted(self, control_pose, weigh) -> _capi.UpdateResult:
        """Amcl.update_weighted over all shards (bb200_sharded_amcl_update_begin / _end): the same `weigh(states, factors)`.

        It is called once per shard that holds particles, in rank order, with shard r's slice of the global particle order,
        inside torch.cuda.device(devices[r]) and torch.cuda.stream(torch.cuda.ExternalStream(view.stream)), so a model
        written for one filter works unchanged.  It is not called when the policies skip the step.  When `weigh` raises,
        every shard's factors are set to 1, the step is closed and the exception propagates."""
        k = len(self.devices)
        views = (_capi.WeighView * k)()
        self._check(self._lib.bb200_sharded_amcl_update_begin(self._h, _dptr(_f64(control_pose)), views))
        res = _capi.UpdateResult()
        if not views[0].updated:
            self._check(self._lib.bb200_sharded_amcl_update_end(self._h, C.byref(res)))
            return res
        try:  # the tensors are made in here too: whatever raises, the step is closed
            import torch

            for device, stream, states, factors in self._weigh_views(views):
                with torch.cuda.device(device), torch.cuda.stream(stream):
                    weigh(states, factors)
        except BaseException:
            try:  # a step without a measurement; end runs even when the fill cannot
                import torch

                for device, stream, _, factors in self._weigh_views(views):
                    with torch.cuda.device(device), torch.cuda.stream(stream):
                        factors.fill_(1.0)
            finally:
                self._lib.bb200_sharded_amcl_update_end(self._h, C.byref(res))
            raise
        self._check(self._lib.bb200_sharded_amcl_update_end(self._h, C.byref(res)))
        return res

    def _weigh_views(self, views):
        """(device, stream, states, factors) of every shard whose view holds particles, in rank order, as torch objects."""
        import torch

        for r, v in enumerate(views):
            if v.n > 0:
                device = torch.device("cuda", self.devices[r])
                yield (device, torch.cuda.ExternalStream(v.stream, device=device), torch.as_tensor(_CudaArray(v.states, (v.n, 4)), device=device),
                       torch.as_tensor(_CudaArray(v.factors, (v.n,)), device=device))

    def cluster_estimate(self, linear: float = 0.20, angular: float = 0.524, percentile: float = 0.90):
        """beluga::cluster_based_estimate over all shards -> (mean[4], cov[3, 3], n_cells, n_clusters)."""
        p = _capi.ClusterParam(linear, angular, percentile)
        est = _capi.Estimate()
        cells, clusters = C.c_uint32(0), C.c_uint32(0)
        self._check(self._lib.bb200_sharded_amcl_cluster_estimate(self._h, C.byref(p), C.byref(est), C.byref(cells), C.byref(clusters)))
        return np.array(est.mean), np.array(est.cov).reshape(3, 3), cells.value, clusters.value

    def update_scan(self, control_pose, ranges, angle_min: float, angle_increment: float, min_range: float = 0.0,
                    max_range: float = float("inf"), max_beams: int = 0, laser_origin=None) -> _capi.UpdateResult:
        """Amcl.update_scan over all shards (bb200_sharded_amcl_update_scan)."""
        scan, keep = _laser_scan(ranges, angle_min, angle_increment, min_range, max_range, max_beams, laser_origin)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_sharded_amcl_update_scan(self._h, _dptr(_f64(control_pose)), C.byref(scan), C.byref(res)))
        return res

    def update_point_cloud(self, control_pose, data, point_step: int, x_offset: int, dtype, origin=None,
                           n_points: int | None = None) -> _capi.UpdateResult:
        """Amcl.update_point_cloud over all shards (bb200_sharded_amcl_update_point_cloud); arguments as point_cloud_to_points."""
        cloud, keep = _point_cloud(data, point_step, x_offset, dtype, origin, n_points)
        res = _capi.UpdateResult()
        self._check(self._lib.bb200_sharded_amcl_update_point_cloud(self._h, _dptr(_f64(control_pose)), C.byref(cloud), C.byref(res)))
        return res

    def particle_histogram(self, linear: float = 1e-3, angular: float = 1e-3):
        """Filter.particle_histogram over all shards, merged in rank order (bb200_sharded_amcl_particle_histogram).
        -> (representatives [m, 4], weights [m], counts [m], first_index [m], max_bin_weight)."""
        n_bins, top = C.c_uint64(0), C.c_double(0.0)
        self._check(self._lib.bb200_sharded_amcl_particle_histogram(self._h, linear, angular, None, 0, C.byref(n_bins), C.byref(top)))
        m = n_bins.value
        arr = (_capi.ClusterCell * max(m, 1))()
        self._check(self._lib.bb200_sharded_amcl_particle_histogram(self._h, linear, angular, arr, m, C.byref(n_bins), C.byref(top)))
        raw = np.frombuffer(arr, dtype=_CELL_DTYPE, count=m)
        return raw["rep"].copy(), raw["weight"].copy(), raw["count"].copy(), raw["first"].copy(), top.value

    def sample_states(self, count: int, step: int = 0xFFFFFFFF) -> np.ndarray:
        """Filter.sample_states over the global particle set (bb200_sharded_amcl_sample_states): the draws one filter holding
        the same particles and weights returns, whatever the shard count."""
        out = np.zeros((count, 4))
        self._check(self._lib.bb200_sharded_amcl_sample_states(self._h, count, step, _dptr(out) if count else None))
        return out

    def cast_rays(self, poses, bearings, max_range: float) -> np.ndarray:
        """Filter.cast_rays on the shards' copies of the map (bb200_sharded_amcl_cast_rays), the poses split over the devices."""
        p, b = _rays(poses, bearings)
        out = np.zeros((len(p), len(b)))
        self._check(self._lib.bb200_sharded_amcl_cast_rays(self._h, _dptr(p) if len(p) else None, len(p), _dptr(b) if len(b) else None, len(b),
                                                           max_range, _dptr(out) if out.size else None))
        return out

    def particles(self):
        """The particle set in global index order (a KLD-sized filter holds fewer than max_particles)."""
        n = sum(f.size() for f in self.shards)
        st = np.zeros((n, 4))
        w = np.zeros(n)
        if n:
            self._check(self._lib.bb200_sharded_amcl_get_particles(self._h, _dptr(st), _dptr(w), n))
        return st, w


_CELL_DTYPE = np.dtype([("rep", "<f8", 4), ("hash", "<u8"), ("first", "<u4"), ("count", "<u4"), ("weight", "<f8"), ("m", "<f8", 9)])


class AmclBatch:
    """bb200_amcl_batch: K independent beluga::Amcl filters on one GPU, each reading one of the batch's maps -- a
    likelihood field, a beam-model map or a landmark map, one for every member (set_*_map) or several (add_*_map and update_map, which
    moves a member to another map as a node's Amcl::update_map does); update() steps every member with a new scan with a fixed
    number of kernel launches and one synchronisation.  Member m's results and particles equal those of a standalone Amcl
    built from params[m] and motions[m] and fed the same inputs.

    Member indices are slots: add_member and remove_member let robots join and leave the running batch without
    disturbing the others.  len() counts the slots, occupied and vacant, and every per-member list keeps that length;
    `params[m]` is None for a vacant slot, whose entries of those lists are not read."""

    def __init__(self, motions, params, adaptive: bool = False, selective: bool = False):
        """`motions[m]`, `params[m]`: member m's motion model and AmclParams (max_particles <= 32768, and
        min_particles == max_particles unless `adaptive`).  adaptive=True (BB200_BATCH_ADAPTIVE) lets members
        have min_particles < max_particles: they resize their particle sets with KLD on every resampling step, and
        particles() and ancestors() then return member_size(m) rows.  selective=True (BB200_BATCH_SELECTIVE) lets members
        have selective_resampling: they resample only when their effective sample size drops below half their particles,
        and each result's `resampled` reports the decision."""
        self._lib = _capi.load()
        k = len(params)
        if len(motions) != k:
            raise ValueError("one motion model per member")
        p = (_capi.AmclParam * max(k, 1))(*[q.c() for q in params])
        m = (_capi.MotionParam * max(k, 1))(*[q.c_motion() for q in motions])
        h = C.c_void_p()
        flags = (_capi.BATCH_ADAPTIVE if adaptive else 0) | (_capi.BATCH_SELECTIVE if selective else 0)
        st = self._lib.bb200_amcl_batch_create_with_flags(p, m, k, flags, C.byref(h))
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_create_error().decode())
        self._h = h
        self.params = list(params)
        self.adaptive = bool(adaptive)
        self.selective = bool(selective)
        self._field_shapes = {}  # (height, width) of each likelihood-field map, by id

    def close(self):
        if getattr(self, "_h", None):
            self._lib.bb200_amcl_batch_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def __len__(self) -> int:
        return self._lib.bb200_amcl_batch_members(self._h)

    def _check(self, st: int):
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_amcl_batch_last_error(self._h).decode())

    def add_member(self, motion, params) -> int:
        """Adds a member configured by `motion` and `params` (AmclParams), validated as the constructor validates one under
        this batch's flags; it takes the lowest vacant slot or appends one, and starts with no map and no particles, as a
        member of a freshly created batch.  Returns its slot.  The other members keep their particles, policies and maps."""
        p, m = params.c(), motion.c_motion()
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_add_member(self._h, C.byref(p), C.byref(m), C.byref(i)))
        if i.value == len(self.params):
            self.params.append(None)
        self.params[i.value] = params
        return i.value

    @classmethod
    def from_states(cls, blobs, adaptive: bool = False, selective: bool = False, device: int = 0) -> "AmclBatch":
        """The batch whose member m is the filter of state blob blobs[m] (bb200_amcl_batch_create_from_states), on `device`,
        validated with the constructor's flags; it has no map (add_*_map, then update_map)."""
        self = cls.__new__(cls)
        self._lib = _capi.load()
        k = len(blobs)
        data = (C.c_void_p * max(k, 1))(*[C.cast(C.c_char_p(b), C.c_void_p) for b in blobs])
        sizes = (C.c_uint64 * max(k, 1))(*[len(b) for b in blobs])
        flags = (_capi.BATCH_ADAPTIVE if adaptive else 0) | (_capi.BATCH_SELECTIVE if selective else 0)
        h = C.c_void_p()
        st = self._lib.bb200_amcl_batch_create_from_states(data, sizes, k, flags, device, C.byref(h))
        if st != _capi.OK:
            raise BelugaB200Error(st, self._lib.bb200_create_error().decode())
        self._h = h
        self.params = [state_params(b)[0] for b in blobs]
        self.adaptive = bool(adaptive)
        self.selective = bool(selective)
        self._field_shapes = {}
        return self

    def export_member(self, member: int) -> bytes:
        """Member `member`'s state blob (bb200_amcl_batch_export_member)."""
        size = C.c_uint64(0)
        self._check(self._lib.bb200_amcl_batch_export_member(self._h, member, None, 0, C.byref(size)))
        buf = C.create_string_buffer(size.value)
        self._check(self._lib.bb200_amcl_batch_export_member(self._h, member, buf, size.value, C.byref(size)))
        return buf.raw

    def export_members(self, present=None) -> list:
        """The fleet checkpoint (bb200_amcl_batch_export_members): the state blob of every member whose `present` entry is
        true (None: every occupied slot), None for the others, with one kernel launch and one synchronisation."""
        mask = self._mask(present)
        k = len(self.params)
        sizes = (C.c_uint64 * k)()
        self._check(self._lib.bb200_amcl_batch_export_members(self._h, mask, None, None, sizes))
        bufs = [C.create_string_buffer(sizes[m]) if sizes[m] else None for m in range(k)]
        out = (C.c_void_p * k)(*[C.cast(b, C.c_void_p) if b is not None else None for b in bufs])
        self._check(self._lib.bb200_amcl_batch_export_members(self._h, mask, out, sizes, sizes))
        return [None if self._skipped(present, m) else bufs[m].raw for m in range(k)]

    def import_member(self, blob: bytes, map_id: int = -1) -> int:
        """add_member with a history (bb200_amcl_batch_import_member): the blob's filter joins in the lowest vacant slot or a
        new one and reads map `map_id` (-1: none).  Returns its slot."""
        params = state_params(blob)[0]
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_import_member(self._h, blob, len(blob), map_id, C.byref(i)))
        if i.value == len(self.params):
            self.params.append(None)
        self.params[i.value] = params
        return i.value

    def remove_member(self, member: int):
        """Makes slot `member` vacant and frees its share of the device buffers; the last member cannot be removed."""
        self._check(self._lib.bb200_amcl_batch_remove_member(self._h, member))
        self.params[member] = None

    def member_active(self, member: int) -> bool:
        """Whether slot `member` holds a member."""
        a = C.c_int(0)
        self._check(self._lib.bb200_amcl_batch_member_active(self._h, member, C.byref(a)))
        return bool(a.value)

    def _skipped(self, present, m) -> bool:
        # not selected: absent from `present`, or a vacant slot when present is None
        return not present[m] if present is not None else self.params[m] is None

    def set_likelihood_field_map(self, params: LikelihoodFieldModelParam, grid: OccupancyGrid, prob: bool = False):
        """One likelihood field for every member: removes every map, adds this one and assigns every member to it."""
        p, g = params.c(), grid.c()
        self._check(self._lib.bb200_amcl_batch_set_likelihood_field_map(self._h, C.byref(p), C.byref(g), int(prob)))
        occupied = next(m for m, q in enumerate(self.params) if q is not None)
        self._field_shapes = {self.member_map(occupied): grid.cells.shape}

    def set_beam_map(self, params: BeamModelParam, grid: OccupancyGrid):
        """The beam model (BeamSensorModel) on `grid` for every member; replaces the map set before, of either model."""
        p, g = params.c(), grid.c()
        self._check(self._lib.bb200_amcl_batch_set_beam_map(self._h, C.byref(p), C.byref(g)))
        self._field_shapes = {}

    def add_likelihood_field_map(self, params: LikelihoodFieldModelParam, grid: OccupancyGrid, prob: bool = False) -> int:
        """Adds a likelihood-field map that no member reads yet; returns its id (0, 1, ... never reused)."""
        p, g = params.c(), grid.c()
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_add_likelihood_field_map(self._h, C.byref(p), C.byref(g), int(prob), C.byref(i)))
        self._field_shapes[i.value] = grid.cells.shape
        return i.value

    def add_beam_map(self, params: BeamModelParam, grid: OccupancyGrid) -> int:
        """Adds a beam-model map that no member reads yet; returns its id."""
        p, g = params.c(), grid.c()
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_add_beam_map(self._h, C.byref(p), C.byref(g), C.byref(i)))
        return i.value

    def set_landmark_map(self, params: LandmarkModelParam, landmark_map: LandmarkMap):
        """The landmark model (LandmarkSensorModel2d) on `landmark_map` for every member; replaces every earlier map."""
        p, m = params.c(), landmark_map.c()
        self._check(self._lib.bb200_amcl_batch_set_landmark_map(self._h, C.byref(p), C.byref(m)))
        self._field_shapes = {}

    def set_bearing_map(self, params: BearingModelParam, landmark_map: LandmarkMap):
        """The bearing model (BearingSensorModel2d) on `landmark_map` for every member; replaces every earlier map."""
        p, m = params.c(), landmark_map.c()
        self._check(self._lib.bb200_amcl_batch_set_bearing_map(self._h, C.byref(p), C.byref(m)))
        self._field_shapes = {}

    def add_landmark_map(self, params: LandmarkModelParam, landmark_map: LandmarkMap) -> int:
        """Adds a landmark-model map that no member reads yet; returns its id."""
        p, m = params.c(), landmark_map.c()
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_add_landmark_map(self._h, C.byref(p), C.byref(m), C.byref(i)))
        return i.value

    def add_bearing_map(self, params: BearingModelParam, landmark_map: LandmarkMap) -> int:
        """Adds a bearing-model map that no member reads yet; returns its id."""
        p, m = params.c(), landmark_map.c()
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_add_bearing_map(self._h, C.byref(p), C.byref(m), C.byref(i)))
        return i.value

    def _built(self, measurements, present, weighed: bool = False):
        """The bb200_measurement table of a step (a None entry: weighed by the caller when `weighed`, no points otherwise),
        with every selected Detections member's detections staged first, and the objects that must outlive the call."""
        k = len(self.params)
        if len(measurements) != k:
            raise ValueError("one measurement per member")
        staged = {m for m in range(k) if isinstance(measurements[m], Detections) and not self._skipped(present, m)}
        if staged:
            arrays = [_landmark_array(measurements[m].positions, measurements[m].categories) if m in staged else (None, 0) for m in range(k)]
            ptrs = (C.POINTER(_capi.Landmark) * k)(*[a if n else None for a, n in arrays])
            counts = (C.c_uint64 * k)(*[n for _, n in arrays])
            mask = (C.c_uint8 * k)(*[1 if m in staged else 0 for m in range(k)])
            self._check(self._lib.bb200_amcl_batch_set_detections(self._h, ptrs, counts, mask))

        def one(m):
            if isinstance(m, Detections):
                return _capi.Measurement(kind=_capi.MEASUREMENT_LANDMARKS), None
            if m is None and weighed:
                return _capi.Measurement(kind=_capi.MEASUREMENT_WEIGHTS), None
            return _measurement(() if m is None else m)

        built = [one(m) for m in measurements]
        return (_capi.Measurement * k)(*[b[0] for b in built]), built

    def update_map(self, member: int, map_id: int):
        """Amcl::update_map for one member: it keeps its particles and policies and reads `map_id` from its next step."""
        self._check(self._lib.bb200_amcl_batch_update_map(self._h, member, map_id))

    def member_map(self, member: int) -> int:
        """The id of the map member `member` reads (-1: none)."""
        i = C.c_int(-1)
        self._check(self._lib.bb200_amcl_batch_member_map(self._h, member, C.byref(i)))
        return i.value

    def remove_map(self, map_id: int):
        """Frees a map that no member reads."""
        self._check(self._lib.bb200_amcl_batch_remove_map(self._h, map_id))
        self._field_shapes.pop(map_id, None)

    def likelihood_field(self, map_id: int) -> np.ndarray:
        """likelihood_field() of a likelihood-field map as a (height, width) float32 array."""
        out = np.zeros(self._field_shapes.get(map_id, (1, 1)), dtype=np.float32)
        size = out.size if map_id in self._field_shapes else 0
        self._check(self._lib.bb200_amcl_batch_get_likelihood_field(self._h, map_id, out.ctypes.data_as(C.POINTER(C.c_float)), size))
        return out

    def initialize(self, member: int, mean_xytheta, cov):
        self._check(self._lib.bb200_amcl_batch_initialize(self._h, member, _dptr(_f64(mean_xytheta)), _dptr(_f64(cov).reshape(9))))

    def initialize_from_map(self, member: int):
        self._check(self._lib.bb200_amcl_batch_initialize_from_map(self._h, member))

    def initialize_states(self, member: int, states, weights=None):
        st = _f64(states).reshape(-1, 4)
        w = None if weights is None else _f64(weights)
        self._check(self._lib.bb200_amcl_batch_initialize_states(self._h, member, _dptr(st), None if w is None else _dptr(w), len(st)))

    def force_update(self, member: int):
        self._check(self._lib.bb200_amcl_batch_force_update(self._h, member))

    def member_size(self, member: int) -> int:
        """Member m's current particle count."""
        n = C.c_uint64(0)
        self._check(self._lib.bb200_amcl_batch_member_size(self._h, member, C.byref(n)))
        return n.value

    def _rows(self, member: int) -> int:
        # a fixed batch keeps its max_particles-row buffers; an adaptive one returns the member's current count
        # (a vacant slot asks the library, which refuses it)
        return self.member_size(member) if self.adaptive or self.params[member] is None else self.params[member].max_particles

    def particles(self, member: int):
        n = self._rows(member)
        st = np.zeros((n, 4))
        w = np.zeros(n)
        self._check(self._lib.bb200_amcl_batch_get_particles(self._h, member, _dptr(st) if n else None, _dptr(w) if n else None, n))
        return st, w

    def ancestors(self, member: int) -> np.ndarray:
        out = np.zeros(self._rows(member), dtype=np.int64)
        self._check(self._lib.bb200_amcl_batch_ancestors(self._h, member, out.ctypes.data_as(C.POINTER(C.c_int64)), len(out)))
        return out

    def cluster_estimate(self, member: int, linear: float = 0.20, angular: float = 0.524, percentile: float = 0.90):
        """beluga::cluster_based_estimate of one member -> (mean[4], cov[3, 3])."""
        p = _capi.ClusterParam(linear, angular, percentile)
        est = _capi.Estimate()
        self._check(self._lib.bb200_amcl_batch_cluster_estimate(self._h, member, C.byref(p), C.byref(est)))
        return np.array(est.mean), np.array(est.cov).reshape(3, 3)

    def cluster_estimates(self, present=None, linear: float = 0.20, angular: float = 0.524, percentile: float = 0.90, with_counts: bool = False):
        """beluga::cluster_based_estimate of every member whose `present` entry is true (None: all), in one call with a fixed
        number of kernel launches -> one (mean[4], cov[3, 3]) per member, None for members not selected; with_counts makes
        each entry (mean, cov, n_cells, n_clusters)."""
        k = len(self.params)
        if present is not None and len(present) != k:
            raise ValueError("one presence flag per member")
        p = _capi.ClusterParam(linear, angular, percentile)
        mask = None if present is None else (C.c_uint8 * k)(*[1 if x else 0 for x in present])
        est = (_capi.Estimate * k)()
        cells, clusters = (C.c_uint32 * k)(), (C.c_uint32 * k)()
        self._check(self._lib.bb200_amcl_batch_cluster_estimates(self._h, C.byref(p), mask, est, cells, clusters))
        out = []
        for m in range(k):
            if self._skipped(present, m):
                out.append(None)
                continue
            e = (np.array(est[m].mean), np.array(est[m].cov).reshape(3, 3))
            out.append((*e, cells[m], clusters[m]) if with_counts else e)
        return out

    def _mask(self, present):
        k = len(self.params)
        if present is not None and len(present) != k:
            raise ValueError("one presence flag per member")
        return None if present is None else (C.c_uint8 * k)(*[1 if x else 0 for x in present])

    def particle_histograms(self, present=None, linear: float = 1e-3, angular: float = 1e-3):
        """Filter.particle_histogram of every member whose `present` entry is true (None: all), in one call with a fixed
        number of kernel launches -> per member (bins, max_bin_weight), None for members not selected.  `bins` is a
        structured array of bb200_cluster_cell records (fields rep[4], hash, first, count, weight, m[9]) in first-occurrence order."""
        mask = self._mask(present)
        k = len(self.params)
        # A member has at most as many bins as particles: buffers of max_particles bins take every histogram in one pass.
        bufs = [np.empty(0 if q is None else q.max_particles, dtype=_CELL_DTYPE) for q in self.params]
        bins = (C.POINTER(_capi.ClusterCell) * k)(*[b.ctypes.data_as(C.POINTER(_capi.ClusterCell)) for b in bufs])
        capacity = (C.c_uint64 * k)(*[len(b) for b in bufs])
        n_bins, top = (C.c_uint64 * k)(), (C.c_double * k)()
        self._check(self._lib.bb200_amcl_batch_particle_histograms(self._h, linear, angular, mask, bins, capacity, n_bins, top))
        return [None if self._skipped(present, m) else (bufs[m][:n_bins[m]].copy(), top[m]) for m in range(k)]

    def sample_states(self, count, step: int = 0xFFFFFFFF, present=None):
        """Filter.sample_states(count, step) of every member whose `present` entry is true (None: all), in one call ->
        per member a (count, 4) array [cos, sin, x, y], None for members not selected.  `count`: one number for every
        member or one per member."""
        mask = self._mask(present)
        k = len(self.params)
        counts = [int(count)] * k if np.isscalar(count) else [int(c) for c in count]
        if len(counts) != k:
            raise ValueError("one sample count per member")
        if any(c < 0 for c in counts):
            raise ValueError("sample counts must not be negative")
        outs = [np.zeros((c, 4)) for c in counts]
        ptrs = (C.POINTER(C.c_double) * k)(*[_dptr(o) if len(o) else None for o in outs])
        self._check(self._lib.bb200_amcl_batch_sample_states(self._h, (C.c_uint64 * k)(*counts), step, mask, ptrs))
        return [None if self._skipped(present, m) else outs[m] for m in range(k)]

    def cast_rays(self, poses, bearings, max_range, present=None, map_ids=None) -> list:
        """Filter.cast_rays for every member whose `present` entry is true (None: every occupied slot), in one launch ->
        per member an (n_poses, n_bearings) array, None for members not selected.  `poses`: per member an (n, 4) array
        (None where not selected); `bearings`: one (m, 2) array for every member, or one per member; `max_range`: one
        number for every member, or one per member; `map_ids`: per member a map id of the batch to cast on, -1 (or
        map_ids None) for the member's own map."""
        mask = self._mask(present)
        k = len(self.params)
        shared = isinstance(bearings, np.ndarray) and bearings.ndim == 2
        if len(poses) != k or (not shared and len(bearings) != k):
            raise ValueError("one pose array and one bearing array per member")
        ranges = [float(max_range)] * k if np.isscalar(max_range) else [float(r) for r in max_range]
        if len(ranges) != k or (map_ids is not None and len(map_ids) != k):
            raise ValueError("one maximum range and one map id per member")
        sel = [not self._skipped(present, m) for m in range(k)]
        rays = [_rays(poses[m], bearings if shared else bearings[m]) if sel[m] else (np.zeros((0, 4)), np.zeros((0, 2))) for m in range(k)]
        outs = [np.zeros((len(p), len(b))) for p, b in rays]
        ptr = lambda a: _dptr(a) if a.size else None  # noqa: E731
        self._check(self._lib.bb200_amcl_batch_cast_rays(
            self._h, mask, None if map_ids is None else (C.c_int * k)(*[int(i) for i in map_ids]),
            (C.POINTER(C.c_double) * k)(*[ptr(p) for p, _ in rays]), (C.c_uint64 * k)(*[len(p) for p, _ in rays]),
            (C.POINTER(C.c_double) * k)(*[ptr(b) for _, b in rays]), (C.c_uint64 * k)(*[len(b) for _, b in rays]),
            (C.c_double * k)(*ranges), (C.POINTER(C.c_double) * k)(*[ptr(o) for o in outs])))
        return [outs[m] if sel[m] else None for m in range(k)]

    def update(self, control_poses, points, present=None) -> list:
        """Amcl::update for every member whose `present` entry is true (None: all).  `control_poses`: K poses [c, s, x, y];
        `points[m]`: member m's (x, y) points.  Returns K UpdateResult blocks; `.updated == 0` for absent members."""
        k = len(self.params)
        poses = _f64(control_poses).reshape(k, 4)
        pts = [_f64(() if p is None else p).reshape(-1, 2) for p in points]
        ptrs = (C.POINTER(C.c_double) * k)(*[_dptr(p) if len(p) else None for p in pts])
        counts = (C.c_uint64 * k)(*[len(p) for p in pts])
        mask = None if present is None else (C.c_uint8 * k)(*[1 if x else 0 for x in present])
        res = (_capi.UpdateResult * k)()
        self._check(self._lib.bb200_amcl_batch_update(self._h, _dptr(poses), ptrs, counts, mask, res))
        return list(res)

    def update_measurements(self, control_poses, measurements, present=None) -> list:
        """update() with each member's measurement as base-frame points ((n, 2) array), a LaserScan, a PointCloud or, for a
        member on a landmark map, Detections, as Amcl.update, Amcl.update_scan, Amcl.update_point_cloud and
        Amcl.update_landmarks take them; scans and clouds are converted on the device.  Results are bit-identical to those
        of update() given scan_to_points / point_cloud_to_points of the same messages."""
        k = len(self.params)
        mask = self._mask(present)
        table, built = self._built(measurements, present)
        poses = _f64(control_poses).reshape(k, 4)
        res = (_capi.UpdateResult * k)()
        self._check(self._lib.bb200_amcl_batch_update_measurements(self._h, _dptr(poses), table, mask, res))
        return list(res)

    def update_clustered(self, control_poses, measurements, present=None, linear: float = 0.20, angular: float = 0.524, percentile: float = 0.90,
                         with_counts: bool = False):
        """update_measurements, then the cluster-based estimate of every member that updated, in one call
        (bb200_amcl_batch_update_clustered): what beluga_ros's Amcl::update returns per member.  Returns (results,
        estimates): the K UpdateResult blocks update_measurements returns, and per member (mean[4], cov[3, 3]) -- with
        with_counts, (mean, cov, n_cells, n_clusters) -- or None for a member that did not update.  The estimates equal
        cluster_estimates(present=updated members) called right after update_measurements, byte for byte."""
        k = len(self.params)
        mask = self._mask(present)
        table, built = self._built(measurements, present)
        poses = _f64(control_poses).reshape(k, 4)
        p = _capi.ClusterParam(linear, angular, percentile)
        res = (_capi.UpdateResult * k)()
        est = (_capi.Estimate * k)()
        cells, clusters = (C.c_uint32 * k)(), (C.c_uint32 * k)()
        self._check(self._lib.bb200_amcl_batch_update_clustered(self._h, _dptr(poses), table, mask, C.byref(p), res, est, cells, clusters))
        out = []
        for m in range(k):
            if not res[m].updated:
                out.append(None)
                continue
            e = (np.array(est[m].mean), np.array(est[m].cov).reshape(3, 3))
            out.append((*e, cells[m], clusters[m]) if with_counts else e)
        return list(res), out

    def update_weighted(self, control_poses, measurements, weigh, present=None, cluster=None):
        """update_measurements with members weighed by the caller's own sensor model (bb200_amcl_batch_update_begin / _end):
        a None measurement marks a weighed member; the others pass points, a LaserScan, a PointCloud or Detections as in
        update_measurements.  `weigh(members, states, factors)` is called once, with the indices of the weighed members that
        update in this step and, per member, torch CUDA tensors over its views without a copy: its propagated states,
        (n, 4) float64, and its factors, (n,) float64, which it fills with L(states[i]).  It runs inside
        torch.cuda.stream(torch.cuda.ExternalStream(stream)) on the batch's stream and is not called when no weighed member
        updates.  When it raises, the step is closed with every factor 1 and the exception propagates.  cluster: None, or
        (linear, angular, percentile) for the cluster estimates of update_clustered; the return value is then (results,
        estimates) as update_clustered returns it, otherwise the results."""
        k = len(self.params)
        mask = self._mask(present)
        table, built = self._built(measurements, present, weighed=True)
        poses = _f64(control_poses).reshape(k, 4)
        views = (_capi.WeighView * k)()
        self._check(self._lib.bb200_amcl_batch_update_begin(self._h, _dptr(poses), table, mask, views))
        res = (_capi.UpdateResult * k)()
        est = (_capi.Estimate * k)()
        cells, clusters = (C.c_uint32 * k)(), (C.c_uint32 * k)()
        p = None if cluster is None else _capi.ClusterParam(*cluster)

        def end():
            return self._lib.bb200_amcl_batch_update_end(self._h, None if p is None else C.byref(p), res, None if p is None else est,
                                                         None if p is None else cells, None if p is None else clusters)

        members = [m for m in range(k) if measurements[m] is None and views[m].updated]
        if members:
            import torch

            device = torch.device("cuda", next(q.device for q in self.params if q is not None))
            states = [torch.as_tensor(_CudaArray(views[m].states, (views[m].n, 4)), device=device) for m in members]
            factors = [torch.as_tensor(_CudaArray(views[m].factors, (views[m].n,)), device=device) for m in members]
            with torch.cuda.stream(torch.cuda.ExternalStream(views[members[0]].stream, device=device)):
                try:
                    weigh(members, states, factors)
                except BaseException:
                    for f in factors:
                        f.fill_(1.0)
                    end()
                    raise
        self._check(end())
        if p is None:
            return list(res)
        out = [None if not res[m].updated else (np.array(est[m].mean), np.array(est[m].cov).reshape(3, 3)) for m in range(k)]
        return list(res), out

    def update_scans(self, control_poses, scans, present=None) -> list:
        """update_measurements with a LaserScan for every member."""
        if any(not isinstance(s, LaserScan) for s in scans):
            raise TypeError("update_scans takes one LaserScan per member")
        return self.update_measurements(control_poses, scans, present)

    def update_point_clouds(self, control_poses, clouds, present=None) -> list:
        """update_measurements with a PointCloud for every member."""
        if any(not isinstance(c, PointCloud) for c in clouds):
            raise TypeError("update_point_clouds takes one PointCloud per member")
        return self.update_measurements(control_poses, clouds, present)

    def launch_count(self) -> int:
        return self._lib.bb200_amcl_batch_launch_count(self._h)
