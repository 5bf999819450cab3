"""Synthetic localisation workload (SURVEY.md section 8(d)): occupancy map, closed trajectory with
perfect odometry, and noisy 360-degree scans converted to base-frame cartesian points the way
beluga_ros does (beluga/sensor/data/laser_scan.hpp:64-91 + beluga_ros/src/amcl.cpp:57-62), and lidar point clouds of the
same scene as packed PointCloud2 records (make_point_cloud).

Pure numpy; deterministic for a given configuration.  Used by bench.py and the tests to drive both
the GPU backend and the CPU oracle with identical inputs.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class Scenario:
    cells: np.ndarray          # int8 [H, W]: 0 free, 100 occupied
    resolution: float
    poses: np.ndarray          # [T, 3] ground-truth / odometry (x, y, theta), T = steps + 1
    scans: list                # T arrays [B, 2] of base-frame points
    initial_mean: np.ndarray   # (x, y, theta)
    initial_cov: np.ndarray    # 3x3


def make_map(size: int, resolution: float = 0.05, seed: int = 42, occupancy: float = 0.10, keep_free=None) -> np.ndarray:
    """Outer walls two cells thick plus random axis-aligned rectangles up to ~`occupancy` of the area.

    `keep_free(x0, y0, x1, y1) -> bool` (metres) vetoes rectangles that would block the robot path."""
    rng = np.random.Generator(np.random.MT19937(seed))
    cells = np.zeros((size, size), dtype=np.int8)
    cells[:2, :] = cells[-2:, :] = 100
    cells[:, :2] = cells[:, -2:] = 100
    target = occupancy * size * size
    guard = 0
    while cells.astype(bool).sum() < target and guard < 100000:
        guard += 1
        w = int(rng.integers(4, max(5, size // 12)))
        h = int(rng.integers(4, max(5, size // 12)))
        x0 = int(rng.integers(2, size - 2 - w))
        y0 = int(rng.integers(2, size - 2 - h))
        if keep_free is not None and keep_free(x0 * resolution, y0 * resolution, (x0 + w) * resolution, (y0 + h) * resolution):
            continue
        cells[y0:y0 + h, x0:x0 + w] = 100
    return cells


def circle_path(center, radius: float, steps: int) -> np.ndarray:
    """Closed circular path, heading tangent to the circle; steps + 1 poses (last == first position)."""
    a = np.linspace(0.0, 2.0 * np.pi, steps + 1)
    x = center[0] + radius * np.cos(a)
    y = center[1] + radius * np.sin(a)
    theta = np.arctan2(np.sin(a + np.pi / 2), np.cos(a + np.pi / 2))
    return np.stack([x, y, theta], axis=1)


def raycast_ranges(cells: np.ndarray, resolution: float, pose, n_beams: int, max_range: float) -> np.ndarray:
    """Range to the first occupied cell along n_beams directions over 360 degrees (marching at a
    quarter cell; synthetic ground truth, not the beam model's Bresenham)."""
    h, w = cells.shape
    angles = pose[2] + np.linspace(-np.pi, np.pi, n_beams, endpoint=False)
    dx, dy = np.cos(angles), np.sin(angles)
    step = 0.25 * resolution
    ranges = np.full(n_beams, max_range)
    alive = np.ones(n_beams, dtype=bool)
    occ = cells != 0
    for k in range(1, int(max_range / step) + 1):
        if not alive.any():
            break
        r = k * step
        xi = np.floor((pose[0] + r * dx[alive]) / resolution).astype(np.int64)
        yi = np.floor((pose[1] + r * dy[alive]) / resolution).astype(np.int64)
        inside = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
        hit = np.zeros(alive.sum(), dtype=bool)
        hit[inside] = occ[yi[inside], xi[inside]]
        stop = hit | ~inside
        idx = np.flatnonzero(alive)
        ranges[idx[hit]] = r
        alive[idx[stop]] = False
    return ranges


def make_scenario(grid_size: int = 500, n_beams: int = 180, steps: int = 100, resolution: float = 0.05, map_seed: int = 42,
                  noise_seed: int = 7, step_length: float = 0.4, scan_max_range: float = 30.0, range_sigma: float = 0.02) -> Scenario:
    extent = grid_size * resolution
    center = (extent / 2.0, extent / 2.0)
    radius = min(step_length * steps / (2.0 * np.pi), extent / 2.0 - 2.0)

    def keep_free(x0, y0, x1, y1):  # veto rectangles closer than 1 m to the path annulus
        cx = np.clip(center[0], x0, x1)
        cy = np.clip(center[1], y0, y1)
        dmin = np.hypot(cx - center[0], cy - center[1])
        corners = [(x0, y0), (x0, y1), (x1, y0), (x1, y1)]
        dmax = max(np.hypot(px - center[0], py - center[1]) for px, py in corners)
        return dmin <= radius + 1.0 and dmax >= radius - 1.0

    cells = make_map(grid_size, resolution, map_seed, keep_free=keep_free)
    poses = circle_path(center, radius, steps)
    rng = np.random.Generator(np.random.MT19937(noise_seed))
    scans = []
    for pose in poses:
        r = raycast_ranges(cells, resolution, pose, n_beams, scan_max_range)
        r = np.clip(r + rng.normal(0.0, range_sigma, n_beams), 0.05, scan_max_range)
        a = np.linspace(-np.pi, np.pi, n_beams, endpoint=False)
        scans.append(np.stack([r * np.cos(a), r * np.sin(a)], axis=1))  # laser_scan.hpp:64-70, laser at the base origin
    cov = np.diag([0.25, 0.25, 0.0685])  # likelihood_params.yaml:83-87
    return Scenario(cells, resolution, poses, scans, poses[0].copy(), cov)


# A packed sensor_msgs/PointCloud2 record of a spinning lidar: x, y, z, intensity (FLOAT32), ring (UINT16), time (FLOAT32)
# at offsets 0, 4, 8, 12, 16, 18, 22 bytes per point -- the Velodyne layout, no padding.  The float64 variant widens x, y, z.
LIDAR_FIELDS = ("x", "y", "z", "intensity", "ring", "time")


def lidar_record(coordinate_type=np.float32) -> np.dtype:
    c = np.dtype(coordinate_type).newbyteorder("<")
    w = c.itemsize
    return np.dtype({"names": list(LIDAR_FIELDS), "formats": [c, c, c, "<f4", "<u2", "<f4"],
                     "offsets": [0, w, 2 * w, 3 * w, 3 * w + 4, 3 * w + 6], "itemsize": 3 * w + 10})


@dataclass
class PointCloud:
    data: np.ndarray           # structured [height * width] array of lidar_record(), row-major (one row per laser ring)
    width: int                 # azimuths per ring
    height: int                # rings
    origin: np.ndarray         # 3x4 [R | t] of the sensor frame in the base frame

    @property
    def point_step(self) -> int:
        return self.data.dtype.itemsize

    @property
    def x_offset(self) -> int:
        return self.data.dtype.fields["x"][1]

    @property
    def datatype(self) -> int:  # sensor_msgs/PointField code of x, y, z
        return 7 if self.data.dtype.fields["x"][0] == np.float32 else 8


def sensor_origin(x: float = 0.2, y: float = -0.05, z: float = 0.8, roll: float = 0.01, pitch: float = -0.015, yaw: float = 0.03) -> np.ndarray:
    """3x4 [R | t] with R = Rz(yaw) Ry(pitch) Rx(roll): a lidar mounted above the base, slightly tilted."""
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    rot = np.array([[cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr],
                    [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr],
                    [-sp, cp * sr, cp * cr]])
    return np.concatenate([rot, np.array([[x], [y], [z]])], axis=1)


def make_point_cloud(sc: Scenario, k: int, rows: int = 16, azimuths: int = 1024, seed: int = 7, origin=None, coordinate_type=np.float32,
                     scan_max_range: float = 30.0, range_sigma: float = 0.02, vertical_fov: float = np.deg2rad(30.0)) -> PointCloud:
    """The lidar cloud seen from pose k of the scenario: `rows` rings x `azimuths` beams over 360 degrees, expressed in the
    sensor frame `origin` (default sensor_origin()).  The map is 2-D, so every ring hits the wall at the same horizontal
    distance: the raycast range from the sensor's position plus the scans' noise (drawn per point), at the ring's
    elevation, which gives each ring its own z.  The base-frame (x, y) of point (ring, j) is that hit; z is the sensor
    height plus distance * tan(elevation).  Deterministic for given arguments."""
    o = sensor_origin() if origin is None else np.asarray(origin, dtype=np.float64).reshape(3, 4)
    rot, t = o[:, :3], o[:, 3]
    yaw = np.arctan2(rot[1, 0], rot[0, 0])
    x, y, theta = sc.poses[k]
    sensor_pose = (x + np.cos(theta) * t[0] - np.sin(theta) * t[1], y + np.sin(theta) * t[0] + np.cos(theta) * t[1], theta + yaw)
    d = raycast_ranges(sc.cells, sc.resolution, sensor_pose, azimuths, scan_max_range)
    rng = np.random.Generator(np.random.MT19937(seed * 100003 + k))
    d = np.clip(d[None, :] + rng.normal(0.0, range_sigma, (rows, azimuths)), 0.05, scan_max_range)
    a = yaw + np.linspace(-np.pi, np.pi, azimuths, endpoint=False)  # beam directions in the base frame
    elevation = np.linspace(-vertical_fov / 2, vertical_fov / 2, rows)[:, None]
    base = np.stack([t[0] + d * np.cos(a), t[1] + d * np.sin(a), t[2] + d * np.tan(elevation)], axis=-1).reshape(-1, 3)
    sensor = (base - t) @ rot  # R^T (p - t), row by row
    out = np.zeros(rows * azimuths, dtype=lidar_record(coordinate_type))
    out["x"], out["y"], out["z"] = sensor[:, 0], sensor[:, 1], sensor[:, 2]
    out["intensity"] = (100.0 / (1.0 + d)).reshape(-1)
    out["ring"] = np.repeat(np.arange(rows, dtype=np.uint16), azimuths)
    out["time"] = np.tile(np.arange(azimuths, dtype=np.float32) / np.float32(azimuths * 10), rows)  # one sweep at 10 Hz
    return PointCloud(out, azimuths, rows, o)
