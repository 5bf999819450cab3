"""Oracle of the landmark and bearing sensor models, in plain Python floats (IEEE doubles, correctly rounded, no
contraction; math.exp / math.atan2 / math.sqrt are the C library's).

Restates, for SE(2) states:
- beluga::LandmarkMap (sensor/data/landmark_map.hpp:40-166): the explicit and implicit bounds (:49-71),
  find_nearest_landmark (:81-110) and find_closest_bearing_landmark (:117-164).  Both searches are std::min_element over
  the landmarks of the detection's category in map order: the first minimum wins, the comparators are strict
  (distance a < b, bearing dot_a > dot_b), and a comparison with a NaN keeps the current candidate.
- LandmarkSensorModel2d (sensor/landmark_sensor_model.hpp:96-156) and BearingSensorModel2d
  (sensor/bearing_sensor_model.hpp:92-140), with the product over detections in libstdc++ 13's grouping of four
  (<numeric>:439-462).

Sophus SO3/SE3 and Eigen are not part of the reference checkout, so this oracle fixes the evaluation order the library
documents (DESIGN.md §1): the rotation about z is the state's stored (cos, sin); R * p adds its row products left to
right without the zero entries of the z rotation; a pose's inverse applied to p is R^T (p - t); dot products and squared
norms add left to right; normalized() is v / sqrt(squaredNorm) when that is > 0 and v itself otherwise (Eigen's rule).
"""
from __future__ import annotations

import math


def dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def normalized(v):
    n = dot(v, v)
    if n > 0.0:
        r = math.sqrt(n)
        return (v[0] / r, v[1] / r, v[2] / r)
    return tuple(v)


def cross_norm(a, b):
    c = (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])
    return math.sqrt(dot(c, c))


def aperture(a, b):
    return math.atan2(cross_norm(a, b), dot(a, b))


def gauss(e, den):
    return math.exp(-e * e / den)


def product_by_fours(values):
    """std::transform_reduce(first, last, 1.0, std::multiplies{}, f) as libstdc++ 13 evaluates it."""
    init, i, n = 1.0, 0, len(values)
    while n - i >= 4:
        init = init * ((values[i] * values[i + 1]) * (values[i + 2] * values[i + 3]))
        i += 4
    for k in range(i, n):
        init = init * values[k]
    return init


class LandmarkMap:
    """landmarks: list of (x, y, z, category) in map order; bounds ((x, y, z), (x, y, z)) or None (implicit)."""

    def __init__(self, landmarks, bounds=None):
        self.landmarks = [(float(x), float(y), float(z), int(c)) for x, y, z, c in landmarks]
        if bounds is not None:
            self.bounds = (tuple(map(float, bounds[0])), tuple(map(float, bounds[1])))
        elif self.landmarks:  # landmark_map.hpp:61-71: cwiseMin / cwiseMax from the first landmark
            lo = list(self.landmarks[0][:3])
            hi = list(self.landmarks[0][:3])
            for l in self.landmarks[1:]:
                for k in range(3):
                    lo[k] = l[k] if l[k] < lo[k] else lo[k]
                    hi[k] = l[k] if hi[k] < l[k] else hi[k]
            self.bounds = (tuple(lo), tuple(hi))
        else:  # a default-constructed AlignedBox3d: empty (min = +max, max = -max)
            big = 1.7976931348623157e308
            self.bounds = ((big, big, big), (-big, -big, -big))

    def map_limits(self):
        return self.bounds

    def _category(self, category):
        return [l for l in self.landmarks if l[3] == category]

    def find_nearest_landmark(self, query, category):
        best, best_key = None, None
        for l in self._category(category):
            e = (l[0] - query[0], l[1] - query[1], l[2] - query[2])
            key = dot(e, e)
            if best is None or key < best_key:
                best, best_key = l, key
        return None if best is None else best[:3]

    def find_closest_bearing_landmark(self, detection, category, frame):
        best, best_key = None, None
        for l in self._category(category):
            key = dot(normalized(to_frame(frame, l)), detection)
            if best is None or key > best_key:
                best, best_key = l, key
        return None if best is None else normalized(to_frame(frame, best))


def robot_frame(state):
    c, s, x, y = state
    return ((c, -s, 0.0, s, c, 0.0, 0.0, 0.0, 1.0), (x, y, 0.0))


def sensor_frame(state, sensor_pose):
    """robot_pose * sensor_pose_in_robot; sensor_pose a 3x4 [R | t] as 12 row-major numbers."""
    c, s, x, y = state
    R = [sensor_pose[0:3], sensor_pose[4:7], sensor_pose[8:11]]
    t = (sensor_pose[3], sensor_pose[7], sensor_pose[11])
    r = [0.0] * 9
    for j in range(3):
        r[j] = c * R[0][j] - s * R[1][j]
        r[3 + j] = s * R[0][j] + c * R[1][j]
        r[6 + j] = R[2][j]
    return (tuple(r), ((c * t[0] - s * t[1]) + x, (s * t[0] + c * t[1]) + y, t[2]))


def to_frame(frame, p):
    """frame^-1 * p = R^T (p - t)."""
    r, t = frame
    dx, dy, dz = p[0] - t[0], p[1] - t[1], p[2] - t[2]
    return ((r[0] * dx + r[3] * dy) + r[6] * dz, (r[1] * dx + r[4] * dy) + r[7] * dz, (r[2] * dx + r[5] * dy) + r[8] * dz)


def landmark_weight(state, detections, lmap: LandmarkMap, sigma_range, sigma_bearing, random_prob):
    """LandmarkSensorModel2d's weight of one state; detections: (x, y, z, category) in the robot frame."""
    frame = robot_frame(state)
    r, t = frame
    range_den = 2. * sigma_range * sigma_range
    bearing_den = 2. * sigma_bearing * sigma_bearing
    factors = []
    for d in detections:
        p = tuple(map(float, d[:3]))
        d_range = math.sqrt(dot(p, p))
        d_bearing = normalized(p)
        query = ((r[0] * p[0] + r[1] * p[1]) + t[0], (r[3] * p[0] + r[4] * p[1]) + t[1], p[2] + t[2])
        l = lmap.find_nearest_landmark(query, int(d[3]))
        if l is None:
            factors.append(random_prob)
            continue
        q = to_frame(frame, l)
        l_range = math.sqrt(dot(q, q))
        l_bearing = normalized(q)
        bearing_error = aperture(l_bearing, d_bearing)
        range_error = d_range - l_range
        factors.append(gauss(range_error, range_den) * gauss(bearing_error, bearing_den) + random_prob)
    return product_by_fours(factors)


def bearing_weight(state, detections, lmap: LandmarkMap, sigma_bearing, sensor_pose):
    """BearingSensorModel2d's weight of one state; detections: (x, y, z, category) bearings in the sensor frame."""
    frame = sensor_frame(state, sensor_pose)
    den = 2. * sigma_bearing * sigma_bearing
    factors = []
    for d in detections:
        p = tuple(map(float, d[:3]))
        b = lmap.find_closest_bearing_landmark(p, int(d[3]), frame)
        if b is None:
            factors.append(0.0)
            continue
        factors.append(gauss(aperture(normalized(p), b), den))
    return product_by_fours(factors)


def box_state(seed, index, step, box, philox):
    """MultivariateUniformDistribution<SE2d, AlignedBox2d> (random/multivariate_uniform_distribution.hpp:43-73) in the
    library's counter-RNG form (DESIGN.md §1): yaw from word a and x from word b of stream 6, y from word a of stream 7,
    each u * (max - min) + min with u = ((bits >> 11) + 0.5) 2^-53.  `box` = (min_x, max_x, min_y, max_y); `philox` is
    Philox4x32-10 (counter, key) -> four uint32 words.  Returns (yaw, x, y)."""
    def draw(stream):
        w = [int(v) for v in philox([index & 0xFFFFFFFF, index >> 32, step, stream], [seed & 0xFFFFFFFF, seed >> 32])]
        return (w[1] << 32) | w[0], (w[3] << 32) | w[2]

    def u(bits):
        return (float(bits >> 11) + 0.5) * 2.0 ** -53

    a, b = draw(6)
    q, _ = draw(7)
    pi = 3.14159265358979323846
    return u(a) * (pi - (-pi)) + (-pi), u(b) * (box[1] - box[0]) + box[0], u(q) * (box[3] - box[2]) + box[2]


IDENTITY_POSE = (1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0)
