"""Laser scans and point clouds in a batch step (bb200_amcl_batch_update_measurements) on the GPU: every member equals, byte for
byte, a standalone Amcl fed update_scan / update_point_cloud / update, and a second batch fed bb200_amcl_batch_update with
the points scan_to_points / point_cloud_to_points return -- update results, particles, weights and ancestors after every
step of a trajectory.  Covered: the likelihood field, the prob model and the beam model (two-pass and fused), one map and
several; K = 1, 16 and 256 with absent members; scans with NaN, +-inf and ranges exactly at min_range / max_range, every
beam filtered out, max_beams 0, 1, 2, n - 1, n and above, no ranges at all, a rotated and translated origin, an origin with
a NaN entry and a scan geometry that changes along the trajectory; float32 and float64 clouds with unaligned records and a
non-zero x_offset at 1, 2049 and 65 537 points; a call mixing all three kinds; the launch count (unchanged for points, one
more with any scan or cloud); and a refused cloud that leaves every member's later steps equal to its twin's."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
SIZES = (1, 33, 256, 2000, 500)
STEPS = 5
INVALID = -1


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


@pytest.fixture(scope="module")
def scene():
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=STEPS + 2)


def origin(yaw=0.3, x=0.2, y=-0.1, z=0.5, pitch=0.02):
    cy, sy, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    r = np.array([[cy * cp, -sy, cy * sp], [sy * cp, cy, sy * sp], [-sp, 0.0, cp]])
    return np.hstack([r, [[x], [y], [z]]])


def ranges(scene, t, n):
    """n ranges of the scene's scan at step t (float32), in beam order."""
    return np.hypot(*np.resize(scene.scans[t % len(scene.scans)], (max(n, 1), 2)).T)[:n].astype(np.float32)


def laser(bb, scene, t, n=181, **kw):
    return bb.LaserScan(ranges(scene, t, n), np.float32(-np.pi), np.float32(2 * np.pi / max(n, 1)), **kw)


def cloud(bb, scene, t, n, coordinate=np.float32, step=22, x_offset=6, with_origin=True, nan_at=None):
    """n packed records of `step` bytes, x, y, z (of `coordinate`) at x_offset: the scene's scan points, z varying."""
    pts = np.resize(scene.scans[t % len(scene.scans)], (max(n, 1), 2))[:n]
    xyz = np.column_stack([pts, 0.01 * np.arange(n) % 0.7]).astype(coordinate)
    if nan_at is not None and n > nan_at:
        xyz[nan_at, 1] = np.nan
    raw = np.zeros((n, step), dtype=np.uint8)
    if n:
        raw[:, x_offset:x_offset + xyz.itemsize * 3] = xyz.view(np.uint8).reshape(n, -1)
    return bb.PointCloud(raw.tobytes(), step, x_offset, coordinate, origin(-0.2) if with_origin else None, n)


def member_spec(bb, scene, m, t):
    """Member m's measurement at step t: a scan, a cloud or points, each edge case on some member."""
    n = 181
    r = ranges(scene, t, n)
    edge = r.copy()
    edge[::7] = np.nan
    edge[1::11] = np.inf
    edge[2::13] = -np.inf
    edge[3::5] = np.float32(0.5)   # exactly min_range
    edge[4::9] = np.float32(30.0)  # exactly max_range
    specs = [
        lambda: laser(bb, scene, t),
        lambda: bb.LaserScan(edge, np.float32(-np.pi), np.float32(2 * np.pi / n), 0.5, 30.0, 0, origin()),
        lambda: laser(bb, scene, t, n, min_range=100.0),  # every beam filtered out
        lambda: laser(bb, scene, t, n, max_beams=1),
        lambda: laser(bb, scene, t, n, max_beams=2, laser_origin=origin(1.0)),
        lambda: laser(bb, scene, t, n, max_beams=n - 1),
        lambda: laser(bb, scene, t, n, max_beams=n),
        lambda: laser(bb, scene, t, n, max_beams=n + 40),
        lambda: laser(bb, scene, t, 0),
        lambda: laser(bb, scene, t, n, laser_origin=np.where(np.arange(12).reshape(3, 4) == 5, np.nan, origin())),
        lambda: laser(bb, scene, t, 90 + 30 * (t % 3), max_beams=60 + 7 * (t % 2)),  # the geometry changes from step to step
        lambda: cloud(bb, scene, t, 2049),
        lambda: cloud(bb, scene, t, 1, coordinate=np.float64, step=27, x_offset=3),
        lambda: cloud(bb, scene, t, 2049, coordinate=np.float64, step=27, x_offset=3, with_origin=False, nan_at=100),
        lambda: np.resize(scene.scans[t % len(scene.scans)], (120, 2)),
        lambda: np.zeros((0, 2)),
        lambda: cloud(bb, scene, t, 0),
    ]
    return specs[m % len(specs)]()


def to_points(bb, spec):
    if isinstance(spec, bb.LaserScan):
        return bb.scan_to_points(spec.ranges, spec.angle_min, spec.angle_increment, spec.min_range, spec.max_range, spec.max_beams, spec.laser_origin)
    if isinstance(spec, bb.PointCloud):
        return bb.point_cloud_to_points(spec.data, spec.point_step, spec.x_offset, spec.dtype, spec.origin, spec.n_points)
    return spec


def twin_update(twin, pose, spec, bb):
    if isinstance(spec, bb.LaserScan):
        return twin.update_scan(pose, spec.ranges, spec.angle_min, spec.angle_increment, spec.min_range, spec.max_range, spec.max_beams,
                                spec.laser_origin)
    if isinstance(spec, bb.PointCloud):
        return twin.update_point_cloud(pose, spec.data, spec.point_step, spec.x_offset, spec.dtype, spec.origin, spec.n_points)
    return twin.update(pose, spec)


def motion(bb, k):
    return [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.OmnidirectionalDriveModelParam(*ALPHAS), bb.StationaryModelParam()][k % 3]


def member_params(bb, k):
    n = SIZES[k % len(SIZES)]
    p = bb.AmclParams(min_particles=n, max_particles=n, seed=300 + k, resample_scheme=k % 2, record_ancestors=True)
    if k % 4 == 3:
        p.resample_interval = 2  # normalising and resampling steps alternate
    return p


def odometry(scene, t, m):
    x, y, th = scene.poses[t]
    th = th + 0.01 * (m % 7)
    return np.array([np.cos(th), np.sin(th), x + 0.02 * (m % 5), y])


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


class Rig:
    """A batch fed measurements, a batch fed host-converted points and standalone twins of the members in `twinned`."""

    def __init__(self, bb, scene, k, maps, twinned):
        self.bb, self.scene, self.k = bb, scene, k
        params = [member_params(bb, m) for m in range(k)]
        motions = [motion(bb, m) for m in range(k)]
        self.a = bb.AmclBatch(motions, params)
        self.b = bb.AmclBatch(motions, params)
        self.twins = {m: bb.Amcl(motions[m], params[m]) for m in twinned}
        for batch in (self.a, self.b):
            ids = [add(batch) for add, _ in maps]
            for m in range(k):
                batch.update_map(m, ids[m % len(ids)])
        for m, twin in self.twins.items():
            maps[m % len(maps)][1](twin)
        for m in range(k):
            mean = scene.initial_mean + np.array([0.02 * (m % 5), 0.0, 0.01 * (m % 7)])
            self.a.initialize(m, mean, scene.initial_cov)
            self.b.initialize(m, mean, scene.initial_cov)
            if m in self.twins:
                self.twins[m].initialize(mean, scene.initial_cov)

    def step(self, t, present=None, specs=None):
        bb, k = self.bb, self.k
        specs = specs or [member_spec(bb, self.scene, m, t) for m in range(k)]
        poses = np.array([odometry(self.scene, t, m) for m in range(k)])
        la, lb = self.a.launch_count(), self.b.launch_count()
        ra = self.a.update_measurements(poses, specs, present)
        rb = self.b.update(poses, [to_points(bb, s) for s in specs], present)
        converted = any(r.updated and not isinstance(s, np.ndarray) for r, s in zip(ra, specs))
        assert self.a.launch_count() - la == self.b.launch_count() - lb + (1 if converted else 0), t
        for m in range(k):
            where = f"step {t}, member {m}"
            assert result_bytes(ra[m]) == result_bytes(rb[m]), where
            if m in self.twins and (present is None or present[m]):
                rt = twin_update(self.twins[m], poses[m], specs[m], bb)
                assert result_bytes(ra[m]) == result_bytes(rt), where
            if not ra[m].updated:
                continue
            sa, wa = self.a.particles(m)
            sb, wb = self.b.particles(m)
            assert sa.tobytes() == sb.tobytes() and wa.tobytes() == wb.tobytes(), where
            if ra[m].resampled:
                assert np.array_equal(self.a.ancestors(m), self.b.ancestors(m)), where
            if m in self.twins:
                ts, tw = self.twins[m].particles()
                n = len(ts)
                assert sa[:n].tobytes() == ts.tobytes() and wa[:n].tobytes() == tw.tobytes(), where
                if ra[m].resampled:
                    assert np.array_equal(self.a.ancestors(m), self.twins[m].filter.ancestors()), where
        return ra


def lfm_map(bb, scene, prob=False):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    sensor = bb.SENSOR_LIKELIHOOD_FIELD_PROB if prob else bb.SENSOR_LIKELIHOOD_FIELD
    return (lambda batch: batch.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid, prob),
            lambda twin: twin.update_map(sensor, bb.LikelihoodFieldModelParam(**LFM), grid))


def beam_map(bb, scene, wide=False):
    cells = np.pad(scene.cells, ((0, 0), (0, 70_000 - scene.cells.shape[1])), constant_values=0) if wide else scene.cells
    grid = bb.OccupancyGrid(cells, scene.resolution)
    beam = bb.BeamModelParam(beam_max_range=20.0)
    return (lambda batch: batch.add_beam_map(beam, grid), lambda twin: twin.update_map(bb.SENSOR_BEAM, beam, grid))


MODELS = {
    "likelihood_field": lambda bb, sc: [lfm_map(bb, sc)],
    "prob": lambda bb, sc: [lfm_map(bb, sc, prob=True)],
    "beam_two_pass": lambda bb, sc: [beam_map(bb, sc)],
    "beam_fused": lambda bb, sc: [beam_map(bb, sc, wide=True)],
    "several_maps": lambda bb, sc: [lfm_map(bb, sc), beam_map(bb, sc), lfm_map(bb, sc, prob=True)],
}


@pytest.mark.parametrize("model", sorted(MODELS))
def test_members_equal_twins_and_host_converted_batch(bb, scene, model):
    k = 17  # every member spec once
    rig = Rig(bb, scene, k, MODELS[model](bb, scene), twinned=range(k))
    for t in range(STEPS):
        present = None if t % 2 == 0 else [m % 3 != t % 3 for m in range(k)]
        rig.step(t, present)


@pytest.mark.parametrize("k", [1, 16, 256])
def test_batch_sizes_with_absent_members(bb, scene, k):
    rig = Rig(bb, scene, k, MODELS["likelihood_field"](bb, scene), twinned=sorted({0, k // 2, k - 1}))
    for t in range(STEPS):
        rig.step(t, None if t == 0 else [(m + t) % 4 != 0 for m in range(k)])


def test_large_clouds(bb, scene):
    k = 3
    rig = Rig(bb, scene, k, MODELS["likelihood_field"](bb, scene), twinned=range(k))
    for t in range(3):
        specs = [cloud(bb, scene, t, 65_537), cloud(bb, scene, t, 65_537, coordinate=np.float64, step=29, x_offset=5, nan_at=65_536),
                 cloud(bb, scene, t, 2049, with_origin=False)]
        rig.step(t, specs=specs)


@pytest.mark.parametrize("k", [1, 16, 256])
def test_launch_counts(bb, scene, k):
    """Points only: the launches of bb200_amcl_batch_update; any scan or cloud among the updating members: one more."""
    rig = Rig(bb, scene, k, MODELS["likelihood_field"](bb, scene), twinned=[])
    points = [np.resize(scene.scans[0], (100, 2))] * k
    for t, specs in enumerate([points, [laser(bb, scene, 1)] + points[1:], [cloud(bb, scene, 2, 10)] * k, points]):
        before = rig.a.launch_count()
        rig.step(t, specs=specs)
        assert rig.a.launch_count() - before == 5 + (0 if specs is points else 1), t


def test_refused_cloud_changes_nothing(bb, scene):
    k = 6
    rig = Rig(bb, scene, k, MODELS["likelihood_field"](bb, scene), twinned=range(k))
    rig.step(0)
    bad = cloud(bb, scene, 1, 10)
    bad.x_offset = 11  # 11 + 12 > 22
    specs = [member_spec(bb, scene, m, 1) for m in range(k)]
    specs[4] = bad
    poses = np.array([odometry(scene, 1, m) for m in range(k)])
    before = rig.a.launch_count()
    with pytest.raises(bb.BelugaB200Error) as e:
        rig.a.update_measurements(poses, specs)
    assert e.value.status == INVALID and rig.a.launch_count() == before
    for dtype in (np.int32, 9):
        bad = cloud(bb, scene, 1, 10)
        bad.dtype = dtype
        specs[4] = bad
        with pytest.raises(bb.BelugaB200Error) as e:
            rig.a.update_measurements(poses, specs, present=[m != 2 for m in range(k)])
        assert e.value.status == INVALID
    for t in range(1, STEPS):
        rig.step(t)
