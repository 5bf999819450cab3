"""update and cluster estimate in one batch call (bb200_amcl_batch_update_clustered) on the GPU.

Two batches are built from the same parameters and fed the same inputs: one steps with update_clustered, its mirror with
update_measurements followed by cluster_estimates over the members that updated.  After every step both are compared
byte for byte -- results, particles, weights, ancestors, the clustered estimates, n_cells and n_clusters -- and, where the
test keeps them, against standalone twins (bb200_amcl, then bb200_filter_cluster_estimate).  Covered: fixed, KLD and
selective members side by side, both resampling schemes, recovery injection, resample_interval = 3, members gated by
on_motion and absent members, both likelihood-field models and both beam forms, several maps, points, scans and clouds,
members of 1, 2000 and 32 768 particles, a degenerate step with NaN weights and a heading on an angular bucket edge (both
take the host fallback, seen in the launch count), a refused parameter block, launch counts at K = 1, 16 and 256, and two
members against the oracle."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
# (min_particles, max_particles, scheme, selective, extra parameters) per member
MEMBERS = [
    (2000, 2000, 1, False, {}),
    (2000, 2000, 0, False, dict(recovery_probability_override=0.05)),
    (500, 2000, 1, False, {}),                                        # KLD
    (2000, 2000, 1, True, {}),                                        # selective
    (1, 1, 0, False, {}),
    (1000, 1000, 0, True, dict(resample_interval=3)),
    (100, 32768, 1, True, {}),                                        # KLD and selective
    (32768, 32768, 0, False, dict(resample_interval=3)),
]


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=14)


def motion(bb, k):
    return [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.OmnidirectionalDriveModelParam(*ALPHAS), bb.StationaryModelParam()][k % 3]


def member_params(bb, k, seed=500):
    lo, hi, scheme, selective, extra = MEMBERS[k % len(MEMBERS)]
    return bb.AmclParams(min_particles=lo, max_particles=hi, seed=seed + k, resample_scheme=scheme, selective_resampling=selective,
                         record_ancestors=True, **extra)


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


def estimate_bytes(e):
    return None if e is None else np.asarray(e[0]).tobytes() + np.asarray(e[1]).tobytes() + struct.pack("<II", e[2], e[3])


def odometry(scene, t, k):
    x, y, th = scene.poses[t - 1 if t % 5 == 4 else t]  # some steps repeat a pose: on_motion gates them
    th = th + 0.01 * k
    return np.array([np.cos(th), np.sin(th), x + 0.02 * k, y])


def feed_twin(bb, twin, pose, meas):
    if isinstance(meas, bb.LaserScan):
        return twin.update_scan(pose, meas.ranges, meas.angle_min, meas.angle_increment, meas.min_range, meas.max_range, meas.max_beams,
                                meas.laser_origin)
    if isinstance(meas, bb.PointCloud):
        return twin.update_point_cloud(pose, meas.data, meas.point_step, meas.x_offset, meas.dtype, meas.origin, meas.n_points)
    return twin.update(pose, meas)


def measurement(bb, scene, t, m):
    pts = scene.scans[t]
    if m % 3 == 1:  # a scan: the ranges of the scene's points at their bearings
        r = np.hypot(pts[:, 0], pts[:, 1]).astype(np.float32)
        return bb.LaserScan(r, np.float32(-np.pi / 2), np.float32(np.pi / (len(r) - 1)), 0.1, 30.0, 0)
    if m % 3 == 2:  # a float32 cloud of the points at z = 0.5
        xyz = np.concatenate([pts, np.full((len(pts), 1), 0.5)], axis=1).astype(np.float32)
        return bb.PointCloud(xyz.tobytes(), 12, 0, np.float32, None, len(xyz))
    return pts


class Pair:
    """A batch stepped with update_clustered and its mirror stepped with update_measurements + cluster_estimates."""

    def __init__(self, bb, motions, params, adaptive=False, selective=False):
        self.bb = bb
        self.a = bb.AmclBatch(motions, params, adaptive=adaptive, selective=selective)
        self.b = bb.AmclBatch(motions, params, adaptive=adaptive, selective=selective)
        self.fallbacks = 0
        self.extra = []  # launches of each update_clustered call beyond its mirror's update_measurements

    def both(self, name, *args, **kwargs):
        getattr(self.a, name)(*args, **kwargs)
        getattr(self.b, name)(*args, **kwargs)

    def step(self, poses, meas, present=None, cluster=None, where=None):
        cluster = cluster or {}
        before = self.a.launch_count()
        got, ests = self.a.update_clustered(poses, meas, present, with_counts=True, **cluster)
        n_a = self.a.launch_count() - before
        before = self.b.launch_count()
        exp = self.b.update_measurements(poses, meas, present)
        n_b = self.b.launch_count() - before
        updated = [bool(r.updated) for r in exp]
        want = self.b.cluster_estimates(present=updated, with_counts=True, **cluster) if any(updated) else [None] * len(exp)
        for m in range(len(exp)):
            assert result_bytes(got[m]) == result_bytes(exp[m]), (where, m)
            assert estimate_bytes(ests[m]) == estimate_bytes(want[m]), (where, m)
            ga, wa = self.a.particles(m)
            gb, wb = self.b.particles(m)
            assert ga.tobytes() == gb.tobytes() and wa.tobytes() == wb.tobytes(), (where, m)
            if exp[m].updated and exp[m].resampled and self.a.params[m].record_ancestors:
                assert self.a.ancestors(m).tobytes() == self.b.ancestors(m).tobytes(), (where, m)
        if any(updated):
            assert n_a in (n_b + 3, n_b + 4), (where, n_a, n_b)
            self.fallbacks += n_a - n_b - 3
            self.extra.append(n_a - n_b)
        else:
            assert n_a == n_b == 0
        return got, ests


def assert_twin(bb, twin, r, est, where):
    exp = r[1]
    assert result_bytes(r[0]) == result_bytes(exp), where
    if exp.updated:
        tm, tc, _, cells, clusters = twin.filter.cluster_estimate(with_ids=True)
        assert estimate_bytes(est) == estimate_bytes((tm, tc, cells, clusters)), where


class Maps:
    def __init__(self, bb, scene, kind):
        cells, self.sensor = scene.cells, bb.SENSOR_LIKELIHOOD_FIELD
        self.params = bb.LikelihoodFieldModelParam(**LFM)
        if kind == "prob":
            self.sensor = bb.SENSOR_LIKELIHOOD_FIELD_PROB
        elif kind in ("beam", "beam_fused"):
            self.sensor = bb.SENSOR_BEAM
            self.params = bb.BeamModelParam(sigma_hit=0.2, lambda_short=0.1, beam_max_range=20.0)
            if kind == "beam_fused":  # wider than 65534 cells: the fused kernel
                cells = np.pad(cells, ((0, 0), (0, 70_000 - cells.shape[1])), constant_values=0)
        self.grid = bb.OccupancyGrid(cells, scene.resolution)

    def set(self, bb, batches, twins):
        for batch in batches:
            if self.sensor == bb.SENSOR_BEAM:
                batch.set_beam_map(self.params, self.grid)
            else:
                batch.set_likelihood_field_map(self.params, self.grid, prob=self.sensor == bb.SENSOR_LIKELIHOOD_FIELD_PROB)
        for t in twins:
            t.update_map(self.sensor, self.params, self.grid)


@pytest.mark.parametrize("kind", ["lfm", "prob", "beam", "beam_fused"])
def test_update_clustered_equals_update_then_cluster_estimates(bb, scene, kind):
    maps = Maps(bb, scene, kind)
    k = len(MEMBERS)
    params = [member_params(bb, m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    pair = Pair(bb, motions, params, adaptive=True, selective=True)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    maps.set(bb, [pair.a, pair.b], twins)
    for m in range(k):
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        pair.both("initialize", m, mean, scene.initial_cov)
        twins[m].initialize(mean, scene.initial_cov)
    resampled, kept, gated = set(), set(), 0
    for t in range(12):
        present = [(t + m) % 5 != 4 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        meas = [measurement(bb, scene, t, m) for m in range(k)]
        for m in range(2, k, 3):  # the stationary members would not update otherwise
            if t % 2 == 0:
                pair.both("force_update", m)
                twins[m].force_update()
        got, ests = pair.step(poses, meas, present, where=(kind, t))
        for m in range(k):
            if not present[m]:
                assert got[m].updated == 0 and ests[m] is None
                continue
            exp = feed_twin(bb, twins[m], poses[m], meas[m])
            assert_twin(bb, twins[m], (got[m], exp), ests[m], (kind, t, m))
            gated += 1 - exp.updated
            if exp.updated:
                (resampled if exp.resampled else kept).add(m)
    assert gated > 0 and pair.fallbacks == 0
    assert {0, 2} <= resampled and 7 in kept


def test_several_maps(bb, scene):
    k = 6
    params = [member_params(bb, m) for m in range(k)]
    motions = [motion(bb, 0) for _ in range(k)]
    pair = Pair(bb, motions, params, adaptive=True, selective=True)
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    beam = bb.BeamModelParam(sigma_hit=0.2, lambda_short=0.1, beam_max_range=20.0)
    for batch in (pair.a, pair.b):
        ids = [batch.add_likelihood_field_map(lfm, grid), batch.add_likelihood_field_map(lfm, grid, prob=True), batch.add_beam_map(beam, grid)]
        for m in range(k):
            batch.update_map(m, ids[m % 3])
    for m in range(k):
        pair.both("initialize", m, scene.initial_mean + np.array([0.02 * m, 0.0, 0.0]), scene.initial_cov)
    for t in range(8):
        if t == 4:
            for batch in (pair.a, pair.b):
                batch.update_map(0, batch.member_map(2))
        pair.step([odometry(scene, t, m) for m in range(k)], [measurement(bb, scene, t, m) for m in range(k)], where=t)
    assert pair.fallbacks == 0


def test_nan_weights_take_the_fallback(bb, scene):
    """A member whose weights are NaN keeps them through a normalising step: its cells' weights are NaN, the device cannot
    promise nth_element's pick, and the host pass runs for it (one launch more) with the same bytes as the mirror."""
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=n, resample_interval=4) for n in (1500, 1200)]
    pair = Pair(bb, [bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 2, params)
    for batch in (pair.a, pair.b):
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    rng = np.random.default_rng(1)
    th = rng.normal(scene.initial_mean[2], 0.2, 1500)
    st = np.stack([np.cos(th), np.sin(th), rng.normal(scene.initial_mean[0], 0.3, 1500), rng.normal(scene.initial_mean[1], 0.3, 1500)], axis=1)
    w = np.ones(1500)
    w[::7] = np.nan
    pair.both("initialize_states", 0, st, w)
    pair.both("initialize", 1, scene.initial_mean, scene.initial_cov)
    for t in range(3):
        pair.step([bb.se2(*scene.poses[t])] * 2, [scene.scans[t]] * 2, where=t)
    assert pair.fallbacks >= 1


def test_heading_on_a_bucket_edge_takes_the_fallback(bb, scene):
    """Every particle of member 0 heads exactly 0.5 rad and a noise-free motion keeps it there: with an angular resolution of
    0.25 the neighbours' headings lie on a bucket edge, where the device's atan2 may differ from glibc's, so the member takes
    the host pass; member 1 does not."""
    params = [bb.AmclParams(min_particles=400, max_particles=400, seed=s, resample_interval=2) for s in (3, 4)]
    pair = Pair(bb, [bb.DifferentialDriveModelParam(0.0, 0.0, 0.0, 0.0), bb.DifferentialDriveModelParam(*ALPHAS[:4])], params)
    for batch in (pair.a, pair.b):
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    rng = np.random.default_rng(2)
    st = np.stack([np.full(400, np.cos(0.5)), np.full(400, np.sin(0.5)), rng.uniform(2.0, 6.0, 400), rng.uniform(2.0, 6.0, 400)], axis=1)
    pair.both("initialize_states", 0, st)
    pair.both("initialize", 1, scene.initial_mean, scene.initial_cov)
    pose = bb.se2(*scene.poses[0])
    for t in range(3):
        pair.both("force_update", 0)
        pair.both("force_update", 1)
        pair.step([pose, pose], [scene.scans[0]] * 2, cluster=dict(angular=0.25), where=t)
    assert pair.fallbacks == 3


def test_refused_parameter_block_changes_nothing(bb, scene):
    from beluga_b200 import _capi

    params = [bb.AmclParams(min_particles=800, max_particles=800, seed=m) for m in range(3)]
    pair = Pair(bb, [bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 3, params)
    for batch in (pair.a, pair.b):
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    for m in range(3):
        pair.both("initialize", m, scene.initial_mean, scene.initial_cov)
    pair.step([bb.se2(*scene.poses[0])] * 3, [scene.scans[0]] * 3, where=0)
    a = pair.a
    before = a.launch_count()
    snapshot = [a.particles(m)[0].tobytes() for m in range(3)]
    for bad in (dict(linear=0.0), dict(angular=-1.0), dict(percentile=1.0), dict(percentile=-0.1), dict(linear=float("nan"))):
        with pytest.raises(bb.BelugaB200Error) as e:
            a.update_clustered([bb.se2(*scene.poses[1])] * 3, [scene.scans[1]] * 3, **bad)
        assert e.value.status == _capi.ERR_INVALID_ARGUMENT and "cluster parameters" in str(e.value)
    assert a.launch_count() == before
    assert [a.particles(m)[0].tobytes() for m in range(3)] == snapshot
    for t in (1, 2):  # the policies did not move: the next steps still match the mirror's
        pair.step([bb.se2(*scene.poses[t])] * 3, [scene.scans[t]] * 3, where=t)


def test_launch_counts(bb, scene):
    """The update's own launches plus 3, whatever K is."""
    for k in (1, 16, 256):
        params = [bb.AmclParams(min_particles=2000, max_particles=2000, seed=m) for m in range(k)]
        pair = Pair(bb, [bb.DifferentialDriveModelParam(*ALPHAS[:4])] * k, params)
        for batch in (pair.a, pair.b):
            batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
        for m in range(k):
            pair.both("initialize", m, scene.initial_mean + np.array([0.01 * (m % 7), 0.0, 0.0]), scene.initial_cov)
        for t in range(2):
            pair.step([bb.se2(*scene.poses[t])] * k, [scene.scans[t]] * k, where=(k, t))
        assert pair.extra == [3, 3], k


def test_two_members_against_the_oracle(bb, orc, scene):
    """The clustered estimates of two members match the oracle's clusterizer over the batch's particles."""
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=n, resample_scheme=s) for n, s in ((3000, 0), (2000, 1))]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 2, params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    for m in range(2):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(6):
        got, ests = batch.update_clustered([bb.se2(*scene.poses[t])] * 2, [scene.scans[t]] * 2)
        for m in range(2):
            if not got[m].updated:
                continue
            s, w = batch.particles(m)
            want_mean, want_cov = orc.cluster_based_estimate(s, w, 0.20, 0.524, 0.90)
            mean, cov = ests[m]
            assert np.allclose(mean, want_mean, rtol=0, atol=1e-9), (t, m)
            finite = np.isfinite(want_cov)
            assert np.array_equal(np.isfinite(cov), finite), (t, m)
            assert np.allclose(cov[finite], want_cov[finite], rtol=1e-9, atol=1e-9), (t, m)
