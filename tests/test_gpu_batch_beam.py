"""The batch of filters with the beam model on the GPU: every member equals a standalone Amcl on the same beam map fed the
same inputs, byte for byte (update results, particles, weights, ancestors and the final cluster estimate), across particle
counts from 1 to 32 768, the three motion models, both resampling schemes, recovery injection, normalising steps, absent
members, steps below update_min_d and scans of 0 to 2049 points (ragged walk chunks of 1024 and mixture chunks of 2048).
The map shapes cover both forms of the step: the two-pass walk (with and without the normaliser table) and the fused
kernel (a grid wider than 65534 cells, a reach of 2^21 cells or more), and a step whose hit words exceed the one-pass
bound of 3 GiB takes the fused kernel while its standalone twins still walk in two passes.  Also: the oracle along a
trajectory, the launch count, map switches, initialize_from_map, rollback and tracking."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
SIZES = (1, 33, 256, 2000, 5000, 32768, 2000, 33)
POINT_COUNTS = (0, 1, 60, 1025, 2049)


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


class Shape:
    """A beam map and the scene scaled to its resolution (scan, poses, sigma_hit, 1 / lambda_short, update_min_d), so that
    rays hit at the usual ranges in cells while beam_max_range stays in metres -- the shapes of the single filter's
    fallback tests."""

    def __init__(self, bb, scene, name):
        cells, res, max_range = scene.cells, scene.resolution, 20.0
        if name == "wide_grid":  # wider than 65534 cells: no padded free-distance copy, fused kernel with the table
            cells = np.pad(cells, ((0, 0), (0, 70_000 - cells.shape[1])), constant_values=0)
        elif name == "long_reach":  # 2^21 cells of reach or more: fused kernel, per-beam normalisers
            res, max_range = 1e-5, 30.0
        elif name == "fine_cells":  # range / resolution too large for the table: two-pass walk, per-beam normalisers
            res, max_range = 0.01, 30.0
        self.scale = res / scene.resolution
        self.grid = bb.OccupancyGrid(cells, res)
        self.beam = bb.BeamModelParam(sigma_hit=0.2 * self.scale, lambda_short=0.1 / self.scale, beam_max_range=max_range)
        self.scene = scene

    def scan(self, t, count):
        return np.resize(self.scene.scans[t], (count, 2)) * self.scale if count else np.zeros((0, 2))

    def mean(self, m):
        return self.scene.initial_mean * np.array([self.scale, self.scale, 1.0]) + np.array([0.02 * m * self.scale, 0.0, 0.01 * m])

    def cov(self):
        return self.scene.initial_cov * np.outer([self.scale, self.scale, 1.0], [self.scale, self.scale, 1.0])

    def odometry(self, t, m):
        """Member m's control: the scene's pose, a little shifted per member; every fifth step repeats the last pose (below
        update_min_d: only a forced update runs)."""
        x, y, th = self.scene.poses[t - 1 if t % 5 == 4 else t]
        th = th + 0.01 * m
        return np.array([np.cos(th), np.sin(th), (x + 0.02 * m) * self.scale, y * self.scale])


def motion(bb, k):
    return [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.OmnidirectionalDriveModelParam(*ALPHAS), bb.StationaryModelParam()][k % 3]


def member_params(bb, k, scale=1.0):
    n = SIZES[k]
    p = bb.AmclParams(min_particles=n, max_particles=n, seed=200 + k, resample_scheme=k % 2, record_ancestors=True,
                      update_min_d=0.25 * scale)
    if k == 3:
        p.recovery_probability_override = 0.05
    if k in (4, 7):
        p.resample_interval = 3  # normalising and resampling steps alternate
    return p


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


def assert_member_equals_twin(batch, m, twin, got, exp, where):
    assert result_bytes(got) == result_bytes(exp), where
    if exp.updated:
        gs, gw = batch.particles(m)
        ts, tw = twin.particles()
        n = len(ts)
        assert gs[:n].tobytes() == ts.tobytes() and gw[:n].tobytes() == tw.tobytes(), where
        if exp.resampled:
            assert np.array_equal(batch.ancestors(m), twin.filter.ancestors()), where


def assert_cluster_estimates_equal(batch, twins):
    for m, twin in enumerate(twins):
        gm, gc = batch.cluster_estimate(m)
        tm, tc = twin.filter.cluster_estimate()
        assert gm.tobytes() == tm.tobytes() and gc.tobytes() == tc.tobytes(), m


@pytest.mark.parametrize("shape, launches", [("normal", 6), ("wide_grid", 5), ("long_reach", 5), ("fine_cells", 6)])
def test_members_equal_standalone_twins(bb, scene, shape, launches):
    sh = Shape(bb, scene, shape)
    k = len(SIZES)
    params = [member_params(bb, m, sh.scale) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    batch.set_beam_map(sh.beam, sh.grid)
    twins = []
    for m in range(k):
        a = bb.Amcl(motions[m], params[m])
        a.update_map(bb.SENSOR_BEAM, sh.beam, sh.grid)
        twins.append(a)
    for m in range(k):
        if m == 7:  # explicit states, fewer than max_particles
            rng = np.random.default_rng(m)
            mean = sh.mean(m)
            th = rng.normal(mean[2], 0.2, 20)
            st = np.stack([np.cos(th), np.sin(th), rng.normal(mean[0], 0.3 * sh.scale, 20), rng.normal(mean[1], 0.3 * sh.scale, 20)], axis=1)
            batch.initialize_states(m, st)
            twins[m].initialize_states(st)
        else:
            batch.initialize(m, sh.mean(m), sh.cov())
            twins[m].initialize(sh.mean(m), sh.cov())
    resampled = normalised = skipped = 0
    for t in range(12):
        present = [(t + m) % 4 != 3 for m in range(k)]
        poses = [sh.odometry(t, m) for m in range(k)]
        pts = [sh.scan(t, POINT_COUNTS[(t + m) % len(POINT_COUNTS)]) for m in range(k)]
        before = batch.launch_count()
        got = batch.update(poses, pts, present)
        if any(r.updated for r in got):
            assert batch.launch_count() - before == launches, t
        for m in range(k):
            if not present[m]:
                assert got[m].updated == 0
                continue
            exp = twins[m].update(poses[m], pts[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            if exp.updated:
                resampled += exp.resampled
                normalised += 1 - exp.resampled
            else:
                skipped += 1
    assert resampled > 0 and normalised > 0 and skipped > 0
    assert_cluster_estimates_equal(batch, twins)


def test_over_the_one_pass_bound_the_batch_takes_the_fused_kernel(bb, scene):
    """4 x 32 768 particles x 6400 points: 3.36 GB of hit words, over the 3 GiB of one pass, so the batch runs the fused
    kernel (5 launches); each standalone twin needs 0.84 GB and walks in two passes.  The results agree byte for byte."""
    n, k, count = 32768, 4, 6400
    sh = Shape(bb, scene, "normal")
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=50 + m, resample_scheme=m % 2, record_ancestors=True) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    batch.set_beam_map(sh.beam, sh.grid)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    for m in range(k):
        twins[m].update_map(bb.SENSOR_BEAM, sh.beam, sh.grid)
        batch.initialize(m, sh.mean(m), sh.cov())
        twins[m].initialize(sh.mean(m), sh.cov())
    for t in range(3):
        poses = [sh.odometry(t, m) for m in range(k)]
        pts = [sh.scan(t + m, count) for m in range(k)]
        for m in range(k):  # every member updates
            batch.force_update(m)
            twins[m].force_update()
        before = batch.launch_count()
        got = batch.update(poses, pts)
        assert batch.launch_count() - before == 5
        for m in range(k):
            exp = twins[m].update(poses[m], pts[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
    assert_cluster_estimates_equal(batch, twins)


def test_oracle_anchor(bb, orc, scene):
    """Two members against oracle::Amcl with the beam model along the synthetic trajectory, with the single filter's
    tolerance: erf/exp differ by ulps between CUDA and glibc, so a handful of CDF boundary flips are allowed."""
    n, steps = 2000, 6
    ap = [dict(update_min_d=0.25, update_min_a=0.2, resample_interval=1, min_particles=n, max_particles=n, seed=77 + m) for m in range(2)]
    schemes = (1, 0)
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 2,
                         [bb.AmclParams(resample_scheme=schemes[m], record_ancestors=True, **ap[m]) for m in range(2)])
    batch.set_beam_map(bb.BeamModelParam(beam_max_range=20.0), bb.OccupancyGrid(scene.cells, scene.resolution))
    oracles = [orc.Amcl(orc.AmclParam(rng_mode=1, scheme=schemes[m], **ap[m]), orc.MotionParam(*ALPHAS[:4])) for m in range(2)]
    for m, o in enumerate(oracles):
        o.set_map(orc.BEAM, orc.BeamParam(beam_max_range=20.0), orc.Grid(scene.cells, scene.resolution))
        o.initialize_normal(scene.initial_mean, scene.initial_cov)
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    mismatched = [0, 0]
    for t in range(steps):
        pose = orc.se2(*scene.poses[t])
        pts = scene.scans[t][::6]
        got = batch.update([pose, pose], [pts, pts])
        for m, o in enumerate(oracles):
            ro = o.update(pose, pts)
            assert got[m].updated == ro.updated == 1 and got[m].resampled == ro.resampled
            mismatched[m] += int((batch.ancestors(m) != o.last_indices()).sum())
            gm, gc = np.array(got[m].estimate.mean), np.array(got[m].estimate.cov)
            assert np.abs(gm - np.array(ro.mean)).max() < 1e-5 and np.abs(gc - np.array(ro.cov)).max() < 1e-5
            if mismatched[m] == 0:
                assert np.abs(gm - np.array(ro.mean)).max() < 1e-10 and np.abs(gc - np.array(ro.cov)).max() < 1e-10
    assert max(mismatched) <= 5
    for m in range(2):
        gm = got[m].estimate.mean
        assert np.hypot(gm[2] - scene.poses[steps - 1][0], gm[3] - scene.poses[steps - 1][1]) < 0.3


@pytest.mark.parametrize("shape, launches", [("normal", 6), ("wide_grid", 5)])
def test_launch_count_does_not_depend_on_the_member_count(bb, scene, shape, launches):
    sh = Shape(bb, scene, shape)
    counts = []
    for k in (1, 16, 256):
        params = [bb.AmclParams(min_particles=500, max_particles=500, seed=m, resample_scheme=1) for m in range(k)]
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam() for _ in range(k)], params)
        batch.set_beam_map(sh.beam, sh.grid)
        for m in range(k):
            batch.initialize(m, sh.mean(0), sh.cov())
        before = batch.launch_count()
        res = batch.update([sh.odometry(0, 0)] * k, [sh.scan(0, 60 + m % 7) for m in range(k)])
        assert all(r.updated for r in res)
        counts.append(batch.launch_count() - before)
    assert counts == [launches] * 3


def test_map_switches(bb, scene):
    """Likelihood field -> beam -> likelihood field on one batch: every step equals twins that switch the same way."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    k = 3
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=30 + n, resample_scheme=n % 2, record_ancestors=True) for n in (700, 2000, 33)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    maps = [(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM)), (bb.SENSOR_BEAM, bb.BeamModelParam(beam_max_range=20.0)),
            (bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM))]
    t = 0
    for phase, (sensor, p) in enumerate(maps):
        if sensor == bb.SENSOR_BEAM:
            batch.set_beam_map(p, grid)
        else:
            batch.set_likelihood_field_map(p, grid)
        for m in range(k):
            twins[m].update_map(sensor, p, grid)
            if phase == 0:
                batch.initialize(m, scene.initial_mean, scene.initial_cov)
                twins[m].initialize(scene.initial_mean, scene.initial_cov)
        for _ in range(3):
            pose = bb.se2(*scene.poses[t])
            for m in range(k):
                batch.force_update(m)
                twins[m].force_update()
            got = batch.update([pose] * k, [scene.scans[t]] * k)
            for m in range(k):
                exp = twins[m].update(pose, scene.scans[t])
                assert exp.updated
                assert_member_equals_twin(batch, m, twins[m], got[m], exp, (phase, t, m))
            t += 1


def test_initialize_from_map_on_a_beam_map(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    beam = bb.BeamModelParam(beam_max_range=20.0)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=n, resample_scheme=1, record_ancestors=True) for n in (1000, 3000)]
    motions = [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.StationaryModelParam()]
    batch = bb.AmclBatch(motions, params)
    batch.set_beam_map(beam, grid)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(2)]
    for m in range(2):
        twins[m].update_map(bb.SENSOR_BEAM, beam, grid)
        batch.initialize_from_map(m)
        twins[m].initialize_from_map()
        assert batch.particles(m)[0].tobytes() == twins[m].particles()[0].tobytes()
    for t in range(3):
        pose = bb.se2(*scene.poses[t])
        got = batch.update([pose, pose], [scene.scans[t]] * 2)
        for m in range(2):
            exp = twins[m].update(pose, scene.scans[t])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))


def test_failed_update_is_rolled_back(bb, scene):
    """An update before any map is set fails; after setting the beam map, a retry gives what a batch that never failed gives."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    beam = bb.BeamModelParam(beam_max_range=20.0)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=3 + n, resample_interval=2) for n in (300, 700)]

    def make(with_map):
        b = bb.AmclBatch([bb.DifferentialDriveModelParam(), bb.StationaryModelParam()], params)
        if with_map:
            b.set_beam_map(beam, grid)
        for m in range(2):
            b.initialize(m, scene.initial_mean, scene.initial_cov)
        return b

    failed, clean = make(False), make(True)
    poses = [bb.se2(*scene.poses[0])] * 2
    with pytest.raises(bb.BelugaB200Error) as e:
        failed.update(poses, [scene.scans[0]] * 2)
    assert e.value.status == -4  # BB200_ERR_STATE
    assert "no map set" in str(e.value)
    failed.set_beam_map(beam, grid)
    for t in range(4):
        poses = [bb.se2(*scene.poses[t])] * 2
        a, b = failed.update(poses, [scene.scans[t]] * 2), clean.update(poses, [scene.scans[t]] * 2)
        assert [result_bytes(r) for r in a] == [result_bytes(r) for r in b]
        for m in range(2):
            assert failed.particles(m)[0].tobytes() == clean.particles(m)[0].tobytes()


def test_every_member_tracks(bb):
    """16 members, each on its own synthetic scene (the scene's noise seed), follow their ground truth with the beam model."""
    from beluga_b200 import synthetic

    k = 16
    scenes = [synthetic.make_scenario(grid_size=300, n_beams=100, steps=30, noise_seed=11 + m) for m in range(k)]
    params = [bb.AmclParams(min_particles=2000, max_particles=2000, seed=m, resample_scheme=1) for m in range(k)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05) for _ in range(k)], params)
    batch.set_beam_map(bb.BeamModelParam(beam_max_range=20.0), bb.OccupancyGrid(scenes[0].cells, scenes[0].resolution))
    for m in range(k):
        batch.initialize(m, scenes[m].initial_mean, scenes[m].initial_cov)
    errors = np.zeros(k)
    for t in range(len(scenes[0].poses)):
        res = batch.update([bb.se2(*s.poses[t]) for s in scenes], [s.scans[t] for s in scenes])
        for m in range(k):
            if res[m].updated:
                errors[m] = np.hypot(res[m].estimate.mean[2] - scenes[m].poses[t][0], res[m].estimate.mean[3] - scenes[m].poses[t][1])
    assert errors.max() < 0.3, errors
