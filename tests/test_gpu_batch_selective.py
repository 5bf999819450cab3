"""Selective-resampling batch members on the GPU (BB200_BATCH_SELECTIVE): every member equals a standalone Amcl built from
the same parameters and fed the same inputs, byte for byte -- update results (resampled, n_particles,
random_state_probability, weight_sum, estimate, weights_degenerate), particles, weights and ancestors after every step,
and cluster estimates, particle histograms and pose samples after kept and after resampled steps.  Every selective
member both resamples and keeps its particles on some step, so both branches of the device's decision run.  Covered:
the scatter and per-slot draws, multinomial, recovery injection, resample_interval = 3, non-selective members next to
selective ones, all motion models, absent members, both likelihood-field models, the beam model in both forms, several
maps with update_map, scans and clouds, selective KLD members, degenerate weights, re-initialisation, launch counts,
a selective batch without selective members against a plain batch, rollback, and two members against the oracle."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
# (min_particles, max_particles, scheme, selective, extra parameters) per member
MEMBERS = [
    (2000, 2000, 1, True, {}),                                          # systematic comb: the scatter draw
    (2000, 2000, 0, True, {}),                                          # multinomial
    (1500, 1500, 1, True, dict(recovery_probability_override=0.05)),    # recovery injection: the per-slot draw
    (1000, 1000, 0, True, dict(resample_interval=3)),                   # the test on every third update only (2-point scans)
    (2000, 2000, 1, False, {}),                                         # an ordinary member next to them
    (777, 777, 0, False, dict(resample_interval=2)),                    # an ordinary member that normalises
    (3000, 3000, 1, True, {}),                                          # starts from 20 explicit states
]
KLD_MEMBERS = [
    (100, 20000, 0, True, {}),
    (1, 32768, 1, True, {}),
    (1000, 1000, 1, True, {}),
    (500, 2000, 1, False, {}),
    (50, 8000, 0, True, dict(spatial_resolution=(0.5, 0.5, 0.5))),
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


def member_params(bb, table, k, seed=300):
    lo, hi, scheme, selective, extra = table[k % len(table)]
    return bb.AmclParams(min_particles=lo, max_particles=hi, seed=seed + k, resample_scheme=scheme, selective_resampling=selective,
                         record_ancestors=True, **extra)


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


def odometry(scene, t, k):
    x, y, th = scene.poses[t - 1 if t % 5 == 4 else t]
    th = th + 0.01 * k
    return np.array([np.cos(th), np.sin(th), x + 0.02 * k, y])


def launches(batch, call):
    before = batch.launch_count()
    out = call()
    return batch.launch_count() - before, out


def initialize(batch, twins, scene, explicit=(6,)):
    for m, twin in enumerate(twins):
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        if m in explicit:
            rng = np.random.default_rng(m)
            th = rng.normal(mean[2], 0.2, 20)
            st = np.stack([np.cos(th), np.sin(th), rng.normal(mean[0], 0.3, 20), rng.normal(mean[1], 0.3, 20)], axis=1)
            batch.initialize_states(m, st)
            twin.initialize_states(st)
        else:
            batch.initialize(m, mean, scene.initial_cov)
            twin.initialize(mean, scene.initial_cov)


def feed_twin(bb, twin, pose, meas):
    if isinstance(meas, bb.LaserScan):
        return twin.update_scan(pose, meas.ranges, meas.angle_min, meas.angle_increment, meas.min_range, meas.max_range, meas.max_beams,
                                meas.laser_origin)
    if isinstance(meas, bb.PointCloud):
        return twin.update_point_cloud(pose, meas.data, meas.point_step, meas.x_offset, meas.dtype, meas.origin, meas.n_points)
    return twin.update(pose, meas)


def assert_member_equals_twin(batch, m, twin, got, exp, where):
    assert result_bytes(got) == result_bytes(exp), where
    gs, gw = batch.particles(m)  # max_particles rows in a batch that is not adaptive
    ts, tw = twin.particles()
    n = batch.member_size(m)
    assert n == len(ts) and len(gs) == (n if batch.adaptive else batch.params[m].max_particles), where
    assert gs[:n].tobytes() == ts.tobytes() and gw[:n].tobytes() == tw.tobytes(), where
    if exp.updated and exp.resampled:
        assert batch.ancestors(m).tobytes() == twin.filter.ancestors().tobytes(), where


def twin_histogram(bb, twin, linear, angular):
    import ctypes as C

    from beluga_b200 import _capi

    f = twin.filter
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, None, 0, C.byref(n), C.byref(top)) == 0
    bins = np.empty(max(n.value, 1), dtype=bb._CELL_DTYPE)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, bins.ctypes.data_as(C.POINTER(_capi.ClusterCell)), n.value,
                                                  C.byref(n), C.byref(top)) == 0
    return bins[:n.value], top.value


def assert_published_equal(bb, batch, twins, step):
    """Cluster estimates, particle histograms and pose samples of every member against its twin; returns the launches of
    the pose samples."""
    est = batch.cluster_estimates()
    hists = batch.particle_histograms(None, 0.05, 0.05)
    counts = [min(700, q.max_particles) for q in batch.params]
    n, samples = launches(batch, lambda: batch.sample_states(counts, step))
    for m, twin in enumerate(twins):
        tm, tc = twin.filter.cluster_estimate()
        assert est[m][0].tobytes() == tm.tobytes() and est[m][1].tobytes() == tc.tobytes(), m
        bins, top = hists[m]
        t_bins, t_top = twin_histogram(bb, twin, 0.05, 0.05)
        assert bins.tobytes() == t_bins.tobytes() and np.float64(top).tobytes() == np.float64(t_top).tobytes(), m
        assert samples[m].tobytes() == twin.filter.sample_states(counts[m], step).tobytes(), m
    return n


class Outcomes:
    """Per selective member, the decisions of the steps on which its resample_interval fired."""

    def __init__(self, params):
        self.params = params
        self.updates = [0] * len(params)
        self.kept = [0] * len(params)
        self.resampled = [0] * len(params)

    def record(self, m, r):
        if not r.updated:
            return
        self.updates[m] += 1
        p = self.params[m]
        if p.selective_resampling and self.updates[m] % p.resample_interval == 0:
            self.kept[m] += r.resampled == 0
            self.resampled[m] += r.resampled == 1
        elif p.resample_interval > 1 and self.updates[m] % p.resample_interval != 0:
            assert r.resampled == 0

    def assert_both(self, members=None):
        for m, p in enumerate(self.params):
            if p.selective_resampling and (members is None or m in members):
                assert self.kept[m] > 0 and self.resampled[m] > 0, (m, self.kept[m], self.resampled[m])


class Maps:
    """The map kinds of the trajectory test, each (sensor, params, grid) and the beam form it takes."""

    def __init__(self, bb, scene, kind):
        cells, self.sensor = scene.cells, bb.SENSOR_LIKELIHOOD_FIELD
        self.params = bb.LikelihoodFieldModelParam(**LFM)
        if kind == "prob":
            self.sensor = bb.SENSOR_LIKELIHOOD_FIELD_PROB
        elif kind in ("beam", "beam_fused"):
            self.sensor = bb.SENSOR_BEAM
            self.params = bb.BeamModelParam(sigma_hit=0.2, lambda_short=0.1, beam_max_range=20.0)
            if kind == "beam_fused":  # wider than 65534 cells: no padded free-distance copy, the fused kernel
                cells = np.pad(cells, ((0, 0), (0, 70_000 - cells.shape[1])), constant_values=0)
        self.grid = bb.OccupancyGrid(cells, scene.resolution)
        self.base = {"lfm": 5, "prob": 5, "beam": 6, "beam_fused": 5}[kind]

    def set(self, bb, batch, twins):
        if self.sensor == bb.SENSOR_BEAM:
            batch.set_beam_map(self.params, self.grid)
        else:
            batch.set_likelihood_field_map(self.params, self.grid, prob=self.sensor == bb.SENSOR_LIKELIHOOD_FIELD_PROB)
        for t in twins:
            t.update_map(self.sensor, self.params, self.grid)


@pytest.mark.parametrize("kind", ["lfm", "prob", "beam", "beam_fused"])
def test_members_equal_standalone_twins(bb, scene, kind):
    maps = Maps(bb, scene, kind)
    k = len(MEMBERS)
    params = [member_params(bb, MEMBERS, m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params, selective=True)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    maps.set(bb, batch, twins)
    initialize(batch, twins, scene)
    outcomes = Outcomes(params)
    skipped = 0
    for t in range(14):
        present = [(t + m) % 5 != 4 for m in range(k)]
        poses = [odometry(scene, t % 12, m) for m in range(k)]
        pts = [scene.scans[t % 12][: 2 if params[m].resample_interval == 3 else 150 + 5 * m] for m in range(k)]
        n, got = launches(batch, lambda: batch.update(poses, pts, present))
        ess = False
        for m in range(k):
            if not present[m]:
                assert got[m].updated == 0
                continue
            exp = twins[m].update(poses[m], pts[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            outcomes.record(m, exp)
            skipped += 1 - exp.updated
            ess |= bool(exp.updated) and params[m].selective_resampling and outcomes.updates[m] % params[m].resample_interval == 0
        if any(r.updated for r in got):
            assert n == maps.base + (2 if ess else 0), (t, n)
        if t in (5, 9, 13):
            assert_published_equal(bb, batch, twins, 0xFFFFFF00 + t)
    assert skipped > 0
    if kind == "lfm":
        outcomes.assert_both()
    # The prob model's weights, exp(sum log pz), are so peaked that its effective sample size always drops below n / 2;
    # with the beam model some members keep their particles on some steps.
    assert all(outcomes.resampled[m] > 0 for m in range(k) if params[m].selective_resampling)
    if kind != "prob":
        assert sum(outcomes.kept) > 0


def test_published_after_kept_and_resampled_steps(bb, scene):
    """cluster_estimates, particle_histograms and sample_states against the twin after a step that kept the particles (whose
    CDF is current: the pose samples take one launch) and after one that resampled (four: the CDF is rebuilt)."""
    params = [bb.AmclParams(min_particles=2000, max_particles=2000, seed=17, selective_resampling=True, record_ancestors=True)]
    motions = [bb.DifferentialDriveModelParam(*ALPHAS[:4])]
    batch = bb.AmclBatch(motions, params, selective=True)
    twins = [bb.Amcl(motions[0], params[0])]
    Maps(bb, scene, "lfm").set(bb, batch, twins)
    initialize(batch, twins, scene, explicit=())
    seen = set()
    for t in range(12):
        pose = odometry(scene, t, 0)
        got = batch.update([pose], [scene.scans[t]])
        exp = twins[0].update(pose, scene.scans[t])
        assert_member_equals_twin(batch, 0, twins[0], got[0], exp, t)
        if exp.updated:
            n = assert_published_equal(bb, batch, twins, 0xFFFFFE00 + t)
            assert n == (4 if exp.resampled else 1), (t, n)
            seen.add(exp.resampled)
    assert seen == {0, 1}


def test_several_maps_scans_and_clouds(bb, scene):
    """Two maps (likelihood field and beam), members moved between them mid-trajectory, and measurements given as points,
    scans and clouds through update_measurements; then re-initialisation of some members."""
    k = len(MEMBERS)
    params = [member_params(bb, MEMBERS, m, seed=500) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params, selective=True)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    lfm, beam = bb.LikelihoodFieldModelParam(**LFM), bb.BeamModelParam(sigma_hit=0.2, lambda_short=0.1, beam_max_range=20.0)
    ids = [batch.add_likelihood_field_map(lfm, grid), batch.add_beam_map(beam, grid)]
    on = [m % 2 for m in range(k)]

    def assign(m):
        batch.update_map(m, ids[on[m]])
        twins[m].update_map(bb.SENSOR_BEAM if on[m] else bb.SENSOR_LIKELIHOOD_FIELD, beam if on[m] else lfm, grid)

    for m in range(k):
        assign(m)
    initialize(batch, twins, scene)

    def measurement(t, m):
        pts = scene.scans[t]
        if m % 3 == 1:  # a scan: the ranges of the scene's points at their bearings, 181 beams over the half circle
            r = np.hypot(pts[:, 0], pts[:, 1]).astype(np.float32)
            return bb.LaserScan(r, np.float32(-np.pi / 2), np.float32(np.pi / (len(r) - 1)), 0.1, 30.0, 0)
        if m % 3 == 2:  # a float32 cloud of the points at z = 0.5
            xyz = np.concatenate([pts, np.full((len(pts), 1), 0.5)], axis=1).astype(np.float32)
            return bb.PointCloud(xyz.tobytes(), 12, 0, np.float32, None, len(xyz))
        return pts

    outcomes = Outcomes(params)
    for t in range(12):
        if t == 5:
            for m in range(0, k, 2):
                on[m] ^= 1
                assign(m)
        if t == 8:
            for m in (0, 1, 4):
                batch.initialize(m, scene.initial_mean, scene.initial_cov)
                twins[m].initialize(scene.initial_mean, scene.initial_cov)
        present = [(t + m) % 5 != 4 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        meas = [measurement(t, m) for m in range(k)]
        got = batch.update_measurements(poses, meas, present)
        for m in range(k):
            if present[m]:
                exp = feed_twin(bb, twins[m], poses[m], meas[m])
                assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
                outcomes.record(m, exp)
    assert_published_equal(bb, batch, twins, 0xFFFFFF40)
    assert sum(outcomes.kept) > 0 and sum(outcomes.resampled) > 0


def test_selective_kld_members(bb, scene):
    """Selective KLD members in an adaptive and selective batch: sizes, recovery probabilities (which a wrong
    commit_update would change) and everything else equal the twins'."""
    k = len(KLD_MEMBERS)
    params = [member_params(bb, KLD_MEMBERS, m, seed=900) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params, adaptive=True, selective=True)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    Maps(bb, scene, "lfm").set(bb, batch, twins)
    initialize(batch, twins, scene, explicit=(0, 4))  # 20 states: the counts grow, and the recovery probability rises
    outcomes = Outcomes(params)
    sizes, probabilities = set(), set()
    for t in range(14):
        present = [(t + m) % 6 != 5 for m in range(k)]
        poses = [odometry(scene, t % 12, m) for m in range(k)]
        pts = [scene.scans[t % 12][: 120 + 5 * m] for m in range(k)]
        n, got = launches(batch, lambda: batch.update(poses, pts, present))
        kld = ess = False
        for m in range(k):
            if not present[m]:
                continue
            exp = twins[m].update(poses[m], pts[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            outcomes.record(m, exp)
            if not exp.updated:
                continue
            fired = outcomes.updates[m] % params[m].resample_interval == 0
            kld |= fired and params[m].min_particles < params[m].max_particles
            ess |= fired and params[m].selective_resampling
            sizes.add(exp.n_particles)
            probabilities.add(exp.random_state_probability)
        if any(r.updated for r in got):
            assert n == 5 + (1 if ess else 0) + (1 if kld else 0) + (1 if kld or ess else 0), (t, n)
    outcomes.assert_both()
    assert len(sizes) > 4 and any(p > 0.0 for p in probabilities)
    assert_published_equal(bb, batch, twins, 0xFFFFFF80)


@pytest.mark.parametrize("kind", ["zero", "nan"])
def test_degenerate_weights(bb, scene, kind):
    """A selective member starting from a weight set with no positive finite weight: the effective sample size is 0, the
    member resamples from the uniform CDF and reports degenerate weights, as its twin does."""
    n = 3000
    rng = np.random.default_rng(12)
    th = rng.normal(scene.initial_mean[2], 0.1, n)
    states = np.stack([np.cos(th), np.sin(th), rng.normal(scene.initial_mean[0], 0.2, n), rng.normal(scene.initial_mean[1], 0.2, n)], 1)
    w = np.full(n, 0.0 if kind == "zero" else np.nan)
    if kind == "zero":
        w[::3] = -0.0
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=31 + m, resample_scheme=m % 2, resample_interval=1 + m, selective_resampling=True,
                            record_ancestors=True) for m in range(2)]
    motions = [bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 2
    batch = bb.AmclBatch(motions, params, selective=True)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(2)]
    Maps(bb, scene, "lfm").set(bb, batch, twins)
    for m in range(2):
        batch.initialize_states(m, states, w)
        twins[m].initialize_states(states, w)
    degenerate = 0
    for t in range(4):
        poses = [odometry(scene, t, m) for m in range(2)]
        got = batch.update(poses, [scene.scans[t]] * 2)
        for m in range(2):
            exp = twins[m].update(poses[m], scene.scans[t])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            degenerate += exp.weights_degenerate
    assert degenerate >= 2


@pytest.mark.parametrize("k", [1, 16, 256])
def test_launch_counts(bb, scene, k):
    """+2 launches when some updating member runs the effective-sample-size test, +3 when some also resamples under KLD, and
    one more with scans; whatever K and the decisions are."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    rows = []
    for lo, selective, interval, scan in ((2000, True, 1, False), (500, True, 1, False), (2000, False, 1, False), (2000, True, 2, False),
                                          (2000, True, 1, True)):
        params = [bb.AmclParams(min_particles=lo, max_particles=2000, seed=m, resample_scheme=m % 2, resample_interval=interval,
                                selective_resampling=selective) for m in range(k)]
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam() for _ in range(k)], params, adaptive=True, selective=True)
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(k):
            batch.initialize(m, scene.initial_mean, scene.initial_cov)
        row, decisions = [], set()
        for t in range(2):
            pts = scene.scans[t]
            if scan:
                r = np.hypot(pts[:, 0], pts[:, 1]).astype(np.float32)
                meas = bb.LaserScan(r, np.float32(-np.pi / 2), np.float32(np.pi / (len(r) - 1)), 0.1, 30.0, 0)
                n, res = launches(batch, lambda: batch.update_measurements([bb.se2(*scene.poses[t])] * k, [meas] * k))
            else:
                n, res = launches(batch, lambda: batch.update([bb.se2(*scene.poses[t])] * k, [pts] * k))
            assert all(r.updated for r in res)
            decisions |= {r.resampled for r in res}
            row.append(n)
        rows.append(row)
    # selective fixed members; selective KLD members; ordinary members; selective members testing on even updates; scans
    assert rows == [[7, 7], [8, 8], [5, 5], [5, 7], [8, 8]]


def test_selective_batch_of_ordinary_members_equals_plain_batch(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    sizes = (1, 33, 2000, 5000, 32768)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=40 + m, resample_scheme=m % 2, record_ancestors=True,
                            resample_interval=1 + m % 2, recovery_probability_override=0.05 if m == 2 else 0.0) for m, n in enumerate(sizes)]
    motions = [motion(bb, m) for m in range(len(sizes))]
    plain, selective = bb.AmclBatch(motions, params), bb.AmclBatch(motions, params, selective=True)
    for b in (plain, selective):
        b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(len(sizes)):
            b.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(8):
        poses = [odometry(scene, t, m) for m in range(len(sizes))]
        n_plain, r_plain = launches(plain, lambda: plain.update(poses, [scene.scans[t]] * len(sizes)))
        n_sel, r_sel = launches(selective, lambda: selective.update(poses, [scene.scans[t]] * len(sizes)))
        assert n_plain == n_sel and [result_bytes(r) for r in r_plain] == [result_bytes(r) for r in r_sel], t
        for m in range(len(sizes)):
            assert plain.particles(m)[0].tobytes() == selective.particles(m)[0].tobytes()
            assert plain.particles(m)[1].tobytes() == selective.particles(m)[1].tobytes()
            assert plain.ancestors(m).tobytes() == selective.ancestors(m).tobytes()


def test_failed_step_is_rolled_back(bb, scene):
    """After selective steps, a step fails (recovery injection on a map without free cells); the members are moved back and
    the batch continues exactly as one that never failed."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    full = bb.OccupancyGrid(np.full_like(scene.cells, 100), scene.resolution)
    params = [bb.AmclParams(min_particles=3000, max_particles=3000, seed=71, selective_resampling=True, record_ancestors=True),
              bb.AmclParams(min_particles=200, max_particles=2500, seed=72, recovery_probability_override=0.1, resample_scheme=1,
                            selective_resampling=True, record_ancestors=True)]
    motions = [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.StationaryModelParam()]

    def make():
        b = bb.AmclBatch(motions, params, adaptive=True, selective=True)
        ids = [b.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid),
               b.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), full)]
        for m in range(2):
            b.update_map(m, ids[0])
            b.initialize(m, scene.initial_mean, scene.initial_cov)
        return b, ids

    (failed, ids), (clean, _) = make(), make()
    for t in range(8):
        poses = [odometry(scene, t, m) for m in range(2)]
        if t == 3:
            sizes = [failed.member_size(m) for m in range(2)]
            failed.update_map(1, ids[1])
            with pytest.raises(bb.BelugaB200Error) as e:
                failed.update(poses, [scene.scans[t]] * 2)
            assert e.value.status == -4  # BB200_ERR_STATE
            assert [failed.member_size(m) for m in range(2)] == sizes
            failed.update_map(1, ids[0])
        a, b = failed.update(poses, [scene.scans[t]] * 2), clean.update(poses, [scene.scans[t]] * 2)
        assert [result_bytes(r) for r in a] == [result_bytes(r) for r in b], t
        for m in range(2):
            assert failed.particles(m)[0].tobytes() == clean.particles(m)[0].tobytes(), (t, m)
            assert failed.particles(m)[1].tobytes() == clean.particles(m)[1].tobytes(), (t, m)
            assert failed.ancestors(m).tobytes() == clean.ancestors(m).tobytes(), (t, m)


def test_oracle_selective_trajectory(bb, orc, scene):
    """Two selective members against oracle::Amcl in counter-RNG mode: equal resampled flags every step, states within
    1e-12 and estimates within 1e-9."""
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    cfg = [dict(scheme=0, seed=77, resample_interval=2, n=8000), dict(scheme=1, seed=78, resample_interval=1, n=5000)]
    params = [bb.AmclParams(min_particles=c["n"], max_particles=c["n"], resample_scheme=c["scheme"], seed=c["seed"], resample_interval=c["resample_interval"],
                            selective_resampling=True, update_min_d=0.25, update_min_a=0.2, record_ancestors=True) for c in cfg]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 2, params, selective=True)
    batch.set_likelihood_field_map(lfm, bb.OccupancyGrid(scene.cells, scene.resolution))
    oracles = [orc.Amcl(orc.AmclParam(rng_mode=1, scheme=c["scheme"], seed=c["seed"], resample_interval=c["resample_interval"], selective_resampling=True,
                                      update_min_d=0.25, update_min_a=0.2, min_particles=c["n"], max_particles=c["n"]), orc.MotionParam(*ALPHAS[:4]))
               for c in cfg]
    for m, o in enumerate(oracles):
        o.set_map(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
        o.initialize_normal(scene.initial_mean, scene.initial_cov)
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    flags = [set(), set()]
    for t in range(10):
        pose = orc.se2(*scene.poses[t])
        got = batch.update([pose, pose], [scene.scans[t], scene.scans[t]])
        for m, o in enumerate(oracles):
            ro = o.update(pose, scene.scans[t])
            assert got[m].updated == ro.updated == 1
            assert got[m].resampled == ro.resampled, (t, m)
            flags[m].add(ro.resampled)
            if ro.resampled:
                assert np.array_equal(batch.ancestors(m), o.last_indices()), (t, m)
            gs = batch.particles(m)[0]
            os_ = np.asarray(o.particles()[0])
            assert np.abs(gs - os_.reshape(gs.shape)).max() < 1e-12, (t, m)
            assert np.abs(np.array(got[m].estimate.mean) - np.array(ro.mean)).max() < 1e-9, (t, m)
    assert flags[1] == {0, 1}
