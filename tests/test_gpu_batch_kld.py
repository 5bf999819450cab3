"""KLD-adaptive batch members on the GPU (bb200_amcl_batch_create_adaptive): every member equals a standalone Amcl built
from the same parameters and fed the same inputs, byte for byte -- update results (n_particles, random_state_probability,
weight_sum, estimate), particles, weights and ancestors after every step, and cluster estimates, particle histograms and
pose samples after KLD steps -- with KLD members of (min, max) from (1, 32768) to (100, 101) next to fixed-size members,
normalising steps, both schemes, all three motion models, recovery injection, members that skip steps, both
likelihood-field models, the beam model in both forms, several maps with update_map, scans and clouds.  Also: launch
counts (+2 on steps where some member resamples under KLD, whatever K is), an adaptive batch of fixed-size members
against a fixed batch, rollback, re-initialisation, and two members against the oracle's take_while_kld."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
FINE = (0.1, 0.1, 0.1)  # spatial resolution with many more buckets than beluga_ros's default
# (min_particles, max_particles, scheme, extra parameters) per member
MEMBERS = [
    (500, 2000, 0, {}),
    (1, 32768, 1, {}),
    (100, 101, 0, {}),
    (2000, 2000, 1, {}),                                              # fixed size
    (300, 5000, 0, dict(resample_interval=3, spatial_resolution=FINE)),  # normalising steps between resampling ones
    (200, 3000, 1, dict(recovery_probability_override=0.05)),          # recovery injection on every resample
    (1000, 1000, 0, dict(resample_interval=3)),                        # fixed size, normalising steps
    (500, 2000, 1, dict(spatial_resolution=FINE)),                     # starts from 20 explicit states
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


def member_params(bb, k, seed=300):
    lo, hi, scheme, extra = MEMBERS[k % len(MEMBERS)]
    return bb.AmclParams(min_particles=lo, max_particles=hi, seed=seed + k, resample_scheme=scheme, record_ancestors=True, **extra)


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


def make_batch(bb, params, motions, adaptive=True):
    return bb.AmclBatch(motions, params, adaptive=adaptive)


def initialize(batch, twins, scene, explicit=(7,)):
    for m, twin in enumerate(twins):
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        if m in explicit:  # explicit states, far fewer than min_particles
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
    gs, gw = batch.particles(m)
    ts, tw = twin.particles()
    assert batch.member_size(m) == len(ts) == len(gs), where
    assert gs.tobytes() == ts.tobytes() and gw.tobytes() == tw.tobytes(), where
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
    """Cluster estimates, particle histograms and pose samples of every member against its twin."""
    est = batch.cluster_estimates()
    hists = batch.particle_histograms(None, 0.05, 0.05)
    counts = [min(700, q.max_particles) for q in batch.params]
    samples = batch.sample_states(counts, step)
    for m, twin in enumerate(twins):
        tm, tc = twin.filter.cluster_estimate()
        assert est[m][0].tobytes() == tm.tobytes() and est[m][1].tobytes() == tc.tobytes(), m
        bins, top = hists[m]
        t_bins, t_top = twin_histogram(bb, twin, 0.05, 0.05)
        assert bins.tobytes() == t_bins.tobytes() and np.float64(top).tobytes() == np.float64(t_top).tobytes(), m
        assert samples[m].tobytes() == twin.filter.sample_states(counts[m], step).tobytes(), m


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
        # launches of a step without KLD members: 4 + the reweight form's
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
    params = [member_params(bb, m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = make_batch(bb, params, motions)
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    maps.set(bb, batch, twins)
    initialize(batch, twins, scene)
    sizes = {m: set() for m in range(k)}
    kld_steps = plain_steps = skipped = 0
    for t in range(12):
        present = [(t + m) % 4 != 3 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        pts = [scene.scans[t][: 40 + 20 * m] for m in range(k)]
        n, got = launches(batch, lambda: batch.update(poses, pts, present))
        kld = False
        for m in range(k):
            if not present[m]:
                assert got[m].updated == 0
                continue
            exp = twins[m].update(poses[m], pts[m])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            skipped += 1 - exp.updated
            kld |= bool(exp.resampled) and params[m].min_particles < params[m].max_particles
            if exp.updated and exp.resampled:
                sizes[m].add(exp.n_particles)
        if any(r.updated for r in got):
            assert n == maps.base + (2 if kld else 0), (t, n)
            kld_steps += kld
            plain_steps += not kld
        if t in (5, 11):
            assert_published_equal(bb, batch, twins, 0xFFFFFF00 + t)
    assert kld_steps > 0 and skipped > 0
    for m in range(k):
        lo, hi = params[m].min_particles, params[m].max_particles
        assert all(lo <= s <= hi for s in sizes[m]), (m, sizes[m])
        if lo == hi:
            assert sizes[m] <= {hi}
    # the count really adapts: several distinct sizes, some below max_particles
    adaptive = set().union(*[sizes[m] for m in range(k) if params[m].min_particles < params[m].max_particles])
    assert len(adaptive) > 1 and any(s < params[m].max_particles for m in range(k) for s in sizes[m] if params[m].min_particles < params[m].max_particles)
    assert any(s < MEMBERS[1][1] for s in sizes[1])  # (1, 32768) shrinks


def test_several_maps_scans_and_clouds(bb, scene):
    """Two maps (likelihood field and beam), members moved between them mid-trajectory, and measurements given as points,
    scans and clouds through update_measurements; then re-initialisation of some members."""
    k = len(MEMBERS)
    params = [member_params(bb, m, seed=500) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = make_batch(bb, params, motions)
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

    for t in range(12):
        if t == 5:
            for m in range(0, k, 2):
                on[m] ^= 1
                assign(m)
        if t == 8:
            for m in (0, 1, 4):
                batch.initialize(m, scene.initial_mean, scene.initial_cov)
                twins[m].initialize(scene.initial_mean, scene.initial_cov)
                assert batch.member_size(m) == params[m].max_particles
        present = [(t + m) % 5 != 4 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        meas = [measurement(t, m) for m in range(k)]
        got = batch.update_measurements(poses, meas, present)
        for m in range(k):
            if present[m]:
                exp = feed_twin(bb, twins[m], poses[m], meas[m])
                assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
    assert_published_equal(bb, batch, twins, 0xFFFFFF40)


@pytest.mark.parametrize("k", [1, 16, 256])
def test_launch_counts(bb, scene, k):
    """+2 launches exactly when some updating member resamples under KLD, whatever K and the accepted counts are."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    rows = []
    for lo, interval in ((500, 1), (2000, 1), (500, 2)):
        params = [bb.AmclParams(min_particles=lo, max_particles=2000, seed=m, resample_scheme=m % 2, resample_interval=interval)
                  for m in range(k)]
        batch = make_batch(bb, params, [bb.DifferentialDriveModelParam() for _ in range(k)])
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(k):
            batch.initialize(m, scene.initial_mean, scene.initial_cov)
        row = []
        for t in range(2):
            n, res = launches(batch, lambda: batch.update([bb.se2(*scene.poses[t])] * k, [scene.scans[t]] * k))
            assert all(r.updated for r in res)
            row.append(n)
        rows.append(row)
    # KLD members resampling every step; fixed-size members; KLD members that normalise on odd steps
    assert rows == [[7, 7], [5, 5], [5, 7]]


def test_adaptive_batch_of_fixed_members_equals_fixed_batch(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    sizes = (1, 33, 2000, 5000, 32768)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=40 + m, resample_scheme=m % 2, record_ancestors=True,
                            resample_interval=1 + m % 2, recovery_probability_override=0.05 if m == 2 else 0.0) for m, n in enumerate(sizes)]
    motions = [motion(bb, m) for m in range(len(sizes))]
    fixed, adaptive = bb.AmclBatch(motions, params), bb.AmclBatch(motions, params, adaptive=True)
    for b in (fixed, adaptive):
        b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(len(sizes)):
            b.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(8):
        poses = [odometry(scene, t, m) for m in range(len(sizes))]
        nf, rf = launches(fixed, lambda: fixed.update(poses, [scene.scans[t]] * len(sizes)))
        na, ra = launches(adaptive, lambda: adaptive.update(poses, [scene.scans[t]] * len(sizes)))
        assert nf == na and [result_bytes(r) for r in rf] == [result_bytes(r) for r in ra], t
        for m in range(len(sizes)):
            assert fixed.particles(m)[0].tobytes() == adaptive.particles(m)[0].tobytes()
            assert fixed.particles(m)[1].tobytes() == adaptive.particles(m)[1].tobytes()
            assert fixed.ancestors(m).tobytes() == adaptive.ancestors(m).tobytes()
            assert fixed.member_size(m) == adaptive.member_size(m)


def test_failed_step_is_rolled_back(bb, scene):
    """After KLD steps, a step fails (recovery injection on a map without free cells); the member is moved back and the
    batch continues exactly as one that never failed, sizes included."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    full = bb.OccupancyGrid(np.full_like(scene.cells, 100), scene.resolution)
    params = [bb.AmclParams(min_particles=300, max_particles=3000, seed=71, record_ancestors=True),
              bb.AmclParams(min_particles=200, max_particles=2500, seed=72, recovery_probability_override=0.1, resample_scheme=1,
                            record_ancestors=True)]
    motions = [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.StationaryModelParam()]

    def make():
        b = make_batch(bb, params, motions)
        ids = [b.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid),
               b.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), full)]
        for m in range(2):
            b.update_map(m, ids[0])
            b.initialize(m, scene.initial_mean, scene.initial_cov)
        return b, ids

    (failed, ids), (clean, _) = make(), make()
    for t in range(6):
        poses = [odometry(scene, t, m) for m in range(2)]
        if t == 3:
            sizes = [failed.member_size(m) for m in range(2)]
            assert sizes[0] < 3000  # the KLD count has moved member 0 off max_particles
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
            assert failed.ancestors(m).tobytes() == clean.ancestors(m).tobytes(), (t, m)


def test_oracle_take_while_kld(bb, orc, scene):
    """Two KLD members against oracle::Amcl in counter-RNG mode: n_particles and ancestors exact, estimates within 1e-9."""
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    res = (0.5, 0.5, float(np.deg2rad(10.0)))
    cfg = [dict(min_particles=500, max_particles=30_000, scheme=1, seed=5), dict(min_particles=200, max_particles=5000, scheme=0, seed=6)]
    params = [bb.AmclParams(min_particles=c["min_particles"], max_particles=c["max_particles"], resample_scheme=c["scheme"], seed=c["seed"],
                            record_ancestors=True, spatial_resolution=res) for c in cfg]
    batch = make_batch(bb, params, [bb.DifferentialDriveModelParam(*ALPHAS[:4])] * 2)
    batch.set_likelihood_field_map(lfm, bb.OccupancyGrid(scene.cells, scene.resolution))
    oracles = [orc.Amcl(orc.AmclParam(rng_mode=1, spatial_resolution_x=res[0], spatial_resolution_y=res[1], spatial_resolution_theta=res[2], **c),
                        orc.MotionParam(*ALPHAS[:4])) for c in cfg]
    for m, o in enumerate(oracles):
        o.set_map(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
        o.initialize_normal(scene.initial_mean, scene.initial_cov)
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    sizes = []
    for t in range(8):
        pose = orc.se2(*scene.poses[t])
        got = batch.update([pose, pose], [scene.scans[t], scene.scans[t]])
        for m, o in enumerate(oracles):
            ro = o.update(pose, scene.scans[t])
            assert got[m].updated == ro.updated == 1
            assert got[m].n_particles == ro.n_particles == batch.member_size(m), (t, m)
            assert got[m].random_state_probability == ro.random_state_probability
            assert np.array_equal(batch.ancestors(m), o.last_indices()), (t, m)
            assert np.abs(np.array(got[m].estimate.mean) - np.array(ro.mean)).max() < 1e-9
            sizes.append(got[m].n_particles)
    assert len(set(sizes)) > 1 and min(sizes) < 5000
