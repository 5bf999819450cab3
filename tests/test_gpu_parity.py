"""GPU parity tests: the CUDA path behind the C ABI against the CPU oracle on the same seeded inputs.

Bit-exact for integer work (CDF, resample indices, hashes) and for weights computed from identical
states; states/estimates that go through libm (sin/cos/log/hypot differ by <= 2 ulp between CUDA and
glibc) are compared at 1e-12 relative, far inside the 1e-5 the north star asks for.
"""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PI = math.pi


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


def grid5(occupied, resolution=0.5):
    cells = np.zeros((5, 5), dtype=np.int8)
    for (r, c) in occupied:
        cells[r, c] = 100
    return cells, resolution


LFM = dict(max_obstacle_distance=2.0, max_laser_distance=20.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)


def gpu_weights(bb, sensor, params, cells, resolution, origin, points, states):
    f = bb.Filter(capacity=max(len(states), 1))
    grid = bb.OccupancyGrid(cells, resolution, origin)
    if sensor == bb.SENSOR_BEAM:
        f.set_beam_map(params, grid)
    else:
        f.set_likelihood_field_map(params, grid, prob=(sensor == bb.SENSOR_LIKELIHOOD_FIELD_PROB))
    f.set_particles(states)
    f.reweight(points)
    return f.particles()[1]


# ---- the reference's known-answer tests, through the C ABI on the GPU -------------------------------
def test_lfm_known_answers(bb, orc):
    """sensor/test_likelihood_field_model.cpp:34-74,160-203 and test_likelihood_field_prob_model.cpp:160-195."""
    cells, res = grid5([(2, 2)])
    p = bb.LikelihoodFieldModelParam(**LFM)
    ident = orc.IDENTITY
    w = lambda pts, st, sensor=bb.SENSOR_LIKELIHOOD_FIELD: gpu_weights(bb, sensor, p, cells, res, ident, pts, [st])[0]  # noqa: E731
    assert w([(1.25, 1.25)], ident) == pytest.approx(2.068, abs=0.003)
    assert w([(2.25, 2.25)], ident) == pytest.approx(1.000, abs=0.003)
    assert w([(-50.0, 50.0)], ident) == pytest.approx(1.000, abs=0.003)
    assert w([(1.20, 1.20), (1.25, 1.25), (1.30, 1.30)], ident) == pytest.approx(4.205, abs=0.01)
    assert w([(0.0, 0.0)], orc.se2(1.25, 1.25, 0.0)) == pytest.approx(2.068, abs=0.003)
    assert w([(1.0, 1.0)], ident) == pytest.approx(2.068577607986223, abs=1e-6)
    assert w([(1.0, 1.0)], ident, bb.SENSOR_LIKELIHOOD_FIELD_PROB) == pytest.approx(1.0223556756973267, abs=1e-6)


def test_lfm_known_answers_with_origin(bb, orc):
    """GridWithOffset / GridWithRotation / GridWithRotationAndOffset (test_likelihood_field_model.cpp:76-158)."""
    cells, res = grid5([(4, 4)], 2.0)
    p = bb.LikelihoodFieldModelParam(**LFM)
    w = lambda origin, pts, st: gpu_weights(bb, bb.SENSOR_LIKELIHOOD_FIELD, p, cells, res, origin, pts, [st])[0]  # noqa: E731
    o = orc.se2(-5, -5, 0.0)
    assert w(o, [(4.5, 4.5)], orc.IDENTITY) == pytest.approx(2.068, abs=0.003)
    assert w(o, [(9.5, 9.5)], o) == pytest.approx(2.068, abs=0.003)
    o = orc.se2(0.0, 0.0, PI / 2)
    assert w(o, [(-9.5, 9.5)], orc.IDENTITY) == pytest.approx(2.068, abs=0.003)
    assert w(o, [(9.5, 9.5)], o) == pytest.approx(2.068, abs=0.003)
    rot = orc.se2(0.0, 0.0, PI / 2)
    t = orc.se2_compose(rot, orc.se2(-5, -5, 0.0))
    o = np.array([rot[0], rot[1], t[2], t[3]])
    assert w(o, [(-4.5, 4.5)], orc.IDENTITY) == pytest.approx(2.068, abs=0.003)
    assert w(o, [(9.5, 9.5)], o) == pytest.approx(2.068, abs=0.003)


def test_beam_known_answers(bb, orc):
    """sensor/test_beam_model.cpp:40-82."""
    cells, res = grid5([(2, 2)])
    p = bb.BeamModelParam(z_hit=0.5, z_short=0.05, z_max=0.05, z_rand=0.5, sigma_hit=0.2, lambda_short=0.1, beam_max_range=60)
    w = lambda pts: gpu_weights(bb, bb.SENSOR_BEAM, p, cells, res, orc.IDENTITY, pts, [orc.IDENTITY])[0]  # noqa: E731
    assert w([(1.0, 1.0)]) == pytest.approx(1.0171643824743635, abs=1e-6)
    assert w([(0.75, 0.75)]) == pytest.approx(0.015905891701088148, abs=1e-6)
    assert w([(2.25, 2.25)]) == pytest.approx(0.000, abs=1e-6)
    assert w([(60.0, 60.0)]) == pytest.approx(0.00012500000000000003, abs=1e-6)


# ---- kernel-level parity against the oracle -----------------------------------------------------------
@pytest.fixture(scope="module")
def scene():
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=12)


def random_states(orc, rng, n, extent):
    xs = rng.uniform(-1.0, extent + 1.0, n)
    ys = rng.uniform(-1.0, extent + 1.0, n)
    th = rng.uniform(-PI, PI, n)
    return np.array([orc.se2(x, y, t) for x, y, t in zip(xs, ys, th)])


def test_likelihood_field_is_identical(bb, orc, scene):
    p = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    for unknown, strict in [(False, False), (True, False), (False, True), (True, True)]:
        cells = scene.cells.copy()
        cells[50:60, 50:60] = -1  # a patch of unknown space
        f = bb.Filter(capacity=8)
        f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(model_unknown_space=unknown, only_obstacle_boundaries=strict, **p),
                                   bb.OccupancyGrid(cells, scene.resolution))
        exp = orc.likelihood_field(orc.LfmParam(model_unknown_space=unknown, only_obstacle_boundaries=strict, **p), orc.Grid(cells, scene.resolution))
        assert np.array_equal(f.likelihood_field(), exp)


@pytest.mark.parametrize("n_points", [0, 1, 3, 4, 5, 181, 2500])
@pytest.mark.parametrize("sensor", [0, 1])
def test_reweight_lfm_bit_exact(bb, orc, scene, n_points, sensor):
    rng = np.random.default_rng(3)
    extent = scene.cells.shape[0] * scene.resolution
    states = random_states(orc, rng, 1500, extent)  # some particles outside the grid
    pts = rng.uniform(-8.0, 8.0, (n_points, 2))
    params = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    origin = orc.se2(0.3, -0.2, 0.1)
    got = gpu_weights(bb, sensor, bb.LikelihoodFieldModelParam(**params), scene.cells, scene.resolution, origin, pts, states)
    exp = orc.sensor_weights(sensor, orc.LfmParam(**params), orc.Grid(scene.cells, scene.resolution, origin), pts, states)
    if sensor == 0:
        assert np.array_equal(got, exp)  # pure +,* arithmetic and float loads: bit-exact
    else:
        normal = exp > 1e-290  # exp(sum log pz) underflows into subnormals for many beams, where ulps are coarse
        assert np.allclose(got[normal], exp[normal], rtol=1e-13, atol=0.0)  # one exp() per particle
        assert np.allclose(got[~normal], exp[~normal], rtol=1e-6, atol=1e-320)


def test_initialize_from_map_matches_oracle(bb, orc, scene):
    """initialize_from_map (beluga_ros/include/beluga_ros/amcl.hpp:192-209): the free cell and yaw of every particle are the
    oracle's (counter stream 6), the first update is forced, and the reference's known answers hold on the GPU
    (test_multivariate_uniform_distribution.cpp:56-124)."""
    n = 50_000
    cells = scene.cells.copy()
    cells[20:40, 20:60] = -1  # unknown space is not free
    g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=n, max_particles=n, seed=21))
    o = orc.Amcl(orc.AmclParam(min_particles=n, max_particles=n, seed=21, rng_mode=1), orc.MotionParam(0.1, 0.05, 0.1, 0.05))
    origin = orc.se2(-3.0, 1.5, 0.3)
    g.update_map(0, bb.LikelihoodFieldModelParam(max_laser_distance=100.0), bb.OccupancyGrid(cells, scene.resolution, origin))
    o.set_map(0, orc.LfmParam(max_laser_distance=100.0), orc.Grid(cells, scene.resolution, origin))
    g.initialize_from_map()
    o.initialize_from_map()
    sg, wg = g.particles()
    so, wo = o.particles()
    assert np.all(wg == 1.0) and len(sg) == n
    assert np.array_equal(sg[:, 2:4], so[:, 2:4])  # cell centroids: plain arithmetic, bit-identical
    assert np.abs(sg[:, 0:2] - so[:, 0:2]).max() < 1e-15
    assert g.update(orc.se2(0.0, 0.0, 0.0), scene.scans[0]).updated == 1  # force_update_ = true
    # GridSomeFreeSlots on the device
    f = bb.Filter(capacity=100_000, seed=4)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(), bb.OccupancyGrid(np.array([[100, 0, 100], [0, 100, 0], [100, 0, 100]], dtype=np.int8), 1.0))
    f.initialize_uniform(100_000)
    st, _ = f.particles()
    buckets, counts = np.unique(st[:, 2:4], axis=0, return_counts=True)
    assert sorted(map(tuple, buckets)) == [(0.5, 1.5), (1.5, 0.5), (1.5, 2.5), (2.5, 1.5)]
    assert np.abs(counts / 100_000 - 0.25).max() < 0.01
    # no free cell: an error, not a crash
    f2 = bb.Filter(capacity=8)
    f2.set_likelihood_field_map(bb.LikelihoodFieldModelParam(), bb.OccupancyGrid(np.full((3, 3), 100, dtype=np.int8), 1.0))
    with pytest.raises(bb.BelugaB200Error):
        f2.initialize_uniform(8)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 257])
@pytest.mark.parametrize("n_points", [7, 1920, 1921])
def test_reweight_ragged_particle_counts(bb, orc, scene, n, n_points):
    """Particle counts around the 32-particle task size of the persistent kernel, and scans on either side of
    the kernel-parameter limit (1920 points: constant bank; 1921: TMA + shared memory)."""
    rng = np.random.default_rng(100 * n + n_points)
    extent = scene.cells.shape[0] * scene.resolution
    states = random_states(orc, rng, n, extent)
    pts = rng.uniform(-6.0, 6.0, (n_points, 2))
    params = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    got = gpu_weights(bb, 0, bb.LikelihoodFieldModelParam(**params), scene.cells, scene.resolution, orc.IDENTITY, pts, states)
    exp = orc.sensor_weights(0, orc.LfmParam(**params), orc.Grid(scene.cells, scene.resolution), pts, states)
    assert np.array_equal(got, exp)


def test_reweight_twice_reuses_the_ticket_counter(bb, orc, scene):
    """Two launches in a row on one filter: the persistent kernel's last warp must rewind its ticket counter."""
    rng = np.random.default_rng(8)
    states = random_states(orc, rng, 5000, scene.cells.shape[0] * scene.resolution)
    pts = rng.uniform(-6.0, 6.0, (64, 2))
    params = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    f = bb.Filter(capacity=len(states))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**params), bb.OccupancyGrid(scene.cells, scene.resolution, orc.IDENTITY))
    f.set_particles(states)
    f.reweight(pts)
    f.reweight(pts)
    once = orc.sensor_weights(0, orc.LfmParam(**params), orc.Grid(scene.cells, scene.resolution), pts, states)
    assert np.array_equal(f.particles()[1], once * once)


def test_reweight_far_away_particles(bb, orc, scene):
    """Coordinates beyond the fast floor range take the general path; all land out of the grid."""
    states = np.array([orc.se2(1e12, -3e11, 0.3), orc.se2(-1e300, 1e300, 1.0), orc.se2(2.0, 2.0, 0.0), orc.se2(5e9, 5e9, 0.0),
                       orc.se2(450.0, -430.0, 2.0), orc.se2(-404.9, 3.0, -1.0), orc.se2(3.0, 409.0, 0.5), orc.se2(float("nan"), 1.0, 0.0)])
    pts = np.array([[1.0, 0.5], [2.0, -1.0], [0.1, 0.1], [3.0, 3.0], [0.0, 0.0]])
    params = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    got = gpu_weights(bb, 0, bb.LikelihoodFieldModelParam(**params), scene.cells, scene.resolution, orc.IDENTITY, pts, states)
    exp = orc.sensor_weights(0, orc.LfmParam(**params), orc.Grid(scene.cells, scene.resolution), pts, states)
    assert np.array_equal(got, exp)


def test_reweight_cell_boundaries(bb, orc, scene):
    """End points exactly on (and one ulp either side of) cell boundaries: the guarded FMA evaluation
    must hand these to the exact operation sequence and land in the reference's cell."""
    res = scene.resolution
    rng = np.random.default_rng(17)
    k = rng.integers(5, 150, (400, 2)).astype(np.float64)
    states = np.array([orc.se2(a * res, b * res, 0.0) for a, b in k])
    states = np.concatenate([states, np.array([orc.se2(a * res, b * res, np.pi / 2) for a, b in k[:200]])])
    m = rng.integers(-40, 40, (96, 2)).astype(np.float64) * res
    pts = np.concatenate([m, np.nextafter(m, np.inf), np.nextafter(m, -np.inf)])
    params = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    got = gpu_weights(bb, 0, bb.LikelihoodFieldModelParam(**params), scene.cells, res, orc.IDENTITY, pts, states)
    exp = orc.sensor_weights(0, orc.LfmParam(**params), orc.Grid(scene.cells, res), pts, states)
    assert np.array_equal(got, exp)


def test_reweight_beam_matches_oracle(bb, orc, scene):
    rng = np.random.default_rng(5)
    extent = scene.cells.shape[0] * scene.resolution
    states = random_states(orc, rng, 600, extent)
    pts = scene.scans[0][::3]
    origin = orc.se2(0.1, 0.05, -0.05)
    got = gpu_weights(bb, bb.SENSOR_BEAM, bb.BeamModelParam(beam_max_range=20.0), scene.cells, scene.resolution, origin, pts, states)
    exp = orc.sensor_weights(orc.BEAM, orc.BeamParam(beam_max_range=20.0), orc.Grid(scene.cells, scene.resolution, origin), pts, states)
    assert np.allclose(got, exp, rtol=1e-11, atol=1e-300)  # erf/exp per beam differ by ulps between CUDA and glibc


@pytest.mark.parametrize("shape, launches", [("wide_grid", 2), ("long_reach", 2), ("fine_cells", 3)])
def test_reweight_beam_fallbacks_match_oracle(bb, orc, scene, shape, launches):
    """Maps whose shape selects the fused beam kernel or the per-beam normalisers instead of the two-pass walk with the
    normaliser table: a grid wider than 65534 cells (fused kernel, table), a reach of 2^21 cells or more (fused kernel,
    per-beam normalisers), and a range / resolution ratio too large for the table (two-pass walk, per-beam normalisers).
    The scene is scaled with the resolution (scan, sigma_hit, 1 / lambda_short) so that its rays hit at the usual ranges
    in cells; beam_max_range stays in metres.  `launches`: begin_step plus 1 (fused) or 2 (walk + mixture)."""
    rng = np.random.default_rng(23)
    if shape == "wide_grid":
        cells = np.where(rng.random((8, 70_000)) < 0.05, 100, 0).astype(np.int8)
        res, max_range = scene.resolution, 20.0
    else:
        cells = scene.cells
        res, max_range = (1e-5, 30.0) if shape == "long_reach" else (0.01, 30.0)
    scale = res / scene.resolution
    height, width = cells.shape
    n = 300
    states = np.array([orc.se2(x, y, t) for x, y, t in zip(rng.uniform(0.0, width * res, n), rng.uniform(0.0, height * res, n),
                                                             rng.uniform(-PI, PI, n))])
    pts = scene.scans[0][::3] * scale
    bp = dict(sigma_hit=0.2 * scale, lambda_short=0.1 / scale, beam_max_range=max_range)
    f = bb.Filter(capacity=n)
    f.set_beam_map(bb.BeamModelParam(**bp), bb.OccupancyGrid(cells, res))
    f.set_particles(states)
    before = f.launch_count()
    f.reweight(pts)
    assert f.launch_count() - before == launches
    exp = orc.sensor_weights(orc.BEAM, orc.BeamParam(**bp), orc.Grid(cells, res), pts, states)
    assert np.allclose(f.particles()[1], exp, rtol=1e-11, atol=1e-300)


def test_propagate_matches_oracle(bb, orc):
    rng = np.random.default_rng(11)
    states = random_states(orc, rng, 5000, 10.0)
    s6 = orc.diff_drive_sampling(orc.MotionParam(0.1, 0.05, 0.1, 0.05), orc.se2(1.3, 0.4, 0.3), orc.se2(1.0, 0.2, 0.1))
    f = bb.Filter(capacity=len(states), seed=99, first_index=1000)
    f.set_particles(states)
    f.propagate(s6, step=7)
    got = f.particles()[0]
    exp = orc.diff_drive_propagate(s6, states, mode=1, seed=99, step=7, first_index=1000)
    assert np.allclose(got, exp, rtol=0.0, atol=1e-12)
    assert np.abs(np.hypot(got[:, 0], got[:, 1]) - 1.0).max() < 1e-15


@pytest.mark.parametrize("model", [1, 2])
def test_propagate_other_motion_models(bb, orc, model):
    """OmnidirectionalDriveModel / StationaryModel (motion/omnidirectional_drive_model.hpp:131-145, stationary_model.hpp:54-59)."""
    rng = np.random.default_rng(12)
    states = random_states(orc, rng, 3000, 10.0)
    alphas = (0.1, 0.05, 0.1, 0.05, 0.02)
    motion = bb.OmnidirectionalDriveModelParam(*alphas) if model == 1 else bb.StationaryModelParam()
    pose, prev = orc.se2(1.3, 0.4, 0.3), orc.se2(1.0, 0.2, 0.1)
    f = bb.Filter(capacity=len(states), seed=99, first_index=500)
    f.set_particles(states)
    f.propagate(bb.motion_sampling(motion, pose, prev), step=4)
    exp = orc.motion_propagate(orc.motion_sampling(model, orc.OmniParam(*alphas), pose, prev), states, mode=1, seed=99, step=4, first_index=500)
    assert np.allclose(f.particles()[0], exp, rtol=0.0, atol=1e-12)


def test_trajectory_omnidirectional(bb, orc, scene):
    n = 6000
    alphas = (0.1, 0.05, 0.1, 0.05, 0.02)
    lfm = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    g = bb.Amcl(bb.OmnidirectionalDriveModelParam(*alphas), bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=1, seed=8, record_ancestors=True))
    o = orc.Amcl(orc.AmclParam(min_particles=n, max_particles=n, scheme=1, seed=8, rng_mode=1), orc.OmniParam(*alphas), motion_model=orc.OMNIDIRECTIONAL)
    g.update_map(0, bb.LikelihoodFieldModelParam(**lfm), bb.OccupancyGrid(scene.cells, scene.resolution))
    o.set_map(0, orc.LfmParam(**lfm), orc.Grid(scene.cells, scene.resolution))
    g.initialize(scene.initial_mean, scene.initial_cov)
    o.initialize_normal(scene.initial_mean, scene.initial_cov)
    for k in range(8):
        pose = orc.se2(*scene.poses[k])
        rg, ro = g.update(pose, scene.scans[k]), o.update(pose, scene.scans[k])
        assert np.array_equal(g.filter.ancestors(), o.last_indices())
        assert np.abs(np.array(rg.estimate.mean) - np.array(ro.mean)).max() < 1e-10


def test_initialize_normal_matches_oracle(bb, orc):
    mean = np.array([3.0, -2.0, 0.7])
    cov = np.array([[0.25, 0.05, 0.0], [0.05, 0.16, 0.01], [0.0, 0.01, 0.0685]])
    n = 4096
    f = bb.Filter(capacity=n, seed=5)
    f.initialize_normal(mean, cov, n)
    got, w = f.particles()
    o = orc.Amcl(orc.AmclParam(max_particles=n, min_particles=n, seed=5, rng_mode=1), orc.MotionParam())
    o.initialize_normal(mean, cov)
    exp, _ = o.particles()
    assert np.all(w == 1.0)
    assert np.allclose(got, exp, rtol=0.0, atol=1e-12)
    # and the sample statistics follow the requested distribution
    th = np.arctan2(got[:, 1], got[:, 0])
    emp = np.cov(np.stack([got[:, 2], got[:, 3], th]))
    assert np.abs(emp - cov).max() < 0.03
    with pytest.raises(bb.BelugaB200Error):  # multivariate_normal_distribution.hpp:114-116
        f.initialize_normal(mean, np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]), n)


@pytest.mark.parametrize("n", [1, 31, 2048, 2049, 100_003])
def test_cdf_and_indices_bit_exact(bb, orc, n):
    rng = np.random.default_rng(n)
    w = rng.gamma(0.5, 2.0, n) + 1e-9
    w[rng.integers(0, n, max(1, n // 50))] = 0.0  # zero-weight particles are never selected
    if not (w > 0).any():
        w[0] = 1.0
    states = np.tile(orc.IDENTITY, (n, 1))
    states[:, 2] = np.arange(n)  # x encodes the particle id
    for scheme in (bb.RESAMPLE_MULTINOMIAL, bb.RESAMPLE_SYSTEMATIC):
        f = bb.Filter(capacity=n, seed=1234, record_ancestors=True)
        f.set_particles(states, w)
        total, ex = f.build_cdf()
        idx, cdf, ex_o = orc.resample_indices(w, scheme, seed=1234, step=3)
        assert ex == ex_o
        assert np.array_equal(f.cdf(), cdf)
        assert total == int(cdf[-1])
        assert f.resample(scheme, step=3, max_particles=n) == n
        anc = f.ancestors()
        assert np.array_equal(anc, idx)
        new_states, new_w = f.particles()
        assert np.array_equal(new_states[:, 2], idx.astype(np.float64))  # the gather moved the right states
        assert np.all(new_w == 1.0)
        assert np.all(w[anc] > 0.0)


@pytest.mark.parametrize("case", ["collapse", "few_heavy", "resize_up", "resize_down"])
def test_systematic_resample_degenerate_weights(bb, orc, case):
    """The scatter-form systematic resample: one particle taking (almost) every slot, a handful of heavy
    particles among dust, and output sizes different from the input size."""
    rng = np.random.default_rng(5)
    n = 20_000
    m = {"resize_up": 50_000, "resize_down": 3_000}.get(case, n)
    w = np.full(n, 1e-12)
    if case == "collapse":
        w[12_345] = 1.0
    elif case == "few_heavy":
        w[rng.integers(0, n, 7)] = rng.uniform(0.5, 2.0, 7)
    else:
        w = rng.gamma(0.3, 1.0, n) + 1e-9
    states = np.tile(orc.IDENTITY, (n, 1))
    states[:, 2] = np.arange(n)
    f = bb.Filter(capacity=max(n, m), seed=77, record_ancestors=True)
    f.set_particles(states, w)
    f.build_cdf()
    idx, _, _ = orc.resample_indices(w, bb.RESAMPLE_SYSTEMATIC, seed=77, step=9, m=m, n_total=max(n, m))  # the exponent follows the capacity
    assert f.resample(bb.RESAMPLE_SYSTEMATIC, step=9, max_particles=m) == m
    assert np.array_equal(f.ancestors(), idx)
    new_states, new_w = f.particles()
    assert np.array_equal(new_states[:, 2], idx.astype(np.float64)) and np.all(new_w == 1.0)
    mean, cov = f.estimate()
    want_mean, want_cov = orc.estimate(states[idx], np.ones(m))
    assert np.allclose(mean, want_mean, atol=1e-9) and np.allclose(cov[:2, :2], want_cov[:2, :2], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("scheme", [0, 1])
def test_injection_never_replaces_the_first_slot(bb, orc, scene, scheme):
    """views::random_intersperse tosses its coin when the view ADVANCES: with probability 1 the output is one
    sampled particle followed by random states only (test_random_intersperse.cpp:88-117)."""
    n = 64
    f = bb.Filter(capacity=n, seed=9, record_ancestors=True)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(max_obstacle_distance=2.0, max_laser_distance=100.0),
                               bb.OccupancyGrid(scene.cells, scene.resolution, orc.IDENTITY))  # the free cells the random states come from
    f.set_particles(np.tile(orc.IDENTITY, (n, 1)), np.ones(n))
    f.build_cdf()
    assert f.resample(scheme, step=4, max_particles=n, random_state_probability=1.0) == n
    anc = f.ancestors()
    assert anc[0] >= 0 and np.all(anc[1:] == -1)
    assert np.array_equal(anc < 0, orc.inject_flags(seed=9, step=4, probability=1.0, m=n).astype(bool))


def test_normalize_and_ess(bb, orc):
    rng = np.random.default_rng(8)
    n = 50_000
    w = rng.uniform(0.5, 3.0, n)
    f = bb.Filter(capacity=n)
    f.set_particles(np.tile(orc.IDENTITY, (n, 1)), w)
    factor, sum_sq = f.normalize()
    got = f.particles()[1]
    assert factor == pytest.approx(w.sum(), rel=1e-11)  # S = T * 2^-e: the quantisation is at 2^-41 of wmax
    assert np.allclose(got, w / factor, rtol=1e-15, atol=0.0)
    assert 1.0 / sum_sq == pytest.approx(orc.effective_sample_size(w), rel=1e-9)


def test_estimate_matches_oracle(bb, orc):
    rng = np.random.default_rng(21)
    n = 30_000
    states = random_states(orc, rng, n, 40.0)
    states[:, 2] += 100.0  # far from the pivot: exercises the shifted moments
    w = rng.uniform(0.0, 2.0, n)
    f = bb.Filter(capacity=n)
    f.set_particles(states, w)
    mean, cov = f.estimate()
    emean, ecov = orc.estimate(states, w)
    assert np.allclose(mean, emean, rtol=0.0, atol=1e-11)
    assert np.allclose(cov, ecov, rtol=1e-10, atol=1e-12)


def test_estimate_known_answers(bb, orc):
    """algorithm/test_estimation.cpp:138-191 (PureTranslation, PureRotation, CancellingOrientations)."""
    f = bb.Filter(capacity=8)
    f.set_particles([orc.se2(1.0, 2.0, 0.0), orc.se2(0.0, 0.0, 0.0)])
    mean, cov = f.estimate()
    assert np.allclose(mean, orc.se2(0.5, 1.0, 0.0), atol=1e-3)
    assert np.allclose(cov, [[0.5, 1.0, 0.0], [1.0, 2.0, 0.0], [0.0, 0.0, 0.0]], atol=1e-3)
    f.set_particles([orc.se2(0.0, 0.0, -PI / 2), orc.se2(0.0, 0.0, 0.0)])
    mean, cov = f.estimate()
    assert np.allclose(mean, orc.se2(0.0, 0.0, -PI / 4), atol=1e-3)
    assert cov[2, 2] == pytest.approx(0.693, abs=1e-3)
    f.set_particles([orc.se2(0.0, 0.0, PI / 2), orc.se2(0.0, 0.0, -PI / 2)])
    mean, cov = f.estimate()
    assert math.isinf(cov[2, 2]) and np.allclose(mean, orc.se2(0.0, 0.0, 0.0), atol=1e-3)


# ---- KLD-adaptive sample size (views/test_take_while_kld.cpp) ------------------------------------------
def kld_count_on_gpu(bb, orc, buckets, min_particles, max_particles, epsilon, z):
    """Runs take_while_kld on the GPU over a prescribed bucket sequence: particle j sits in bucket
    buckets[j]; equal weights + the systematic comb make output slot j a copy of particle j."""
    buckets = np.asarray(buckets)
    n = len(buckets)
    assert n == max_particles
    states = np.tile(orc.IDENTITY, (n, 1))
    states[:, 2] = buckets * 10.0 + 0.5  # 10 m apart: distinct x buckets of a 1 m spatial hash
    f = bb.Filter(capacity=n, seed=9, record_ancestors=True)
    f.set_particles(states)
    m = f.resample(bb.RESAMPLE_SYSTEMATIC, step=1, max_particles=max_particles, min_particles=min_particles, kld_epsilon=epsilon, kld_z=z,
                   spatial_resolution=(1.0, 1.0, 1.0))
    assert np.array_equal(f.ancestors(), np.arange(m))
    hashes = [orc.spatial_hash(s, 1.0, 1.0, 1.0) for s in states[:: max(1, n // 64)]]  # sanity: buckets really differ
    assert len(set(hashes)) == len(set(buckets[:: max(1, n // 64)].tolist()))
    return m


@pytest.mark.parametrize(
    "z,clusters,expected",
    [(1.28155156327703, 3, 228), (1.28155156327703, 4, 311), (1.28155156327703, 5, 388), (1.28155156327703, 6, 461),
     (1.28155156327703, 7, 531), (1.28155156327703, 100, 5871), (2.32634787735669, 3, 462), (2.32634787735669, 4, 569),
     (2.32634787735669, 5, 666), (2.32634787735669, 6, 756), (2.32634787735669, 7, 843), (2.32634787735669, 100, 6733)],
)
def test_kld_known_answers(bb, orc, z, clusters, expected):
    """KldConditionWithParam.Limit (views/test_take_while_kld.cpp:119-148): exact counts."""
    n = 8192
    buckets = np.minimum(np.arange(1, n + 1), clusters)
    assert kld_count_on_gpu(bb, orc, buckets, 0, n, 0.01, z) == expected


def test_kld_take_limits(bb, orc):
    """TakeMaximum / TakeLimit / TakeMinimum (views/test_take_while_kld.cpp:159-188)."""
    assert kld_count_on_gpu(bb, orc, np.ones(1200, dtype=int), 200, 1200, 0.05, 3.0) == 1200
    seq = np.tile([1, 3, 2, 3], 300)
    assert kld_count_on_gpu(bb, orc, seq, 0, 1200, 0.05, 3.0) == 135
    assert kld_count_on_gpu(bb, orc, seq, 200, 1200, 0.05, 3.0) == 200


def test_kld_multi_chunk(bb, orc):
    """A cutoff beyond the first chunk of candidates (chunks double from 65536 slots)."""
    n = 300_000
    rng = np.random.default_rng(2)
    buckets = rng.integers(0, 15000, n)  # ~15000 buckets: target(k) ~ 10 k = 150k > first chunk
    got = kld_count_on_gpu(bb, orc, buckets, 1000, n, 0.05, 3.0)
    states_x = buckets * 10.0 + 0.5
    hashes = [orc.spatial_hash(np.array([1.0, 0.0, x, 0.0]), 1.0, 1.0, 1.0) for x in states_x]
    assert got == orc.kld_take_count(hashes, 1000, n, 0.05, 3.0)
    assert got > 65536


# ---- whole-filter parity along a seeded trajectory ------------------------------------------------------
def run_trajectory(bb, orc, scene, sensor, scheme, n, steps, selective=False, interval=1, beam_stride=1):
    motion = dict(alpha1=0.1, alpha2=0.05, alpha3=0.1, alpha4=0.05)
    lfm = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    ap = dict(update_min_d=0.25, update_min_a=0.2, resample_interval=interval, selective_resampling=selective, min_particles=n,
              max_particles=n, seed=77)
    g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(resample_scheme=scheme, record_ancestors=True, **ap))
    o = orc.Amcl(orc.AmclParam(rng_mode=1, scheme=scheme, **ap), orc.MotionParam(**motion))
    if sensor == bb.SENSOR_BEAM:
        g.update_map(sensor, bb.BeamModelParam(beam_max_range=20.0), bb.OccupancyGrid(scene.cells, scene.resolution))
        o.set_map(orc.BEAM, orc.BeamParam(beam_max_range=20.0), orc.Grid(scene.cells, scene.resolution))
    else:
        g.update_map(sensor, bb.LikelihoodFieldModelParam(**lfm), bb.OccupancyGrid(scene.cells, scene.resolution))
        o.set_map(sensor, orc.LfmParam(**lfm), orc.Grid(scene.cells, scene.resolution))
    g.initialize(scene.initial_mean, scene.initial_cov)
    o.initialize_normal(scene.initial_mean, scene.initial_cov)
    mismatched = 0
    for k in range(steps):
        pose = orc.se2(*scene.poses[k])
        pts = scene.scans[k][::beam_stride]
        rg = g.update(pose, pts)
        ro = o.update(pose, pts)
        assert rg.updated == ro.updated == 1
        assert rg.resampled == ro.resampled
        assert rg.n_particles == ro.n_particles == n
        if rg.resampled:
            a_g, a_o = g.filter.ancestors(), o.last_indices()
            mismatched += int((a_g != a_o).sum())
        gm, gc = np.array(rg.estimate.mean), np.array(rg.estimate.cov)
        om, oc = np.array(ro.mean), np.array(ro.cov)
        assert np.abs(gm - om).max() < 1e-5 and np.abs(gc - oc).max() < 1e-5  # the north-star bound
        if mismatched == 0:
            assert np.abs(gm - om).max() < 1e-10 and np.abs(gc - oc).max() < 1e-10
            assert rg.weight_sum == pytest.approx(ro.weight_sum, rel=1e-12)
    # the filter actually tracks the ground truth
    assert np.hypot(gm[2] - scene.poses[steps - 1][0], gm[3] - scene.poses[steps - 1][1]) < 0.3
    return mismatched


@pytest.mark.parametrize("scheme", [0, 1])
def test_trajectory_lfm(bb, orc, scene, scheme):
    assert run_trajectory(bb, orc, scene, bb.SENSOR_LIKELIHOOD_FIELD, scheme, n=20_000, steps=12) == 0


def test_trajectory_lfm_prob(bb, orc, scene):
    # 60 beams keep exp(sum log pz) inside the double range
    assert run_trajectory(bb, orc, scene, bb.SENSOR_LIKELIHOOD_FIELD_PROB, 1, n=5_000, steps=8, beam_stride=3) <= 5


def test_trajectory_selective_resampling(bb, orc, scene):
    assert run_trajectory(bb, orc, scene, bb.SENSOR_LIKELIHOOD_FIELD, 0, n=8_000, steps=10, selective=True, interval=2) == 0


def test_trajectory_beam(bb, orc, scene):
    # erf/exp differ by ulps between CUDA and glibc, so a handful of CDF boundary flips are tolerated
    assert run_trajectory(bb, orc, scene, bb.SENSOR_BEAM, 1, n=2_000, steps=6, beam_stride=6) <= 5


def test_trajectory_kld_adaptive(bb, orc, scene):
    """min_particles < max_particles: the particle count follows take_while_kld step by step."""
    motion = dict(alpha1=0.1, alpha2=0.05, alpha3=0.1, alpha4=0.05)
    lfm = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    ap = dict(min_particles=500, max_particles=40_000, kld_epsilon=0.05, kld_z=3.0, seed=5)
    res = (0.5, 0.5, float(np.deg2rad(10.0)))  # beluga_ros defaults (amcl.hpp:91-97)
    g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(resample_scheme=1, record_ancestors=True, spatial_resolution=res, **ap))
    o = orc.Amcl(orc.AmclParam(rng_mode=1, scheme=1, spatial_resolution_x=res[0], spatial_resolution_y=res[1], spatial_resolution_theta=res[2], **ap),
                 orc.MotionParam(**motion))
    g.update_map(0, bb.LikelihoodFieldModelParam(**lfm), bb.OccupancyGrid(scene.cells, scene.resolution))
    o.set_map(0, orc.LfmParam(**lfm), orc.Grid(scene.cells, scene.resolution))
    g.initialize(scene.initial_mean, scene.initial_cov)
    o.initialize_normal(scene.initial_mean, scene.initial_cov)
    sizes = []
    for k in range(8):
        pose = orc.se2(*scene.poses[k])
        rg, ro = g.update(pose, scene.scans[k]), o.update(pose, scene.scans[k])
        assert rg.n_particles == ro.n_particles
        assert rg.random_state_probability == ro.random_state_probability  # Thrun estimator reacts to the size change
        a_g, a_o = g.filter.ancestors(), o.last_indices()
        assert np.array_equal(a_g, a_o)
        assert np.abs(np.array(rg.estimate.mean) - np.array(ro.mean)).max() < 1e-9
        sizes.append(rg.n_particles)
    assert min(sizes) < 40_000 and len(set(sizes)) > 1  # the count really adapts


def test_update_policy_and_force_update(bb, orc, scene):
    """amcl_core.hpp:166-172: no particles -> nullopt; no motion -> nullopt unless forced."""
    n = 1000
    g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=n, max_particles=n))
    g.update_map(0, bb.LikelihoodFieldModelParam(max_laser_distance=100.0), bb.OccupancyGrid(scene.cells, scene.resolution))
    pose = orc.se2(*scene.poses[0])
    assert g.update(pose, scene.scans[0]).updated == 0  # not initialised: particles_.empty()
    g.initialize(scene.initial_mean, scene.initial_cov)
    assert g.update(pose, scene.scans[0]).updated == 1  # first update is forced by initialize()
    assert g.update(pose, scene.scans[0]).updated == 0  # same pose: on_motion says no
    g.force_update()
    assert g.update(pose, scene.scans[0]).updated == 1
    assert g.update(orc.se2(*scene.poses[1]), scene.scans[1]).updated == 1  # moved 0.4 m > update_min_d


def test_update_scan_equals_update_with_points(bb, orc, scene):
    """Amcl::update(pose, laser_scan) (beluga_ros/src/amcl.cpp:54-64) == update(pose, converted points)."""
    n = 2000
    mk = lambda: bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=n, max_particles=n, seed=4))  # noqa: E731
    a, b = mk(), mk()
    for f in (a, b):
        f.update_map(0, bb.LikelihoodFieldModelParam(max_laser_distance=100.0), bb.OccupancyGrid(scene.cells, scene.resolution))
        f.initialize(scene.initial_mean, scene.initial_cov)
    ranges = np.hypot(scene.scans[0][:, 0], scene.scans[0][:, 1]).astype(np.float32)
    args = dict(angle_min=-PI, angle_increment=2 * PI / len(ranges), min_range=0.1, max_range=25.0, max_beams=60)
    ra = a.update_scan(bb.se2(*scene.poses[0]), ranges, **args)
    rb = b.update(bb.se2(*scene.poses[0]), bb.scan_to_points(ranges, **args))
    assert ra.updated == rb.updated == 1
    assert np.array_equal(np.array(ra.estimate.mean), np.array(rb.estimate.mean))
    assert np.array_equal(a.particles()[0], b.particles()[0])


def test_large_scale_properties(bb):
    """BASELINE config 2 shapes (1M particles x 1080 beams) through size-independent properties:
    weights reset to 1, ancestors sorted for the systematic comb, states stay unit-norm, and the
    estimate tracks the ground truth."""
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=500, n_beams=1080, steps=6)
    n = 1_000_000
    g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05),
                bb.AmclParams(min_particles=n, max_particles=n, resample_scheme=bb.RESAMPLE_SYSTEMATIC, record_ancestors=True, seed=3))
    g.update_map(0, bb.LikelihoodFieldModelParam(max_obstacle_distance=2.0, max_laser_distance=100.0), bb.OccupancyGrid(sc.cells, sc.resolution))
    g.initialize(sc.initial_mean, sc.initial_cov)
    for k in range(6):
        r = g.update(bb.se2(*sc.poses[k]), sc.scans[k])
        assert r.updated == 1 and r.resampled == 1 and r.n_particles == n
        anc = g.filter.ancestors()
        assert np.all(np.diff(anc) >= 0) and anc.min() >= 0 and anc.max() < n
    st, w = g.particles()
    assert np.all(w == 1.0)
    assert np.abs(np.hypot(st[:, 0], st[:, 1]) - 1.0).max() < 1e-14
    assert np.hypot(r.estimate.mean[2] - sc.poses[5][0], r.estimate.mean[3] - sc.poses[5][1]) < 0.5  # posterior sigma ~0.3 m (1 + sum pz^3 is a weak likelihood)


def test_estimate_of_a_fresh_filter_is_its_own(bb, scene):
    """The host polls a completion ticket in the filter's pinned summary block.  Pinned allocations are recycled with their
    old contents: a new filter must not take a destroyed filter's last ticket (and its estimate) for its own first step."""
    lfm = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
    for shift in (0.0, 3.0, -2.5, 1.0):
        g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=5000, max_particles=5000, resample_scheme=1, seed=3))
        g.update_map(0, bb.LikelihoodFieldModelParam(**lfm), bb.OccupancyGrid(scene.cells, scene.resolution))
        mean = np.array(scene.initial_mean, dtype=float)
        mean[0] += shift
        g.initialize(mean, scene.initial_cov * 0.01)
        r = g.update(bb.se2(*scene.poses[0]), scene.scans[0])
        assert r.updated == 1 and r.resampled == 1
        assert abs(r.estimate.mean[2] - mean[0]) < 0.3 and abs(r.estimate.mean[3] - mean[1]) < 0.3
        del g
