"""The point-cloud input on the GPU: Amcl.update_point_cloud against update(pose, point_cloud_to_points(...)), and the reweight
kernels at cloud sizes against the CPU oracle.

A 64-ring lidar gives about 65k points per step.  Scans longer than 1920 points reach the likelihood-field kernels through
shared memory, 2048 points (one TMA bulk copy, one mbarrier phase) at a time; 2049, 4097, 65536 and 65537 points take 2, 3, 32
and 33 of those chunks, with a ragged last chunk except at 65536, and the libstdc++ groups of four run across every chunk
boundary.  The beam model at 4097 points and 390 000 particles needs two passes of its walk / mixture pair."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
MOTION = (0.1, 0.05, 0.1, 0.05)
# rings x azimuths of the synthetic clouds with these point counts
CLOUD_SHAPES = {2049: (3, 683), 4097: (17, 241), 65536: (64, 1024), 65537: (1, 65537)}


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=12)


def cloud_points(bb, scene, n_points, k=3):
    from beluga_b200 import synthetic

    rows, azimuths = CLOUD_SHAPES[n_points]
    pc = synthetic.make_point_cloud(scene, k, rows=rows, azimuths=azimuths)
    return bb.point_cloud_to_points(pc.data, pc.point_step, pc.x_offset, pc.datatype, pc.origin)


def se2_array(x, y, theta):
    c, s = np.cos(theta), np.sin(theta)
    n = np.hypot(c, s)
    return np.stack([c / n, s / n, x, y], axis=1)


def mixed_states(scene, n, seed, k=3):
    """Particle 0 at the true pose, the first half around it (posterior-like), the rest uniform over and around the map."""
    rng = np.random.default_rng(seed)
    extent = scene.cells.shape[0] * scene.resolution
    x0, y0, t0 = scene.poses[k]
    near = n // 2 + 1
    xs = np.concatenate([x0 + rng.normal(0.0, 0.05, near), rng.uniform(-1.0, extent + 1.0, n - near)])[:n]
    ys = np.concatenate([y0 + rng.normal(0.0, 0.05, near), rng.uniform(-1.0, extent + 1.0, n - near)])[:n]
    ts = np.concatenate([t0 + rng.normal(0.0, 0.02, near), rng.uniform(-math.pi, math.pi, n - near)])[:n]
    xs[0], ys[0], ts[0] = x0, y0, t0
    return se2_array(xs, ys, ts)


def gpu_weights(bb, sensor, params, scene, points, states):
    f = bb.Filter(capacity=len(states))
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    if sensor == bb.SENSOR_BEAM:
        f.set_beam_map(params, grid)
    else:
        f.set_likelihood_field_map(params, grid, prob=(sensor == bb.SENSOR_LIKELIHOOD_FIELD_PROB))
    f.set_particles(states)
    f.reweight(points)
    return f.particles()[1]


# ---- update_point_cloud is update on the converted points ------------------------------------------------
@pytest.mark.parametrize("coordinate_type", [np.float32, np.float64])
@pytest.mark.parametrize("sensor", [0, 1, 2])
def test_update_point_cloud_equals_update_with_points(bb, scene, sensor, coordinate_type):
    """Amcl::update(pose, point_cloud) (beluga_ros/src/amcl.cpp:67-81) == update(pose, converted points), step after step."""
    from beluga_b200 import synthetic

    n = 2000
    params = bb.BeamModelParam(beam_max_range=20.0) if sensor == bb.SENSOR_BEAM else bb.LikelihoodFieldModelParam(**LFM)
    mk = lambda: bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=n, max_particles=n, seed=4))  # noqa: E731
    a, b = mk(), mk()
    for f in (a, b):
        f.update_map(sensor, params, bb.OccupancyGrid(scene.cells, scene.resolution))
        f.initialize(scene.initial_mean, scene.initial_cov)
    for k in range(3):
        pc = synthetic.make_point_cloud(scene, k, rows=4, azimuths=128, coordinate_type=coordinate_type)
        pose = bb.se2(*scene.poses[k])
        ra = a.update_point_cloud(pose, pc.data, pc.point_step, pc.x_offset, pc.datatype, origin=pc.origin)
        rb = b.update(pose, bb.point_cloud_to_points(pc.data, pc.point_step, pc.x_offset, pc.datatype, pc.origin))
        assert ra.updated == rb.updated == 1 and ra.resampled == rb.resampled
        assert np.array_equal(np.array(ra.estimate.mean), np.array(rb.estimate.mean))
        assert np.array_equal(np.array(ra.estimate.cov), np.array(rb.estimate.cov))
        sa, wa = a.particles()
        sb, wb = b.particles()
        assert np.array_equal(sa, sb) and np.array_equal(wa, wb)
    with pytest.raises(bb.BelugaB200Error) as e:
        a.update_point_cloud(bb.se2(*scene.poses[5]), pc.data, pc.point_step, pc.x_offset, 5)  # PointField INT32
    assert e.value.status == -1


# ---- the reweight kernels at cloud sizes ---------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 33, 257, 10_000])
@pytest.mark.parametrize("n_points", [2049, 4097, 65536, 65537])
@pytest.mark.parametrize("source", ["uniform", "cloud"])
@pytest.mark.parametrize("sensor", [0, 1])
def test_reweight_lfm_at_cloud_sizes(bb, orc, scene, sensor, source, n_points, n):
    """One to 33 shared-memory chunks with ragged tails, particle counts around the 32-particle task size and 10 000 on the
    200^2 scene.  The likelihood field (sum of cubes) is bit-exact.  The prob model sums the logs in the same order, bit-exact,
    and ends with one exp() per particle, which differs by an ulp or so between CUDA and glibc: compared at 1e-15, which a
    difference in the order of the sum (an ulp of a sum of hundreds of logs) would exceed."""
    rng = np.random.default_rng(1000 * n + n_points + 7 * sensor)
    states = mixed_states(scene, n, seed=n_points + n)
    pts = rng.uniform(-6.0, 6.0, (n_points, 2)) if source == "uniform" else cloud_points(bb, scene, n_points)
    got = gpu_weights(bb, sensor, bb.LikelihoodFieldModelParam(**LFM), scene, pts, states)
    exp = orc.sensor_weights(sensor, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution), pts, states)
    if sensor == 0:
        assert np.array_equal(got, exp)
        return
    normal = exp > 1e-290
    assert np.array_equal(got[exp == 0.0], exp[exp == 0.0])
    assert np.allclose(got[normal], exp[normal], rtol=1e-15, atol=0.0)
    assert np.allclose(got[~normal], exp[~normal], rtol=1e-6, atol=1e-320)
    if source == "cloud" and n_points <= 4097:
        assert normal[0]  # the particle at the true pose keeps a weight that the comparison above sees


def test_reweight_beam_two_passes_at_cloud_size(bb, orc, scene):
    """4097 points: the walk / mixture pair runs over the particles in passes of 196 544 (3 GiB of hit words), so 390 000
    particles take two passes, two launches more than the single pass that 2049 points need.  A sample of 1500 particles from
    both passes is compared with the oracle at rtol 1e-11 (erf/exp per beam differ by ulps between CUDA and glibc)."""
    n = 390_000
    states = mixed_states(scene, n, seed=41)
    params = dict(beam_max_range=20.0)
    pts = cloud_points(bb, scene, 4097)
    f = bb.Filter(capacity=n)
    f.set_beam_map(bb.BeamModelParam(**params), bb.OccupancyGrid(scene.cells, scene.resolution))
    f.set_particles(states)
    before = f.launch_count()
    f.reweight(cloud_points(bb, scene, 2049))
    one_pass = f.launch_count() - before
    f.set_particles(states)
    before = f.launch_count()
    f.reweight(pts)
    assert f.launch_count() - before == one_pass + 2
    got = f.particles()[1]
    sample = np.random.default_rng(5).choice(n, 1500, replace=False)
    sample[0] = 0  # the particle at the true pose
    exp = orc.sensor_weights(orc.BEAM, orc.BeamParam(**params), orc.Grid(scene.cells, scene.resolution), pts, states[sample])
    assert np.allclose(got[sample], exp, rtol=1e-11, atol=1e-300)
    assert exp[0] > 0.0


# ---- a whole trajectory on synthetic clouds --------------------------------------------------------------
def test_trajectory_on_synthetic_clouds(bb, orc, scene):
    """Amcl driven by 16 x 256 lidar clouds along the closed path, next to oracle::Amcl fed the converted points: the same
    resample indices and estimates, and the filter tracks the ground truth within test_large_scale_properties' 0.5 m."""
    from beluga_b200 import synthetic

    n = 10_000
    ap = dict(min_particles=n, max_particles=n, seed=17)
    g = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(resample_scheme=1, record_ancestors=True, **ap))
    o = orc.Amcl(orc.AmclParam(rng_mode=1, scheme=1, **ap), orc.MotionParam(*MOTION))
    g.update_map(0, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    o.set_map(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
    g.initialize(scene.initial_mean, scene.initial_cov)
    o.initialize_normal(scene.initial_mean, scene.initial_cov)
    steps = len(scene.poses) - 1
    for k in range(steps):
        pc = synthetic.make_point_cloud(scene, k, rows=16, azimuths=256)
        pose = bb.se2(*scene.poses[k])
        rg = g.update_point_cloud(pose, pc.data, pc.point_step, pc.x_offset, pc.datatype, origin=pc.origin)
        ro = o.update(pose, bb.point_cloud_to_points(pc.data, pc.point_step, pc.x_offset, pc.datatype, pc.origin))
        assert rg.updated == ro.updated == 1 and rg.resampled == ro.resampled == 1
        assert np.array_equal(g.filter.ancestors(), o.last_indices())
        assert np.abs(np.array(rg.estimate.mean) - np.array(ro.mean)).max() < 1e-10
        assert np.abs(np.array(rg.estimate.cov) - np.array(ro.cov)).max() < 1e-10
    mean = np.array(rg.estimate.mean)
    assert np.hypot(mean[2] - scene.poses[steps - 1][0], mean[3] - scene.poses[steps - 1][1]) < 0.5
