"""The batch of filters on the GPU: every member equals a standalone Amcl built from the same parameters and fed the same
inputs, bit for bit (update results and particles), across particle counts from 1 to 32 768, all three motion models, both
resampling schemes, recovery injection, normalising steps between resampling ones, scans of 0 to 4097 points (1 to 3
shared-memory chunks), members that skip steps, steps below update_min_d, both likelihood-field models and maps on both
sides of kFixedMaxSide.  Also: the oracle over a trajectory, cluster estimates, the launch count, atomicity and tracking."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
SIZES = (1, 33, 256, 2000, 5000, 32768, 2000, 33, 5000)
POINT_COUNTS = (0, 1, 180, 1080, 4097)


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


def member_params(bb, k):
    n = SIZES[k]
    p = bb.AmclParams(min_particles=n, max_particles=n, seed=100 + k, resample_scheme=k % 2, record_ancestors=True)
    if k == 3:
        p.recovery_probability_override = 0.05
    if k in (4, 7):
        p.resample_interval = 3  # normalising and resampling steps alternate
    return p


def result_bytes(r):
    return struct.pack("<iiQ13ddd i", r.updated, r.resampled, r.n_particles, *r.estimate.mean, *r.estimate.cov, r.random_state_probability,
                       r.weight_sum, r.weights_degenerate)


def scan(scene, t, count):
    return np.resize(scene.scans[t], (count, 2)) if count else np.zeros((0, 2))


def odometry(scene, t, k):
    """Member k's control: the scene's pose, a little shifted per member; every fifth step repeats the last pose (below
    update_min_d: only a forced update runs)."""
    x, y, th = scene.poses[t - 1 if t % 5 == 4 else t]
    th = th + 0.01 * k
    return np.array([np.cos(th), np.sin(th), x + 0.02 * k, y])


@pytest.mark.parametrize("prob", [False, True])
@pytest.mark.parametrize("wide", [False, True])
def test_members_equal_standalone_filters(bb, scene, prob, wide):
    cells = scene.cells
    if wide:  # wider than kFixedMaxSide: the general lookup kernel with the tiled table
        cells = np.pad(cells, ((0, 0), (0, 8100 - cells.shape[1])), constant_values=0)
    grid = bb.OccupancyGrid(cells, scene.resolution)
    k = len(SIZES)
    params = [member_params(bb, m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid, prob=prob)
    twins = []
    for m in range(k):
        a = bb.Amcl(motions[m], params[m])
        a.update_map(bb.SENSOR_LIKELIHOOD_FIELD_PROB if prob else bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        twins.append(a)
    for m in range(k):
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        if m == 8:  # explicit states, fewer than max_particles
            rng = np.random.default_rng(m)
            th = rng.normal(mean[2], 0.2, 1000)
            st = np.stack([np.cos(th), np.sin(th), rng.normal(mean[0], 0.3, 1000), rng.normal(mean[1], 0.3, 1000)], axis=1)
            batch.initialize_states(m, st)
            twins[m].initialize_states(st)
        else:
            batch.initialize(m, mean, scene.initial_cov)
            twins[m].initialize(mean, scene.initial_cov)
    resampled = normalised = skipped = 0
    for t in range(12):
        present = [(t + m) % 4 != 3 for m in range(k)]
        poses = [odometry(scene, t, m) for m in range(k)]
        pts = [scan(scene, t, POINT_COUNTS[(t + m) % len(POINT_COUNTS)]) for m in range(k)]
        got = batch.update(poses, pts, present)
        for m in range(k):
            if not present[m]:
                assert got[m].updated == 0
                continue
            exp = twins[m].update(poses[m], pts[m])
            assert result_bytes(got[m]) == result_bytes(exp), (t, m)
            if exp.updated:
                resampled += exp.resampled
                normalised += 1 - exp.resampled
                gs, gw = batch.particles(m)
                ts, tw = twins[m].particles()
                n = len(ts)
                assert gs[:n].tobytes() == ts.tobytes() and gw[:n].tobytes() == tw.tobytes(), (t, m)
                if exp.resampled:
                    assert np.array_equal(batch.ancestors(m), twins[m].filter.ancestors()), (t, m)
            else:
                skipped += 1
    assert resampled > 0 and normalised > 0 and skipped > 0
    for m in range(k):  # the cluster estimate of each member equals its twin's
        gm, gc = batch.cluster_estimate(m)
        tm, tc = twins[m].filter.cluster_estimate()
        assert gm.tobytes() == tm.tobytes() and gc.tobytes() == tc.tobytes(), m


def test_oracle_anchor(bb, orc, scene):
    """Two members against oracle::Amcl over the synthetic trajectory: resample indices bit-exact, estimates within 1e-9."""
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    params = [bb.AmclParams(min_particles=3000, max_particles=3000, resample_scheme=1, seed=8, record_ancestors=True),
              bb.AmclParams(min_particles=2000, max_particles=2000, resample_scheme=0, seed=9, record_ancestors=True)]
    batch = bb.AmclBatch([bb.OmnidirectionalDriveModelParam(*ALPHAS), bb.DifferentialDriveModelParam(*ALPHAS[:4])], params)
    batch.set_likelihood_field_map(lfm, bb.OccupancyGrid(scene.cells, scene.resolution))
    oracles = [orc.Amcl(orc.AmclParam(min_particles=3000, max_particles=3000, scheme=1, seed=8, rng_mode=1), orc.OmniParam(*ALPHAS),
                        motion_model=orc.OMNIDIRECTIONAL),
               orc.Amcl(orc.AmclParam(min_particles=2000, max_particles=2000, scheme=0, seed=9, rng_mode=1), orc.MotionParam(*ALPHAS[:4]))]
    for m, o in enumerate(oracles):
        o.set_map(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
        o.initialize_normal(scene.initial_mean, scene.initial_cov)
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(8):
        pose = orc.se2(*scene.poses[t])
        got = batch.update([pose, pose], [scene.scans[t], scene.scans[t]])
        for m, o in enumerate(oracles):
            ro = o.update(pose, scene.scans[t])
            assert got[m].updated == ro.updated == 1
            assert np.array_equal(batch.ancestors(m), o.last_indices()), (t, m)
            assert np.abs(np.array(got[m].estimate.mean) - np.array(ro.mean)).max() < 1e-9


def test_launch_count_does_not_depend_on_the_member_count(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    counts = []
    for k in (1, 16, 256):
        params = [bb.AmclParams(min_particles=500, max_particles=500, seed=m, resample_scheme=1) for m in range(k)]
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam() for _ in range(k)], params)
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(k):
            batch.initialize(m, scene.initial_mean, scene.initial_cov)
        before = batch.launch_count()
        res = batch.update([bb.se2(*scene.poses[0])] * k, [scene.scans[0]] * k)
        assert all(r.updated for r in res)
        counts.append(batch.launch_count() - before)
    assert counts[0] == counts[1] == counts[2] == 5


def test_failed_update_is_rolled_back(bb, scene):
    """An update before any map is set fails; after setting the map, a retry gives what a batch that never failed gives."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=3 + n, resample_interval=2) for n in (300, 700)]

    def make(with_map):
        b = bb.AmclBatch([bb.DifferentialDriveModelParam(), bb.StationaryModelParam()], params)
        if with_map:
            b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(2):
            b.initialize(m, scene.initial_mean, scene.initial_cov)
        return b

    failed, clean = make(False), make(True)
    poses = [bb.se2(*scene.poses[0])] * 2
    with pytest.raises(bb.BelugaB200Error) as e:
        failed.update(poses, [scene.scans[0]] * 2)
    assert e.value.status == -4  # BB200_ERR_STATE
    failed.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
    for t in range(4):
        poses = [bb.se2(*scene.poses[t])] * 2
        a, b = failed.update(poses, [scene.scans[t]] * 2), clean.update(poses, [scene.scans[t]] * 2)
        assert [result_bytes(r) for r in a] == [result_bytes(r) for r in b]
        for m in range(2):
            assert failed.particles(m)[0].tobytes() == clean.particles(m)[0].tobytes()


def test_every_member_tracks(bb):
    """64 members, each on its own synthetic scene (the scene's noise seed), follow their ground truth."""
    from beluga_b200 import synthetic

    k = 64
    scenes = [synthetic.make_scenario(grid_size=300, n_beams=100, steps=30, noise_seed=11 + m) for m in range(k)]
    params = [bb.AmclParams(min_particles=2000, max_particles=2000, seed=m, resample_scheme=1) for m in range(k)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05) for _ in range(k)], params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scenes[0].cells, scenes[0].resolution))
    for m in range(k):
        batch.initialize(m, scenes[m].initial_mean, scenes[m].initial_cov)
    errors = np.zeros(k)
    for t in range(len(scenes[0].poses)):
        res = batch.update([bb.se2(*s.poses[t]) for s in scenes], [s.scans[t] for s in scenes])
        for m in range(k):
            if res[m].updated:
                errors[m] = np.hypot(res[m].estimate.mean[2] - scenes[m].poses[t][0], res[m].estimate.mean[3] - scenes[m].poses[t][1])
    assert errors.max() < 0.3, errors
