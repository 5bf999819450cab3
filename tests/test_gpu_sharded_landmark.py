"""The landmark and bearing models on a sharded filter (bb200_sharded_amcl_set_landmark_map / _set_bearing_map /
_update_landmarks, ShardedAmcl.update_map and .update_landmarks), with all shards on ONE device as in
tests/test_gpu_sharded_publish.py.  Every case runs twins: the sharded filter and a single Amcl with the same parameters, seed,
map and detections.  Particles and weights are compared byte for byte after every step, the update results by their
decisions, counts and normalisation factor bit for bit (same_step) and the estimate to rounding: it sums the same terms
grouped per shard.  A refused call must leave every shard's particles and policies as they were, which the twins show by
still comparing equal on the steps after it."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_sharded_local import MODES  # noqa: E402
from test_gpu_sharded_publish import same_bytes, same_particles, same_step  # noqa: E402

pytestmark = pytest.mark.gpu

MOTION = (0.1, 0.05, 0.1, 0.05)
INVALID, STATE = -1, -4
N = 12_000  # divisible by 2, 3, 4 and 8
SHARDS = [2, 3, 4, 8]
MODELS = ["landmark", "bearing"]
SENSOR_POSE = (0.0, 0.0, 1.0, 0.2, -1.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.5)  # a camera looking along the robot's x
STEPS = 6
EMPTY_STEP = 3  # the step without detections
ABSENT_STEP = 1  # the step with a detection of a category the map lacks (the bearing model weighs it 0: a degenerate step)


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


# ---- maps and detections ------------------------------------------------------------------------------------------------
def fiducial_map(bb):
    """24 landmarks in 6 categories, explicit bounds."""
    rng = np.random.default_rng(5)
    pos = np.stack([rng.uniform(-6, 6, 24), rng.uniform(-5, 5, 24), rng.uniform(0.0, 2.0, 24)], axis=1)
    return bb.LandmarkMap(pos, np.arange(24, dtype=np.uint32) % 6, [-8.0, -7.0, 0.0], [8.0, 7.0, 2.0])


def reflector_map(bb, n=600):
    """n landmarks of one category (more than 256: several candidate chunks per detection), the landmarks' own bounds."""
    rng = np.random.default_rng(6)
    pos = np.stack([rng.uniform(-10, 10, n), rng.uniform(-10, 10, n), np.zeros(n)], axis=1)
    return bb.LandmarkMap(pos, np.zeros(n, dtype=np.uint32))


MAPS = {"fiducial": (fiducial_map, 6), "reflector": (reflector_map, 1)}


def detections(kind, k):
    """Step k's detections on a map of `kind`, cycling through its categories; at ABSENT_STEP the last one is of a category
    the map lacks, at EMPTY_STEP there are none."""
    n_categories = MAPS[kind][1]
    if k == EMPTY_STEP:
        return np.zeros((0, 3)), np.zeros(0, dtype=np.uint32)
    rng = np.random.default_rng(100 + k)
    n = 8 if kind == "fiducial" else 16
    pos = np.stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(0.0, 2.0, n)], axis=1)
    cat = (np.arange(n) % n_categories).astype(np.uint32)
    if k == ABSENT_STEP:
        cat[-1] = 9
    return pos, cat


def model_params(bb, model):
    if model == "landmark":
        return bb.SENSOR_LANDMARK, bb.LandmarkModelParam(0.5, 0.3, 1e-3)
    return bb.SENSOR_BEARING, bb.BearingModelParam(0.3, SENSOR_POSE)


def control(bb, k):
    th = 0.1 * (k + 1)
    return np.array([math.cos(th), math.sin(th), 0.3 * (k + 1), 0.1 * k])


def make_twins(bb, model, kind, shards, n=N, init="normal", devices=None, **kw):
    """(sharded filter, single Amcl) with the same parameters, seed, map and initial particles."""
    ap = dict(min_particles=n, max_particles=n, seed=41, update_min_d=0.0, update_min_a=0.0)
    ap.update(kw)
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap), devices=devices or [0] * shards)
    sensor, params = model_params(bb, model)
    lmap = MAPS[kind][0](bb)
    for f in (single, group):
        f.update_map(sensor, params, lmap)
        if init == "normal":
            f.initialize([0.5, -0.5, 0.3], np.diag([0.5, 0.5, 0.2]))
        else:
            f.initialize_from_map()
    assert same_particles(group, single)
    return group, single


def same_estimate(a, b):
    np.testing.assert_allclose(np.array(a.estimate.mean), np.array(b.estimate.mean), rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(np.array(a.estimate.cov), np.array(b.estimate.cov), rtol=1e-9, atol=1e-12)


def step_twins(bb, group, single, kind, k):
    det = detections(kind, k)
    pose = control(bb, k)
    rg, rs = group.update_landmarks(pose, *det), single.update_landmarks(pose, *det)
    assert same_step(rg, rs), k
    assert rg.weights_degenerate == rs.weights_degenerate
    if rg.updated:
        same_estimate(rg, rs)
    assert same_particles(group, single), k
    return rg


def run_twins(bb, group, single, kind, steps=STEPS, first=0):
    return [step_twins(bb, group, single, kind, k) for k in range(first, first + steps)]


# ---- steps ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("init", ["normal", "map"])
@pytest.mark.parametrize("shards", SHARDS)
@pytest.mark.parametrize("kind", sorted(MAPS))
@pytest.mark.parametrize("model", MODELS)
def test_steps_follow_the_single_filter(bb, model, kind, shards, init):
    group, single = make_twins(bb, model, kind, shards, init=init, resample_scheme=1)
    results = run_twins(bb, group, single, kind)
    assert all(r.updated == 1 and r.resampled == 1 for r in results)


@pytest.mark.parametrize("shards", [2, 3, 8])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("model", MODELS)
def test_resampling_modes(bb, model, mode, shards):
    """Systematic and multinomial resampling, recovery injection from the box, every_n and selective resampling."""
    group, single = make_twins(bb, model, "fiducial", shards, **MODES[mode])
    run_twins(bb, group, single, "fiducial")


@pytest.mark.parametrize("model", MODELS)
def test_injection_draws_the_box(bb, model):
    """recovery_probability_override = 1: every slot but the first takes a state of the map's box."""
    group, single = make_twins(bb, model, "fiducial", 4, recovery_probability_override=1.0, resample_scheme=0)
    r = step_twins(bb, group, single, "fiducial", 0)
    assert r.resampled == 1
    st = group.particles()[0]
    inside = (st[1:, 2] >= -8.0) & (st[1:, 2] <= 8.0) & (st[1:, 3] >= -7.0) & (st[1:, 3] <= 7.0)
    assert inside.all() and np.unique(st[1:, 2]).size == N - 1


@pytest.mark.parametrize("shards,scheme", [(2, 1), (3, 0), (4, 1)])
@pytest.mark.parametrize("model", MODELS)
def test_kld(bb, model, shards, scheme):
    group, single = make_twins(bb, model, "reflector", shards, n=4000 * shards, init="map", min_particles=300, resample_scheme=scheme)
    run_twins(bb, group, single, "reflector")


def test_kld_with_an_empty_shard(bb):
    """take_while_kld settles on 41 particles: 6 on each of the first six shards, 5 on the seventh, none on the last, which
    then steps with no particles."""
    group, single = make_twins(bb, "landmark", "fiducial", 8, n=8 * 1000, min_particles=41, resample_scheme=1, seed=31, kld_epsilon=1.0)
    sizes = []
    for k in range(4):
        step_twins(bb, group, single, "fiducial", k)
        sizes.append([f.size() for f in group.shards])
    assert any(s[-1] == 0 and sum(s) > 0 for s in sizes), sizes


def test_bearing_pose_is_not_the_identity(bb):
    """The bearing model's sensor pose takes part in the weights: the same filter with the identity pose differs."""
    group, single = make_twins(bb, "bearing", "fiducial", 2, resample_scheme=1)
    other = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=N, max_particles=N, seed=41, update_min_d=0.0,
                                                                                  update_min_a=0.0, resample_scheme=1), devices=[0, 0])
    other.update_map(bb.SENSOR_BEARING, bb.BearingModelParam(0.3), fiducial_map(bb))
    other.initialize([0.5, -0.5, 0.3], np.diag([0.5, 0.5, 0.2]))
    step_twins(bb, group, single, "fiducial", 0)
    other.update_landmarks(control(bb, 0), *detections("fiducial", 0))
    assert not same_particles(group, other)


# ---- publishing and weighed steps ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shards", [3, 8])
@pytest.mark.parametrize("model", MODELS)
def test_publishing_on_a_landmark_map(bb, model, shards):
    """cluster_estimate, particle_histogram and sample_states after a resampling step (unit weights) and after one that
    keeps its particles (resample_interval = 2)."""
    group, single = make_twins(bb, model, "fiducial", shards, init="map", resample_interval=2, resample_scheme=1)
    for k in range(2):
        step_twins(bb, group, single, "fiducial", k)
        for kw in (dict(), dict(linear=0.5, angular=0.3, percentile=0.5)):
            ms, cs, _, cells_s, clusters_s = single.filter.cluster_estimate(with_ids=True, **kw)
            mg, cg, cells_g, clusters_g = group.cluster_estimate(**kw)
            assert (cells_g, clusters_g) == (cells_s, clusters_s)
            np.testing.assert_allclose(mg, ms, rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(cg, cs, rtol=1e-9, atol=1e-12)
        hg, hs = group.particle_histogram(0.5, 0.3), single.filter.particle_histogram(0.5, 0.3)
        for name, a, b in zip(("rep", "weight", "count", "first"), hg[:4], hs[:4]):
            if name == "weight" and k == 0:
                np.testing.assert_allclose(a, b, rtol=1e-12, atol=0)  # a cell that spans shards adds its weights per shard
            else:
                assert same_bytes(a, b), (k, name)
        for count, stp in ((1, 0), (500, 7), (N, 3)):
            assert same_bytes(group.sample_states(count, step=stp), single.filter.sample_states(count, step=stp)), (k, count)


@pytest.mark.parametrize("model", MODELS)
def test_weighed_step_with_all_ones(bb, model):
    """A weighed step with factors 1 on a landmark map equals the single filter's; the landmark steps after it too."""
    pytest.importorskip("torch")
    group, single = make_twins(bb, model, "fiducial", 4, resample_scheme=1)
    run_twins(bb, group, single, "fiducial", steps=2)
    pose = control(bb, 2)
    rg = group.update_weighted(pose, lambda s, f: f.fill_(1.0))
    rs = single.update_weighted(pose, lambda s, f: f.fill_(1.0))
    assert rg.updated == 1 and same_step(rg, rs)
    same_estimate(rg, rs)
    assert same_particles(group, single)
    run_twins(bb, group, single, "fiducial", steps=2, first=3)


# ---- refusals --------------------------------------------------------------------------------------------------------------
def refused(bb, call, status):
    with pytest.raises(bb.BelugaB200Error) as e:
        call()
    assert e.value.status == status
    return str(e.value)


def launches(group):
    return [f.launch_count() for f in group.shards]


def test_update_landmarks_on_a_grid_map(bb):
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=100, n_beams=60, steps=4)
    ap = dict(min_particles=N, max_particles=N, seed=41, resample_scheme=1)
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap), devices=[0] * 3)
    for f in (single, group):
        f.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(), bb.OccupancyGrid(sc.cells, sc.resolution))
        f.initialize(sc.initial_mean, sc.initial_cov)
    before = launches(group)
    refused(bb, lambda: group.update_landmarks(bb.se2(*sc.poses[0]), *detections("fiducial", 0)), STATE)
    assert launches(group) == before and same_particles(group, single)
    for k in range(3):
        pose = bb.se2(*sc.poses[k])
        rg, rs = group.update(pose, sc.scans[k]), single.update(pose, sc.scans[k])
        assert same_step(rg, rs) and same_particles(group, single)


@pytest.mark.parametrize("model", MODELS)
def test_grid_calls_on_a_landmark_map(bb, model):
    """Point, scan and cloud steps and ray casts on a landmark map: BB200_ERR_STATE, nothing launched, nothing moved."""
    group, single = make_twins(bb, model, "fiducial", 4, resample_scheme=0)
    step_twins(bb, group, single, "fiducial", 0)
    before = launches(group)
    pose = control(bb, 1)
    ranges = np.full(30, 2.0, dtype=np.float32)
    cloud = np.ones((10, 3), dtype=np.float32)
    refused(bb, lambda: group.update(pose, np.ones((10, 2))), STATE)
    refused(bb, lambda: group.update(pose, np.zeros((0, 2))), STATE)
    refused(bb, lambda: group.update_scan(pose, ranges, -1.0, 0.05), STATE)
    refused(bb, lambda: group.update_point_cloud(pose, cloud, 12, 0, np.float32), STATE)
    refused(bb, lambda: group.cast_rays(np.array([[1.0, 0.0, 0.0, 0.0]]), np.array([[1.0, 0.0]]), 5.0), STATE)
    assert launches(group) == before and same_particles(group, single)
    run_twins(bb, group, single, "fiducial", steps=3, first=1)


@pytest.mark.parametrize("model", MODELS)
def test_refused_maps_leave_every_shard_s_map(bb, model):
    """A bad sigma or a sensor pose that is not a rotation: the single filter's status and message, and every shard keeps
    the map it had."""
    group, single = make_twins(bb, model, "fiducial", 3, resample_scheme=1)
    step_twins(bb, group, single, "fiducial", 0)
    lmap = reflector_map(bb)
    bad = [(bb.SENSOR_LANDMARK, bb.LandmarkModelParam(0.0, 1.0, 0.1)),
           (bb.SENSOR_LANDMARK, bb.LandmarkModelParam(1.0, float("nan"), 0.1)),
           (bb.SENSOR_BEARING, bb.BearingModelParam(-1.0)),
           (bb.SENSOR_BEARING, bb.BearingModelParam(1.0, np.diag([1.0, 1.0, 1.0 + 1e-6, 0.0])[:3]))]
    other = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=16, max_particles=16))
    for sensor, params in bad:
        got = refused(bb, lambda: group.update_map(sensor, params, lmap), INVALID)
        assert got == refused(bb, lambda: other.update_map(sensor, params, lmap), INVALID)
    run_twins(bb, group, single, "fiducial", steps=3, first=1)


def test_too_many_detections_are_refused_before_reading_them(bb):
    """n >= 2^32 - 1 with a one-element array: refused before any detection is read or any buffer grows."""
    from beluga_b200 import _capi

    lib = _capi.load()
    group, single = make_twins(bb, "landmark", "fiducial", 2, resample_scheme=1)
    step_twins(bb, group, single, "fiducial", 0)
    before = launches(group)
    det = (_capi.Landmark * 1)()
    pose = np.ascontiguousarray(control(bb, 1))
    res = _capi.UpdateResult()
    for n in (2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1):
        assert lib.bb200_sharded_amcl_update_landmarks(group._h, pose.ctypes.data_as(C.POINTER(C.c_double)), det, n, C.byref(res)) == INVALID
        assert res.updated == 0
    assert lib.bb200_sharded_amcl_update_landmarks(group._h, pose.ctypes.data_as(C.POINTER(C.c_double)), None, 1, C.byref(res)) == INVALID
    assert launches(group) == before and same_particles(group, single)
    run_twins(bb, group, single, "fiducial", steps=2, first=1)


def test_new_calls_refused_while_a_weighed_step_is_open(bb):
    pytest.importorskip("torch")
    from beluga_b200 import _capi

    lib = _capi.load()
    group, single = make_twins(bb, "landmark", "fiducial", 3, resample_scheme=1)
    step_twins(bb, group, single, "fiducial", 0)
    lmap = fiducial_map(bb).c()
    lp, bp = bb.LandmarkModelParam(0.5, 0.3, 1e-3).c(), bb.BearingModelParam(0.3).c()
    det = (_capi.Landmark * 1)()
    pose = np.ascontiguousarray(control(bb, 1))
    res = _capi.UpdateResult()
    statuses = []

    def weigh(states, factors):
        statuses.append(lib.bb200_sharded_amcl_set_landmark_map(group._h, C.byref(lp), C.byref(lmap)))
        statuses.append(lib.bb200_sharded_amcl_set_bearing_map(group._h, C.byref(bp), C.byref(lmap)))
        statuses.append(lib.bb200_sharded_amcl_update_landmarks(group._h, pose.ctypes.data_as(C.POINTER(C.c_double)), det, 1, C.byref(res)))
        factors.fill_(1.0)

    rg = group.update_weighted(pose, weigh)
    rs = single.update_weighted(pose, lambda s, f: f.fill_(1.0))
    assert statuses == [STATE] * 9
    assert same_step(rg, rs) and same_particles(group, single)
    run_twins(bb, group, single, "fiducial", steps=2, first=2)


def test_skipped_step_launches_nothing(bb):
    """A step the policies skip (the robot has not moved) returns updated = 0 and launches nothing: the staging is a copy."""
    group, single = make_twins(bb, "bearing", "fiducial", 4, resample_scheme=1)
    step_twins(bb, group, single, "fiducial", 0)
    before = launches(group)
    det = detections("fiducial", 1)
    rg, rs = group.update_landmarks(control(bb, 0), *det), single.update_landmarks(control(bb, 0), *det)
    assert rg.updated == 0 and rs.updated == 0 and bytes(rg) == bytes(rs)
    assert launches(group) == before and same_particles(group, single)
    run_twins(bb, group, single, "fiducial", steps=2, first=1)


# ---- the bench shape, launch counts, two devices ------------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
def test_bench_shape(bb, model):
    """One step at 1M particles x 16 detections on the 1000-landmark reflector map over 8 shards."""
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=1 << 20, max_particles=1 << 20, seed=3, resample_scheme=1))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=1 << 20, max_particles=1 << 20, seed=3,
                                                                                  resample_scheme=1), devices=[0] * 8)
    sensor, params = model_params(bb, model)
    lmap = reflector_map(bb, 1000)
    for f in (single, group):
        f.update_map(sensor, params, lmap)
        f.initialize_from_map()
    det = detections("reflector", 0)
    rg, rs = group.update_landmarks(control(bb, 0), *det), single.update_landmarks(control(bb, 0), *det)
    assert rg.updated == 1 and rg.resampled == 1 and same_step(rg, rs)
    same_estimate(rg, rs)
    assert same_particles(group, single)


def lfm_twins(bb, sc, shards, **kw):
    ap = dict(min_particles=N, max_particles=N, seed=41, update_min_d=0.0, update_min_a=0.0, **kw)
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap), devices=[0] * shards)
    for f in (single, group):
        f.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(), bb.OccupancyGrid(sc.cells, sc.resolution))
        f.initialize(sc.initial_mean, sc.initial_cov)
    return group, single


@pytest.mark.parametrize("mode", ["systematic", "multinomial", "every-3"])
@pytest.mark.parametrize("model", MODELS)
def test_launch_count(bb, model, mode):
    """Per shard, a landmark step launches what the single filter's landmark step launches plus what sharding adds to a
    step, which the likelihood-field twins measure: the exchanges are the same whatever weighs the particles, and staging
    the detections launches nothing.  Below 32768 particles per filter no step builds a schedule."""
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=100, n_beams=60, steps=4)
    shards = 2
    group, single = make_twins(bb, model, "fiducial", shards, **MODES[mode])
    lfm_group, lfm_single = lfm_twins(bb, sc, shards, **MODES[mode])
    for k in range(4):
        lg, ls, fg, fs = launches(group), single.filter.launch_count(), launches(lfm_group), lfm_single.filter.launch_count()
        step_twins(bb, group, single, "fiducial", k)
        pose = control(bb, k)
        assert lfm_group.update(pose, sc.scans[k]).updated == 1
        lfm_single.update(pose, sc.scans[k])
        sharding = [x - y - (lfm_single.filter.launch_count() - fs) for x, y in zip(launches(lfm_group), fg)]
        landmark = [x - y for x, y in zip(launches(group), lg)]
        assert landmark == [single.filter.launch_count() - ls + s for s in sharding], (k, landmark, sharding)


@pytest.mark.parametrize("model", MODELS)
def test_two_devices(bb, model):
    if bb.device_count() < 2:
        pytest.skip("one GPU: the two-device case needs two")
    group, single = make_twins(bb, model, "reflector", 2, devices=[0, 1], resample_scheme=1)
    run_twins(bb, group, single, "reflector", steps=4)
