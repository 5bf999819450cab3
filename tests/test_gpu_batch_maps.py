"""Several maps in one batch on the GPU: members that read different maps -- likelihood field, its prob variant on a grid
the fixed-point kernel does not take, a beam map the two-pass walk takes and one it does not -- each equal a standalone
Amcl on their own map fed the same inputs, byte for byte (update results, particles, weights, ancestors and the cluster
estimates that follow).  Also: update_map in the middle of a trajectory (recovery injection then draws from the new
map's free cells), initialize_from_map on each member's own map, the launch count of every mix of reweight forms and
its independence of K, set_*_map after add_*_map, the refusals of bad ids, maps in use and null arguments, rollback,
and likelihood_field(id)."""
import ctypes as C
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
SIZES = (1, 33, 256, 2000, 5000, 32768, 2000, 33, 700)
POINT_COUNTS = (0, 1, 60, 1025, 2049)
STATE, INVALID = -4, -1


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


def make_maps(bb, scene):
    """(sensor, params, grid) of the four map kinds: the likelihood field; its prob variant on a grid wider than
    kFixedMaxSide (the general kernel); the beam model on the scene (two-pass walk); the beam model on the scene padded to
    70 000 cells wide (no padded free-distance copy: the fused kernel)."""
    cells, res = scene.cells, scene.resolution
    wide_lfm = np.pad(cells, ((0, 0), (0, 8200 - cells.shape[1])), constant_values=0)
    wide_beam = np.pad(cells, ((0, 0), (0, 70_000 - cells.shape[1])), constant_values=0)
    beam = bb.BeamModelParam(beam_max_range=20.0)
    return [(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(cells, res)),
            (bb.SENSOR_LIKELIHOOD_FIELD_PROB, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(wide_lfm, res)),
            (bb.SENSOR_BEAM, beam, bb.OccupancyGrid(cells, res)),
            (bb.SENSOR_BEAM, beam, bb.OccupancyGrid(wide_beam, res))]


def add_map(bb, batch, sensor, params, grid):
    if sensor == bb.SENSOR_BEAM:
        return batch.add_beam_map(params, grid)
    return batch.add_likelihood_field_map(params, grid, prob=sensor == bb.SENSOR_LIKELIHOOD_FIELD_PROB)


def motion(bb, k):
    return [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.OmnidirectionalDriveModelParam(*ALPHAS), bb.StationaryModelParam()][k % 3]


def member_params(bb, k):
    n = SIZES[k]
    p = bb.AmclParams(min_particles=n, max_particles=n, seed=300 + k, resample_scheme=k % 2, record_ancestors=True)
    if k in (3, 6):
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


def odometry(scene, t, m):
    """Member m's control: the scene's pose, a little shifted per member; every fifth step repeats the last pose (below
    update_min_d: only a forced update runs)."""
    x, y, th = scene.poses[t - 1 if t % 5 == 4 else t]
    th = th + 0.01 * m
    return np.array([np.cos(th), np.sin(th), x + 0.02 * m, y])


def scan(scene, t, count):
    return np.resize(scene.scans[t], (count, 2)) if count else np.zeros((0, 2))


def expected_launches(forms):
    """4 + 1 (likelihood field) + 2 (two-pass beam) + 1 (fused beam) for the forms present."""
    return 4 + (1 if "field" in forms else 0) + (2 if "walk" in forms else 0) + (1 if "fused" in forms else 0)


FORM_OF_MAP = ("field", "field", "walk", "fused")


def test_members_on_four_maps_equal_standalone_twins(bb, scene):
    maps = make_maps(bb, scene)
    k = len(SIZES)
    params = [member_params(bb, m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    ids = [add_map(bb, batch, *mp) for mp in maps]
    assert ids == [0, 1, 2, 3]
    twins = []
    for m in range(k):
        batch.update_map(m, ids[m % 4])
        assert batch.member_map(m) == ids[m % 4]
        a = bb.Amcl(motions[m], params[m])
        a.update_map(*maps[m % 4])
        twins.append(a)
    for m in range(k):
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        if m == 7:  # explicit states, fewer than max_particles
            rng = np.random.default_rng(m)
            th = rng.normal(mean[2], 0.2, 20)
            st = np.stack([np.cos(th), np.sin(th), rng.normal(mean[0], 0.3, 20), rng.normal(mean[1], 0.3, 20)], axis=1)
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
        before = batch.launch_count()
        got = batch.update(poses, pts, present)
        forms = {FORM_OF_MAP[m % 4] for m in range(k) if got[m].updated}
        assert batch.launch_count() - before == (expected_launches(forms) if forms else 0), t
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
    present = [m % 2 == 0 for m in range(k)]
    for m, e in enumerate(batch.cluster_estimates(present)):
        if present[m]:
            tm, tc = twins[m].filter.cluster_estimate()
            assert e[0].tobytes() == tm.tobytes() and e[1].tobytes() == tc.tobytes(), m


def test_update_map_mid_trajectory(bb, scene):
    """Member 0 moves from map A to map B at step 3 and keeps its particles; its recovery injection then draws from B's
    free cells (B is the scene with 150 free columns added).  Member 1 stays on A, member 2 reads B throughout."""
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid_a = bb.OccupancyGrid(scene.cells, scene.resolution)
    grid_b = bb.OccupancyGrid(np.pad(scene.cells, ((0, 0), (0, 150)), constant_values=0), scene.resolution)
    k = 3
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=40 + n, resample_scheme=n % 2, record_ancestors=True,
                            recovery_probability_override=0.3) for n in (2000, 700, 1500)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    a, b = batch.add_likelihood_field_map(lfm, grid_a), batch.add_likelihood_field_map(lfm, grid_b)
    start = [a, a, b]
    twins = []
    for m in range(k):
        batch.update_map(m, start[m])
        tw = bb.Amcl(motions[m], params[m])
        tw.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid_a if start[m] == a else grid_b)
        twins.append(tw)
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
        twins[m].initialize(scene.initial_mean, scene.initial_cov)
    injected_on_b = False
    for t in range(8):
        if t == 3:
            batch.update_map(0, b)
            twins[0].update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, grid_b)
            assert batch.member_map(0) == b
        pose = bb.se2(*scene.poses[t])
        for m in range(k):
            batch.force_update(m)
            twins[m].force_update()
        got = batch.update([pose] * k, [scene.scans[t]] * k)
        for m in range(k):
            exp = twins[m].update(pose, scene.scans[t])
            assert exp.updated
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))
            if m == 0 and t >= 3 and exp.resampled and exp.random_state_probability > 0.0:
                injected_on_b = True
    assert injected_on_b
    assert_cluster_estimates_equal(batch, twins)


def test_initialize_from_map_samples_each_members_map(bb, scene):
    maps = make_maps(bb, scene)[:3]
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=n, resample_scheme=1, record_ancestors=True) for n in (1000, 3000, 1500)]
    motions = [bb.DifferentialDriveModelParam(*ALPHAS[:4]), bb.StationaryModelParam(), bb.DifferentialDriveModelParam(*ALPHAS[:4])]
    batch = bb.AmclBatch(motions, params)
    ids = [add_map(bb, batch, *mp) for mp in maps]
    twins = []
    for m in range(3):
        batch.update_map(m, ids[m])
        twins.append(bb.Amcl(motions[m], params[m]))
        twins[m].update_map(*maps[m])
        batch.initialize_from_map(m)
        twins[m].initialize_from_map()
        assert batch.particles(m)[0].tobytes() == twins[m].particles()[0].tobytes(), m
    assert batch.particles(1)[0][:, 2].max() > scene.cells.shape[1] * scene.resolution  # member 1 samples the wide map
    for t in range(3):
        pose = bb.se2(*scene.poses[t])
        got = batch.update([pose] * 3, [scene.scans[t]] * 3)
        for m in range(3):
            exp = twins[m].update(pose, scene.scans[t])
            assert_member_equals_twin(batch, m, twins[m], got[m], exp, (t, m))


@pytest.mark.parametrize("k", [1, 16, 256])
def test_launch_count_of_each_mix(bb, scene, k):
    """One map in use while the others exist: 5 (likelihood field) or 6 (two-pass beam) launches; for mixes of forms the
    documented count; none of them depends on K."""
    maps = make_maps(bb, scene)
    params = [bb.AmclParams(min_particles=500, max_particles=500, seed=m, resample_scheme=1) for m in range(k)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam() for _ in range(k)], params)
    ids = [add_map(bb, batch, *mp) for mp in maps]
    mixes = [(0,), (1,), (2,), (3,), (0, 1)]
    if k > 1:
        mixes += [(0, 3), (0, 2), (2, 3), (0, 2, 3), (1, 2, 3)]
    for mix in mixes:
        for m in range(k):
            batch.update_map(m, ids[mix[m % len(mix)]])
            batch.initialize(m, scene.initial_mean, scene.initial_cov)
        before = batch.launch_count()
        res = batch.update([bb.se2(*scene.poses[0])] * k, [scan(scene, 0, 60 + m % 7) for m in range(k)])
        assert all(r.updated for r in res)
        forms = {FORM_OF_MAP[i] for i in mix[:k]}
        assert batch.launch_count() - before == expected_launches(forms), mix
    assert expected_launches({"field"}) == 5 and expected_launches({"walk"}) == 6


def test_set_map_after_add_and_the_refusals(bb, scene):
    maps = make_maps(bb, scene)
    lfm_sensor, lfm, grid = maps[0]
    k = 3
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=7 + n, resample_interval=2, record_ancestors=True) for n in (300, 700, 1200)]
    motions = [motion(bb, m) for m in range(k)]

    def make(with_map):
        b = bb.AmclBatch(motions, params)
        if with_map:
            b.set_likelihood_field_map(lfm, grid)
        for m in range(k):
            b.initialize(m, scene.initial_mean, scene.initial_cov)
        return b

    failed, clean = make(False), make(True)
    ids = [add_map(bb, failed, *mp) for mp in maps[1:]]
    assert ids == [0, 1, 2]
    failed.update_map(0, ids[0])
    failed.update_map(1, ids[2])
    poses = [bb.se2(*scene.poses[0])] * k
    with pytest.raises(bb.BelugaB200Error) as e:  # member 2 has no map
        failed.update(poses, [scene.scans[0]] * k)
    assert e.value.status == STATE
    with pytest.raises(bb.BelugaB200Error) as e:
        failed.remove_map(ids[0])  # member 0 reads it
    assert e.value.status == STATE
    failed.remove_map(ids[1])
    for bad in (ids[1], 17, -1):
        with pytest.raises(bb.BelugaB200Error) as e:
            failed.update_map(0, bad)
        assert e.value.status == INVALID
        with pytest.raises(bb.BelugaB200Error) as e:
            failed.remove_map(bad)
        assert e.value.status == INVALID
        with pytest.raises(bb.BelugaB200Error) as e:
            failed.likelihood_field(bad)
        assert e.value.status == INVALID
    with pytest.raises(bb.BelugaB200Error) as e:
        failed.update_map(k, ids[0])
    assert e.value.status == INVALID
    assert [failed.member_map(m) for m in range(k)] == [ids[0], ids[2], -1]
    # every member back on one map: the new map takes the next id and the failed update left no trace
    failed.set_likelihood_field_map(lfm, grid)
    assert [failed.member_map(m) for m in range(k)] == [3] * k
    for bad in ids:
        with pytest.raises(bb.BelugaB200Error) as e:
            failed.update_map(0, bad)
        assert e.value.status == INVALID
    twins = [bb.Amcl(motions[m], params[m]) for m in range(k)]
    for m in range(k):
        twins[m].update_map(lfm_sensor, lfm, grid)
        twins[m].initialize(scene.initial_mean, scene.initial_cov)
    for t in range(4):
        poses = [bb.se2(*scene.poses[t])] * k
        before = failed.launch_count()
        a, b = failed.update(poses, [scene.scans[t]] * k), clean.update(poses, [scene.scans[t]] * k)
        assert failed.launch_count() - before == 5
        assert [result_bytes(r) for r in a] == [result_bytes(r) for r in b]
        for m in range(k):
            exp = twins[m].update(poses[m], scene.scans[t])
            assert_member_equals_twin(failed, m, twins[m], a[m], exp, (t, m))
            assert failed.particles(m)[0].tobytes() == clean.particles(m)[0].tobytes()


def test_likelihood_field_of_each_map(bb, scene):
    maps = make_maps(bb, scene)
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam()], [bb.AmclParams(min_particles=100, max_particles=100)])
    ids = [add_map(bb, batch, *mp) for mp in maps]
    for i, (sensor, p, grid) in zip(ids, maps):
        if sensor == bb.SENSOR_BEAM:
            with pytest.raises(bb.BelugaB200Error) as e:
                batch.likelihood_field(i)
            assert e.value.status == STATE
            continue
        twin = bb.Amcl(bb.DifferentialDriveModelParam(), bb.AmclParams(min_particles=100, max_particles=100))
        twin.update_map(sensor, p, grid)
        got, exp = batch.likelihood_field(i), twin.filter.likelihood_field()
        assert got.shape == exp.shape == grid.cells.shape and got.dtype == np.float32
        assert got.tobytes() == exp.tobytes()


def test_null_arguments_with_a_real_handle_are_refused(bb, scene):
    """Each pointer argument of the new entry points, null with a live batch: BB200_ERR_INVALID_ARGUMENT, nothing written,
    and the batch unchanged (no map added, the member's map kept)."""
    from beluga_b200 import _capi

    lib = _capi.load()
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam()], [bb.AmclParams(min_particles=100, max_particles=100)])
    first = batch.add_likelihood_field_map(lfm, grid)
    batch.update_map(0, first)
    h = batch._h
    p, g, beam = lfm.c(), grid.c(), bb.BeamModelParam().c()
    i = C.c_int(-7)
    for prob in (0, 1):
        assert lib.bb200_amcl_batch_add_likelihood_field_map(h, None, C.byref(g), prob, C.byref(i)) == INVALID
        assert lib.bb200_amcl_batch_add_likelihood_field_map(h, C.byref(p), None, prob, C.byref(i)) == INVALID
        assert lib.bb200_amcl_batch_add_likelihood_field_map(h, C.byref(p), C.byref(g), prob, None) == INVALID
    assert lib.bb200_amcl_batch_add_beam_map(h, None, C.byref(g), C.byref(i)) == INVALID
    assert lib.bb200_amcl_batch_add_beam_map(h, C.byref(beam), None, C.byref(i)) == INVALID
    assert lib.bb200_amcl_batch_add_beam_map(h, C.byref(beam), C.byref(g), None) == INVALID
    assert lib.bb200_amcl_batch_member_map(h, 0, None) == INVALID
    assert lib.bb200_amcl_batch_get_likelihood_field(h, first, None, grid.cells.size) == INVALID
    assert i.value == -7
    # nothing was added: the next map takes the next id, and member 0 still reads the first map
    assert batch.add_likelihood_field_map(lfm, grid) == first + 1
    assert batch.member_map(0) == first
