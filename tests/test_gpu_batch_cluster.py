"""The batched cluster estimate (bb200_amcl_batch_cluster_estimates) on the GPU: every selected member's estimate is byte-equal to
the per-member call and to a standalone filter's over the same particles, across member sizes from 1 to 32 768, non-unit weights
and recovery injection; cell-count extremes agree with the CPU oracle; masks leave the other members' entries alone; errors are
raised before any launch; and the launch count depends neither on K nor on the cells."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

from test_oracle_cluster import multicluster_dataset

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
SIZES = (1, 33, 256, 2000, 5000, 32768, 2000, 33)


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
    p = bb.AmclParams(min_particles=n, max_particles=n, seed=200 + k, resample_scheme=k % 2)
    if k == 3:
        p.recovery_probability_override = 0.05
    if k in (4, 5, 7):
        p.resample_interval = 3  # non-unit weights between resampling steps: the cell weight replays the particle order
    return p


def odometry(scene, t, k):
    x, y, th = scene.poses[t]
    th = th + 0.01 * k
    return np.array([np.cos(th), np.sin(th), x + 0.02 * k, y])


def estimate_bytes(mean, cov):
    return np.asarray(mean).tobytes() + np.asarray(cov).tobytes()


def test_estimates_equal_standalone_filters(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    k = len(SIZES)
    params = [member_params(bb, m) for m in range(k)]
    motions = [motion(bb, m) for m in range(k)]
    batch = bb.AmclBatch(motions, params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
    twins = []
    for m in range(k):
        a = bb.Amcl(motions[m], params[m])
        a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        batch.initialize(m, mean, scene.initial_cov)
        a.initialize(mean, scene.initial_cov)
        twins.append(a)
    non_unit = 0
    for t in range(10):
        poses = [odometry(scene, t, m) for m in range(k)]
        for m in range(2, k, 3):  # the stationary members would not update otherwise
            batch.force_update(m)
            twins[m].force_update()
        got = batch.update(poses, [scene.scans[t]] * k)
        for m in range(k):
            twins[m].update(poses[m], scene.scans[t])
        assert any(r.updated for r in got)
        ests = batch.cluster_estimates(with_counts=True)
        for m in range(k):
            mean, cov, cells, clusters = ests[m]
            one = batch.cluster_estimate(m)
            tm, tc, _, t_cells, t_clusters = twins[m].filter.cluster_estimate(with_ids=True)
            assert estimate_bytes(mean, cov) == estimate_bytes(*one), (t, m)
            assert estimate_bytes(mean, cov) == estimate_bytes(tm, tc), (t, m)
            assert (cells, clusters) == (t_cells, t_clusters), (t, m)
            if m in (4, 5, 7):
                non_unit += int(np.any(batch.particles(m)[1] != 1.0))
    assert non_unit > 0


def own_cells(n, spacing=1.5):
    side = int(math.ceil(math.sqrt(n)))
    ix, iy = np.arange(n) % side, np.arange(n) // side
    th = 0.3 * np.ones(n)
    return np.stack([np.cos(th), np.sin(th), 0.5 + spacing * ix, 0.5 + spacing * iy], axis=1)


def test_cell_count_extremes(bb, orc):
    """One batch call over members whose cells span the range: 32 768 cells (the full 15-bit sort key), one cell, more than 256
    cells (two radix passes), and the reference's four-peak grid with its non-unit weights."""
    linear, angular, percentile = 1.0, math.pi / 2, 0.9
    rng = np.random.default_rng(5)
    spread = own_cells(32768)
    th = rng.uniform(0.0, 0.2, 1000)
    one = np.stack([np.cos(th), np.sin(th), rng.uniform(3.1, 3.9, 1000), rng.uniform(7.1, 7.9, 1000)], axis=1)
    th = rng.uniform(-math.pi, math.pi, 2000)
    many = np.stack([np.cos(th), np.sin(th), rng.uniform(0.0, 30.0, 2000), rng.uniform(0.0, 30.0, 2000)], axis=1)
    peaks, peak_w = multicluster_dataset(0.0, 36.0, 0.0, 36.0, 1.0)
    members = [(spread, rng.uniform(0.5, 1.5, len(spread))), (one, None), (many, rng.uniform(0.0, 1.0, 2000)), (peaks, peak_w)]
    params = [bb.AmclParams(min_particles=len(s), max_particles=len(s), seed=m) for m, (s, _) in enumerate(members)]
    batch = bb.AmclBatch([bb.StationaryModelParam() for _ in members], params)
    for m, (s, w) in enumerate(members):
        batch.initialize_states(m, s, w)
    ests = batch.cluster_estimates(linear=linear, angular=angular, percentile=percentile, with_counts=True)
    cells = [e[2] for e in ests]
    assert cells[0] == 32768 and cells[1] == 1 and cells[2] > 256
    for m, (s, w) in enumerate(members):
        mean, cov, n_cells, n_clusters = ests[m]
        weights = np.ones(len(s)) if w is None else w
        f = bb.Filter(capacity=len(s))
        f.set_particles(s, weights)
        fm, fc, _, f_cells, f_clusters = f.cluster_estimate(linear=linear, angular=angular, percentile=percentile, with_ids=True)
        assert estimate_bytes(mean, cov) == estimate_bytes(fm, fc), m
        assert (n_cells, n_clusters) == (f_cells, f_clusters), m
        want_mean, want_cov = orc.cluster_based_estimate(s, weights, linear, angular, percentile)
        assert np.allclose(mean, want_mean, rtol=0, atol=1e-9), m
        finite = np.isfinite(want_cov)
        assert np.array_equal(np.isfinite(cov), finite), m
        assert np.allclose(cov[finite], want_cov[finite], rtol=1e-9, atol=1e-9), m


def raw_call(bb, batch, present, linear=0.2, angular=0.524, percentile=0.9, sentinel=12345.0, cell_sentinel=0xDEADBEEF):
    from beluga_b200 import _capi

    k = len(batch)
    p = _capi.ClusterParam(linear, angular, percentile)
    out = (_capi.Estimate * k)()
    for e in out:
        for i in range(4):
            e.mean[i] = sentinel
        for i in range(9):
            e.cov[i] = sentinel
    cells = (C.c_uint32 * k)(*([cell_sentinel] * k))
    clusters = (C.c_uint32 * k)(*([cell_sentinel] * k))
    mask = None if present is None else (C.c_uint8 * k)(*[1 if x else 0 for x in present])
    st = batch._lib.bb200_amcl_batch_cluster_estimates(batch._h, C.byref(p), mask, out, cells, clusters)
    return st, out, list(cells), list(clusters)


def test_masks_and_errors(bb, scene):
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=n) for n in (600, 900, 1200)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam() for _ in params], params)
    batch.initialize(0, scene.initial_mean, scene.initial_cov)
    batch.initialize(2, scene.initial_mean, scene.initial_cov)
    before = batch.launch_count()
    st, _, _, _ = raw_call(bb, batch, None)  # member 1 holds no particles
    assert st == -4 and "member 1" in batch._lib.bb200_amcl_batch_last_error(batch._h).decode()
    assert batch.launch_count() == before
    st, out, cells, clusters = raw_call(bb, batch, [1, 0, 1])
    assert st == 0
    assert list(out[1].mean) == [12345.0] * 4 and list(out[1].cov) == [12345.0] * 9
    assert cells[1] == clusters[1] == 0xDEADBEEF
    for m in (0, 2):
        assert cells[m] != 0xDEADBEEF and clusters[m] != 0xDEADBEEF
        mean, cov = batch.cluster_estimate(m)
        assert np.array(out[m].mean).tobytes() == mean.tobytes() and np.array(out[m].cov).tobytes() == cov.tobytes()
    assert batch.cluster_estimates(present=[True, False, True])[1] is None
    before = batch.launch_count()
    for bad in (dict(linear=0.0), dict(angular=-1.0), dict(percentile=1.0), dict(percentile=-0.1), dict(linear=float("nan"))):
        st, out, cells, _ = raw_call(bb, batch, [1, 0, 1], **bad)
        assert st == -1, bad
        assert "cluster parameters" in batch._lib.bb200_amcl_batch_last_error(batch._h).decode()
        assert cells == [0xDEADBEEF] * 3
    assert batch.launch_count() == before
    st, _, _, _ = raw_call(bb, batch, [0, 0, 0])  # nothing selected: nothing to do
    assert st == 0 and batch.launch_count() == before


def test_launch_count_does_not_depend_on_members_or_cells(bb, scene):
    counts = []
    for k in (1, 16, 256):
        params = [bb.AmclParams(min_particles=500, max_particles=500, seed=m) for m in range(k)]
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam() for _ in range(k)], params)
        for m in range(k):
            batch.initialize(m, scene.initial_mean, scene.initial_cov)
        before = batch.launch_count()
        assert all(e is not None for e in batch.cluster_estimates())
        counts.append(batch.launch_count() - before)
    params = [bb.AmclParams(min_particles=4000, max_particles=4000, seed=1)]
    batch = bb.AmclBatch([bb.StationaryModelParam()], params)
    per_cloud = []
    for spread in (True, False):
        if spread:
            batch.initialize(0, scene.initial_mean, np.diag([25.0, 25.0, 3.0]))
        else:
            batch.initialize_states(0, np.tile(bb.se2(*scene.initial_mean), (4000, 1)))
        before = batch.launch_count()
        _, _, cells, _ = batch.cluster_estimates(with_counts=True)[0]
        per_cloud.append((batch.launch_count() - before, cells))
    assert per_cloud[0][1] > 256 and per_cloud[1][1] == 1
    assert counts[0] == counts[1] == counts[2] == per_cloud[0][0] == per_cloud[1][0] == 2


def test_estimates_follow_the_step(bb, scene):
    """update then cluster_estimates, the beluga_ros-shaped round, for members that skip steps: an absent member's entry is None."""
    k = 4
    params = [bb.AmclParams(min_particles=1500, max_particles=1500, seed=m, resample_scheme=1) for m in range(k)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS[:4]) for _ in range(k)], params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    for m in range(k):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
    for t in range(6):
        present = [(t + m) % 3 != 0 for m in range(k)]
        res = batch.update([bb.se2(*scene.poses[t])] * k, [scene.scans[t]] * k, present)
        updated = [bool(r.updated) for r in res]
        ests = batch.cluster_estimates(present=updated)
        for m in range(k):
            if not updated[m]:
                assert ests[m] is None
                continue
            assert struct.pack("<4d9d", *ests[m][0], *ests[m][1].ravel()) == struct.pack("<4d9d", *batch.cluster_estimate(m)[0],
                                                                                          *batch.cluster_estimate(m)[1].ravel())
