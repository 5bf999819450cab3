"""Batched particle-cloud publication on the GPU (bb200_amcl_batch_particle_histograms and bb200_amcl_batch_sample_states):
every selected member's bins, bin count, heaviest bin and pose samples are byte-equal to a standalone twin's
particle_histogram and sample_states, in every CDF state a member can be in (stale after an initialisation or a
resampling step, current after a normalising step or a rebuild); masks leave the other members' buffers alone; errors come
before any launch; the launch count depends neither on K nor on the counts; and sampling changes no member's later steps."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
SIZES = (1, 33, 2000, 32768, 2000, 33)
STATE, CAPACITY, INVALID = -4, -5, -1


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


def odometry(scene, t, k):
    x, y, th = scene.poses[t]
    th = th + 0.01 * k
    return np.array([np.cos(th), np.sin(th), x + 0.02 * k, y])


def twin_histogram(bb, twin, linear=1e-3, angular=1e-3):
    """bb200_filter_particle_histogram of a standalone filter -> (bins as raw records, n_bins, max_bin_weight)."""
    from beluga_b200 import _capi

    f = twin.filter
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, None, 0, C.byref(n), C.byref(top)) == 0
    bins = np.empty(max(n.value, 1), dtype=bb._CELL_DTYPE)
    assert f._lib.bb200_filter_particle_histogram(f._h, linear, angular, bins.ctypes.data_as(C.POINTER(_capi.ClusterCell)), n.value,
                                                  C.byref(n), C.byref(top)) == 0
    return bins[:n.value], n.value, top.value


def assert_same_cloud(bb, batch, twins, counts, step, present=None, linear=1e-3, angular=1e-3):
    hists = batch.particle_histograms(present, linear, angular)
    samples = batch.sample_states(counts, step, present)
    for m, twin in enumerate(twins):
        if present is not None and not present[m]:
            assert hists[m] is None and samples[m] is None
            continue
        bins, top = hists[m]
        t_bins, t_n, t_top = twin_histogram(bb, twin, linear, angular)
        assert len(bins) == t_n and bins.tobytes() == t_bins.tobytes(), m
        assert np.float64(top).tobytes() == np.float64(t_top).tobytes(), m
        want = twin.filter.sample_states(counts[m], step)
        assert samples[m].shape == (counts[m], 4) and samples[m].tobytes() == want.tobytes(), m


def launches(batch, call):
    before = batch.launch_count()
    call()
    return batch.launch_count() - before


def make_pair(bb, params, motions, grid):
    batch = bb.AmclBatch(motions, params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
    twins = []
    for m in range(len(params)):
        a = bb.Amcl(motions[m], params[m])
        a.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        twins.append(a)
    return batch, twins


def step_both(batch, twins, scene, t, present=None):
    k = len(twins)
    poses = [odometry(scene, t, m) for m in range(k)]
    for m in range(k):
        batch.force_update(m)
        twins[m].force_update()
    got = batch.update(poses, [scene.scans[t]] * k, present)
    for m in range(k):
        if present is None or present[m]:
            twins[m].update(poses[m], scene.scans[t])
    return got


def test_cloud_equals_standalone_filters(bb, scene):
    """Member sizes 1 to 32 768, both schemes, recovery injection, three motion models; members with resample_interval = 3
    sample from their normalising steps' CDFs (one launch), the others from rebuilt ones; the steps after many publishes
    stay byte-identical to the twins'."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    k = len(SIZES)
    params = []
    for m, n in enumerate(SIZES):
        p = bb.AmclParams(min_particles=n, max_particles=n, seed=300 + m, resample_scheme=m % 2)
        if m == 2:
            p.recovery_probability_override = 0.05
        if m in (1, 3, 4):
            p.resample_interval = 3
        params.append(p)
    motions = [motion(bb, m) for m in range(k)]
    batch, twins = make_pair(bb, params, motions, grid)
    for m in range(k):
        mean = scene.initial_mean + np.array([0.02 * m, 0.0, 0.01 * m])
        batch.initialize(m, mean, scene.initial_cov)
        twins[m].initialize(mean, scene.initial_cov)
    assert_same_cloud(bb, batch, twins, [n for n in SIZES], 0xFFFFFFFF)  # right after initialize: every CDF stale
    all_current = 0
    for t in range(8):
        got = step_both(batch, twins, scene, t)
        resampled = [bool(r.resampled) for r in got]
        counts = [(SIZES[m], 1, 0, 777)[(t + m) % 4] for m in range(k)]
        counts = [min(c, SIZES[m]) for m, c in enumerate(counts)]
        assert_same_cloud(bb, batch, twins, counts, 0xFFFFFFFF - t)
        if not any(resampled):
            all_current += 1
        for m in range(k):
            if not resampled[m] and params[m].resample_interval == 3:
                assert np.any(batch.particles(m)[1] != 1.0) or SIZES[m] == 1, (t, m)
        # the same call again: every CDF is current now
        assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 0xFFFFFFFF - t)) == 2 + (1 if any(counts) else 0)
        for m in range(k):
            st, w = batch.particles(m)
            t_st, t_w = twins[m].particles()
            assert st.tobytes() == t_st[:SIZES[m]].tobytes() and w.tobytes() == t_w[:SIZES[m]].tobytes(), (t, m)
    # only the interval-3 members selected after a normalising step (their tenth update): one launch for the draws
    step_both(batch, twins, scene, 8)
    got = step_both(batch, twins, scene, 9)
    current = [not r.resampled for r in got]
    assert any(current)
    n = batch.launch_count()
    assert_same_cloud(bb, batch, twins, [1] * k, 5, present=current)
    assert batch.launch_count() - n == 2 + 1


def raw_samples(batch, counts, step, present, sentinel=-7.25):
    k = len(batch)
    outs = [np.full((max(c, 1), 4), sentinel) for c in counts]
    ptrs = (C.POINTER(C.c_double) * k)(*[o.ctypes.data_as(C.POINTER(C.c_double)) for o in outs])
    mask = None if present is None else (C.c_uint8 * k)(*present)
    st = batch._lib.bb200_amcl_batch_sample_states(batch._h, (C.c_uint64 * k)(*counts), step, mask, ptrs)
    return st, outs


def raw_histograms(bb, batch, present, capacity, linear=1e-3, angular=1e-3, sentinel=0xDEADBEEF):
    from beluga_b200 import _capi

    k = len(batch)
    bufs = [np.zeros(max(c, 1), dtype=bb._CELL_DTYPE) for c in capacity]
    bins = (C.POINTER(_capi.ClusterCell) * k)(*[b.ctypes.data_as(C.POINTER(_capi.ClusterCell)) for b in bufs])
    n_bins = (C.c_uint64 * k)(*([sentinel] * k))
    top = (C.c_double * k)(*([-1.0] * k))
    mask = None if present is None else (C.c_uint8 * k)(*present)
    st = batch._lib.bb200_amcl_batch_particle_histograms(batch._h, linear, angular, mask, bins, (C.c_uint64 * k)(*capacity), n_bins, top)
    return st, bufs, list(n_bins), list(top)


def test_cdf_states(bb, scene):
    """Every CDF state: after initialize, after initialize_states with non-unit and with all-zero weights (degenerate: the
    uniform CDF), after a resampling step, after a normalising step, a second call after a rebuild, and a mix in one call."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=40 + m, resample_interval=(1, 3, 3)[m]) for m, n in enumerate((500, 900, 1300))]
    motions = [motion(bb, m) for m in range(3)]
    batch, twins = make_pair(bb, params, motions, grid)
    counts = [500, 64, 1300]
    for m in range(3):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
        twins[m].initialize(scene.initial_mean, scene.initial_cov)
    assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 11)) == 2 + 4  # stale after initialize
    assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 12)) == 2 + 1  # current after the rebuild
    rng = np.random.default_rng(3)
    states = np.tile(bb.se2(*scene.initial_mean), (900, 1)) + rng.normal(0, 0.05, (900, 4))
    weights = rng.uniform(0.1, 3.0, 900)
    batch.initialize_states(1, states, weights)
    twins[1].initialize_states(states, weights)
    assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 13)) == 2 + 4  # member 1 stale, the others current
    zero = np.zeros(900)
    batch.initialize_states(1, states, zero)
    twins[1].initialize_states(states, zero)
    assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 14)) == 2 + 4  # degenerate weights
    assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 15)) == 2 + 1
    batch.initialize_states(1, states, weights)
    twins[1].initialize_states(states, weights)
    for t in range(3):  # member 0 resamples every step; members 1 and 2 normalise twice, then resample
        got = step_both(batch, twins, scene, t)
        stale = [bool(r.resampled) for r in got]
        assert stale[0] and stale[1] == stale[2] == (t == 2)
        want = 4 if any(stale) else 1
        assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 100 + t)) == 2 + want, t
        assert launches(batch, lambda: assert_same_cloud(bb, batch, twins, counts, 200 + t)) == 2 + 1, t
        if not stale[1]:
            assert np.any(batch.particles(1)[1] != 1.0) and np.any(batch.particles(2)[1] != 1.0)


def test_counts_masks_and_errors(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=n) for n in (600, 900, 1200)]
    motions = [motion(bb, 0)] * 3
    batch, twins = make_pair(bb, params, motions, grid)
    for m in (0, 2):
        batch.initialize(m, scene.initial_mean, scene.initial_cov)
        twins[m].initialize(scene.initial_mean, scene.initial_cov)
    before = batch.launch_count()
    # member 1 holds no particles
    assert raw_samples(batch, [1, 1, 1], 0, None)[0] == STATE
    assert "member 1" in batch._lib.bb200_amcl_batch_last_error(batch._h).decode()
    assert raw_histograms(bb, batch, None, [600, 900, 1200])[0] == STATE
    # counts above max_particles, a null buffer with a positive count
    assert raw_samples(batch, [601, 0, 1], 0, [1, 0, 1])[0] == CAPACITY
    k = 3
    ptrs = (C.POINTER(C.c_double) * k)()
    assert batch._lib.bb200_amcl_batch_sample_states(batch._h, (C.c_uint64 * k)(1, 0, 0), 0, (C.c_uint8 * k)(1, 0, 1), ptrs) == INVALID
    assert batch._lib.bb200_amcl_batch_sample_states(batch._h, None, 0, None, ptrs) == INVALID
    for lin, ang in ((0.0, 1e-3), (1e-3, -1.0), (float("nan"), 1e-3)):
        st, _, n_bins, _ = raw_histograms(bb, batch, [1, 0, 1], [600, 900, 1200], lin, ang)
        assert st == INVALID and n_bins == [0xDEADBEEF] * 3
    assert batch.launch_count() == before
    assert raw_samples(batch, [0, 5, 0], 0, [1, 0, 1])[0] == 0 and batch.launch_count() == before  # nothing to draw
    # counts 0, 1 and max_particles; member 1 is not selected and keeps its sentinels
    st, outs = raw_samples(batch, [0, 7, 1200], 9, [1, 0, 1])
    assert st == 0
    assert np.all(outs[0] == -7.25) and np.all(outs[1] == -7.25)
    assert outs[2].tobytes() == twins[2].filter.sample_states(1200, 9).tobytes()
    st, outs = raw_samples(batch, [1, 0, 0], 9, [1, 0, 1])
    assert st == 0 and outs[0].tobytes() == twins[0].filter.sample_states(1, 9).tobytes()
    # histograms: a buffer too small for member 2 -> BB200_ERR_CAPACITY, every count still written, member 0's bins filled
    _, t_n2, _ = twin_histogram(bb, twins[2])
    st, bufs, n_bins, top = raw_histograms(bb, batch, [1, 0, 1], [600, 900, t_n2 - 1])
    assert st == CAPACITY and n_bins[2] == t_n2 and n_bins[1] == 0xDEADBEEF and top[1] == -1.0
    t_bins0, t_n0, t_top0 = twin_histogram(bb, twins[0])
    assert n_bins[0] == t_n0 and bufs[0][:t_n0].tobytes() == t_bins0.tobytes() and top[0] == t_top0
    # counts only: bins NULL
    n = (C.c_uint64 * 3)(*([0xDEADBEEF] * 3))
    assert batch._lib.bb200_amcl_batch_particle_histograms(batch._h, 1e-3, 1e-3, (C.c_uint8 * 3)(1, 0, 1), None, None, n, None) == 0
    assert list(n) == [t_n0, 0xDEADBEEF, t_n2]


def test_launch_count_does_not_depend_on_members(bb, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    rows = []
    for k in (1, 16, 64):
        params = [bb.AmclParams(min_particles=700, max_particles=700, seed=m, resample_interval=1 + m % 2) for m in range(k)]
        batch = bb.AmclBatch([motion(bb, 0)] * k, params)
        batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
        for m in range(k):
            batch.initialize(m, scene.initial_mean, scene.initial_cov)
        row = [launches(batch, lambda: batch.particle_histograms()),
               launches(batch, lambda: batch.sample_states(700)),       # all stale
               launches(batch, lambda: batch.sample_states(3))]         # all current
        for m in range(k):
            batch.force_update(m)
        res = batch.update([bb.se2(*scene.poses[0])] * k, [scene.scans[0]] * k)
        assert any(r.resampled for r in res) and (k == 1 or not all(r.resampled for r in res))
        row.append(launches(batch, lambda: batch.sample_states([1 + m for m in range(k)])))  # stale and current mixed (k > 1)
        row.append(launches(batch, lambda: batch.sample_states(1)))
        rows.append(row)
    assert rows[0] == rows[1] == rows[2] == [2, 4, 1, 4, 1]
