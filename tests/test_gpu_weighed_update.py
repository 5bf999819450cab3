"""Steps weighed by the caller's own sensor model (bb200_amcl_update_begin / _end, Amcl.update_weighted).

With factors bit-equal to a stock model's likelihoods (the oracle's sensor_weights on the propagated states the step
hands out) a weighed step must be byte-identical to the built-in update with that model: particles, weights, CDF,
ancestors, the result block and the cluster estimate, for every motion model, both resampling schemes, KLD, selective
resampling and recovery injection, and at the bench's shape.  Also: the stream ordering of a torch model, the rules for
factors a sensor model cannot produce, the open step's refusals and the rollback of a refused step."""
import ctypes as C
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DBL_MAX = sys.float_info.max
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
BEAM = dict(z_hit=0.5, z_short=0.05, z_max=0.05, z_rand=0.5, sigma_hit=0.2, lambda_short=0.1, beam_max_range=60.0)
ALPHAS = (0.1, 0.05, 0.1, 0.05)
STATE = -4  # BB200_ERR_STATE


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


@pytest.fixture(scope="module")
def orc():
    from oracle import pyoracle

    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="module")
def scene():
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=21)


def motion_of(bb, name):
    if name == "diff":
        return bb.DifferentialDriveModelParam(*ALPHAS)
    if name == "omni":
        return bb.OmnidirectionalDriveModelParam(0.1, 0.05, 0.1, 0.05, 0.1)
    return bb.StationaryModelParam()


def the_map(bb, sensor, scene):
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    if sensor == "beam":
        return bb.SENSOR_BEAM, bb.BeamModelParam(**BEAM), grid
    return (bb.SENSOR_LIKELIHOOD_FIELD_PROB if sensor == "prob" else bb.SENSOR_LIKELIHOOD_FIELD), bb.LikelihoodFieldModelParam(**LFM), grid


def oracle_weigh(orc, sensor, scene, points):
    """A weigh callable computing the stock model's likelihoods with the oracle on the states the step hands out."""
    kind = {"lfm": orc.LFM, "prob": orc.LFM_PROB, "beam": orc.BEAM}[sensor]
    param = orc.BeamParam(**BEAM) if sensor == "beam" else orc.LfmParam(**LFM)
    grid = orc.Grid(scene.cells, scene.resolution)

    def weigh(states, factors):
        import torch

        f = orc.sensor_weights(kind, param, grid, points, states.cpu().numpy())
        factors.copy_(torch.from_numpy(f))

    return weigh


def result_tuple(r):
    return (r.updated, r.resampled, r.n_particles, tuple(r.estimate.mean), tuple(r.estimate.cov), r.random_state_probability, r.weight_sum,
            r.weights_degenerate)


def assert_twins_equal(a, b, exact=True):
    sa, wa = a.filter.particles()
    sb, wb = b.filter.particles()
    if exact:
        assert sa.tobytes() == sb.tobytes() and wa.tobytes() == wb.tobytes()
    else:
        assert sa.shape == sb.shape
        np.testing.assert_allclose(sa, sb, rtol=0, atol=1e-9)
        np.testing.assert_allclose(wa, wb, rtol=1e-11, atol=1e-300)


CONFIGS = {
    "multinomial": dict(resample_scheme=0),
    "systematic": dict(resample_scheme=1),
    "kld": dict(resample_scheme=0, min_particles=500),
    "selective": dict(resample_scheme=1, selective_resampling=True),
    "injection": dict(resample_scheme=0, recovery_probability_override=0.05),
    "every_3": dict(resample_scheme=1, resample_interval=3),
}


def twins(bb, scene, motion, sensor, config, n=2000, seed=17):
    ap = dict(min_particles=n, max_particles=n, seed=seed, record_ancestors=True, update_min_d=0.05)
    ap.update(CONFIGS[config])
    out = []
    for _ in range(2):
        g = bb.Amcl(motion_of(bb, motion), bb.AmclParams(**ap))
        g.update_map(*the_map(bb, sensor, scene))
        g.initialize(scene.initial_mean, scene.initial_cov)
        out.append(g)
    return out


def run_twins(bb, orc, scene, a, b, sensor, steps, exact=True):
    for k in range(steps):
        pose = bb.se2(*scene.poses[k % len(scene.poses)])
        ra = a.update(pose, scene.scans[k % len(scene.scans)])
        rb = b.update_weighted(pose, oracle_weigh(orc, sensor, scene, scene.scans[k % len(scene.scans)]))
        if exact:
            assert result_tuple(ra) == result_tuple(rb), k
        else:
            assert (ra.updated, ra.resampled, ra.n_particles) == (rb.updated, rb.resampled, rb.n_particles)
        assert_twins_equal(a, b, exact)
        if ra.updated and exact:
            if ra.resampled:
                assert np.array_equal(a.filter.ancestors(), b.filter.ancestors())
            else:
                assert np.array_equal(a.filter.cdf(), b.filter.cdf())
    if exact:
        ca, cb = a.filter.cluster_estimate(), b.filter.cluster_estimate()
        assert ca[0].tobytes() == cb[0].tobytes() and ca[1].tobytes() == cb[1].tobytes()


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("motion", ["diff", "omni", "stationary"])
def test_weighed_steps_equal_builtin_steps(bb, orc, scene, motion, config):
    a, b = twins(bb, scene, motion, "lfm", config)
    run_twins(bb, orc, scene, a, b, "lfm", 20)


def test_weighed_steps_equal_builtin_prob_model(bb, orc, scene):
    a, b = twins(bb, scene, "diff", "prob", "systematic")
    run_twins(bb, orc, scene, a, b, "prob", 10)


def test_weighed_steps_follow_the_beam_model(bb, orc, scene):
    """The beam model matches the oracle to rtol 1e-11, not bit for bit: one normalising step, compared with that tolerance."""
    a, b = twins(bb, scene, "diff", "beam", "every_3")
    run_twins(bb, orc, scene, a, b, "beam", 1, exact=False)


def test_bench_shape(bb, orc):
    """One resampling step at 1M particles x 1080 beams on the 2000^2 map: the built-in step takes the scheduled, binned
    path; the weighed one the plain propagate."""
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=4)
    n = 1 << 20
    ap = dict(min_particles=n, max_particles=n, seed=3, record_ancestors=True, resample_scheme=1)
    a, b = (bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(**ap)) for _ in range(2))
    for g in (a, b):
        g.update_map(*the_map(bb, "lfm", sc))
        g.initialize(sc.initial_mean, sc.initial_cov)
    for k in range(2):  # the second step predicts its schedule from the first one's estimate
        pose = bb.se2(*sc.poses[k])
        ra = a.update(pose, sc.scans[k])
        rb = b.update_weighted(pose, oracle_weigh(orc, "lfm", sc, sc.scans[k]))
        assert ra.resampled == 1 and result_tuple(ra) == result_tuple(rb)
        assert_twins_equal(a, b)
        assert np.array_equal(a.filter.ancestors(), b.filter.ancestors())


def test_torch_model_is_ordered_on_the_step_stream(bb, scene):
    """A Gaussian position fix written in torch, issued on the step's stream with no synchronisation, against a twin
    handed the same factor bytes after an explicit synchronisation."""
    import torch

    fix = torch.tensor([scene.poses[3][0], scene.poses[3][1]], dtype=torch.float64)
    saved = []

    def model(states, factors):
        d = states[:, 2:4] - fix.to(states.device, non_blocking=True)
        factors.copy_(torch.exp(-(d * d).sum(dim=1) / (2 * 0.3 ** 2)))
        saved.append(factors.clone())

    def replay(states, factors):
        torch.cuda.synchronize()
        factors.copy_(saved[-1].cpu().to(factors.device))
        torch.cuda.synchronize()

    a, b = twins(bb, scene, "diff", "lfm", "multinomial", n=50000)
    for k in range(6):
        pose = bb.se2(*scene.poses[k])
        ra = a.update_weighted(pose, model)
        rb = b.update_weighted(pose, replay)
        assert ra.updated == 1 and result_tuple(ra) == result_tuple(rb)
        assert_twins_equal(a, b)


def test_edge_factors(bb, orc):
    """0, -1, NaN, +-inf, DBL_MAX and subnormal factors: the CDF of a normalising step and the indices of a resampling one
    equal the oracle's on w * factor, and weights_degenerate is set exactly when no weight can be selected."""
    import torch

    n = 4096
    rng = np.random.default_rng(9)
    specials = np.array([0.0, -1.0, np.nan, np.inf, -np.inf, DBL_MAX, 5e-324, 1e-310, -0.0])
    sets = {
        "mixed": np.where(rng.random(n) < 0.2, specials[rng.integers(0, len(specials), n)], rng.uniform(0.0, 2.0, n)),
        "max_and_dust": np.where(np.arange(n) == 77, DBL_MAX, 5e-324 * rng.integers(0, 3, n)),
        "none_selectable": specials[np.arange(n) % 5],
    }
    w0 = rng.uniform(0.5, 1.5, n)
    states = np.tile(np.array([1.0, 0.0, 0.0, 0.0]), (n, 1))
    states[:, 2] = np.arange(n)
    for name, f in sets.items():
        with np.errstate(over="ignore", invalid="ignore"):
            w = w0 * f
        valid = bool(np.any((w > 0.0) & (w <= DBL_MAX)))
        for scheme, interval in ((0, 2), (0, 1), (1, 1)):
            ap = dict(min_particles=n, max_particles=n, seed=12, record_ancestors=True, resample_scheme=scheme, resample_interval=interval)
            g = bb.Amcl(bb.StationaryModelParam(), bb.AmclParams(**ap))
            g.initialize_states(states, w0)
            r = g.update_weighted(bb.se2(0.0, 0.0, 0.0), lambda s, fac: fac.copy_(torch.from_numpy(f)))
            assert r.updated == 1 and r.weights_degenerate == (0 if valid else 1), name
            idx, cdf, _, ok = orc.resample_indices(w, scheme, seed=12, step=1, return_valid=True)
            assert ok == valid
            if interval == 2:
                assert r.resampled == 0 and np.array_equal(g.filter.cdf(), cdf), name
            else:
                assert r.resampled == 1 and np.array_equal(g.filter.ancestors(), idx), name


def test_open_step_refuses_every_other_call(bb, scene):
    lib = bb._capi.load()
    a, b = twins(bb, scene, "diff", "lfm", "multinomial")
    h = a._h
    f = lib.bb200_amcl_filter(h)
    view, res = bb._capi.WeighView(), bb._capi.UpdateResult()
    pose = np.ascontiguousarray(bb.se2(*scene.poses[0]))
    dp = pose.ctypes.data_as(C.POINTER(C.c_double))
    assert lib.bb200_amcl_update_end(h, C.byref(res)) == STATE  # end without begin
    before = a.export_state()
    assert lib.bb200_amcl_update_begin(h, dp, C.byref(view)) == 0 and view.updated == 1 and view.n == 2000
    pts = np.ascontiguousarray(scene.scans[0])
    buf = np.zeros(8 * 2000)
    n = C.c_uint64(0)
    size = C.c_uint64(0)
    refused = [
        lib.bb200_amcl_update_begin(h, dp, C.byref(view)),
        lib.bb200_amcl_update(h, dp, pts.ctypes.data_as(C.POINTER(C.c_double)), len(pts), C.byref(res)),
        lib.bb200_amcl_initialize_from_map(h),
        lib.bb200_amcl_export_state(h, None, 0, C.byref(size)),
        lib.bb200_amcl_plan_update(h, dp, C.byref(bb._capi.StepPlan())),
        lib.bb200_filter_get_particles(f, buf.ctypes.data_as(C.POINTER(C.c_double)), None, 10),
        lib.bb200_filter_size(f, C.byref(n)),
        lib.bb200_filter_synchronize(f),
    ]
    assert refused == [STATE] * len(refused)
    lib.bb200_amcl_force_update(h)
    b_view = bb._capi.WeighView()
    assert lib.bb200_amcl_update_begin(b._h, dp, C.byref(b_view)) == 0  # the twin's step opens independently
    import torch

    for v in (view, b_view):
        torch.as_tensor(bb._CudaArray(v.factors, (v.n,)), device="cuda").fill_(1.0)
    torch.cuda.synchronize()
    ra, rb = bb._capi.UpdateResult(), bb._capi.UpdateResult()
    assert lib.bb200_amcl_update_end(h, C.byref(ra)) == 0 and lib.bb200_amcl_update_end(b._h, C.byref(rb)) == 0
    assert result_tuple(ra) == result_tuple(rb)
    assert_twins_equal(a, b)
    assert lib.bb200_amcl_update_end(h, C.byref(res)) == STATE  # closed
    assert a.export_state() != before
    # a step the policies skip: nothing reaches the device, end still closes it
    launches = a.filter.launch_count()
    snap = a.export_state()
    assert lib.bb200_amcl_update_begin(h, dp, C.byref(view)) == 0 and view.updated == 0
    assert lib.bb200_amcl_initialize_from_map(h) == STATE
    assert lib.bb200_amcl_update_end(h, C.byref(res)) == 0 and res.updated == 0
    assert a.filter.launch_count() == launches and a.export_state() == snap
    # destroy with an open step
    assert lib.bb200_amcl_update_begin(h, np.ascontiguousarray(bb.se2(*scene.poses[2])).ctypes.data_as(C.POINTER(C.c_double)), C.byref(view)) == 0
    a.close()
    b.close()


def test_refused_begin_rolls_back(bb, scene):
    """A step that would inject random states needs a map: begin refuses it before any device work, the policies stay as
    they were, and the next update equals a twin's that never saw the refused call."""
    n = 3000
    ap = dict(min_particles=n, max_particles=n, seed=4, record_ancestors=True, recovery_probability_override=0.1)
    a, b = (bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(**ap)) for _ in range(2))
    for g in (a, b):
        g.initialize(scene.initial_mean, scene.initial_cov)
    launches = a.filter.launch_count()
    with pytest.raises(bb.BelugaB200Error) as e:
        a.update_weighted(bb.se2(*scene.poses[1]), lambda s, f: None)
    assert e.value.status == STATE and a.filter.launch_count() == launches
    # no map and no injection: a weighed step runs; the twins stay equal
    for g in (a, b):
        g.update_map(*the_map(bb, "lfm", scene))
    pose = bb.se2(*scene.poses[1])
    ra, rb = a.update(pose, scene.scans[1]), b.update(pose, scene.scans[1])
    assert result_tuple(ra) == result_tuple(rb)
    assert_twins_equal(a, b)
    assert np.array_equal(a.filter.ancestors(), b.filter.ancestors())


def test_weighed_steps_without_a_map(bb, scene):
    """A filter without a map takes weighed steps (no injection), and a sharded filter refuses them."""
    import torch

    n = 2000
    g = bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(min_particles=n, max_particles=n, seed=2))
    g.initialize(scene.initial_mean, scene.initial_cov)
    r = g.update_weighted(bb.se2(*scene.poses[1]), lambda s, f: f.copy_(torch.exp(-s[:, 2].abs())))
    assert r.updated == 1 and r.resampled == 1 and r.n_particles == n
    s = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(min_particles=2 * n, max_particles=2 * n, seed=2), [0, 0])
    lib = bb._capi.load()
    view = bb._capi.WeighView()
    pose = np.ascontiguousarray(bb.se2(*scene.poses[1]))
    assert lib.bb200_amcl_update_begin(lib.bb200_sharded_amcl_shard(s._h, 0), pose.ctypes.data_as(C.POINTER(C.c_double)), C.byref(view)) == STATE


# ---- batches: members weighed by the caller next to members with points ------------------------------------------
BATCH_PARAMS = [
    dict(resample_scheme=1, selective_resampling=True),  # weighed, selective
    dict(resample_scheme=0, min_particles=500),          # weighed, KLD
    dict(resample_scheme=1, resample_interval=2),        # points
    dict(resample_scheme=0, recovery_probability_override=0.05),  # weighed, injection
]
WEIGHED = [0, 1, 3]


def batch_params(bb, n=2000):
    out = []
    for m, extra in enumerate(BATCH_PARAMS):
        ap = dict(min_particles=n, max_particles=n, seed=40 + m, record_ancestors=True, update_min_d=0.05)
        ap.update(extra)
        out.append(bb.AmclParams(**ap))
    return out


def make_batch(bb, scene, params):
    b = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS) for _ in params], params, adaptive=True, selective=True)
    b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    for m in range(len(params)):
        b.initialize(m, scene.initial_mean, scene.initial_cov)
    return b


def batch_oracle_weigh(orc, scene, points):
    param, grid = orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution)

    def weigh(members, states, factors):
        import torch

        for s, f in zip(states, factors):
            f.copy_(torch.from_numpy(orc.sensor_weights(orc.LFM, param, grid, points, s.cpu().numpy())))

    return weigh


def test_mixed_batch_equals_standalone_twins(bb, orc, scene):
    params = batch_params(bb)
    batch = make_batch(bb, scene, params)
    twins_ = []
    for p in params:
        g = bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), p)
        g.update_map(*the_map(bb, "lfm", scene))
        g.initialize(scene.initial_mean, scene.initial_cov)
        twins_.append(g)
    for k in range(12):
        pose = bb.se2(*scene.poses[k])
        poses = np.stack([pose] * len(params))
        meas = [None if m in WEIGHED else scene.scans[k] for m in range(len(params))]
        rb = batch.update_weighted(poses, meas, batch_oracle_weigh(orc, scene, scene.scans[k]))
        for m, g in enumerate(twins_):
            rt = g.update(pose, scene.scans[k])
            assert result_tuple(rb[m]) == result_tuple(rt), (k, m)
            sb, wb = batch.particles(m)
            st, wt = g.filter.particles()
            assert sb.tobytes() == st.tobytes() and wb.tobytes() == wt.tobytes(), (k, m)
            if rt.updated and rt.resampled:
                assert np.array_equal(batch.ancestors(m), g.filter.ancestors())


def test_weighed_end_with_cluster_equals_update_clustered(bb, orc, scene):
    params = batch_params(bb)
    a, b = make_batch(bb, scene, params), make_batch(bb, scene, params)
    for k in range(6):
        poses = np.stack([bb.se2(*scene.poses[k])] * len(params))
        ra, ea = a.update_clustered(poses, [scene.scans[k]] * len(params))
        meas = [None if m in WEIGHED else scene.scans[k] for m in range(len(params))]
        rb, eb = b.update_weighted(poses, meas, batch_oracle_weigh(orc, scene, scene.scans[k]), cluster=(0.20, 0.524, 0.90))
        for m in range(len(params)):
            assert result_tuple(ra[m]) == result_tuple(rb[m])
            assert (ea[m] is None) == (eb[m] is None)
            if ea[m] is not None:
                assert ea[m][0].tobytes() == eb[m][0].tobytes() and ea[m][1].tobytes() == eb[m][1].tobytes()


def test_batch_without_weighed_members_launches_as_before(bb, scene):
    params = batch_params(bb)
    a, b = make_batch(bb, scene, params), make_batch(bb, scene, params)
    for k in range(6):
        poses = np.stack([bb.se2(*scene.poses[k])] * len(params))
        la, lb = a.launch_count(), b.launch_count()
        ra = a.update_measurements(poses, [scene.scans[k]] * len(params))
        rb = b.update_weighted(poses, [scene.scans[k]] * len(params), lambda *args: pytest.fail("nothing to weigh"))
        assert a.launch_count() - la == b.launch_count() - lb
        assert [result_tuple(r) for r in ra] == [result_tuple(r) for r in rb]
        for m in range(len(params)):
            assert a.particles(m)[0].tobytes() == b.particles(m)[0].tobytes()


def test_open_batch_step_refuses_other_calls(bb, scene):
    lib = bb._capi.load()
    params = batch_params(bb)
    batch = make_batch(bb, scene, params)
    k = len(params)
    poses = np.ascontiguousarray(np.stack([bb.se2(*scene.poses[0])] * k))
    table = (bb._capi.Measurement * k)(*[bb._capi.Measurement(kind=bb._capi.MEASUREMENT_WEIGHTS) for _ in range(k)])
    views = (bb._capi.WeighView * k)()
    res = (bb._capi.UpdateResult * k)()
    dp = poses.ctypes.data_as(C.POINTER(C.c_double))
    assert lib.bb200_amcl_batch_update_end(batch._h, None, res, None, None, None) == STATE
    assert lib.bb200_amcl_batch_update_begin(batch._h, dp, table, None, views) == 0
    assert all(views[m].updated == 1 and views[m].n == 2000 for m in range(k))
    assert lib.bb200_amcl_batch_update_begin(batch._h, dp, table, None, views) == STATE
    assert lib.bb200_amcl_batch_update_measurements(batch._h, dp, table, None, res) == STATE
    assert lib.bb200_amcl_batch_initialize_from_map(batch._h, 0) == STATE
    n = C.c_uint64(0)
    assert lib.bb200_amcl_batch_member_size(batch._h, 0, C.byref(n)) == STATE
    import torch

    for m in range(k):
        torch.as_tensor(bb._CudaArray(views[m].factors, (views[m].n,)), device="cuda").fill_(1.0)
    torch.cuda.synchronize()
    assert lib.bb200_amcl_batch_update_end(batch._h, None, res, None, None, None) == 0
    assert all(res[m].updated == 1 for m in range(k))
    assert lib.bb200_amcl_batch_update_end(batch._h, None, res, None, None, None) == STATE
    # a weighed member with no map takes steps; one whose step may inject is refused before any device work
    nomap = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS)], [bb.AmclParams(min_particles=1000, max_particles=1000, seed=1)])
    nomap.initialize(0, scene.initial_mean, scene.initial_cov)
    r = nomap.update_weighted(poses[:1], [None], lambda members, s, f: f[0].copy_(torch.exp(-s[0][:, 2].abs())))
    assert r[0].updated == 1 and r[0].resampled == 1
