"""Sharded steps weighed by the caller's own sensor model (bb200_sharded_amcl_update_begin / _end, ShardedAmcl.update_weighted).

With factors bit-equal to a stock model's likelihoods (the oracle's sensor_weights on the states each shard hands out) a
weighed sharded step must be byte-identical to the built-in sharded step: particles, weights, the result block and the
cluster estimate, under every resampling mode, KLD (a shard left empty included), the prob and beam models and the
bench's shape.  A weighed sharded filter must follow a weighed single filter whatever the shard count.  Also: the edge
factors, a sensor model slower than the exchanges' timeout, the open step's refusals, rollback and the launch count."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_sharded_local import MODES
from test_gpu_weighed_update import ALPHAS, DBL_MAX, STATE, oracle_weigh, result_tuple, the_map

pytestmark = pytest.mark.gpu


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=21)


def sharded_twins(bb, scene, shards, n, sensor="lfm", devices=None, with_map=True, **kw):
    """A built-in and a weighed ShardedAmcl with the same parameters."""
    ap = dict(min_particles=n, max_particles=n, seed=99)
    ap.update(kw)
    out = []
    for _ in range(2):
        g = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(**ap), devices=devices or [0] * shards)
        if with_map:
            g.update_map(*the_map(bb, sensor, scene))
        g.initialize(scene.initial_mean, scene.initial_cov)
        out.append(g)
    return out


def assert_sharded_equal(a, b, exact=True):
    sa, wa = a.particles()
    sb, wb = b.particles()
    if exact:
        assert sa.tobytes() == sb.tobytes() and wa.tobytes() == wb.tobytes()
    else:
        assert sa.shape == sb.shape
        np.testing.assert_allclose(sa, sb, rtol=0, atol=1e-9)
        np.testing.assert_allclose(wa, wb, rtol=1e-11, atol=1e-300)


def counting(weigh, calls):
    def wrapped(states, factors):
        calls.append(len(factors))
        weigh(states, factors)

    return wrapped


def run_sharded_twins(bb, orc, scene, a, b, sensor, steps, exact=True):
    """Steps `a` built in and `b` weighed; returns the particle count of every shard's view at every step."""
    views = []
    for k in range(steps):
        pose = bb.se2(*scene.poses[k % len(scene.poses)])
        pts = scene.scans[k % len(scene.scans)]
        sizes = [f.size() for f in b.shards]
        calls = []
        ra = a.update(pose, pts)
        rb = b.update_weighted(pose, counting(oracle_weigh(orc, sensor, scene, pts), calls))
        if rb.updated:
            assert calls == [n for n in sizes if n > 0], k  # once per shard with particles, in rank order
            views.append(sizes)
        if exact:
            assert result_tuple(ra) == result_tuple(rb), k
        else:
            assert (ra.updated, ra.resampled, ra.n_particles) == (rb.updated, rb.resampled, rb.n_particles)
        assert_sharded_equal(a, b, exact)
    if exact:
        ca, cb = a.cluster_estimate(), b.cluster_estimate()
        assert ca[0].tobytes() == cb[0].tobytes() and ca[1].tobytes() == cb[1].tobytes()
    return views


@pytest.mark.parametrize("shards", [2, 3, 4])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_weighed_shards_equal_builtin_shards(bb, orc, scene, shards, mode):
    a, b = sharded_twins(bb, scene, shards, 3000 * shards, **MODES[mode])
    run_sharded_twins(bb, orc, scene, a, b, "lfm", 6)


@pytest.mark.parametrize("shards,scheme", [(2, 1), (3, 0), (4, 1)])
def test_weighed_kld_shards_equal_builtin_shards(bb, orc, scene, shards, scheme):
    a, b = sharded_twins(bb, scene, shards, 12_000 * shards, min_particles=600, resample_scheme=scheme, seed=31)
    run_sharded_twins(bb, orc, scene, a, b, "lfm", 6)


def test_weighed_kld_with_an_empty_shard(bb, orc, scene):
    """take_while_kld settles on 41 particles: 6 on each of the first six shards, 5 on the seventh, none on the last.  The
    next step hands the last shard a view of n = 0, and its weigh is not called."""
    a, b = sharded_twins(bb, scene, 8, 8 * 1000, min_particles=41, resample_scheme=1, seed=31, kld_epsilon=1.0)
    views = run_sharded_twins(bb, orc, scene, a, b, "lfm", 4)
    assert any(v[-1] == 0 and sum(v) > 0 for v in views), views


def test_weighed_shards_prob_model(bb, orc, scene):
    a, b = sharded_twins(bb, scene, 2, 6000, sensor="prob", resample_scheme=1)
    run_sharded_twins(bb, orc, scene, a, b, "prob", 5)


def test_weighed_eight_shards_beam_model(bb, orc, scene):
    """The beam model matches the oracle to rtol 1e-11, not bit for bit: one normalising step, compared with that tolerance."""
    a, b = sharded_twins(bb, scene, 8, 8 * 512, sensor="beam", resample_scheme=1, resample_interval=3)
    run_sharded_twins(bb, orc, scene, a, b, "beam", 1, exact=False)


def test_weighed_shards_bench_shape(bb, orc):
    """One resampling step at 1M particles x 1080 beams on the 2000^2 map over 4 shards."""
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=2)
    a, b = sharded_twins(bb, sc, 4, 1 << 20, resample_scheme=1, seed=3)
    pose = bb.se2(*sc.poses[0])
    ra = a.update(pose, sc.scans[0])
    rb = b.update_weighted(pose, oracle_weigh(orc, "lfm", sc, sc.scans[0]))
    assert ra.resampled == 1 and result_tuple(ra) == result_tuple(rb)
    assert_sharded_equal(a, b)


def position_fix(fix, sigma=0.3):
    import torch

    def model(states, factors):
        d = states[:, 2:4] - torch.tensor(fix, dtype=torch.float64, device=states.device)
        torch.exp(-(d * d).sum(dim=1) / (2 * sigma ** 2), out=factors)

    return model


@pytest.mark.parametrize("shards", [2, 4])
@pytest.mark.parametrize("mode", ["systematic", "multinomial", "selective", "every-3"])
def test_shard_count_does_not_matter(bb, scene, shards, mode):
    """A torch position fix drives a weighed ShardedAmcl and a weighed single Amcl: the run_pair tolerances."""
    n = 8192 * shards
    ap = dict(min_particles=n, max_particles=n, seed=99, **MODES[mode])
    single = bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(**ap), devices=[0] * shards)
    for f in (single, group):
        f.initialize(scene.initial_mean, scene.initial_cov)
    for k in range(7):
        pose = bb.se2(*scene.poses[k])
        model = position_fix(scene.poses[k][:2])
        rs, rg = single.update_weighted(pose, model), group.update_weighted(pose, model)
        assert rs.updated == rg.updated and rs.resampled == rg.resampled and rs.n_particles == rg.n_particles
        assert rs.random_state_probability == rg.random_state_probability and rs.weight_sum == rg.weight_sum
        ss, ws = single.particles()
        sg, wg = group.particles()
        assert ss.tobytes() == sg.tobytes() and ws.tobytes() == wg.tobytes(), k
        assert np.abs(np.array(rs.estimate.mean) - np.array(rg.estimate.mean)).max() < 1e-12
        assert np.abs(np.array(rs.estimate.cov) - np.array(rg.estimate.cov)).max() < 1e-12


def test_edge_factors_spread_over_shards(bb):
    """The factor sets of the single filter's edge test, spread over 4 shards, equal the single weighed filter."""
    import torch

    n, shards = 4096, 4
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
        for scheme, interval in ((0, 2), (0, 1), (1, 1)):
            ap = bb.AmclParams(min_particles=n, max_particles=n, seed=12, resample_scheme=scheme, resample_interval=interval)
            single = bb.Amcl(bb.StationaryModelParam(), ap)
            group = bb.ShardedAmcl(bb.StationaryModelParam(), ap, devices=[0] * shards)
            single.initialize_states(states, w0)
            lib = bb._capi.load()
            m = n // shards
            for r in range(shards):
                st, w = np.ascontiguousarray(states[r * m:(r + 1) * m]), np.ascontiguousarray(w0[r * m:(r + 1) * m])
                assert lib.bb200_amcl_initialize_states(lib.bb200_sharded_amcl_shard(group._h, r), st.ctypes.data_as(C.POINTER(C.c_double)),
                                                        w.ctypes.data_as(C.POINTER(C.c_double)), m) == 0
            pose = bb.se2(0.0, 0.0, 0.0)
            rs = single.update_weighted(pose, lambda s, fac: fac.copy_(torch.from_numpy(f)))
            first = [0]

            def weigh(s, fac):  # called in rank order: the shards' slices follow each other in the global order
                fac.copy_(torch.from_numpy(f[first[0]:first[0] + len(fac)]))
                first[0] += len(fac)

            rg = group.update_weighted(pose, weigh)
            assert rs.updated == rg.updated == 1 and rs.resampled == rg.resampled, name
            assert rs.weights_degenerate == rg.weights_degenerate, name
            assert rs.weight_sum == rg.weight_sum or (np.isnan(rs.weight_sum) and np.isnan(rg.weight_sum)), name
            ss, ws = single.particles()
            sg, wg = group.particles()
            assert ss.tobytes() == sg.tobytes() and ws.tobytes() == wg.tobytes(), (name, scheme, interval)


def test_slow_model_completes_the_step(bb, scene):
    """Shard 0's model keeps its stream busy for about 5 s, longer than the exchanges' 4 s timeout: every shard's exchanges
    wait for every shard's factors, so the step completes and equals a twin weighed without the delay.  Run once."""
    import torch

    n, shards = 8192, 2
    ap = bb.AmclParams(min_particles=n * shards, max_particles=n * shards, seed=5, resample_scheme=1)
    slow, fast = (bb.ShardedAmcl(bb.DifferentialDriveModelParam(*ALPHAS), ap, devices=[0] * shards) for _ in range(2))
    for g in (slow, fast):
        g.initialize(scene.initial_mean, scene.initial_cov)
    cycles = 10_000_000_000  # SM clock cycles: at least 5 s at the H100's top clock of 1.98 GHz
    model = position_fix(scene.poses[1][:2])
    calls = []

    def slow_model(states, factors):
        if not calls:
            torch.cuda._sleep(cycles)
        calls.append(1)
        model(states, factors)

    pose = bb.se2(*scene.poses[1])
    rs = slow.update_weighted(pose, slow_model)
    rf = fast.update_weighted(pose, model)
    assert rs.updated == 1 and result_tuple(rs) == result_tuple(rf)
    assert_sharded_equal(slow, fast)


def weigh_ones(bb, views, k):
    import torch

    for r in range(k):
        if views[r].n:
            torch.as_tensor(bb._CudaArray(views[r].factors, (views[r].n,)), device="cuda").fill_(1.0)
    torch.cuda.synchronize()


def test_open_step_refuses_every_other_call(bb, scene):
    lib = bb._capi.load()
    k = 3
    a, b = sharded_twins(bb, scene, k, 3000 * k, resample_scheme=0)
    h = a._h
    views, res = (bb._capi.WeighView * k)(), bb._capi.UpdateResult()
    pose = np.ascontiguousarray(bb.se2(*scene.poses[0]))
    dp = pose.ctypes.data_as(C.POINTER(C.c_double))
    assert lib.bb200_sharded_amcl_update_end(h, C.byref(res)) == STATE  # end without begin
    assert lib.bb200_sharded_amcl_update_begin(h, dp, views) == 0
    assert all(views[r].updated == 1 and views[r].n == 3000 for r in range(k))
    assert len({views[r].states for r in range(k)}) == k and len({views[r].stream for r in range(k)}) == k
    pts = np.ascontiguousarray(scene.scans[0])
    dpts = pts.ctypes.data_as(C.POINTER(C.c_double))
    buf = np.zeros(8 * 3000 * k)
    dbuf = buf.ctypes.data_as(C.POINTER(C.c_double))
    shard = lib.bb200_sharded_amcl_shard(h, 1)
    f = lib.bb200_amcl_filter(shard)
    n = C.c_uint64(0)
    mean, cov = np.ascontiguousarray(scene.initial_mean, dtype=np.float64), np.ascontiguousarray(scene.initial_cov, dtype=np.float64)
    refused = [
        lib.bb200_sharded_amcl_update_begin(h, dp, views),
        lib.bb200_sharded_amcl_update(h, dp, dpts, len(pts), C.byref(res)),
        lib.bb200_sharded_amcl_initialize(h, mean.ctypes.data_as(C.POINTER(C.c_double)), cov.ctypes.data_as(C.POINTER(C.c_double))),
        lib.bb200_sharded_amcl_initialize_from_map(h),
        lib.bb200_sharded_amcl_get_particles(h, dbuf, None, 10),
        lib.bb200_sharded_amcl_sample_states(h, 10, 0, dbuf),
        lib.bb200_sharded_amcl_cluster_estimate(h, C.byref(bb._capi.ClusterParam(0.2, 0.524, 0.9)), C.byref(bb._capi.Estimate()), None, None),
        lib.bb200_sharded_amcl_particle_histogram(h, 1e-3, 1e-3, None, 0, C.byref(n), None),
        lib.bb200_amcl_update(shard, dp, dpts, len(pts), C.byref(res)),
        lib.bb200_amcl_update_begin(shard, dp, C.byref(bb._capi.WeighView())),
        lib.bb200_amcl_update_end(shard, C.byref(res)),
        lib.bb200_amcl_initialize_from_map(shard),
        lib.bb200_filter_size(f, C.byref(n)),
        lib.bb200_filter_synchronize(f),
    ]
    assert refused == [STATE] * len(refused)
    lib.bb200_sharded_amcl_force_update(h)  # ignored
    b_views = (bb._capi.WeighView * k)()
    assert lib.bb200_sharded_amcl_update_begin(b._h, dp, b_views) == 0
    weigh_ones(bb, views, k)
    weigh_ones(bb, b_views, k)
    ra, rb = bb._capi.UpdateResult(), bb._capi.UpdateResult()
    assert lib.bb200_sharded_amcl_update_end(h, C.byref(ra)) == 0 and lib.bb200_sharded_amcl_update_end(b._h, C.byref(rb)) == 0
    assert ra.updated == 1 and result_tuple(ra) == result_tuple(rb)
    assert_sharded_equal(a, b)
    assert lib.bb200_sharded_amcl_update_end(h, C.byref(res)) == STATE  # closed
    # a step the policies skip: nothing reaches any shard, end still closes it
    launches = [s.launch_count() for s in a.shards]
    before = a.particles()
    assert lib.bb200_sharded_amcl_update_begin(h, dp, views) == 0 and all(views[r].updated == 0 for r in range(k))
    assert lib.bb200_sharded_amcl_initialize_from_map(h) == STATE
    assert lib.bb200_sharded_amcl_update_end(h, C.byref(res)) == 0 and res.updated == 0
    assert [s.launch_count() for s in a.shards] == launches
    after = a.particles()
    assert before[0].tobytes() == after[0].tobytes() and before[1].tobytes() == after[1].tobytes()
    # destroy with an open step
    p2 = np.ascontiguousarray(bb.se2(*scene.poses[2]))
    assert lib.bb200_sharded_amcl_update_begin(h, p2.ctypes.data_as(C.POINTER(C.c_double)), views) == 0
    a.close()
    b.close()


def test_refused_begin_on_one_shard_moves_no_shard(bb, scene):
    """Only shard 0 has a map (set through its filter view) and the plan injects: shard 0 passes begin's checks, shard 1
    refuses.  Every shard's checks run before any shard's propagate, so no shard launches anything, and the filter equals a
    twin that never saw the refused call, particles included."""
    k = 3
    a, b = sharded_twins(bb, scene, k, 1000 * k, with_map=False, recovery_probability_override=0.1, seed=4)
    sensor, params, grid = the_map(bb, "lfm", scene)
    for g in (a, b):
        g.shards[0].set_likelihood_field_map(params, grid, prob=False)
    launches = [s.launch_count() for s in a.shards]
    with pytest.raises(bb.BelugaB200Error) as e:
        a.update_weighted(bb.se2(*scene.poses[1]), lambda s, f: pytest.fail("a refused step weighs nothing"))
    assert e.value.status == STATE and [s.launch_count() for s in a.shards] == launches
    assert_sharded_equal(a, b)
    for g in (a, b):
        g.update_map(sensor, params, grid)
    for step in (1, 2):
        pose = bb.se2(*scene.poses[step])
        ra, rb = a.update(pose, scene.scans[step]), b.update(pose, scene.scans[step])
        assert result_tuple(ra) == result_tuple(rb)
        assert_sharded_equal(a, b)


def test_refused_begin_rolls_back(bb, scene):
    """A step that would inject random states needs a map: begin refuses it before any device work, and the filter then
    equals a twin that never saw the refused call."""
    n = 3 * 1000
    a, b = sharded_twins(bb, scene, 3, n, with_map=False, recovery_probability_override=0.1, seed=4)
    launches = [s.launch_count() for s in a.shards]
    with pytest.raises(bb.BelugaB200Error) as e:
        a.update_weighted(bb.se2(*scene.poses[1]), lambda s, f: pytest.fail("a refused step weighs nothing"))
    assert e.value.status == STATE and [s.launch_count() for s in a.shards] == launches
    for g in (a, b):
        g.update_map(*the_map(bb, "lfm", scene))
    for k in (1, 2):
        pose = bb.se2(*scene.poses[k])
        ra, rb = a.update(pose, scene.scans[k]), b.update(pose, scene.scans[k])
        assert result_tuple(ra) == result_tuple(rb)
        assert_sharded_equal(a, b)


def test_raising_weigh_equals_all_ones(bb, scene):
    a, b = sharded_twins(bb, scene, 2, 6000, resample_scheme=1)

    def broken(states, factors):
        raise ValueError("sensor offline")

    pose = bb.se2(*scene.poses[1])
    with pytest.raises(ValueError):
        a.update_weighted(pose, broken)
    rb = b.update_weighted(pose, lambda s, f: f.fill_(1.0))
    assert rb.updated == 1
    assert_sharded_equal(a, b)
    pose = bb.se2(*scene.poses[2])  # the step was closed: the next one runs
    assert result_tuple(a.update(pose, scene.scans[2])) == result_tuple(b.update(pose, scene.scans[2]))
    assert_sharded_equal(a, b)


@pytest.mark.parametrize("mode", ["systematic", "selective"])
def test_launch_count(bb, orc, scene, mode):
    """Per shard, a weighed step launches what the built-in step launches, with the schedule and reweight launches
    replaced by the one apply_factors launch.  A shard below 32768 particles has no schedule: both steps then launch
    begin_step, propagate and one sensor kernel (reweight_lfm or apply_factors), and the counts are equal."""
    shards = 2
    a, b = sharded_twins(bb, scene, shards, 6000 * shards, **MODES[mode])
    for k in range(4):
        pose = bb.se2(*scene.poses[k])
        la, lb = [s.launch_count() for s in a.shards], [s.launch_count() for s in b.shards]
        ra = a.update(pose, scene.scans[k])
        b.update_weighted(pose, oracle_weigh(orc, "lfm", scene, scene.scans[k]))
        if not ra.updated:
            continue
        da = [s.launch_count() - x for s, x in zip(a.shards, la)]
        db = [s.launch_count() - x for s, x in zip(b.shards, lb)]
        assert db == da, (k, da, db)


def test_launch_count_of_scheduled_shards(bb, orc, scene):
    """At 40960 particles per shard the built-in step schedules its reweight.  Every step resamples, so the host predicts
    the pose bins: the binned propagate, finish_schedule (2 launches) and reweight_lfm are 4 launches against the weighed
    step's propagate and apply_factors, 2.  Per shard the weighed step takes exactly 2 launches fewer (DESIGN.md §5)."""
    shards = 2
    a, b = sharded_twins(bb, scene, shards, 40960 * shards, resample_scheme=1)
    for k in range(3):
        pose = bb.se2(*scene.poses[k])
        la, lb = [s.launch_count() for s in a.shards], [s.launch_count() for s in b.shards]
        ra = a.update(pose, scene.scans[k])
        rb = b.update_weighted(pose, oracle_weigh(orc, "lfm", scene, scene.scans[k]))
        assert ra.updated == rb.updated == 1 and ra.resampled == 1 and result_tuple(ra) == result_tuple(rb)
        da = [s.launch_count() - x for s, x in zip(a.shards, la)]
        db = [s.launch_count() - x for s, x in zip(b.shards, lb)]
        assert [x - y for x, y in zip(da, db)] == [2] * shards, (k, da, db)


def test_two_devices(bb, orc, scene):
    if bb.device_count() < 2:
        pytest.skip("one GPU: the two-device case needs two")
    a, b = sharded_twins(bb, scene, 2, 12_000, devices=[0, 1], resample_scheme=1)
    run_sharded_twins(bb, orc, scene, a, b, "lfm", 4)
