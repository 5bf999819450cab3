"""The weight pipeline after the sensor models -- largest weight, fixed-point CDF, normalisation factor S = T * 2^-e,
resampling, the step's moments -- against the oracle at the edges of the double range: largest weights from the smallest
subnormal to DBL_MAX, dust spread over ~1100 binades, zero, -0, negative, NaN and infinite weights among them, weight sets
in which no weight can be selected (the uniform fallback CDF), and the 1080-beam prob model whose exp(sum log pz)
underflows.  Every place a CDF gets built is covered: Filter::build_cdf, the fused single-filter step, the batch step and
the rebuild inside batch sample_states.

CDFs, totals, exponents, ancestors and normalised weights are bit-exact (w / S is one IEEE division on both sides);
estimates use the tolerances of test_gpu_parity.py."""
import math
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DBL_MAX = sys.float_info.max
WMAX = [5e-324, 2.2250738585072014e-308, 1e-300, 1.0, 1e300, DBL_MAX]
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
ALPHAS = (0.1, 0.05, 0.1, 0.05)
DEGENERATE_ERROR = "no positive finite weight (uniform CDF substituted)"


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=6)


@pytest.fixture(scope="module")
def bench_scene():
    """The bench's scan (1080 beams) on a smaller grid of the same generator."""
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=500, n_beams=1080, steps=4)


def selectable(w):
    return (w > 0.0) & (w <= DBL_MAX)


def ceil_log2(n):
    return max(int(n) - 1, 0).bit_length()


def id_states(n):
    """Identity rotations with x = the particle's index: a resampled state names its ancestor."""
    states = np.tile(np.array([1.0, 0.0, 0.0, 0.0]), (n, 1))
    states[:, 2] = np.arange(n)
    return states


def edge_weights(rng, n, wmax, plus_inf=True):
    """wmax at one position; the rest dust over ~1100 binades below it (subnormals and zeros included) and, at scattered
    positions, 0.0, -0.0, negatives, NaN, -inf and +inf."""
    w = np.ldexp(wmax * rng.uniform(0.5, 1.0, n), -rng.integers(0, 1100, n))
    specials = [0.0, -0.0, -1.0, -DBL_MAX, -5e-324, float("nan"), -float("inf")] + ([float("inf")] if plus_inf else [])
    if n > 1:
        pos = rng.permutation(n)[: max(len(specials), n // 40)]
        w[pos] = np.resize(np.array(specials), len(pos))
    w[rng.integers(0, n)] = wmax
    return w


def same_doubles(a, b):
    """Equal as doubles, NaN matching NaN and the sign of zero included."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and np.array_equal(np.signbit(a), np.signbit(b))


def last_error(f):
    return f._lib.bb200_last_error(f._h).decode()


def free_map(bb):
    """A small map with free cells, for the recovery injection of the per-slot resample form."""
    cells = np.zeros((20, 20), dtype=np.int8)
    cells[0, :] = 100
    return bb.OccupancyGrid(cells, 0.5)


def check_resample(bb, orc, states, w, capacity, seed, step, scheme, m, p_inject=0.0):
    """One resample on a fresh filter against the oracle's comb over its CDF."""
    f = bb.Filter(capacity=capacity, seed=seed, record_ancestors=True)
    if p_inject > 0.0:
        f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), free_map(bb))
    f.set_particles(states, w)
    total, ex = f.build_cdf()
    idx, cdf, ex_o, valid = orc.resample_indices(w, scheme, seed=seed, step=step, m=m, n_total=capacity, return_valid=True)
    assert valid
    assert ex == ex_o and total == int(cdf[-1])
    assert np.array_equal(f.cdf(), cdf)
    assert np.all(np.diff(cdf.astype(np.float64)) >= 0.0)
    assert f.resample(scheme, step=step, max_particles=m, random_state_probability=p_inject) == m
    anc = f.ancestors()
    want = idx.copy()
    if p_inject > 0.0:
        want[orc.inject_flags(seed=seed, step=step, probability=p_inject, m=m).astype(bool)] = -1
    assert np.array_equal(anc, want)
    new_states, new_w = f.particles()
    kept = anc >= 0
    assert np.array_equal(new_states[kept, 2], anc[kept].astype(np.float64)) and np.all(new_w == 1.0)
    assert np.all(selectable(w[anc[kept]]))  # no excluded weight is ever an ancestor


# ---- a. Filter level ---------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2048, 2049, 100_003])
@pytest.mark.parametrize("wmax", WMAX)
@pytest.mark.parametrize("inf", ["finite_specials", "plus_inf"])
def test_filter_cdf_resample_normalize_at_the_edges(bb, orc, wmax, n, inf):
    rng = np.random.default_rng(n + WMAX.index(wmax))
    w = edge_weights(rng, n, wmax, plus_inf=(inf == "plus_inf"))
    assert w.max(initial=0.0, where=selectable(w)) == wmax
    capacity = 3 * n + 5  # the exponent follows the capacity, not the particle count
    states = id_states(n)
    seed = 1000 + n
    check_resample(bb, orc, states, w, capacity, seed, 3, bb.RESAMPLE_MULTINOMIAL, n)
    check_resample(bb, orc, states, w, capacity, seed, 4, bb.RESAMPLE_SYSTEMATIC, n)  # scatter form
    check_resample(bb, orc, states, w, capacity, seed, 5, bb.RESAMPLE_SYSTEMATIC, 2 * n + 1)  # scatter form, more slots than particles
    check_resample(bb, orc, states, w, capacity, seed, 6, bb.RESAMPLE_SYSTEMATIC, n, p_inject=0.3)  # per-slot form
    check_resample(bb, orc, states, w, capacity, seed, 7, bb.RESAMPLE_MULTINOMIAL, n, p_inject=0.3)
    if n <= 2049:  # KLD-sized: take_while_kld over the comb of max_particles slots
        f = bb.Filter(capacity=n, seed=seed, record_ancestors=True)
        f.set_particles(states, w)
        res = (0.5, 0.5, 0.5)
        got = f.resample(bb.RESAMPLE_SYSTEMATIC, step=8, max_particles=n, min_particles=max(n // 8, 1), spatial_resolution=res)
        idx, _, _ = orc.resample_indices(w, bb.RESAMPLE_SYSTEMATIC, seed=seed, step=8, m=n)
        hashes = [orc.spatial_hash(states[i], *res) for i in idx]
        assert got == orc.kld_take_count(hashes, max(n // 8, 1), n, 0.05, 3.0)
        assert np.array_equal(f.ancestors(), idx[:got])
    # normalisation: w / S with S = T * 2^-e, one IEEE division per weight (S overflows to inf when the weights sum past
    # DBL_MAX, as the reference's sum does); the ESS on the same set with every weight that cannot be selected set to 0
    for ws in (w, np.where(selectable(w), w, 0.0)):
        f = bb.Filter(capacity=capacity, seed=seed)
        f.set_particles(states, ws)
        factor, sum_sq = f.normalize()
        _, cdf, ex = orc.resample_indices(ws, bb.RESAMPLE_MULTINOMIAL, seed=seed, step=1, n_total=capacity)
        with np.errstate(over="ignore", invalid="ignore"):
            s = float(np.ldexp(float(int(cdf[-1])), -ex))  # inf past DBL_MAX, like std::ldexp
            want = ws / s
        assert factor == s
        assert same_doubles(f.particles()[1], want)
        if np.all(ws >= 0.0) and sum_sq > 0.0:
            assert sum_sq == pytest.approx(float(np.sum(want * want)), rel=1e-12)
            assert 1.0 / sum_sq == pytest.approx(orc.effective_sample_size(want), rel=1e-9)


# ---- b. degenerate weight sets: the uniform fallback -------------------------------------------------
DEGENERATE = {"zero": 0.0, "nan": float("nan"), "negative": None, "minus_inf": -float("inf"), "plus_inf": float("inf")}


def degenerate_weights(kind, n, rng):
    if kind == "negative":
        return -rng.uniform(0.5, 2.0, n)
    w = np.full(n, DEGENERATE[kind])
    if kind == "zero":
        w[::3] = -0.0
    return w


@pytest.mark.parametrize("kind", list(DEGENERATE))
def test_degenerate_sets_take_the_uniform_cdf(bb, orc, kind):
    rng = np.random.default_rng(11)
    n, capacity = 2049, 4096
    w = degenerate_weights(kind, n, rng)
    states = id_states(n)
    for scheme, m in ((bb.RESAMPLE_MULTINOMIAL, n), (bb.RESAMPLE_SYSTEMATIC, n), (bb.RESAMPLE_SYSTEMATIC, 3000)):
        f = bb.Filter(capacity=capacity, seed=21, record_ancestors=True)
        f.set_particles(states, w)
        total, ex = f.build_cdf()
        assert last_error(f) == DEGENERATE_ERROR
        assert np.array_equal(f.cdf(), (np.arange(n, dtype=np.uint64) + 1) << np.uint64(20))
        assert total == n << 20 and ex == min(52, 62 - ceil_log2(capacity))
        idx, cdf, ex_o, valid = orc.resample_indices(w, scheme, seed=21, step=2, m=m, n_total=capacity, return_valid=True)
        assert not valid and ex_o == ex and np.array_equal(f.cdf(), cdf)
        assert f.resample(scheme, step=2, max_particles=m) == m
        assert np.array_equal(f.ancestors(), idx)
    # normalising leaves the weights as they are; the estimate is the reference's 0 / 0 where the weights sum to 0, NaN or inf
    f = bb.Filter(capacity=capacity)
    f.set_particles(states, w)
    factor, _ = f.normalize()
    assert factor == math.ldexp(float(n << 20), -ex)
    assert same_doubles(f.particles()[1], w)
    mean, _ = f.estimate()
    if kind == "negative":
        want, _ = orc.estimate(states, w)
        assert np.allclose(mean, want, rtol=0.0, atol=1e-9)
    else:
        assert np.isnan(mean[2]) and np.isnan(mean[3])


@pytest.mark.parametrize("interval", [1, 2])
@pytest.mark.parametrize("kind", list(DEGENERATE))
def test_degenerate_amcl_steps_match_the_oracle(bb, orc, scene, kind, interval):
    """A whole Amcl step on a degenerate set: weights_degenerate, the uniform comb's ancestors, and a normalising step that
    leaves the weights untouched -- all as oracle::Amcl does it."""
    n = 3000
    rng = np.random.default_rng(12)
    th = rng.normal(scene.initial_mean[2], 0.1, n)
    states = np.stack([np.cos(th), np.sin(th), rng.normal(scene.initial_mean[0], 0.2, n), rng.normal(scene.initial_mean[1], 0.2, n)], 1)
    w = degenerate_weights(kind, n, rng)
    ap = dict(min_particles=n, max_particles=n, seed=31, resample_interval=interval)
    g = bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(resample_scheme=1, record_ancestors=True, **ap))
    o = orc.Amcl(orc.AmclParam(rng_mode=1, scheme=1, **ap), orc.MotionParam(*ALPHAS))
    g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    o.set_map(orc.LFM, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
    g.initialize_states(states, w)
    o.set_particles(states, w)
    degenerate = True  # until a resample from the uniform comb gives every particle weight 1
    for k in range(3):
        pose = orc.se2(*scene.poses[k])
        rg, ro = g.update(pose, scene.scans[k]), o.update(pose, scene.scans[k])
        assert rg.updated == ro.updated == 1 and rg.resampled == ro.resampled
        assert rg.weights_degenerate == int(degenerate), k
        assert rg.weight_sum == pytest.approx(ro.weight_sum, rel=1e-12)
        if rg.resampled:
            assert np.array_equal(g.filter.ancestors(), o.last_indices()), k
        elif degenerate:  # reweighted, never normalised
            gw, ow = g.particles()[1], o.particles()[1]
            if kind == "negative":
                assert np.all(gw < 0.0) and np.allclose(gw, ow, rtol=1e-12, atol=0.0)
            else:
                assert same_doubles(gw, ow)
        if rg.resampled or kind == "negative" or not degenerate:
            assert np.abs(np.array(rg.estimate.mean) - np.array(ro.mean)).max() < 1e-10, k
        else:
            assert np.isnan(rg.estimate.mean[2]) and np.isnan(ro.mean[2])
        degenerate = degenerate and not rg.resampled


# ---- c. the fused single-filter step: the exponent from the reweight kernel's wmax_bits -------------------
def extreme_initial_weights(shape, rng, n):
    """Weights that, after one likelihood-field reweight (a factor in [1, 182] with 181 beams), put the largest weight in a
    subnormal, next to DBL_MAX, or overflow some weights to +inf."""
    if shape == "subnormal":
        return 5e-324 * rng.integers(1, 40, n).astype(np.float64)
    if shape == "near_max":  # two heavy particles (their sum stays below DBL_MAX) among ordinary ones
        w = rng.uniform(0.5, 1.0, n)
        w[rng.permutation(n)[:2]] = DBL_MAX / 400.0
        return w
    w = 1e300 * rng.uniform(0.5, 1.0, n)
    w[rng.permutation(n)[:50]] = DBL_MAX * 0.9  # overflow to +inf in the reweight
    return w


def normal_cloud(rng, mean, n, spread=0.2):
    th = rng.normal(mean[2], 0.1, n)
    return np.stack([np.cos(th), np.sin(th), rng.normal(mean[0], spread, n), rng.normal(mean[1], spread, n)], 1)


@pytest.mark.parametrize("interval", [1, 3])
@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("shape", ["subnormal", "near_max", "plus_inf"])
def test_fused_step_with_extreme_weights(bb, orc, scene, shape, scheme, interval):
    n = 5000
    rng = np.random.default_rng(40 + scheme)
    states = normal_cloud(rng, scene.initial_mean, n)
    w = extreme_initial_weights(shape, rng, n)
    ap = dict(min_particles=n, max_particles=n, seed=55, resample_interval=interval)
    g = bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(resample_scheme=scheme, record_ancestors=True, **ap))
    o = orc.Amcl(orc.AmclParam(rng_mode=1, scheme=scheme, **ap), orc.MotionParam(*ALPHAS))
    g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    o.set_map(orc.LFM, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
    g.initialize_states(states, w)
    o.set_particles(states, w)
    resampled = 0
    for k in range(4):
        pose = orc.se2(*scene.poses[k])
        rg, ro = g.update(pose, scene.scans[k]), o.update(pose, scene.scans[k])
        assert rg.updated == ro.updated == 1 and rg.resampled == ro.resampled
        assert rg.weights_degenerate == 0
        assert rg.weight_sum == pytest.approx(ro.weight_sum, rel=1e-12)
        if rg.resampled:
            resampled += 1
            anc = g.filter.ancestors()
            assert np.array_equal(anc, o.last_indices())
        gm, om = np.array(rg.estimate.mean), np.array(ro.mean)
        if np.all(np.isfinite(om)):  # a normalising step's estimate with a +inf weight is not pinned
            assert np.abs(gm - om).max() < 1e-10
    assert resampled == (4 if interval == 1 else 1)


# ---- d. the prob model at 1080 beams -----------------------------------------------------------------
def test_prob_model_partial_underflow(bb, orc, bench_scene):
    """exp(sum log pz) over 1080 beams: near the pose the likelihood is ~1e-5, farther out it underflows; with initial
    weights of 1e-304 the largest weight is subnormal and many are 0.  The GPU's own weights go to the oracle's CDF, so
    libm ulps stay out of the check of the integer pipeline."""
    sc = bench_scene
    n = 4000
    rng = np.random.default_rng(5)
    states = normal_cloud(rng, sc.poses[0], n, spread=0.08)
    states[:, 2] += np.where(np.arange(n) % 4 == 0, 0.5, 0.0)  # a quarter far enough out to underflow
    w0 = np.full(n, 1e-304)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    f = bb.Filter(capacity=n, seed=8, record_ancestors=True)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid, prob=True)
    f.set_particles(states, w0)
    f.reweight(sc.scans[0])
    got = f.particles()[1]
    exp = w0 * orc.sensor_weights(orc.LFM_PROB, orc.LfmParam(**LFM), orc.Grid(sc.cells, sc.resolution), sc.scans[0], states)
    assert 0.0 < got.max() < 2.2250738585072014e-308 and (got == 0.0).any()
    assert np.allclose(got, exp, rtol=1e-6, atol=1e-320)  # test_reweight_lfm_bit_exact's bound for subnormal weights
    for scheme in (bb.RESAMPLE_MULTINOMIAL, bb.RESAMPLE_SYSTEMATIC):
        g = bb.Filter(capacity=n, seed=8, record_ancestors=True)
        g.set_particles(id_states(n), got)
        total, ex = g.build_cdf()
        idx, cdf, ex_o, valid = orc.resample_indices(got, scheme, seed=8, step=2, return_valid=True)
        assert valid and ex == ex_o and total == int(cdf[-1]) and np.array_equal(g.cdf(), cdf)
        assert g.resample(scheme, step=2, max_particles=n) == n
        anc = g.ancestors()
        assert np.array_equal(anc, idx) and np.all(got[anc] > 0.0)


def test_prob_model_full_underflow(bb, orc, bench_scene):
    """Poses far from every obstacle: every weight underflows to 0, the step takes the uniform comb; once the filter is back
    near the walls the next step is an ordinary one."""
    sc = bench_scene
    n = 3000
    rng = np.random.default_rng(6)
    ap = dict(min_particles=n, max_particles=n, seed=66)
    g = bb.Amcl(bb.DifferentialDriveModelParam(*ALPHAS), bb.AmclParams(resample_scheme=1, record_ancestors=True, **ap))
    g.update_map(bb.SENSOR_LIKELIHOOD_FIELD_PROB, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(sc.cells, sc.resolution))
    far = normal_cloud(rng, (-400.0, 300.0, 0.0), n)
    g.initialize_states(far)
    r = g.update(orc.se2(*sc.poses[0]), sc.scans[0])
    assert r.updated == 1 and r.resampled == 1 and r.weights_degenerate == 1
    idx, _, _, valid = orc.resample_indices(np.zeros(n), orc.SYSTEMATIC, seed=66, step=1, return_valid=True)
    assert not valid and np.array_equal(g.filter.ancestors(), idx)
    g.initialize_states(normal_cloud(rng, sc.poses[0], n, spread=0.03))  # the next update moves them by poses[0] -> poses[1]
    r = g.update(orc.se2(*sc.poses[1]), sc.scans[1])
    assert r.updated == 1 and r.weights_degenerate == 0
    assert np.hypot(r.estimate.mean[2] - sc.poses[1][0], r.estimate.mean[3] - sc.poses[1][1]) < 0.2


# ---- e. the batch -------------------------------------------------------------------------------------
BATCH_MEMBERS = [("subnormal", 1, 1), ("plus_inf", 1, 1), ("near_max", 0, 3), ("zero", 1, 1), ("nan", 0, 2), ("ordinary", 1, 1),
                 ("plus_inf", 0, 3)]


def test_batch_members_with_extreme_weights_match_the_oracle(bb, orc, scene):
    """AmclBatch members holding the shapes of the fused-step and degenerate tests next to ordinary members, each compared
    with oracle::Amcl directly; then sample_states rebuilding a member's CDF from extreme weights."""
    rng = np.random.default_rng(70)
    k = len(BATCH_MEMBERS)
    sizes = [2000 + 700 * m for m in range(k)]
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=90 + m, resample_scheme=s, resample_interval=iv, record_ancestors=True)
              for m, ((_, s, iv), n) in enumerate(zip(BATCH_MEMBERS, sizes))]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(*ALPHAS)] * k, params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    oracles = []
    for m, ((shape, s, iv), n) in enumerate(zip(BATCH_MEMBERS, sizes)):
        states = normal_cloud(rng, scene.initial_mean, n)
        if shape in ("zero", "nan"):
            w = degenerate_weights(shape, n, rng)
        elif shape == "ordinary":
            w = rng.uniform(0.5, 3.0, n)
        else:
            w = extreme_initial_weights(shape, rng, n)
        batch.initialize_states(m, states, w)
        o = orc.Amcl(orc.AmclParam(rng_mode=1, scheme=s, min_particles=n, max_particles=n, seed=90 + m, resample_interval=iv), orc.MotionParam(*ALPHAS))
        o.set_map(orc.LFM, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution))
        o.set_particles(states, w)
        oracles.append(o)
    degenerate = [shape in ("zero", "nan") for shape, _, _ in BATCH_MEMBERS]
    for t in range(3):
        poses = [orc.se2(*scene.poses[t])] * k
        got = batch.update(poses, [scene.scans[t]] * k)
        for m, o in enumerate(oracles):
            ro = o.update(poses[m], scene.scans[t])
            rg = got[m]
            assert rg.updated == ro.updated == 1 and rg.resampled == ro.resampled, (t, m)
            assert rg.weights_degenerate == int(degenerate[m]), (t, m)
            degenerate[m] = degenerate[m] and not rg.resampled
            assert rg.weight_sum == pytest.approx(ro.weight_sum, rel=1e-12), (t, m)
            if rg.resampled:
                assert np.array_equal(batch.ancestors(m), o.last_indices()), (t, m)
            gm, om = np.array(rg.estimate.mean), np.array(ro.mean)
            if np.all(np.isfinite(om)):  # a normalising step's estimate with a +inf or NaN weight is not pinned
                assert np.abs(gm - om).max() < 1e-10, (t, m)
    # sample_states: members whose CDF must be rebuilt from extreme weights (and one degenerate set)
    count = 1500
    sets = {}
    for m in range(k):
        n = sizes[m]
        shape = BATCH_MEMBERS[m][0]
        w = edge_weights(rng, n, WMAX[m % len(WMAX)]) if shape != "zero" else degenerate_weights("zero", n, rng)
        batch.initialize_states(m, id_states(n), w)
        sets[m] = w
    draws = batch.sample_states(count, step=77)
    for m in range(k):
        idx, _, _, valid = orc.resample_indices(sets[m], orc.MULTINOMIAL, seed=90 + m, step=77, m=count, n_total=sizes[m], return_valid=True)
        assert valid == (BATCH_MEMBERS[m][0] != "zero")
        assert np.array_equal(draws[m][:, 2], idx.astype(np.float64)), m
        if valid:
            assert np.all(selectable(sets[m][idx]))
