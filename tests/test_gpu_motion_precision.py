"""The kernels that write particle states, against the high-precision restatement of test_motion_precision_cpu.py.

a. The motion update (`propagate_one` through `propagate_kernel`) of every motion model and every edge case of
   `motion_cases`: each output within the per-particle bound `motion_bound` (K_MOTION = 32) of the mpmath result on a
   fixed subsample, within the sum of the device's and the oracle's bounds of the oracle on the whole array, and with
   |c^2 + s^2 - 1| <= K_UNIT eps = 8 eps.
b. The launch paths of `propagate_one` -- `propagate_kernel` without and with the device-built schedule,
   `propagate_binned_kernel` in the fused step, the batch kernel and the per-shard launches -- give the same states
   byte for byte, and the reweight after each weighs every particle exactly once, bit for bit like the oracle.
c. `initialize_normal_kernel` given the filter's transform T (K_INIT = 32), and the free-space draws of
   `initialize_from_map` and of the recovery injection (K_FREE = 16).
"""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_motion_precision_cpu import (  # noqa: E402
    CASE_ROWS, COVARIANCES, EPS, FIRST, INIT_MEAN, K_UNIT, SEED, STEP, draws_double, edge_states, exact_free_state,
    exact_normal_init, exact_propagate, free_cells, free_state_grid, motion_bound, motion_cases, sampling10, subsample,
    transform_defect, unit_defect, worst_ratio)

pytestmark = pytest.mark.gpu

SUBSAMPLE_GPU = 2000
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
WORST = {}  # case -> worst device error / bound, printed at the end of the module


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=4)


@pytest.fixture(scope="module")
def cases(orc):
    return motion_cases(orc)


def device_sampling(s):
    from beluga_b200 import _capi
    import ctypes as C

    s = np.asarray(s, dtype=np.float64)
    return _capi.MotionSampling(int(s[8]), (C.c_double * 3)(*s[0:3]), (C.c_double * 3)(*s[3:6]), (C.c_double * 2)(*s[6:8]))


def as_sampling10(ms) -> np.ndarray:
    return sampling10(ms.model, list(ms.mean), list(ms.stddev), list(ms.first_rotation))


def propagate_on_device(bb, states, s, seed, step, first_index):
    f = bb.Filter(capacity=len(states), seed=seed, first_index=first_index)
    f.set_particles(states)
    f.propagate(device_sampling(s), step)
    return f.particles()[0]


# ---- a. the motion update against the exact reference ------------------------------------------------------------------
MOTION_CASES = [f"{m}-{t}" for m in ("diff", "omni", "stationary")
                for t in ("zero-noise", "first-pi", "first-pi-ulp", "sigma10", "sigma1e3", "below-threshold", "at-threshold", "jump-100m")
                if not (m == "stationary" and t in ("below-threshold", "at-threshold", "jump-100m"))]


@pytest.mark.parametrize("name", MOTION_CASES)
def test_motion_update_inside_the_bound(bb, orc, cases, name):
    """propagate_kernel without a schedule (Filter.propagate: begin_step + propagate = 2 launches) on CASE_ROWS edge
    states whose global indices cross 2^32.  Holds every output to motion_bound (K_MOTION = 32): against mpmath on
    SUBSAMPLE_GPU rows, against the oracle on all rows (the two bounds added), and |c^2 + s^2 - 1| <= 8 eps."""
    s = cases[name]
    model = int(s[8])
    states = edge_states(CASE_ROWS)
    f = bb.Filter(capacity=CASE_ROWS, seed=SEED, first_index=FIRST)
    f.set_particles(states)
    before = f.launch_count()
    f.propagate(device_sampling(s), STEP)
    assert f.launch_count() - before == 2
    got = f.particles()[0]
    defect = unit_defect(got)
    assert defect.max() <= K_UNIT * EPS, f"{name}: |c^2 + s^2 - 1| = {defect.max() / EPS:.3g} eps at row {int(np.argmax(defect))}"
    exp = orc.motion_propagate(s, states, mode=1, seed=SEED, step=STEP, first_index=FIRST)
    d, rs = draws_double(states, s, SEED, STEP, FIRST)
    ratio_o, row, comp = worst_ratio(got, exp, 2.0 * motion_bound(model, states, d, rs))
    assert ratio_o <= 1.0, f"{name}: device vs oracle at row {row} component {'csxy'[comp]}: {ratio_o:.3g} x (2 x bound)"
    rows = subsample(CASE_ROWS, SUBSAMPLE_GPU)
    exact, d, rs = exact_propagate(states, s, SEED, STEP, FIRST, rows)
    ratio, row, comp = worst_ratio(got[rows], exact, motion_bound(model, states[rows], d, rs))
    WORST[name] = ratio
    assert ratio <= 1.0, f"{name}: device vs exact at row {rows[row]} component {'csxy'[comp]}: {ratio:.3g} x bound"


def test_device_and_oracle_motion_sampling_agree(bb, orc, cases):
    """bb.motion_sampling (the library's control -> sampling) gives the oracle's sampling for the threshold cases."""
    import test_motion_precision_cpu as cpu

    for model, motion in ((0, bb.DifferentialDriveModelParam(*cpu.ALPHAS[:4], cpu.DISTANCE_THRESHOLD)),
                          (1, bb.OmnidirectionalDriveModelParam(*cpu.ALPHAS, cpu.DISTANCE_THRESHOLD))):
        for dist in (0.5 * cpu.DISTANCE_THRESHOLD, cpu.DISTANCE_THRESHOLD, 100.0):
            pose, prev = cpu.control_pair(dist)
            got = as_sampling10(bb.motion_sampling(motion, pose, prev))
            exp = orc.motion_sampling(model, orc.OmniParam(*cpu.ALPHAS, distance_threshold=cpu.DISTANCE_THRESHOLD), pose, prev)
            assert np.array_equal(got[:9], exp[:9]), (model, dist)


# ---- b. every launch path gives the same states ------------------------------------------------------------------------
def scene_states(n: int, extent: float, seed: int, kind: str = "spread") -> np.ndarray:
    rng = np.random.default_rng(seed)
    th = rng.uniform(-math.pi, math.pi, n)
    xy = rng.uniform(0.0, extent, (n, 2))
    if kind == "point":  # one pose: every particle in one schedule bin
        th[:], xy[:] = 0.3, (0.4 * extent, 0.6 * extent)
    elif kind == "wide":  # most particles far outside the cloud's core: the edge bins
        xy = rng.standard_cauchy((n, 2)) * extent
    out = np.stack([np.cos(th), np.sin(th), xy[:, 0], xy[:, 1]], axis=1)
    if kind == "nan-far":
        out[::97] = (np.nan, np.nan, np.nan, np.nan)
        out[5::101, 2] = 1e300
        out[7::103, 3] = -1e300
    return out


PATH_SAMPLING = sampling10(0, (0.2, 0.5, -0.1), (0.1, 0.05, 0.1))


@pytest.mark.parametrize("n,kind", [(3000, "spread"), (32768, "spread"), (32769, "point"), (100_003, "wide"), (32769, "nan-far")])
def test_filter_paths_agree_and_weigh_each_particle_once(bb, orc, scene, n, kind):
    """Filter.propagate (propagate_kernel, no schedule: 2 launches) against Filter.propagate_reweight on a twin: below
    32 768 particles propagate_kernel + reweight (3 launches); from 32 768 on propagate_kernel with the moment sums and
    the device-built schedule (begin_step 1 + propagate 2 + schedule 4 + reweight 1 = 8 launches).  Both filters start
    at first_index 2^32 - 1000, as a shard's would.  States are byte-identical; every weight equals the oracle's
    likelihood-field weight of the device's own propagated state, bit for bit -- the schedule's permutation weighed
    each particle exactly once.  No bound constant: equality."""
    first = (1 << 32) - 1000
    extent = scene.cells.shape[0] * scene.resolution
    states = scene_states(n, extent, n, kind)
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    pts = scene.scans[0][::4]
    a = bb.Filter(capacity=n, seed=SEED, first_index=first)
    a.set_particles(states)
    a.propagate(device_sampling(PATH_SAMPLING), STEP)
    b = bb.Filter(capacity=n, seed=SEED, first_index=first)
    b.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid)
    b.set_particles(states)
    before = b.launch_count()
    b.propagate_reweight(device_sampling(PATH_SAMPLING), STEP, pts)
    assert b.launch_count() - before == (3 if n < 32768 else 8)
    sa, sb = a.particles()[0], b.particles()[0]
    assert sa.tobytes() == sb.tobytes()
    w = b.particles()[1]
    exp = orc.sensor_weights(orc.LFM, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution), pts, sb)
    assert w.tobytes() == exp.tobytes(), f"{int((w != exp).sum())} weights differ"


@pytest.mark.parametrize("n,init", [(3000, "normal"), (32768, "states"), (32768, "normal"), (32769, "zero-cov"),
                                    (100_003, "wide-cov"), (32769, "heading-noise")])
def test_fused_step_paths_agree(bb, orc, scene, n, init):
    """Amcl.update's fused step with the stationary model (noise 0.02 on every draw from the first update):
    after initialize_states the schedule is built on the device (propagate_kernel); after initialize (a known normal
    cloud) the host predicts the bins and propagate_binned_kernel runs -- three launches fewer, asserted against the
    device-built twin; below 32 768 there is no schedule.  The cloud may collapse to one bin (zero covariance), fill
    the edge bins (a covariance of 1e4 m^2), or have no meaningful mean heading (100 rad^2 in theta).  The resampled
    states equal a standalone Filter.propagate of the same initial states gathered by the ancestors, byte for byte,
    and the ancestors equal the oracle's multinomial draw over the oracle's weights of those propagated states, which
    holds only if each particle was weighed exactly once.  No bound constant: equality."""
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    extent = scene.cells.shape[0] * scene.resolution
    cov = {"normal": np.diag([0.25, 0.25, 0.0685]), "zero-cov": np.zeros((3, 3)), "wide-cov": np.diag([1e4, 1e4, 0.5]),
           "heading-noise": np.diag([0.5, 0.5, 100.0])}.get(init)
    mean = np.array([0.45 * extent, 0.55 * extent, 0.7])
    ap = dict(min_particles=n, max_particles=n, seed=SEED, resample_scheme=bb.RESAMPLE_MULTINOMIAL, alpha_slow=0.0,
              alpha_fast=0.0, record_ancestors=True)
    launches = {}
    for setup in ("states", "normal") if init in ("normal", "states") and n >= 32768 else (init,):
        g = bb.Amcl(bb.StationaryModelParam(), bb.AmclParams(**ap))
        g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        if setup == "states":
            g.initialize_states(scene_states(n, extent, n))
        else:
            g.initialize(mean, cov if cov is not None else np.diag([0.25, 0.25, 0.0685]))
        start = g.particles()[0]
        pose = bb.se2(*scene.poses[0])
        before = g.filter.launch_count()
        r = g.update(pose, scene.scans[0][::4])
        launches[setup] = g.filter.launch_count() - before
        assert r.updated == 1 and r.resampled == 1
        sampling = bb.motion_sampling(bb.StationaryModelParam(), pose, pose)
        twin = bb.Filter(capacity=n, seed=SEED)
        twin.set_particles(start)
        twin.propagate(sampling, 1)
        prop = twin.particles()[0]
        anc = g.filter.ancestors()
        assert g.particles()[0].tobytes() == prop[anc].tobytes(), setup
        w = orc.sensor_weights(orc.LFM, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution), scene.scans[0][::4], prop)
        idx, _, _ = orc.resample_indices(w, orc.MULTINOMIAL, seed=SEED, step=1)
        assert np.array_equal(anc, idx), f"{setup}: {int((anc != idx).sum())} ancestors differ"
    if len(launches) == 2:
        assert launches["states"] - launches["normal"] == 3, launches


@pytest.mark.parametrize("first", [(1 << 32) - 1000, (1 << 32) + 5])
def test_first_index_across_the_word_boundary(bb, first):
    """propagate_kernel keyed by first_index + i with first_index at 2^32 - 1000 (the launch crosses into the high word)
    and 2^32 + 5: n = 3000 states against the mpmath restatement keyed by the global index, within K_MOTION = 32."""
    n = 3000
    s = sampling10(0, (0.2, 0.5, -0.1), (0.3, 0.2, 0.3))
    states = edge_states(n, seed=3)
    got = propagate_on_device(bb, states, s, SEED, STEP, first)
    rows = np.union1d(subsample(n, 300), np.arange(990, 1010))
    exact, d, rs = exact_propagate(states, s, SEED, STEP, first, rows)
    ratio, row, comp = worst_ratio(got[rows], exact, motion_bound(0, states[rows], d, rs))
    assert ratio <= 1.0, f"first_index {first}: row {rows[row]} component {'csxy'[comp]} at {ratio:.3g} x bound"


def test_batch_member_keys_by_its_local_index(bb, scene):
    """batch_propagate_kernel keys a member's particle i by i alone (no first_index): after a normalising first step
    (resample_interval 3) with the stationary model, each member's states equal a standalone Filter.propagate with
    first_index 0 and the member's seed, byte for byte, and lie within K_MOTION = 32 of the exact reference."""
    n = 4096
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=s, resample_interval=3) for s in (SEED, 77)]
    batch = bb.AmclBatch([bb.StationaryModelParam()] * 2, params)
    batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    extent = scene.cells.shape[0] * scene.resolution
    starts = [scene_states(n, extent, 40 + m) for m in range(2)]
    for m in range(2):
        batch.initialize_states(m, starts[m])
    pose = bb.se2(*scene.poses[0])
    res = batch.update([pose, pose], [scene.scans[0][::4]] * 2)
    sampling = bb.motion_sampling(bb.StationaryModelParam(), pose, pose)
    for m, p in enumerate(params):
        assert res[m].updated == 1 and res[m].resampled == 0
        got = batch.particles(m)[0]
        assert got.tobytes() == propagate_on_device(bb, starts[m], as_sampling10(sampling), p.seed, 1, 0).tobytes()
        rows = subsample(n, 200)
        exact, d, rs = exact_propagate(starts[m], as_sampling10(sampling), p.seed, 1, 0, rows)
        assert worst_ratio(got[rows], exact, motion_bound(2, starts[m][rows], d, rs))[0] <= 1.0


@pytest.mark.parametrize("shards", [2, 3])
def test_shards_key_by_the_global_index(bb, scene, shards):
    """A sharded filter on one device (2 shards of 36 000 particles: each shard's fused step predicts its bins and runs
    propagate_binned_kernel; 3 shards of 24 000: propagate_kernel without a schedule), each shard keyed from its own
    first_index.  After one normalising step its states equal the single filter's byte for byte, and so do the
    normalised weights.  No bound constant: equality."""
    n = 72_000
    ap = dict(min_particles=n, max_particles=n, seed=SEED, resample_interval=3)
    single = bb.Amcl(bb.StationaryModelParam(), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.StationaryModelParam(), bb.AmclParams(**ap), devices=[0] * shards)
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    for f in (single, group):
        f.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        f.initialize(scene.initial_mean, scene.initial_cov)
    pose = bb.se2(*scene.poses[0])
    rs, rg = single.update(pose, scene.scans[0][::4]), group.update(pose, scene.scans[0][::4])
    assert rs.resampled == rg.resampled == 0
    (ss, ws), (sg, wg) = single.particles(), group.particles()
    assert ss.tobytes() == sg.tobytes()
    assert ws.tobytes() == wg.tobytes()


# ---- c. the drawn states -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("first", [0, (1 << 32) - 2000])
@pytest.mark.parametrize("name", list(COVARIANCES))
def test_initialize_normal_given_its_transform(bb, orc, name, first):
    """initialize_normal_kernel (1 launch) against exact_normal_init with the filter's cyclic Jacobi transform T
    (the oracle's normal_transform runs the same sweep), within K_INIT = 32; T T^T within K_COV = 64 eps ||C||_F."""
    cov, n = COVARIANCES[name], 4096
    f = bb.Filter(capacity=n, seed=5, first_index=first)
    before = f.launch_count()
    f.initialize_normal(INIT_MEAN, cov, n)
    assert f.launch_count() - before == 1
    got = f.particles()[0]
    t = orc.normal_transform(cov)
    worst, bound = transform_defect(cov, t)
    assert worst <= bound
    assert unit_defect(got).max() <= K_UNIT * EPS
    rows = np.union1d(subsample(n, 400), np.arange(1990, 2010))
    exact, bnd = exact_normal_init(INIT_MEAN, t, 5, first, rows)
    ratio, row, comp = worst_ratio(got[rows], exact, bnd)
    assert ratio <= 1.0, f"{name}: row {rows[row]} component {'csxy'[comp]} at {ratio:.3g} x bound"


def test_singular_covariance_refusal_boundary(bb, orc):
    """A singular PSD covariance is accepted or refused exactly as the reference's check decides on its rounded
    eigenvalues (an eigenvalue rounded to -tiny is refused, multivariate_normal_distribution.hpp:114-116): the filter
    and the oracle run the same Jacobi sweep, so they agree matrix by matrix, and both outcomes occur."""
    rng = np.random.default_rng(4)
    outcomes = set()
    for _ in range(40):
        v = rng.normal(size=3)
        cov = np.outer(v, v)  # rank 1: two eigenvalues are zero before rounding
        try:
            orc.normal_transform(cov)
            ok = True
        except RuntimeError:
            ok = False
        f = bb.Filter(capacity=8, seed=1)
        if ok:
            f.initialize_normal((0.0, 0.0, 0.0), cov, 8)
        else:
            with pytest.raises(bb.BelugaB200Error):
                f.initialize_normal((0.0, 0.0, 0.0), cov, 8)
        outcomes.add(ok)
    assert outcomes == {True, False}


@pytest.mark.parametrize("first", [0, (1 << 32) - 100])
@pytest.mark.parametrize("kind", ["one", "prime", "many"])
def test_initialize_from_map_states(bb, kind, first):
    """initialize_uniform_kernel (1 launch): particle i is random_free_state of counter_draw(seed, first_index + i, 0,
    kStreamRandomState), against exact_free_state within K_FREE = 16, on rotated origins far from zero."""
    cells, res, origin = free_state_grid(kind)
    n = 3000
    f = bb.Filter(capacity=n, seed=11, first_index=first)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(cells, res, origin))
    before = f.launch_count()
    f.initialize_uniform(n)
    assert f.launch_count() - before == 1
    got = f.particles()[0]
    rows = subsample(n, 600)
    exact, bound = exact_free_state(free_cells(cells), cells.shape[1], res, origin, 11, np.uint64(first) + rows.astype(np.uint64), 0)
    ratio, row, comp = worst_ratio(got[rows], exact, bound)
    assert ratio <= 1.0, f"{kind}: row {rows[row]} component {'csxy'[comp]} at {ratio:.3g} x bound"


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("kind", ["one", "prime", "many"])
def test_injected_states(bb, orc, kind, scheme):
    """The recovery injection of the resample (resample.cuh): slot j is injected by the oracle's coin, and an injected
    slot holds random_free_state of counter_draw(seed, j, step, kStreamRandomState), against exact_free_state within
    K_FREE = 16, for the per-slot multinomial (0) and the systematic (1) resample."""
    cells, res, origin = free_state_grid(kind)
    n, step, p = 5000, 4, 0.3
    f = bb.Filter(capacity=n, seed=9, record_ancestors=True)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(cells, res, origin))
    f.set_particles(np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)), np.random.default_rng(2).uniform(0.5, 2.0, n))
    f.build_cdf()
    assert f.resample(scheme, step=step, max_particles=n, random_state_probability=p) == n
    anc = f.ancestors()
    assert np.array_equal(anc < 0, orc.inject_flags(seed=9, step=step, probability=p, m=n).astype(bool))
    slots = np.flatnonzero(anc < 0)
    got = f.particles()[0][slots]
    exact, bound = exact_free_state(free_cells(cells), cells.shape[1], res, origin, 9, slots, step)
    ratio, row, comp = worst_ratio(got, exact, bound)
    assert ratio <= 1.0, f"{kind}: slot {slots[row]} component {'csxy'[comp]} at {ratio:.3g} x bound"


def test_zz_report_worst_ratios():
    """Prints the worst device error / bound of every motion case (pytest -s shows it)."""
    print("device worst error / bound:", ", ".join(f"{k}: {v:.3f}" for k, v in WORST.items()))
