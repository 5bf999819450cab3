"""The landmark and bearing sensor models on the device (bb200_filter_set_landmark_map / _set_bearing_map,
bb200_filter_reweight_landmarks, bb200_amcl_update_landmarks) against the oracle of tests/_landmark_oracle.py.

Weights are held to rtol 1e-11: the landmark each detection is matched to is the oracle's bit for bit (only correctly
rounded +, -, *, /, sqrt decide it), and the factor goes through exp and atan2, where CUDA's double-precision functions
are within 2 ulp of the correctly rounded result (CUDA C++ Programming Guide, "Mathematical Functions": exp 1 ulp,
atan2 2 ulp) and glibc's within 1 ulp.  A factor is exp(-a) * exp(-b) + c with a and b carrying an atan2 error of at most
3 ulp through a square, so one factor is within about (1 + 1 + 2 * 3 * |a or b|) ulp, and a product of 64 factors within
64 times that.  With |a|, |b| <= 10 here that is below 1e-11 relative; a different landmark choice moves a factor by far
more."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _landmark_oracle as lo  # noqa: E402

pytestmark = pytest.mark.gpu

STATE, INVALID = -4, -1
RTOL = 1e-11


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


def yaw_to_state(x, y, th):
    return np.stack([np.cos(th), np.sin(th), x, y], axis=1)


def random_states(rng, n, extent=10.0):
    return yaw_to_state(rng.uniform(-extent, extent, n), rng.uniform(-extent, extent, n), rng.uniform(-np.pi, np.pi, n))


def random_map(rng, n, n_categories, extent=10.0):
    pos = np.stack([rng.uniform(-extent, extent, n), rng.uniform(-extent, extent, n), rng.uniform(0.0, 2.0, n)], axis=1)
    cat = rng.integers(0, n_categories, n).astype(np.uint32)
    return pos, cat


def random_detections(rng, n, n_categories, extra_category=False):
    pos = np.stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(0.0, 2.0, n)], axis=1)
    cat = rng.integers(0, n_categories + (1 if extra_category else 0), n).astype(np.uint32)
    return pos, cat


SENSOR_POSE = (0.0, 0.0, 1.0, 0.2, -1.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.5)  # a camera looking along the robot's x


def oracle_weights(model, states, det, lmap_pos, lmap_cat, sigma=(0.5, 0.3, 1e-3)):
    lmap = lo.LandmarkMap([(*p, c) for p, c in zip(lmap_pos.tolist(), lmap_cat.tolist())])
    dets = [(*p, c) for p, c in zip(det[0].tolist(), det[1].tolist())]
    out = []
    for s in states.tolist():
        if model == "landmark":
            out.append(lo.landmark_weight(s, dets, lmap, sigma[0], sigma[1], sigma[2]))
        else:
            out.append(lo.bearing_weight(s, dets, lmap, sigma[1], SENSOR_POSE))
    return np.array(out)


def set_model(bb, f, model, pos, cat, sigma=(0.5, 0.3, 1e-3)):
    m = bb.LandmarkMap(pos, cat)
    if model == "landmark":
        f.set_landmark_map(bb.LandmarkModelParam(*sigma), m)
    else:
        f.set_bearing_map(bb.BearingModelParam(sigma[1], SENSOR_POSE), m)


def device_weights(bb, model, states, w0, det, pos, cat):
    f = bb.Filter(capacity=len(states), seed=1)
    set_model(bb, f, model, pos, cat)
    f.set_particles(states, w0)
    f.reweight_landmarks(*det)
    got = f.particles()[1]
    f.close()
    return got


def check(got, want, w0):
    want = w0 * want
    bad = ~np.isclose(got, want, rtol=RTOL, atol=0.0) & ~(np.isnan(got) & np.isnan(want))
    assert not bad.any(), (np.flatnonzero(bad)[:5], got[bad][:5], want[bad][:5])


SHAPES = [  # particles, detections, landmarks, categories, particles checked against the oracle
    (1, 1, 1, 1, None),
    (1000, 64, 64, 64, None),
    (4096, 16, 1000, 1, 300),     # four shared-memory chunks of candidates per detection
    (2000, 5, 10000, 1, 40),      # 40 chunks
    (1 << 20, 16, 1000, 1, 150),  # 1M particles
    (3000, 33, 200, 7, 300),      # detection chunks of 32 and categories the detections do not all find
]


@pytest.mark.parametrize("model", ["landmark", "bearing"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}x{s[2]}c{s[3]}")
def test_weights_match_oracle(bb, model, shape):
    n, d, l, c, checked = shape
    rng = np.random.default_rng(n + d + l + c)
    states = random_states(rng, n)
    w0 = rng.uniform(0.5, 2.0, n)
    pos, cat = random_map(rng, l, c)
    det = random_detections(rng, d, c, extra_category=(c == 7))
    got = device_weights(bb, model, states, w0, det, pos, cat)
    idx = np.arange(n) if checked is None else np.unique(np.concatenate([[0, n - 1], rng.integers(0, n, checked)]))
    check(got[idx], oracle_weights(model, states[idx], det, pos, cat), w0[idx])


@pytest.mark.parametrize("model", ["landmark", "bearing"])
def test_ties_zero_vectors_nan_and_far_states(bb, model):
    """Exact distance ties (four landmarks at distance 1 of an integer query point), exact bearing ties (landmarks on one ray
    from the sensor), a detection at the origin, a landmark at the particle, an empty category, NaN and far-away states."""
    rng = np.random.default_rng(7)
    pts = []
    for q in [(3.0, 1.0), (-2.0, 4.0)]:
        for dx, dy in [(1, 0), (0, 1), (-1, 0), (0, -1)]:
            pts.append((q[0] + dx, q[1] + dy, 0.0))
    pts += [(2.0, 0.0, 0.5), (4.0, 0.0, 1.0), (8.0, 0.0, 2.0), (0.0, 0.0, 0.0), (1.0, 1.0, 0.0)]
    pos = np.array(pts * 40)  # the same landmarks many times over: every candidate slice holds exact duplicates
    cat = np.array([k % 3 for k in range(len(pos))], dtype=np.uint32)
    xs = np.array([0.0, 1.0, -2.0, 3.0, 0.2, 0.0, 1e300, np.nan, 5e15, -0.0])
    ys = np.array([0.0, 1.0, 3.0, 0.0, -0.3, 0.0, 1.0, 0.0, -5e15, 0.0])
    ths = np.array([0.0, 0.0, np.pi / 2, np.pi, 0.1, np.nan, 0.0, 0.0, 1.0, -np.pi / 2])
    states = np.concatenate([yaw_to_state(xs, ys, ths), random_states(rng, 500, extent=4.0)])
    states[:4, 0], states[:4, 1] = [1.0, 1.0, 0.0, -1.0], [0.0, 0.0, 1.0, 0.0]  # exact rotations
    det_pos = np.array([[3.0, 1.0, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.5], [-2.0, 4.0, 0.0], [1.0, 1.0, 0.0], [0.5, 0.5, 0.5]])
    det_cat = np.array([0, 1, 2, 0, 1, 5, 2], dtype=np.uint32)  # category 5: no landmark
    w0 = np.ones(len(states))
    got = device_weights(bb, model, states, w0, (det_pos, det_cat), pos, cat)
    check(got, oracle_weights(model, states, (det_pos, det_cat), pos, cat), w0)


def test_empty_map_and_no_detections(bb):
    rng = np.random.default_rng(3)
    states = random_states(rng, 100)
    w0 = rng.uniform(0.5, 2.0, 100)
    det = random_detections(rng, 3, 2)
    empty = (np.zeros((0, 3)), np.zeros(0, dtype=np.uint32))
    assert np.array_equal(device_weights(bb, "landmark", states, w0, det, *empty), w0 * ((1e-3 * 1e-3) * 1e-3))
    assert np.array_equal(device_weights(bb, "bearing", states, w0, det, *empty), np.zeros(100))
    pos, cat = random_map(rng, 10, 2)
    assert np.array_equal(device_weights(bb, "landmark", states, w0, empty, pos, cat), w0)


def make_amcl(bb, model, pos, cat, **kw):
    params = bb.AmclParams(update_min_d=0.0, update_min_a=0.0, **kw)
    a = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), params)
    sensor = bb.SENSOR_LANDMARK if model == "landmark" else bb.SENSOR_BEARING
    m = bb.LandmarkMap(pos, cat)
    a.update_map(sensor, bb.LandmarkModelParam(0.5, 0.3, 1e-3) if model == "landmark" else bb.BearingModelParam(0.3, SENSOR_POSE), m)
    a.initialize([0.5, -0.5, 0.3], np.diag([0.5, 0.5, 0.2]))
    return a


AMCL_CASES = {
    "multinomial": dict(min_particles=800, max_particles=800),
    "systematic": dict(min_particles=800, max_particles=800, resample_scheme=1),
    "selective": dict(min_particles=800, max_particles=800, selective_resampling=True),
    "kld": dict(min_particles=100, max_particles=800),
}


@pytest.mark.parametrize("model", ["landmark", "bearing"])
@pytest.mark.parametrize("case", sorted(AMCL_CASES))
def test_amcl_trajectory_matches_oracle_factors(bb, model, case):
    """Amcl.update_landmarks against the same filter stepped by Amcl.update_weighted with the oracle's likelihoods of the
    states the step hands out: the whole Amcl step (policies, resampling, KLD, estimate) around the device model."""
    pytest.importorskip("torch")
    import torch

    rng = np.random.default_rng(11)
    pos, cat = random_map(rng, 30, 4, extent=6.0)
    a = make_amcl(bb, model, pos, cat, seed=5, **AMCL_CASES[case])
    b = make_amcl(bb, model, pos, cat, seed=5, **AMCL_CASES[case])
    pose = np.array([1.0, 0.0, 0.0, 0.0])
    for step in range(6):
        th = 0.1 * (step + 1)
        pose = np.array([math.cos(th), math.sin(th), 0.3 * (step + 1), 0.1 * step])
        det = random_detections(rng, 4, 4)
        ra = a.update_landmarks(pose, *det)

        def weigh(states, factors):
            f = oracle_weights(model, states.cpu().numpy(), det, pos, cat)
            factors.copy_(torch.from_numpy(f))

        rb = b.update_weighted(pose, weigh)
        assert (ra.updated, ra.resampled, ra.n_particles, ra.weights_degenerate) == (rb.updated, rb.resampled, rb.n_particles, rb.weights_degenerate)
        sa, wa = a.particles()
        sb, wb = b.particles()
        np.testing.assert_allclose(sa, sb, rtol=0, atol=1e-12)
        np.testing.assert_allclose(wa, wb, rtol=1e-10, atol=0)
        np.testing.assert_allclose(np.array(ra.estimate.mean), np.array(rb.estimate.mean), rtol=0, atol=1e-9)


def test_bearing_step_without_matches_is_degenerate(bb):
    rng = np.random.default_rng(2)
    pos, cat = random_map(rng, 20, 2)
    a = make_amcl(bb, "bearing", pos, cat, min_particles=500, max_particles=500)
    r = a.update_landmarks([1.0, 0.0, 0.5, 0.0], np.array([[1.0, 0.0, 0.0]]), np.array([9], dtype=np.uint32))
    assert r.updated == 1 and r.weights_degenerate == 1
    assert np.isfinite(a.particles()[0]).all()


def test_refusals_leave_the_filter_unchanged(bb):
    from beluga_b200 import BelugaB200Error

    rng = np.random.default_rng(4)
    pos, cat = random_map(rng, 20, 2)
    a = make_amcl(bb, "landmark", pos, cat, min_particles=500, max_particles=500)
    before = a.particles()
    blob = a.export_state()

    def refused(call, status=STATE):
        with pytest.raises(BelugaB200Error) as e:
            call()
        assert e.value.status == status

    refused(lambda: a.update([1.0, 0.0, 0.5, 0.0], np.ones((10, 2))))
    refused(lambda: a.update([1.0, 0.0, 0.5, 0.0], np.zeros((0, 2))))
    refused(lambda: a.filter.reweight(np.ones((10, 2))))
    refused(lambda: a.cast_rays(np.array([[1.0, 0.0, 0.0, 0.0]]), np.array([[1.0, 0.0]]), 5.0))
    field = (C.c_float * 16)()
    assert a.filter._lib.bb200_filter_get_likelihood_field(a.filter._h, field, 16) == STATE
    after = a.particles()
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    assert a.export_state() == blob  # the policies too: a retried step sees the same step
    # with the refused calls behind it, the step runs as on a fresh filter
    b = make_amcl(bb, "landmark", pos, cat, min_particles=500, max_particles=500)
    det = random_detections(rng, 3, 2)
    ra, rb = a.update_landmarks([1.0, 0.0, 0.5, 0.0], *det), b.update_landmarks([1.0, 0.0, 0.5, 0.0], *det)
    assert np.array_equal(a.particles()[0], b.particles()[0]) and tuple(ra.estimate.mean) == tuple(rb.estimate.mean)

    grid = bb.OccupancyGrid(np.zeros((20, 20), dtype=np.int8), 0.1)
    g = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=100, max_particles=100))
    g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(), grid)
    g.initialize([0.5, 0.5, 0.0], np.diag([0.1, 0.1, 0.1]))
    gb = g.particles()
    refused(lambda: g.update_landmarks([1.0, 0.0, 0.5, 0.0], *det))
    refused(lambda: g.filter.reweight_landmarks(*det))
    assert np.array_equal(gb[0], g.particles()[0]) and np.array_equal(gb[1], g.particles()[1])


def test_argument_validation(bb):
    from beluga_b200 import BelugaB200Error

    f = bb.Filter(capacity=16)
    m = bb.LandmarkMap(np.zeros((2, 3)), np.zeros(2, dtype=np.uint32))
    bad = [
        lambda: f.set_landmark_map(bb.LandmarkModelParam(0.0, 1.0, 0.1), m),
        lambda: f.set_landmark_map(bb.LandmarkModelParam(1.0, float("nan"), 0.1), m),
        lambda: f.set_landmark_map(bb.LandmarkModelParam(1.0, 1.0, 1.5), m),
        lambda: f.set_landmark_map(bb.LandmarkModelParam(1.0, 1.0, -0.1), m),
        lambda: f.set_bearing_map(bb.BearingModelParam(-1.0), m),
        lambda: f.set_bearing_map(bb.BearingModelParam(1.0, np.diag([1.0, 1.0, 1.0 + 1e-6, 0.0])[:3]), m),
        lambda: f.set_bearing_map(bb.BearingModelParam(1.0, np.diag([1.0, 1.0, -1.0, 0.0])[:3]), m),
    ]
    for call in bad:
        with pytest.raises(BelugaB200Error) as e:
            call()
        assert e.value.status == INVALID
    lib = f._lib
    assert lib.bb200_filter_reweight_landmarks(f._h, None, 3) == INVALID
    f.set_landmark_map(bb.LandmarkModelParam(), m)


def philox():
    from oracle import pyoracle

    pyoracle.build()
    return pyoracle.philox4x32_10


@pytest.mark.parametrize("explicit", [True, False])
def test_initialize_from_map_draws_the_box(bb, explicit):
    """initialize_from_map on a landmark map: MultivariateUniformDistribution<SE2d, AlignedBox2d> over the explicit bounds
    or the landmarks' own; x and y bit-exact against the counter-RNG definition, the rotation to 1e-12."""
    rng = np.random.default_rng(21)
    pos, cat = random_map(rng, 25, 3)
    lo_b, hi_b = (np.array([-3.0, -1.5, 0.0]), np.array([4.0, 2.5, 1.0])) if explicit else (None, None)
    a = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=3000, max_particles=3000, seed=17))
    a.update_map(bb.SENSOR_LANDMARK, bb.LandmarkModelParam(), bb.LandmarkMap(pos, cat, lo_b, hi_b))
    a.initialize_from_map()
    st = a.particles()[0]
    m = lo.LandmarkMap([(*p, int(c)) for p, c in zip(pos.tolist(), cat.tolist())],
                       None if lo_b is None else (tuple(lo_b), tuple(hi_b)))
    (x0, y0, _), (x1, y1, _) = m.map_limits()
    ph = philox()
    for i in list(range(50)) + [2999]:
        yaw, x, y = lo.box_state(17, i, 0, (x0, x1, y0, y1), ph)
        assert st[i, 2] == x and st[i, 3] == y
        np.testing.assert_allclose(st[i, :2], [math.cos(yaw), math.sin(yaw)], rtol=0, atol=1e-12)
    assert (st[:, 2] >= x0).all() and (st[:, 2] <= x1).all() and (st[:, 3] >= y0).all() and (st[:, 3] <= y1).all()


@pytest.mark.parametrize("model", ["landmark", "bearing"])
def test_injection_forced_by_override_draws_the_box(bb, model):
    """recovery_probability_override = 1: every slot but the first takes a state of the box (random_intersperse), and the
    step runs instead of being refused."""
    rng = np.random.default_rng(5)
    pos, cat = random_map(rng, 30, 4, extent=6.0)
    a = make_amcl(bb, model, pos, cat, min_particles=1000, max_particles=1000, recovery_probability_override=1.0)
    det = random_detections(rng, 4, 4)
    r = a.update_landmarks([1.0, 0.0, 0.3, 0.0], *det)
    assert r.updated == 1 and r.resampled == 1
    st = a.particles()[0]
    x0, x1, y0, y1 = pos[:, 0].min(), pos[:, 0].max(), pos[:, 1].min(), pos[:, 1].max()
    inside = (st[1:, 2] >= x0) & (st[1:, 2] <= x1) & (st[1:, 3] >= y0) & (st[1:, 3] <= y1)
    assert inside.all()
    assert np.unique(st[1:, 2]).size == 999  # independent draws, not copies of resampled particles


def test_kld_growth_with_the_recovery_estimator_keeps_stepping(bb):
    """KLD with the default recovery estimator: a step where the particle count grows makes the estimator inject; on a
    landmark map that draws from the box, so the filter keeps stepping."""
    rng = np.random.default_rng(8)
    pos, cat = random_map(rng, 30, 4, extent=6.0)
    a = make_amcl(bb, "landmark", pos, cat, min_particles=100, max_particles=3000)
    sizes = []
    for step in range(12):
        det = random_detections(rng, 3, 4)
        th = 0.3 * step
        r = a.update_landmarks([math.cos(th), math.sin(th), 0.5 * step, 0.0], *det)
        assert r.updated == 1
        sizes.append(r.n_particles)
    assert np.isfinite(a.particles()[0]).all()


def test_empty_box_refuses_initialize_from_map(bb):
    from beluga_b200 import BelugaB200Error

    a = bb.Amcl(bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05), bb.AmclParams(min_particles=100, max_particles=100))
    a.update_map(bb.SENSOR_LANDMARK, bb.LandmarkModelParam(), bb.LandmarkMap(np.zeros((0, 3)), np.zeros(0, dtype=np.uint32)))
    with pytest.raises(BelugaB200Error) as e:
        a.initialize_from_map()
    assert e.value.status == STATE
    a.update_map(bb.SENSOR_LANDMARK, bb.LandmarkModelParam(), bb.LandmarkMap(np.zeros((0, 3)), np.zeros(0, dtype=np.uint32), [1, 1, 0], [0, 2, 0]))
    with pytest.raises(BelugaB200Error):
        a.initialize_from_map()
