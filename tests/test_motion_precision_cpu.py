"""A high-precision restatement of every kernel that writes particle states, and the error bound the kernels are held to.

The motion update (`propagate_one`, propagate.cuh), the normal initialisation (`initialize_normal_kernel`) and the
free-space draw (`random_free_state`, used by `initialize_from_map` and by the recovery injection of the resample) all
start from Philox4x32-10 counter draws.  Given the draw, each is a short real-valued formula, so the exact result can be
computed: the functions below do it in mpmath at `DPS` significant digits from the double uniforms the kernels draw
(`uniform01`; from 1/2 up they are rounded, which both the device and the oracle share).

Neither the device nor the oracle computes that formula exactly.  The oracle rounds 2*pi*u before cos / sin, divides
through hypot and applies Sophus' 2 / (1 + |z|^2) rescale; the device uses cospi / sincospi, sqrt and a reciprocal,
and skips the rescale (se2_math.cuh:102-148).  Both are held to one first-order bound per particle and component
(`motion_bound`), with eps = 2^-53:

    |c - c*|, |s - s*| <= K eps * PHI
    |x - x*|, |y - y*| <= K eps * (|x| + |y| + LIN + LEVER * PHI)

    PHI   = 1 + sum over the sampled angles   (|d_k| + r_k sigma_k)
    LIN   =     sum over the sampled lengths  (|d_k| + r_k sigma_k)
    LEVER =     sum over the sampled lengths   |d_k|

r_k is the Box-Muller radius of draw k, so r_k sigma_k bounds the absolute error a relative error of the normal carries
into d_k = z_k sigma_k + mu_k; the angles are d0 (and d2 for the differential drive), the lengths d1 (and d2 for the
omnidirectional and stationary models).  LEVER * PHI is a heading error swung through the translation.  K = K_MOTION
= 32 covers about a dozen roundings per term: the Box-Muller angle (the oracle's rounded 2*pi*u costs up to ~8.5 eps
times r), the log / sqrt of the radius, sincos, two or three rotation products with their normalisation, and the
additions of the composition.  |c^2 + s^2 - 1| <= K_UNIT eps = 8 eps holds for every normalised output.

The tests here pin the restatement to the oracle before any device number is read: the NumPy Philox to the oracle's,
and the oracle (`orc.motion_propagate`, counter mode) inside the bound on every case the GPU tests use.
"""
from __future__ import annotations

import math
import os
import sys

import mpmath
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

EPS = 2.0 ** -53
DPS = 50
K_MOTION = 32.0
K_UNIT = 8.0
K_INIT = 32.0
K_FREE = 16.0
K_COV = 64.0
PI = math.pi

# Stream identifiers of the counter (se2_math.cuh `Stream`).
INIT0, INIT1, MOTION0, MOTION1, RESAMPLE, SYSTEMATIC, RANDOM_STATE = range(7)

_M32 = np.uint64(0xFFFFFFFF)


# ---- Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11), vectorised ---------------------------------------------------
def philox4x32_10(ctr, key) -> np.ndarray:
    """ctr (..., 4) and key (..., 2) of uint32 -> (..., 4) uint32."""
    c = np.asarray(ctr, dtype=np.uint64)
    k = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (c[..., i].copy() for i in range(4))
    k0, k1 = k[..., 0].copy(), k[..., 1].copy()
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0  # < 2^64: the full 32x32 product
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def counter_draw(seed: int, index, step: int, stream: int):
    """counter_draw (se2_math.cuh:176): counter (index lo, index hi, step, stream), key = seed -> two uint64 words."""
    idx = np.atleast_1d(np.asarray(index, dtype=np.uint64))
    ctr = np.stack([idx & _M32, idx >> np.uint64(32), np.full_like(idx, step), np.full_like(idx, stream)], axis=-1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64), (len(idx), 2))
    v = philox4x32_10(ctr, key).astype(np.uint64)
    return (v[:, 1] << np.uint64(32)) | v[:, 0], (v[:, 3] << np.uint64(32)) | v[:, 2]


def uniform01(bits) -> np.ndarray:
    """uniform01 (se2_math.cuh:194) as the kernels compute it: ((bits >> 11) + 0.5) * 2^-53 in double.  The sum is exact
    below 1/2 only: from 2^52 on, k + 0.5 needs 54 bits and rounds to even (the top word rounds to exactly 1.0)."""
    k = np.asarray(bits, dtype=np.uint64) >> np.uint64(11)
    return (k.astype(np.float64) + 0.5) * 2.0 ** -53


def uniform01_mp(bits: int):
    """The double uniform01 returns, as an exact mpmath number: every later step of the restatement is exact."""
    return mpmath.mpf(float(uniform01(bits)))


def mulhi64(a: int, b: int) -> int:
    return (int(a) * int(b)) >> 64


# ---- exact SE(2) --------------------------------------------------------------------------------------------------------
def _unit(c, s):
    h = mpmath.sqrt(c * c + s * s)
    return c / h, s / h


def _rot_mul(a, b):
    """Sophus SO2 product: complex product, then normalised (the 2 / (1 + |z|^2) rescale cancels exactly)."""
    return _unit(a[0] * b[0] - a[1] * b[1], a[0] * b[1] + a[1] * b[0])


def _pose_mul(a, b):
    """Sophus SE2 product: the translation is rotated by a's stored (unnormalised) complex."""
    c, s = _rot_mul(a[:2], b[:2])
    return (c, s, a[2] + a[0] * b[2] - a[1] * b[3], a[3] + a[1] * b[2] + a[0] * b[3])


def _exp(theta):
    return mpmath.cos(theta), mpmath.sin(theta)


def motion_apply_exact(model: int, st, d, first):
    """motion_apply (se2_math.cuh:88-99) in exact arithmetic; st and first hold the stored doubles."""
    mp = mpmath.mpf
    st = tuple(mp(float(v)) for v in st)
    if model == 1:
        f = (mp(float(first[0])), mp(float(first[1])))
        second = _rot_mul(_exp(d[0]), _unit(f[0], -f[1]))
        a = _pose_mul(st, (f[0], f[1], mp(0), mp(0)))
        return _pose_mul(a, (second[0], second[1], d[1], -d[2]))
    if model == 2:
        r = _exp(d[0])
        return _pose_mul(st, (r[0], r[1], d[1], d[2]))
    r1, r2 = _exp(d[0]), _exp(d[2])
    a = _pose_mul(st, (r1[0], r1[1], mp(0), mp(0)))
    return _pose_mul(a, (r2[0], r2[1], d[1], mp(0)))


def _box_muller_exact(a_bits: int, b_bits: int):
    r = mpmath.sqrt(-2 * mpmath.log(uniform01_mp(a_bits)))
    ang = 2 * mpmath.pi * uniform01_mp(b_bits)
    return r, r * mpmath.cos(ang), r * mpmath.sin(ang)


def exact_propagate(states, sampling10, seed: int, step: int, first_index: int, rows=None):
    """The exact motion update of states[rows] (default all), keyed by the global index first_index + row.

    Returns (exact states (m, 4) rounded to double, draws d (m, 3), r_k sigma_k (m, 3)); the latter two feed
    `motion_bound`.  The exact states are rounded only at the end, so they are within half an ulp of the real value."""
    states = np.asarray(states, dtype=np.float64).reshape(-1, 4)
    rows = np.arange(len(states)) if rows is None else np.asarray(rows)
    s = np.asarray(sampling10, dtype=np.float64)
    mean, std, first, model = s[0:3], s[3:6], s[6:8], int(s[8])
    idx = np.uint64(first_index) + rows.astype(np.uint64)
    a0, b0 = counter_draw(seed, idx, step, MOTION0)
    a1, b1 = counter_draw(seed, idx, step, MOTION1)
    out, dd, rs = np.zeros((len(rows), 4)), np.zeros((len(rows), 3)), np.zeros((len(rows), 3))
    with mpmath.workdps(DPS):
        for j, i in enumerate(rows):
            r0, z0, z1 = _box_muller_exact(a0[j], b0[j])
            r1, z2, _ = _box_muller_exact(a1[j], b1[j])
            d = [z0 * mpmath.mpf(std[0]) + mpmath.mpf(mean[0]), z1 * mpmath.mpf(std[1]) + mpmath.mpf(mean[1]),
                 z2 * mpmath.mpf(std[2]) + mpmath.mpf(mean[2])]
            out[j] = [float(v) for v in motion_apply_exact(model, states[i], d, first)]
            dd[j] = [float(v) for v in d]
            rs[j] = [float(r0 * std[0]), float(r0 * std[1]), float(r1 * std[2])]
    return out, dd, rs


def draws_double(states, sampling10, seed: int, step: int, first_index: int):
    """d (n, 3) and r_k sigma_k (n, 3) of every row in double: the magnitudes `motion_bound` needs for a whole array."""
    n = len(np.asarray(states).reshape(-1, 4))
    s = np.asarray(sampling10, dtype=np.float64)
    idx = np.uint64(first_index) + np.arange(n, dtype=np.uint64)
    a0, b0 = counter_draw(seed, idx, step, MOTION0)
    a1, b1 = counter_draw(seed, idx, step, MOTION1)
    r0, r1 = np.sqrt(-2.0 * np.log(uniform01(a0))), np.sqrt(-2.0 * np.log(uniform01(a1)))
    t0, t1 = 2.0 * PI * uniform01(b0), 2.0 * PI * uniform01(b1)
    z = np.stack([r0 * np.cos(t0), r0 * np.sin(t0), r1 * np.cos(t1)], axis=1)
    return z * s[3:6] + s[0:3], np.stack([r0, r0, r1], axis=1) * s[3:6]


def motion_bound(model: int, states, d, rs):
    """Per-particle, per-component error bound (module docstring) -> (m, 4): c, s, x, y."""
    st = np.abs(np.asarray(states, dtype=np.float64).reshape(-1, 4))
    ad = np.abs(d)
    angles, lengths = ([0, 2], [1]) if model == 0 else ([0], [1, 2])
    phi = 1.0 + sum(ad[:, k] + rs[:, k] for k in angles)
    lin = sum(ad[:, k] + rs[:, k] for k in lengths)
    lever = sum(ad[:, k] for k in lengths)
    rot = K_MOTION * EPS * phi
    xy = K_MOTION * EPS * (st[:, 2] + st[:, 3] + lin + lever * phi)
    return np.stack([rot, rot, xy, xy], axis=1)


def unit_defect(states) -> np.ndarray:
    """|c^2 + s^2 - 1| of each state, in extended precision where the platform has it."""
    c = np.asarray(states)[:, 0].astype(np.longdouble)
    s = np.asarray(states)[:, 1].astype(np.longdouble)
    return np.abs(c * c + s * s - 1).astype(np.float64)


def worst_ratio(got, exact, bound) -> tuple[float, int, int]:
    """The largest |got - exact| / bound over every finite row and component, and where it is."""
    err = np.abs(np.asarray(got) - exact)
    ratio = np.where(np.isfinite(exact), err / bound, 0.0)
    k = int(np.argmax(ratio))
    return float(ratio.flat[k]), k // 4, k % 4


# ---- the normal initialisation ------------------------------------------------------------------------------------------
def exact_normal_init(mean, transform, seed: int, first_index: int, rows):
    """initialize_normal_kernel (propagate.cu:18-31) given its transform T: (x, y, theta) = mean + T delta with the exact
    Box-Muller normals of streams 0 and 1 at step 0 -> (exact states, bound (m, 4))."""
    mean = np.asarray(mean, dtype=np.float64)
    t = np.asarray(transform, dtype=np.float64).reshape(3, 3)
    rows = np.asarray(rows)
    idx = np.uint64(first_index) + rows.astype(np.uint64)
    a0, b0 = counter_draw(seed, idx, 0, INIT0)
    a1, b1 = counter_draw(seed, idx, 0, INIT1)
    out, bound = np.zeros((len(rows), 4)), np.zeros((len(rows), 4))
    with mpmath.workdps(DPS):
        for j in range(len(rows)):
            r0, z0, z1 = _box_muller_exact(a0[j], b0[j])
            r1, z2, _ = _box_muller_exact(a1[j], b1[j])
            delta, radius = (z0, z1, z2), (r0, r0, r1)
            v = [mpmath.mpf(mean[r]) + sum(mpmath.mpf(t[r, k]) * delta[k] for k in range(3)) for r in range(3)]
            c, s = _exp(v[2])
            out[j] = [float(c), float(s), float(v[0]), float(v[1])]
            mag = [abs(mean[r]) + sum(abs(t[r, k]) * float(radius[k]) for k in range(3)) for r in range(3)]
            bound[j] = K_INIT * EPS * np.array([1.0 + mag[2], 1.0 + mag[2], mag[0], mag[1]])
    return out, bound


def transform_defect(cov, transform) -> tuple[float, float]:
    """max |T T^T - C| in exact arithmetic, and the bound it is held to: K_COV eps ||C||_F."""
    t = np.asarray(transform, dtype=np.float64).reshape(3, 3)
    c = np.asarray(cov, dtype=np.float64).reshape(3, 3)
    with mpmath.workdps(DPS):
        worst = max(abs(sum(mpmath.mpf(t[i, k]) * mpmath.mpf(t[j, k]) for k in range(3)) - mpmath.mpf(c[i, j]))
                    for i in range(3) for j in range(3))
    return float(worst), K_COV * EPS * float(np.linalg.norm(c))


# ---- the free-space draw ------------------------------------------------------------------------------------------------
def exact_free_state(free_cells, width: int, resolution: float, origin, seed: int, slots, step: int):
    """random_free_state (propagate.cuh:23-31) for counter_draw(seed, slot, step, kStreamRandomState): the free cell
    mulhi64(a, n_free), its centroid in the origin frame, yaw = u(b) 2 pi - pi -> (exact states, bound (m, 4))."""
    free = np.asarray(free_cells)
    o = np.asarray(origin, dtype=np.float64)
    slots = np.asarray(slots, dtype=np.uint64)
    a, b = counter_draw(seed, slots, step, RANDOM_STATE)
    out, bound = np.zeros((len(slots), 4)), np.zeros((len(slots), 4))
    with mpmath.workdps(DPS):
        for j in range(len(slots)):
            cell = int(free[mulhi64(a[j], len(free))])
            lx = (mpmath.mpf(cell % width) + mpmath.mpf(0.5)) * mpmath.mpf(resolution)
            ly = (mpmath.mpf(cell // width) + mpmath.mpf(0.5)) * mpmath.mpf(resolution)
            yaw = uniform01_mp(b[j]) * 2 * mpmath.pi - mpmath.pi
            c, s = _exp(yaw)
            x = mpmath.mpf(o[0]) * lx - mpmath.mpf(o[1]) * ly + mpmath.mpf(o[2])
            y = mpmath.mpf(o[1]) * lx + mpmath.mpf(o[0]) * ly + mpmath.mpf(o[3])
            out[j] = [float(c), float(s), float(x), float(y)]
            mag = abs(o[0]) * float(lx) + abs(o[1]) * float(ly)
            bound[j] = K_FREE * EPS * np.array([4.0, 4.0, mag + abs(o[2]), mag + abs(o[3])])
    return out, bound


# ---- the cases the motion tests run -------------------------------------------------------------------------------------
ALPHAS = (0.1, 0.05, 0.1, 0.05, 0.02)
DISTANCE_THRESHOLD = 0.01


def edge_states(n: int, seed: int = 7) -> np.ndarray:
    """n states mixing the pose-range edges: near the origin, at |x|, |y| ~ 1e4 and 1e6 m, headings at and next to
    +-pi, and rotations stored through float32 (c^2 + s^2 - 1 ~ 1e-8, as a pose read from a float message is)."""
    rng = np.random.default_rng(seed)
    th = rng.uniform(-PI, PI, n)
    scale = np.array([10.0, 1e4, 1e6])[np.arange(n) % 3]
    xy = rng.uniform(-1.0, 1.0, (n, 2)) * scale[:, None]
    k = np.arange(n) % 7
    th[k == 1] = PI
    th[k == 2] = np.nextafter(PI, 0.0)
    th[k == 3] = -np.nextafter(PI, 0.0)
    out = np.stack([np.cos(th), np.sin(th), xy[:, 0], xy[:, 1]], axis=1)
    out[k == 1, :2] = (-1.0, 0.0)
    f32 = k >= 5
    out[f32, :2] = out[f32, :2].astype(np.float32).astype(np.float64)
    return out


def sampling10(model: int, mean, std, first=(1.0, 0.0)) -> np.ndarray:
    return np.array([*mean, *std, *first, float(model), 0.0], dtype=np.float64)


def control_pair(distance: float, heading: float = 0.4, turn: float = 0.3):
    """(pose, previous pose) as data() vectors: a move of `distance` along `heading` while turning by `turn`."""
    prev = np.array([math.cos(0.1), math.sin(0.1), 2.0, -1.0])
    th = 0.1 + turn
    pose = np.array([math.cos(th), math.sin(th), 2.0 + distance * math.cos(heading), -1.0 + distance * math.sin(heading)])
    return pose, prev


def motion_cases(orc) -> dict:
    """name -> sampling10 of every motion case: each model with zero noise, a first rotation of exactly pi and of
    pi - 1 ulp, translations below, at and far above distance_threshold (from control poses through the motion model),
    and angular sigmas of 10 and 1e3 rad."""
    pi_down = float(np.nextafter(PI, 0.0))
    cases = {}
    for model, name in ((0, "diff"), (1, "omni"), (2, "stationary")):
        cases[f"{name}-zero-noise"] = sampling10(model, (0.3, 1.0, -0.2) if model != 1 else (0.3, 1.0, 0.0), (0.0, 0.0, 0.0),
                                                 (math.cos(0.7), math.sin(0.7)) if model == 1 else (1.0, 0.0))
        for tag, a in (("pi", PI), ("pi-ulp", pi_down)):
            if model == 1:  # the first rotation of the omnidirectional model is the deterministic heading rotation
                cases[f"{name}-first-{tag}"] = sampling10(1, (0.2, 1.5, 0.0), (0.05, 0.1, 0.05), (math.cos(a), math.sin(a)))
            else:
                cases[f"{name}-first-{tag}"] = sampling10(model, (a, 1.5, -0.3) if model == 0 else (a, 0.2, -0.1), (0.05, 0.1, 0.05))
        for tag, sigma in (("sigma10", 10.0), ("sigma1e3", 1e3)):
            std = (sigma, 0.1, sigma) if model == 0 else (sigma, 0.1, 0.1)
            cases[f"{name}-{tag}"] = sampling10(model, (0.2, 1.0, 0.1) if model != 1 else (0.2, 1.0, 0.0), std,
                                                (math.cos(-2.0), math.sin(-2.0)) if model == 1 else (1.0, 0.0))
        if model != 2:
            for tag, dist in (("below-threshold", 0.5 * DISTANCE_THRESHOLD), ("at-threshold", DISTANCE_THRESHOLD), ("jump-100m", 100.0)):
                pose, prev = control_pair(dist)
                cases[f"{name}-{tag}"] = orc.motion_sampling(model, orc.OmniParam(*ALPHAS, distance_threshold=DISTANCE_THRESHOLD), pose, prev)
    return cases


CASE_ROWS = 6000        # states per case (the device and the oracle run all of them)
SUBSAMPLE_CPU = 300     # rows per case checked against mpmath here
SEED, STEP, FIRST = 0x1234_5678_9ABC, 7, (1 << 32) - 3000  # the case rows cross the 2^32 index boundary


def subsample(n: int, m: int) -> np.ndarray:
    return np.unique(np.linspace(0, n - 1, m).astype(np.int64))


# ---- tests --------------------------------------------------------------------------------------------------------------
def test_philox_matches_oracle(orc):
    rng = np.random.default_rng(1)
    edges = [(1 << 32) - 1, 1 << 32, (1 << 32) + 1, 0, (1 << 64) - 1]
    counters = [(idx & 0xFFFFFFFF, idx >> 32, step, stream) for idx in edges for step in (0, 0xFFFFFFFF) for stream in range(7)]
    counters += [tuple(int(v) for v in rng.integers(0, 1 << 32, 4)) for _ in range(200)]
    keys = [tuple(int(v) for v in rng.integers(0, 1 << 32, 2)) for _ in counters]
    keys[:3] = [(0, 0), (0xFFFFFFFF, 0xFFFFFFFF), (1, 0)]
    got = philox4x32_10(np.array(counters, dtype=np.uint64), np.array(keys, dtype=np.uint64))
    for c, k, g in zip(counters, keys, got):
        assert np.array_equal(g, orc.philox4x32_10(c, k)), (c, k)


def test_uniform01_rounds_at_and_above_one_half():
    """uniform01 is the exact (k + 1/2) 2^-53 below 1/2; above, k + 1/2 rounds to even, and the largest word gives
    exactly 1.0 (log(1) = 0: a zero Box-Muller radius, not a fault).  The restatement starts from these doubles."""
    lo = np.array([0, 1, (1 << 63) - 1], dtype=np.uint64) | np.uint64(0x7FF)
    with mpmath.workdps(DPS):
        for b in lo:
            assert mpmath.mpf(float(uniform01(b))) == (mpmath.mpf(int(b) >> 11) + mpmath.mpf(0.5)) * mpmath.mpf(2) ** -53
    assert float(uniform01(np.uint64((1 << 64) - 1))) == 1.0
    assert float(uniform01(np.uint64(1 << 63))) == 0.5  # 2^52 + 1/2 rounds to even
    assert float(uniform01(np.uint64(3 << 62))) == 0.75


def test_counter_draw_keys_the_index_in_two_words(orc):
    """The high word of the index reaches the counter: indices 2^32 apart draw different numbers, and the draw at
    2^32 + i is the oracle's Philox of (i, 1, step, stream)."""
    a_lo, _ = counter_draw(5, [3], 9, MOTION0)
    a_hi, b_hi = counter_draw(5, [(1 << 32) + 3], 9, MOTION0)
    assert a_lo[0] != a_hi[0]
    v = orc.philox4x32_10((3, 1, 9, MOTION0), (5, 0)).astype(np.uint64)
    assert a_hi[0] == (int(v[1]) << 32) | int(v[0]) and b_hi[0] == (int(v[3]) << 32) | int(v[2])


def test_restatement_reproduces_the_oracle_at_high_precision(orc):
    """At zero noise and unit-norm states the exact composition and the oracle differ only by rounding: the
    restatement's SE(2) algebra (order of products, inverse of the first rotation, the sign of the strafe) is the
    oracle's."""
    states = edge_states(200)
    for model in (0, 1, 2):
        s = sampling10(model, (0.8, 2.0, -0.6), (0.0, 0.0, 0.0), (math.cos(1.1), math.sin(1.1)) if model == 1 else (1.0, 0.0))
        exact, d, rs = exact_propagate(states, s, seed=3, step=1, first_index=0)
        got = orc.motion_propagate(s, states, mode=1, seed=3, step=1, first_index=0)
        ratio, row, comp = worst_ratio(got, exact, motion_bound(model, states, d, rs))
        assert ratio <= 1.0, f"model {model}: row {row} component {comp} at {ratio:.3g} x bound"
    # a wrong sign of the strafe is far outside the bound
    s = sampling10(1, (0.0, 0.0, 0.5), (0.0, 0.0, 0.0))
    exact, d, rs = exact_propagate(states[:10], s, 3, 1, 0)
    flipped = orc.motion_propagate(sampling10(1, (0.0, 0.0, -0.5), (0.0, 0.0, 0.0)), states[:10], mode=1, seed=3)
    assert worst_ratio(flipped, exact, motion_bound(1, states[:10], d, rs))[0] > 1e6


def test_oracle_motion_update_stays_inside_the_bound(orc):
    """orc.motion_propagate (counter mode) on every motion case of the GPU tests: each subsampled particle against the
    mpmath restatement, within K_MOTION = 32 eps of the bound, and |c^2 + s^2 - 1| <= K_UNIT = 8 eps everywhere."""
    states = edge_states(CASE_ROWS)
    rows = subsample(CASE_ROWS, SUBSAMPLE_CPU)
    report = []
    for name, s in motion_cases(orc).items():
        got = orc.motion_propagate(s, states, mode=1, seed=SEED, step=STEP, first_index=FIRST)
        assert np.all(unit_defect(got) <= K_UNIT * EPS), name
        exact, d, rs = exact_propagate(states, s, SEED, STEP, FIRST, rows)
        ratio, row, comp = worst_ratio(got[rows], exact, motion_bound(int(s[8]), states[rows], d, rs))
        report.append(f"{name}: {ratio:.3f}")
        assert ratio <= 1.0, f"{name}: row {rows[row]} component {'csxy'[comp]} at {ratio:.3g} x bound"
    print("oracle worst error / bound:", ", ".join(report))


def test_motion_cases_take_the_threshold_branches(orc):
    """Below distance_threshold the models keep no heading: the differential drive's first rotation mean and the
    omnidirectional first rotation are zero / identity; above it they follow the motion."""
    cases = motion_cases(orc)
    assert cases["diff-below-threshold"][0] == 0.0 and cases["diff-jump-100m"][0] != 0.0
    assert tuple(cases["omni-below-threshold"][6:8]) == (1.0, 0.0) and tuple(cases["omni-jump-100m"][6:8]) != (1.0, 0.0)
    assert cases["diff-jump-100m"][1] == pytest.approx(100.0)


COVARIANCES = {
    "ros-default": np.diag([0.25, 0.25, 0.0685]),  # repeated eigenvalue
    "zero-theta": np.diag([0.3, 0.1, 0.0]),
    "scale-1e-12": np.array([[2.0, 0.3, 0.1], [0.3, 1.0, 0.05], [0.1, 0.05, 0.5]]) * 1e-12,
    "scale-1e6": np.array([[2.0, 0.3, 0.1], [0.3, 1.0, 0.05], [0.1, 0.05, 0.5]]) * 1e6,
    "xy-correlated": np.array([[1.0, 0.999, 0.0], [0.999, 1.0, 0.0], [0.0, 0.0, 0.1]]),
}
INIT_MEAN = np.array([1.5e3, -2.5e4, 2.9])


@pytest.mark.parametrize("name", list(COVARIANCES))
def test_normal_transform_reproduces_the_covariance(orc, name):
    """T T^T = C within K_COV eps ||C||_F = 64 eps ||C||_F (exact arithmetic on the stored T), for the cyclic Jacobi
    transform the filter (filter.cu:25-78) and the oracle both compute."""
    cov = COVARIANCES[name]
    t = orc.normal_transform(cov)
    worst, bound = transform_defect(cov, t)
    assert worst <= bound, f"{name}: |T T^T - C| = {worst:.3g} > {bound:.3g}"


@pytest.mark.parametrize("name", list(COVARIANCES))
def test_oracle_normal_init_stays_inside_the_bound(orc, name):
    """The oracle's counter-mode initial states against exact_normal_init given T, within K_INIT = 32 eps."""
    cov, n = COVARIANCES[name], 512
    o = orc.Amcl(orc.AmclParam(max_particles=n, min_particles=n, seed=5, rng_mode=1), orc.MotionParam())
    o.initialize_normal(INIT_MEAN, cov)
    got, _ = o.particles()
    rows = subsample(n, 100)
    exact, bound = exact_normal_init(INIT_MEAN, orc.normal_transform(cov), 5, 0, rows)
    ratio, row, comp = worst_ratio(got[rows], exact, bound)
    assert ratio <= 1.0, f"{name}: row {rows[row]} component {'csxy'[comp]} at {ratio:.3g} x bound"


def free_state_grid(kind: str):
    """(cells, resolution, origin) of the free-space cases: one free cell, a prime number of them (397), and more than
    2^16 (90 000) under a rotated origin far from zero."""
    if kind == "one":
        cells = np.full((7, 9), 100, dtype=np.int8)
        cells[4, 6] = 0
        return cells, 0.25, np.array([math.cos(2.5), math.sin(2.5), -3.0, 4.0])
    if kind == "prime":
        cells = np.zeros((20, 20), dtype=np.int8)
        cells[0, :3] = 100  # 397 free cells
        return cells, 0.05, np.array([math.cos(-0.4), math.sin(-0.4), 1.2e3, -7.5e2])
    cells = np.zeros((300, 300), dtype=np.int8)
    return cells, 0.1, np.array([math.cos(1.9), math.sin(1.9), 2.0e5, 3.5e5])


def free_cells(cells) -> np.ndarray:
    return np.flatnonzero(np.asarray(cells).ravel() == 0).astype(np.uint32)


@pytest.mark.parametrize("kind", ["one", "prime", "many"])
def test_oracle_free_states_stay_inside_the_bound(orc, kind):
    """The oracle's initialize_from_map states (random_state_counter at step 0, slot = particle index) against
    exact_free_state, within K_FREE = 16 eps."""
    cells, res, origin = free_state_grid(kind)
    assert len(free_cells(cells)) == {"one": 1, "prime": 397, "many": 90_000}[kind]
    n = 400
    o = orc.Amcl(orc.AmclParam(max_particles=n, min_particles=n, seed=11, rng_mode=1), orc.MotionParam())
    o.set_map(orc.LFM, orc.LfmParam(max_obstacle_distance=2.0, max_laser_distance=20.0), orc.Grid(cells, res, origin))
    o.initialize_from_map()
    got, _ = o.particles()
    exact, bound = exact_free_state(free_cells(cells), cells.shape[1], res, origin, 11, np.arange(n), 0)
    ratio, row, comp = worst_ratio(got, exact, bound)
    assert ratio <= 1.0, f"{kind}: row {row} component {'csxy'[comp]} at {ratio:.3g} x bound"
