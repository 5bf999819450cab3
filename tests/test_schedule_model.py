"""Executable version of the argument behind the execution schedule of the reweight kernel (csrc/kernels.cuh:
schedule_from_moments, csrc/kernels.cu: schedule_bin): particles are counting-sorted over pose bins and every warp takes 32
neighbours of that order, so the 32 end points of one beam land in a few cache lines.  The schedule decides only WHICH
THREAD handles a particle -- any permutation gives the same results -- so what there is to check is that the bin function
always yields a valid bin, that consecutive bins are neighbours (boustrophedon order), and that the equal-mass bins do what
they are for: on a normal cloud, 32 schedule neighbours span a smaller box than with equal-size bins of the same count.

CPU only; a numpy restatement of the two functions, it does not run the kernel."""
import math

import numpy as np
import pytest

MAX_BINS = 1 << 19
PER_BIN = 4.0  # kSchedulePerBin
X_SPLIT = 8.0  # kScheduleXSplit


def schedule_from_moments(cbar, sbar, mx, my, vx, vy, n, mean_range, min_bin):
    r = math.hypot(cbar, sbar)
    c0, s0, sigma_theta = 1.0, 0.0, math.pi
    if r > 1e-9:
        c0, s0 = cbar / r, sbar / r
        sigma_theta = math.sqrt(-2.0 * math.log(r)) if r < 1.0 else 0.0
    half_theta = min(2.0, max(3.0 * sigma_theta, 1e-4))
    half_u = 2.0 * math.tan(0.5 * half_theta)
    half_x, half_y = max(3.0 * math.sqrt(max(vx, 0.0)), min_bin), max(3.0 * math.sqrt(max(vy, 0.0)), min_bin)
    lever = max(mean_range, 1.0)
    centre = 1.0 / (3.0 * 0.4255)
    ext_t, ext_x, ext_y = centre * half_u * lever, centre * half_x, centre * half_y
    q = max(np.cbrt(X_SPLIT * ext_t * ext_x * ext_y / max(n / PER_BIN, 1.0)), min_bin)
    while True:
        nt = int(min(max(math.ceil(ext_t / q), 1.0), 65536.0))
        nx = int(min(max(math.ceil(X_SPLIT * ext_x / q), 1.0), 65536.0))
        ny = int(min(max(math.ceil(ext_y / q), 1.0), 65536.0))
        if nt * nx * ny <= MAX_BINS:
            break
        q *= 1.3
    return dict(c0=c0, s0=s0, half_u=half_u, mx=mx, my=my, kt=np.float32(1.702 * 3.0 / half_u), kx=np.float32(1.702 * 3.0 / half_x),
                ky=np.float32(1.702 * 3.0 / half_y), nt=nt, nx=nx, ny=ny, n_bins=nt * nx * ny)


def heading_u(g, c, s):
    """Heading relative to the grid's mean as u = 2 tan(dtheta / 2)."""
    cr, sr = c * g["c0"] + s * g["s0"], s * g["c0"] - c * g["s0"]
    return np.where(cr > -0.4, 2.0 * sr / (1.0 + cr), np.where(sr >= 0.0, 1e6, -1e6))


def boustrophedon(g, bt, by, bx):
    """-> (bin, bt, by, bx); (by, bx) are the coordinates AFTER the flips of odd planes and rows."""
    by = np.where(bt & 1, g["ny"] - 1 - by, by)
    row = bt * g["ny"] + by
    bx = np.where(row & 1, g["nx"] - 1 - bx, bx)
    return row * g["nx"] + bx, bt, by, bx


def schedule_bin(g, c, s, x, y):
    """-> (bin, bt, by, bx) per particle; (by, bx) are the coordinates AFTER the boustrophedon flips."""
    with np.errstate(all="ignore"):
        u = heading_u(g, c, s)

        def cdf_bin(z, count):
            f = np.float32(count) / (np.float32(1.0) + np.exp(-z.astype(np.float32)))
            f = np.where(np.isnan(f), np.float32(0.0), f)  # __float2int_rz(NaN) = 0
            return np.clip(np.trunc(np.clip(f, -2e9, 2e9)).astype(np.int64), 0, count - 1)

        bt = cdf_bin(u.astype(np.float32) * g["kt"], g["nt"])
        bx = cdf_bin((x - g["mx"]).astype(np.float32) * g["kx"], g["nx"])
        by = cdf_bin((y - g["my"]).astype(np.float32) * g["ky"], g["ny"])
    return boustrophedon(g, bt, by, bx)


def normal_cloud(rng, n, sx=0.5, sy=0.55, st=0.2, mean=(30.0, 40.0, 1.1)):
    theta = mean[2] + st * rng.standard_normal(n)
    return np.cos(theta), np.sin(theta), mean[0] + sx * rng.standard_normal(n), mean[1] + sy * rng.standard_normal(n), theta


def grid_for(cloud, n, mean_range=21.0, res=0.05):
    c, s, x, y, _ = cloud
    return schedule_from_moments(c.mean(), s.mean(), x.mean(), y.mean(), x.var(), y.var(), float(n), mean_range, 0.5 * res)


def test_every_pose_gets_a_valid_bin():
    rng = np.random.default_rng(4)
    n = 200_000
    cloud = normal_cloud(rng, n)
    g = grid_for(cloud, n)
    assert 0 < g["n_bins"] <= MAX_BINS
    c, s, x, y, _ = cloud
    # outliers: far away, opposite heading, non-finite
    c, s, x, y = (np.concatenate([a, b]) for a, b in ((c, [-1.0, 0.0, np.nan, 1.0]), (s, [0.0, -1.0, 0.0, np.nan]), (x, [1e30, -1e30, np.nan, np.inf]),
                                                      (y, [-np.inf, 5.0, 1e300, np.nan])))
    b, *_ = schedule_bin(g, c, s, x, y)
    assert b.min() >= 0 and b.max() < g["n_bins"]


def test_consecutive_bins_are_neighbours():
    """Boustrophedon order: bin k and bin k + 1 differ by one step along one axis, at row ends and plane ends too."""
    g = dict(nt=3, ny=4, nx=5)
    coords = {}
    for bt in range(g["nt"]):
        for by in range(g["ny"]):
            for bx in range(g["nx"]):
                fy = g["ny"] - 1 - by if bt & 1 else by
                row = bt * g["ny"] + fy
                fx = g["nx"] - 1 - bx if row & 1 else bx
                coords[row * g["nx"] + fx] = (bt, by, bx)  # physical cell of a linear index
    assert sorted(coords) == list(range(g["nt"] * g["ny"] * g["nx"]))
    for k in range(len(coords) - 1):
        a, b = coords[k], coords[k + 1]
        assert sum(abs(p - q) for p, q in zip(a, b)) == 1, (k, a, b)


def warp_extents(cloud, bins, mean_range):
    """Median extent, over warps of 32 schedule neighbours, of (lever * heading, x, y) in metres."""
    c, s, x, y, theta = cloud
    order = np.argsort(bins, kind="stable")
    m = (len(order) // 32) * 32
    o = order[:m].reshape(-1, 32)
    ext = lambda v: np.median(v[o].max(axis=1) - v[o].min(axis=1))  # noqa: E731
    return ext(theta * mean_range), ext(x), ext(y)


def equal_size_bins(cloud, n, mean_range=21.0, res=0.05, per_bin=16.0):
    """Baseline of the test below, not product code: bins of equal physical size tiling the +-3 sigma box of
    (mean_range * u, x, y), about `per_bin` particles each, in the same boustrophedon order.  -> (bins, bin count)"""
    c, s, x, y, _ = cloud
    g = grid_for(cloud, n, mean_range, res)  # mean heading and half_u
    min_bin = 0.5 * res
    half_x, half_y = max(3.0 * math.sqrt(x.var()), min_bin), max(3.0 * math.sqrt(y.var()), min_bin)
    lows = (-g["half_u"], x.mean() - half_x, y.mean() - half_y)
    widths = (2.0 * g["half_u"], 2.0 * half_x, 2.0 * half_y)
    ext = (widths[0] * max(mean_range, 1.0), widths[1], widths[2])
    q = max(np.cbrt(np.prod(ext) / max(n / per_bin, 1.0)), min_bin)
    counts = [max(math.ceil(e / q), 1) for e in ext]
    bt, bx, by = (np.clip(np.floor((v - lo) * (k / w)).astype(np.int64), 0, k - 1)
                  for v, lo, w, k in zip((heading_u(g, c, s), x, y), lows, widths, counts))
    bins, *_ = boustrophedon(dict(nt=counts[0], nx=counts[1], ny=counts[2]), bt, by, bx)
    return bins, int(np.prod(counts))


def test_equal_mass_bins_tighten_the_warps_of_a_normal_cloud():
    rng = np.random.default_rng(9)
    n = 400_000
    cloud = normal_cloud(rng, n)
    c, s, x, y, _ = cloud
    bu, n_bins_u = equal_size_bins(cloud, n)
    shaped = grid_for(cloud, n)
    bs, *_ = schedule_bin(shaped, c, s, x, y)
    # equal mass: the fullest bin is a small multiple of the mean; equal size over a normal cloud: the centre is ~13x over-full
    count_u, count_s = np.bincount(bu, minlength=n_bins_u), np.bincount(bs, minlength=shaped["n_bins"])
    assert count_s.max() < 8 * n / shaped["n_bins"]
    assert count_u.max() > 8 * n / n_bins_u
    eu, es = warp_extents(cloud, bu, 21.0), warp_extents(cloud, bs, 21.0)
    # the box a warp's 32 particles span shrinks in volume, and no side grows by more than a quarter
    assert np.prod(es) < 0.6 * np.prod(eu), (eu, es)
    assert all(b < 1.25 * a for a, b in zip(eu, es)), (eu, es)


def test_degenerate_clouds_collapse_to_few_bins():
    """A cloud without spread (all particles equal) and a cloud without a mean heading (uniform on the circle)."""
    n = 10_000
    g = schedule_from_moments(1.0, 0.0, 3.0, 4.0, 0.0, 0.0, float(n), 10.0, 0.025)
    assert g["n_bins"] >= 1 and g["nt"] * g["nx"] * g["ny"] == g["n_bins"] <= MAX_BINS
    b, *_ = schedule_bin(g, np.ones(5), np.zeros(5), np.full(5, 3.0), np.full(5, 4.0))
    assert len(set(b.tolist())) == 1
    g = schedule_from_moments(0.0, 0.0, 0.0, 0.0, 1.0, 1.0, float(n), 10.0, 0.025)
    theta = np.linspace(-math.pi, math.pi, 1000, endpoint=False)
    b, *_ = schedule_bin(g, np.cos(theta), np.sin(theta), np.zeros(1000), np.zeros(1000))
    assert b.min() >= 0 and b.max() < g["n_bins"]
