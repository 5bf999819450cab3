"""Integer model of the empty-space skipping in cast_ray (csrc/reweight_beam.cuh): the beam kernel walks the reference's
standard Bresenham line (algorithm/raycasting/bresenham.hpp:84-160) but advances d steps at once where the
Chebyshev free-distance map says the next d - 1 cells cannot stop the ray, updating (x, y, error) in closed form
(with the 32-bit reciprocal-multiply-and-correct quotient the kernel uses).  Checked here against a plain cell-by-cell
walk over the oracle's Bresenham cells on random maps and rays.  CPU only."""
import numpy as np
import pytest
from scipy import ndimage


def free_distance_map(cells):
    """map_host.cpp:make_free_distance -- Chebyshev distance to the nearest non-free or outside cell, capped at 255."""
    free = np.pad(cells == 0, 1, constant_values=False)
    d = ndimage.distance_transform_cdt(free, metric="chessboard")[1:-1, 1:-1]
    return np.minimum(d, 255).astype(np.int64)


def skip_walk(dist, sx, sy, fx, fy):
    """The loop of cast_ray: -> (cx, cy) of the first non-free cell, or None on a miss."""
    h, w = dist.shape
    xspan, xstep = fx - sx, 1
    if xspan < 0:
        xspan, xstep = -xspan, -1
    yspan, ystep = fy - sy, 1
    if yspan < 0:
        yspan, ystep = -yspan, -1
    x, y, reversed_ = sx, sy, False
    if xspan < yspan:
        x, y = y, x
        xspan, yspan = yspan, xspan
        xstep, ystep = ystep, xstep
        reversed_ = True
    dxspan, dyspan = 2 * xspan, 2 * yspan
    recip = 0xFFFFFFFF // dxspan if dxspan else 0  # ray_begin: floor((2^32 - 1) / dxspan)
    error, step = xspan, 0
    while True:
        cx, cy = (y, x) if reversed_ else (x, y)
        if not (0 <= cx < w and 0 <= cy < h):
            return None
        d = int(dist[cy, cx])
        if d == 0:
            return cx, cy
        k = min(d, xspan - step)
        if k == 0:
            return None
        step += k
        x += k * xstep
        t = error + k * dyspan
        assert 0 <= t - 1 < 2 ** 32
        m = ((t - 1) * recip) >> 32  # __umulhi(t - 1, recip): the quotient or one below it
        r = (t - 1) - m * dxspan
        assert 0 <= r < 2 * dxspan
        if r >= dxspan:
            m += 1
        assert m == (t - 1) // dxspan  # one remainder check makes the quotient exact
        y += m * ystep
        error = t - m * dxspan
        assert 0 < error <= dxspan


def plain_walk(orc, cells, sx, sy, fx, fy):
    h, w = cells.shape
    for cx, cy in orc.bresenham((sx, sy), (fx, fy)):
        if not (0 <= cx < w and 0 <= cy < h):
            return None
        if cells[cy, cx] != 0:
            return int(cx), int(cy)
    return None


@pytest.mark.parametrize("seed", range(6))
def test_skipping_finds_the_same_cell(orc, seed):
    rng = np.random.default_rng(seed)
    h, w = 90, 120
    cells = np.zeros((h, w), dtype=np.int8)
    for _ in range(int(rng.integers(3, 25))):
        x0, y0 = int(rng.integers(0, w - 6)), int(rng.integers(0, h - 6))
        cells[y0:y0 + int(rng.integers(1, 6)), x0:x0 + int(rng.integers(1, 6))] = 100 if rng.random() < 0.8 else -1
    dist = free_distance_map(cells)
    for _ in range(400):
        sx, sy = int(rng.integers(0, w)), int(rng.integers(0, h))
        fx, fy = int(rng.integers(-40, w + 40)), int(rng.integers(-40, h + 40))
        assert skip_walk(dist, sx, sy, fx, fy) == plain_walk(orc, cells, sx, sy, fx, fy), (sx, sy, fx, fy)


def test_degenerate_rays(orc):
    cells = np.zeros((8, 8), dtype=np.int8)
    cells[4, 6] = 100
    dist = free_distance_map(cells)
    for ray in [(2, 2, 2, 2), (2, 4, 7, 4), (2, 4, 6, 4), (6, 4, 6, 4), (0, 0, 7, 7), (7, 0, 0, 7), (3, 3, 3, 30), (3, 3, -30, 3)]:
        assert skip_walk(dist, *ray) == plain_walk(orc, cells, *ray), ray
