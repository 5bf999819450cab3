"""Executable version of the argument behind the unclamped lookup of the fixed-point reweight kernels (csrc/reweight_lfm.cuh,
fixed_lookup<true>): a warp whose particles pass the in-grid test reads the table without clamping its cell coordinates and
without removing their bias, from a base pointer moved back by fixed_index_bias(pitch).

Two claims, replayed on the CPU with IEEE doubles for the reference's operation sequence and exact integers for the
index arithmetic:
- a particle that passes the in-grid test has every end point's reference cell inside the grid, so the clamp is the
  identity there;
- for every cell, the biased index is the clamped index plus the bias, with no wrap past 2^32, whenever the upload-time
  check (DeviceMap::upload) accepts the pitch -- and that check rejects a table where some biased index would wrap.
CPU only; it models the arithmetic, it does not run the kernel."""
import math

import numpy as np
import pytest

from test_fixed_point_lookup_model import BIAS_X, BIAS_Y, bordered_index, kernel_cells, kernel_index, reference_cells

M32 = 1 << 32


def in_grid(tx, ty, inv, radius, width, height):
    """fixed_pose_setup: the square of points_radius * inv + 2 cells around the position lies inside the grid."""
    cells = radius * inv + 2.0
    gx, gy = tx * inv, ty * inv
    return gx - cells >= 0.0 and gx + cells < width and gy - cells >= 0.0 and gy + cells < height


def fixed_index_bias(pitch):
    return (BIAS_Y * (4 * pitch) + BIAS_X) % M32


def accepts(pitch, table_size):
    """DeviceMap::upload: the moved-back base is used only if no element's biased index passes 2^32."""
    return fixed_index_bias(pitch) + table_size <= M32


def clamped_index(ux4, uy, kx, width, height):
    """fixed_lookup<false>: the words minus their bias, clamped to the far border."""
    return kernel_index(min(ux4 % M32, 4 * (width + 1) + 3), min(uy % M32, height + 1), kx)


def biased_index(ux4, uy, kx):
    """fixed_lookup<true>: lop3 and multiply-add on the words with their bias still in, modulo 2^32."""
    hx, hy = (ux4 + BIAS_X) % M32, (uy + BIAS_Y) % M32
    low = (hx & ~3) | (hy & 3)
    return ((hy & ~3) * (4 << kx) + low) % M32


def kx_of(width):
    return max(0, math.ceil(math.log2(-(-(width + 2) // 4))))


def edge_particles(rng, width, height, res, radius):
    """(tx, ty, theta, d): positions d cells from one edge and well inside the others, at any heading.  d runs from one cell
    either side of the in-grid test's limit (reach = radius / res + 2) down to end points that reach the last cell of
    the grid, cross the edge by one cell, and by several."""
    inv = 1.0 / res
    r = radius * inv
    reach = r + 2.0
    for d in (reach + 1.0, reach + 0.5, reach, reach - 0.5, reach - 1.0, r + 0.5, r - 0.5, r - 4.5):
        for edge in range(4):
            along = float(rng.uniform(reach + 1.0, min(width, height) - reach - 1.0))
            gx, gy = [(d, along), (width - d, along), (along, d), (along, height - d)][edge]
            # a quarter-turn heading puts an axis end point (|x| or |y| = radius) square onto the edge's normal
            theta = float(rng.integers(-1, 3)) * math.pi / 2 if d < r + 1.0 else float(rng.uniform(-math.pi, math.pi))
            yield gx * res, gy * res, theta, d


@pytest.mark.parametrize("width, height, res", [(200, 120, 0.05), (2000, 2000, 0.05), (37, 61, 1.0 / 3.0)])
def test_in_grid_particles_only_reach_cells_inside_the_grid(width, height, res):
    rng = np.random.default_rng(width)
    inv = 1.0 / res
    radius = 1.5 if width > 50 else 4.0  # |x| + |y| of the farthest end point
    reach = radius * inv + 2.0
    kx = kx_of(width)
    for tx, ty, theta, d in edge_particles(rng, width, height, res, radius):
        c, s = math.cos(theta), math.sin(theta)
        # the end points that reach farthest: the corners and axis points of the |x| + |y| <= radius diamond
        ends = [(radius, 0.0), (-radius, 0.0), (0.0, radius), (0.0, -radius)]
        ends += [(a * radius, (1.0 - abs(a)) * radius * sgn) for a in rng.uniform(-1.0, 1.0, 12) for sgn in (1.0, -1.0)]
        accepted = in_grid(tx, ty, inv, radius, width, height)
        if abs(d - reach) >= 0.5:  # the test is exactly the square of `reach` cells: each bound of each axis, both sides
            assert accepted == (d > reach), (tx, ty, d)
        inside = [0 <= xr < width and 0 <= yr < height for xr, yr in (reference_cells(px, py, c, s, tx, ty, inv) for px, py in ends)]
        if d < radius * inv:  # an end point crosses the edge: only the clamped loop may take this particle
            assert not all(inside)
        elif d < radius * inv + 1.0:  # an end point lands in the last cell before the edge
            assert all(inside)
        if not accepted:
            continue
        for px, py in ends:
            xr, yr = reference_cells(px, py, c, s, tx, ty, inv)
            assert 0 <= xr < width and 0 <= yr < height, (tx, ty, theta, px, py)
            xk, yk, amb = kernel_cells(px, py, c, s, tx, ty, inv)
            if not amb:
                assert (xk, yk) == (xr, yr)
            # whatever the kernel's cell (ambiguous ones are off by at most one), it is one the clamp leaves alone
            assert -1 <= xk <= width and -1 <= yk <= height
            ux4, uy = 4 * (xk + 1) + 2, yk + 1
            assert clamped_index(ux4, uy, kx, width, height) == bordered_index(xk + 1, yk + 1, kx)


@pytest.mark.parametrize("width, height", [(5, 7), (64, 33), (200, 200), (1998, 1998), (7998, 7998)])
def test_biased_index_is_the_clamped_index_plus_the_bias(width, height):
    """For every in-grid cell (all of them on small maps, a sample on large ones) and every value of x's fraction bits."""
    kx = kx_of(width)
    size = (-(-(height + 2) // 4)) << (kx + 4)
    assert accepts(1 << kx, size)  # every map the fixed-point kernel takes
    bias = fixed_index_bias(1 << kx)
    rng = np.random.default_rng(kx)
    if width * height <= 40000:
        cells = [(x, y) for y in range(-1, height + 1) for x in range(-1, width + 1)]
    else:
        cells = [(int(x), int(y)) for x, y in zip(rng.integers(-1, width + 1, 20000), rng.integers(-1, height + 1, 20000))]
        cells += [(-1, -1), (width, height), (-1, height), (width, -1)]
    for x, y in cells:
        for frac in range(4):
            ux4, uy = 4 * (x + 1) + frac, y + 1
            e = clamped_index(ux4, uy, kx, width, height)
            assert e < size
            assert biased_index(ux4, uy, kx) == e + bias  # no wrap: the moved-back base finds element e


def test_upload_check_rejects_a_pitch_whose_biased_index_wraps():
    """A table with 2^5 tiles per row and more than 2^32 - bias elements: the largest biased index would wrap, and the
    moved-back base would miss the element.  The check refuses it; a smaller table with the same pitch passes."""
    kx = 5
    bias = fixed_index_bias(1 << kx)
    assert bias == 0xDD180000
    size = M32 - bias + 16  # the last tile row's elements pass 2^32
    assert not accepts(1 << kx, size)
    assert accepts(1 << kx, M32 - bias)
    e = size - 1  # the largest element: padded cell (x, y) with bordered_index(x, y) = e
    py = (e >> (kx + 4)) * 4 + (e & 3)
    px = ((e >> 4) & ((1 << kx) - 1)) * 4 + ((e >> 2) & 3)
    assert bordered_index(px, py, kx) == e
    assert biased_index(4 * px, py, kx) != e + bias  # wrapped
