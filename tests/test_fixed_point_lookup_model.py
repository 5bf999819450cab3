"""Executable version of the argument behind reweight_lfm_fixed_*_kernel (csrc/reweight_lfm.cuh): the kernel finds the
likelihood-field CELL of a beam end point with two FMAs per coordinate and a magic-number add instead of the
reference's rounded operation sequence -- the magic number riding in the FMAs' addend -- and claims the same cell
whenever the fraction word it reads is at least 5.

This test replays both evaluations on the CPU -- IEEE doubles for the reference sequence, exact rationals rounded
once for the FMAs -- on random and adversarial (cell-edge) inputs and checks the claim, plus how often the
fallback would be taken.  CPU only; it models the arithmetic, it does not run the kernel."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

MAGIC_X, MAGIC_Y = 393216.0, 1572864.0  # 1.5 * 2^18, 1.5 * 2^20 (kFixedMagicX / kFixedMagicY)
BIAS_X, BIAS_Y = 0x41180000, 0x41380000
# Folding the magic add into the FMA chain costs three roundings at the magic's ulp (2^-34 for x, 2^-32 for y) instead of
# one: the computed fixed-point value lies within 3 half-ulps + 2^-36 of the reference's.  Two ulps of guard are added to
# the offset, so that the uncertainty interval sits entirely BELOW the computed value: the cell is the reference's
# whenever the fraction word is at least 5 (kFixedGuardX / kFixedGuardY / kFixedAmbiguous in the kernel).
GUARD_X, GUARD_Y = 2.0 ** -33, 2.0 ** -31
AMBIGUOUS_BELOW = 4


def fma(a: float, b: float, c: float) -> float:
    return float(Fraction(a) * Fraction(b) + Fraction(c))  # one rounding, to nearest even


def words(t: float):
    bits = struct.unpack("<Q", struct.pack("<d", t))[0]
    return bits >> 32, bits & 0xFFFFFFFF


def reference_cells(px, py, c, s, tx, ty, inv):
    x = (px * c - py * s) + tx  # likelihood_field_model.hpp:82-83, every operation rounded
    y = (px * s + py * c) + ty
    return math.floor(x * inv), math.floor(y * inv)  # regular_grid.hpp:75-78


def kernel_cells(px, py, c, s, tx, ty, inv):
    """-> (cell x, cell y, ambiguous) as fixed_lookup computes them (before clamping to the border)."""
    cx, sx = c * inv, s * inv
    # the magic constants ride in the FMAs' addend: (offset + 1 border cell) + (magic + guard), each sum rounded once
    ox, oy = (tx * inv + 1.0) + (MAGIC_X + GUARD_X), (ty * inv + 1.0) + (MAGIC_Y + GUARD_Y)
    gx = fma(px, cx, fma(-py, sx, ox))
    gy = fma(px, sx, fma(py, cx, oy))
    hx, lx = words(gx)
    hy, ly = words(gy)
    ux = (hx - BIAS_X) & 0xFFFFFFFF  # 4 * padded x + 2 fraction bits (padded x = cell + 1, for cells >= -1)
    uy = (hy - BIAS_Y) & 0xFFFFFFFF  # padded y
    to_signed = lambda u: u - (1 << 32) if u >= (1 << 31) else u  # noqa: E731
    return (to_signed(ux) >> 2) - 1, to_signed(uy) - 1, (lx <= AMBIGUOUS_BELOW or ly <= AMBIGUOUS_BELOW)


def random_case(rng, res):
    theta = rng.uniform(-math.pi, math.pi)
    c, s = math.cos(theta), math.sin(theta)
    tx, ty = rng.uniform(-20.0, 120.0, 2)
    r = rng.uniform(0.0, 100.0)
    a = rng.uniform(-math.pi, math.pi)
    return r * math.cos(a), r * math.sin(a), c, s, float(tx), float(ty), 1.0 / res


@pytest.mark.parametrize("res", [0.05, 0.025, 0.1, 1.0 / 3.0])
def test_random_end_points(res):
    rng = np.random.default_rng(int(res * 1e6))
    ambiguous = 0
    for _ in range(6000):
        case = random_case(rng, res)
        xr, yr = reference_cells(*case)
        xk, yk, amb = kernel_cells(*case)
        ambiguous += amb
        if not amb:
            assert (xk, yk) == (xr, yr), case
    assert ambiguous <= 1  # 5 * 2^-32 per coordinate


def test_end_points_on_and_around_cell_edges():
    """Axis-aligned and quarter-turn poses with end points exactly on cell edges, one ulp either side, and a few
    thousand ulps away: the fraction word must flag every case it cannot decide, and decide the others right."""
    rng = np.random.default_rng(1)
    res = 0.05
    inv = 1.0 / res
    flagged = decided = 0
    for theta in (0.0, math.pi / 2, math.pi, -math.pi / 2):
        c, s = math.cos(theta), math.sin(theta)
        for _ in range(400):
            tx, ty = float(rng.integers(0, 2000)) * res, float(rng.integers(0, 2000)) * res
            # px on a cell edge (before the +-k ulp nudges), py well inside a cell; the quarter turns swap their roles,
            # so both the x word (fraction bits after 1.5*2^18) and the y word (after 1.5*2^20) meet edges
            px = float(rng.integers(-400, 400)) * res
            py = (float(rng.integers(-400, 400)) + float(rng.uniform(0.2, 0.8))) * res  # y: well inside a cell
            for k in (0, 1, -1, 3, -3, 4096, -4096):
                ppx = px
                for _ in range(abs(k)) if abs(k) < 10 else ():
                    ppx = math.nextafter(ppx, math.inf if k > 0 else -math.inf)
                if abs(k) >= 10:
                    ppx = px + k * math.ulp(px if px != 0.0 else res)
                case = (ppx, py, c, s, tx, ty, inv)
                xr, yr = reference_cells(*case)
                xk, yk, amb = kernel_cells(*case)
                if amb:
                    flagged += 1
                else:
                    decided += 1
                    assert (xk, yk) == (xr, yr), case
    assert flagged > 100 and decided > 100  # both branches exercised


def test_range_limit_of_the_argument():
    """The kernel only trusts the fixed-point words while every term stays below 2^13 cells (reach < 8100)."""
    rng = np.random.default_rng(3)
    res = 0.05
    for _ in range(3000):
        theta = rng.uniform(-math.pi, math.pi)
        c, s = math.cos(theta), math.sin(theta)
        tx, ty = rng.uniform(-200.0, 200.0, 2)  # up to 4000 cells
        r = rng.uniform(0.0, 200.0)  # plus up to 4000 cells of beam: reach <= 8000
        a = rng.uniform(-math.pi, math.pi)
        case = (r * math.cos(a), r * math.sin(a), c, s, float(tx), float(ty), 1.0 / res)
        xr, yr = reference_cells(*case)
        xk, yk, amb = kernel_cells(*case)
        if not amb:
            assert (xk, yk) == (xr, yr), case


def test_end_points_a_hair_either_side_of_an_edge_at_any_heading():
    """Arbitrary headings (every product rounds): end points placed within 2^-30 .. 2^-36 cells of a cell edge, on both
    sides.  Three roundings at the magic's ulp can move the computed word either way; the guard keeps every such case
    either flagged or decided like the reference."""
    rng = np.random.default_rng(11)
    res = 0.05
    inv = 1.0 / res
    flagged = decided = 0
    for _ in range(1500):
        theta = rng.uniform(-math.pi, math.pi)
        c, s = math.cos(theta), math.sin(theta)
        tx, ty = float(rng.uniform(0.0, 100.0)), float(rng.uniform(0.0, 100.0))
        py = float(rng.uniform(-30.0, 30.0))
        if abs(c) < 0.2:
            continue
        cell = int(rng.integers(10, 1990))
        for eps in (0.0, 2.0 ** -36, -2.0 ** -36, 2.0 ** -34, -2.0 ** -34, 2.0 ** -33, -2.0 ** -33, 1.5 * 2.0 ** -32, -1.5 * 2.0 ** -32,
                    2.0 ** -31, -2.0 ** -31, 2.0 ** -30, -2.0 ** -30):
            target = (Fraction(cell) + Fraction(eps)) / Fraction(inv)
            # x word: solve (px * c - py * s + tx) * inv = cell + eps for px in exact arithmetic, then round px once
            px = float((target - Fraction(tx) + Fraction(py) * Fraction(s)) / Fraction(c))
            # y word (other magic constant): solve (qx * s + qy * c + ty) * inv = cell + eps for qy
            qx = py
            qy = float((target - Fraction(ty) - Fraction(qx) * Fraction(s)) / Fraction(c))
            for case in ((px, py, c, s, tx, ty, inv), (qx, qy, c, s, tx, ty, inv)):
                xr, yr = reference_cells(*case)
                xk, yk, amb = kernel_cells(*case)
                if amb:
                    flagged += 1
                else:
                    decided += 1
                    assert (xk, yk) == (xr, yr), (case, eps)
    assert flagged > 200 and decided > 200


def bordered_index(px: int, py: int, kx: int) -> int:
    """kernels.cuh: bordered_index -- 4 x 4 tiles, 2^kx tiles per row, y fastest inside a tile."""
    return ((py >> 2) << (kx + 4)) | ((px >> 2) << 4) | ((px & 3) << 2) | (py & 3)


def kernel_index(ux4: int, uy: int, kx: int) -> int:
    """fixed_lookup's integer tail: x arrives as 4 * padded x + two fraction bits, y as padded y; one bit-select (lop3 0xB8 with
    the immediate 3), one mask, one multiply-add with row_pitch = 4 * 2^kx."""
    low = (ux4 & ~3) | (uy & 3)
    return ((uy & ~3) * (4 << kx) + low) & 0xFFFFFFFF


def test_tile_index_is_the_bordered_layout():
    """The three integer operations of the lookup reproduce bordered_index for every padded cell and every value of the two
    fraction bits, the layout is a bijection onto the table, and clamped coordinates stay inside it."""
    for width, height in ((5, 7), (64, 33), (200, 200)):
        kx = max(0, math.ceil(math.log2(-(-(width + 2) // 4))))
        seen = set()
        for py in range(height + 2):
            for px in range(width + 2):
                want = bordered_index(px, py, kx)
                for frac in range(4):
                    assert kernel_index(4 * px + frac, py, kx) == want
                seen.add(want)
        assert len(seen) == (width + 2) * (height + 2)  # no two cells share an element
        rows = -(-(height + 2) // 4)
        assert max(seen) < rows * (16 << kx)
        # what __viaddmin_u32 leaves of wild coordinates: x_max = 4 (width + 1) + 3, y_max = height + 1 -> the far border
        x_max, y_max = 4 * (width + 1) + 3, height + 1
        for raw_x, raw_y in ((-5, 3), (2**31, 1), (7, -1), (4 * (width + 9), height + 40)):
            ux4 = min(raw_x & 0xFFFFFFFF, x_max)
            uy = min(raw_y & 0xFFFFFFFF, y_max)
            idx = kernel_index(ux4, uy, kx)
            assert idx in seen
            assert ((raw_x & 0xFFFFFFFF) <= x_max) or idx == bordered_index(width + 1, uy, kx)


def test_lop3_truth_table_is_a_bit_select():
    """lop3.b32 d, a, b, c, 0xB8 with b = 3: the immLut is f(a, b, c) evaluated on the masks 0xF0, 0xCC, 0xAA."""
    ta, tb, tc = 0xF0, 0xCC, 0xAA
    assert ((ta & ~tb) | (tc & tb)) & 0xFF == 0xB8
