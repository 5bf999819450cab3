"""Executable version of the argument behind reweight_lfm_fixed_*_kernel (csrc/reweight_lfm.cuh): the kernel finds the
likelihood-field CELL of a beam end point with two FMAs per coordinate and a magic-number add instead of the
reference's rounded operation sequence -- the magic number riding in the FMAs' addend -- and claims the same cell
whenever the fraction word it reads is at least 5.

This test replays both evaluations on the CPU -- IEEE doubles for the reference sequence, exact rationals rounded
once for the FMAs -- on random and adversarial (cell-edge) inputs and checks the claim, plus how often the
fallback would be taken.  CPU only; it models the arithmetic, it does not run the kernel.  The model and the case
generator live in tests/_cell_edges.py, which test_gpu_lfm_cell_edges.py runs on the device."""
import math
from fractions import Fraction

import numpy as np
import pytest

import _cell_edges as ce
from _cell_edges import kernel_cells, reference_cells


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


# The shared generator (tests/_cell_edges.py) at the edges of the argument: end points 500 cells from poses 7550 cells
# along a 7998-cell strip (every term near 2^13 cells, where the error bound is largest), and a 1/3 m grid (an inverse that
# is not exact).  Every edge counts as one that changes the value read.
HAIR_MAPS = {"strip": ((96, 7998), 0.05, 25.0, ((500, 7550), (-300, 400))), "third": ((300, 300), 1.0 / 3.0, 20.0, ((63, 237), (63, 237)))}
_hair = {}


def hair_set(name):
    if name not in _hair:
        shape, res, radius, box = HAIR_MAPS[name]
        rng = np.random.default_rng(list(HAIR_MAPS).index(name) + 1)
        emap = ce.EdgeMap.from_values(np.zeros(shape), res, thresh=-1.0)
        r = radius * np.sqrt(rng.uniform(0.0, 1.0, 181))
        a = rng.uniform(-math.pi, math.pi, 181)
        pts = np.stack([r * np.cos(a), r * np.sin(a)], axis=1)
        pts *= np.minimum(1.0, radius / np.abs(pts).sum(axis=1))[:, None]
        _, poses = ce.hair_cloud(rng, emap, pts, box, 500, quarter_share=0.3)
        _hair[name] = emap, pts, poses
    return _hair[name]


@pytest.mark.parametrize("name", list(HAIR_MAPS))
def test_hair_clouds_near_the_range_limit_and_at_an_inexact_inverse(name):
    emap, pts, poses = hair_set(name)
    reach = (np.abs(pts).sum(axis=1).max() + np.abs(poses[:, 2:]).max()) * emap.inv + 2.0
    assert reach < ce.REACH_LIMIT and (name != "strip" or reach > 8000.0)
    b = ce.cloud_bands(emap, pts, poses)
    assert b.wrong == 0, b
    assert min(b.guard_x, b.guard_y, b.flagged) >= 150 and b.decided_particles >= 150 and b.flagged_particles >= 150, b


@pytest.mark.parametrize("mutation", ["no_guard", "no_ambiguity"])
def test_the_hair_clouds_catch_a_weaker_lookup(mutation):
    """Without the two ulps of guard, or with only a zero fraction word taken as ambiguous, the model predicts a wrong cell
    for some decided lookup of the generated cases: the device test built on them fails under either change."""
    guard, ambiguous = ((0.0, 0.0), ce.AMBIGUOUS_BELOW) if mutation == "no_guard" else ((ce.GUARD_X, ce.GUARD_Y), 0)
    wrong = sum(ce.cloud_bands(emap, pts, poses, guard, ambiguous).wrong for emap, pts, poses in map(hair_set, HAIR_MAPS))
    assert wrong >= 1


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
