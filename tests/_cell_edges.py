"""Cell-edge cases for the fixed-point likelihood-field lookup (csrc/reweight_lfm.cuh: fixed_lookup, fixed_pose_setup).

The kernel finds an end point's cell from two FMAs per coordinate with a magic number in the addend, and trusts that cell
when the low "fraction word" it reads is above AMBIGUOUS_BELOW; a particle with any smaller word has its beams redone with
the reference's own operation sequence.  This module replays both evaluations on the CPU -- IEEE doubles for the
reference sequence, exact rationals rounded once for each FMA -- and builds particles whose end points lie a hair either
side of a cell edge at any heading, so that the CPU model (test_fixed_point_lookup_model.py) and the device
(test_gpu_lfm_cell_edges.py) meet the same cases.

A lookup is *flagged* when one of its fraction words is at most AMBIGUOUS_BELOW (the particle is redone exactly), in the
*guard band* when a word lies in 5..GUARD_BAND (decided by the fast path close to an edge), and *plain* otherwise.  The
fallback redoes a whole particle per staged chunk of the scan, so a lookup is *decided* only when no lookup of its
particle in the same chunk is flagged."""
import math
import struct
from dataclasses import dataclass
from fractions import Fraction

import numpy as np

MAGIC_X, MAGIC_Y = 393216.0, 1572864.0  # 1.5 * 2^18, 1.5 * 2^20 (kFixedMagicX / kFixedMagicY)
BIAS_X, BIAS_Y = 0x41180000, 0x41380000
# Folding the magic add into the FMA chain costs three roundings at the magic's ulp (2^-34 for x, 2^-32 for y) instead of
# one: the computed fixed-point value lies within 3 half-ulps + 2^-36 of the reference's.  Two ulps of guard are added to
# the offset, so that the uncertainty interval sits entirely BELOW the computed value: the cell is the reference's
# whenever the fraction word is at least 5 (kFixedGuardX / kFixedGuardY / kFixedAmbiguous in the kernel).
GUARD_X, GUARD_Y = 2.0 ** -33, 2.0 ** -31
AMBIGUOUS_BELOW = 4
GUARD_BAND = 64  # fraction words 5..64: the fast path decides within 64 words of an edge
REACH_LIMIT = 8100.0  # fixed_pose_setup: every term below 2^13 cells
CHUNK = 2048  # kChunkBeams: the fallback redoes one staged chunk of the scan
FAR = 1 << 31  # the word recorded for a lookup too far from every edge to be replayed exactly
# Offsets (cells) of a reference value from the edge it is placed at, on both sides: 1..8 ulps of the x word (2^-34) and of
# the y word (2^-32), two coarser steps, and fractions of an x ulp down to 2^-38 -- the offsets at which three roundings
# can carry the fixed-point value across the edge.  All are at least 2^-38 cells, far above the one-ulp heading difference
# the device's hypot may make (points_radius / res * 2^-51 cells), so the oracle and the device agree on the side of the
# edge.  GUARDED_X / GUARDED_Y: the offsets whose word lands in the guard band (at least 4 ulps above the edge).
EPS = tuple(sorted({sg * k * 2.0 ** e for sg in (1, -1) for k in range(1, 9) for e in (-34, -32)}
                   | {sg * 2.0 ** e for sg in (1, -1) for e in (-38, -37, -36, -35, -30, -28)}))
GUARDED_X = tuple(e for e in EPS if e >= 2.0 ** -32)
GUARDED_Y = tuple(e for e in EPS if e >= 2.0 ** -30)
FINE = tuple(e for e in EPS if abs(e) < 2.0 ** -34)  # drawn more often: without the guard they can give a wrong cell


def fma(a: float, b: float, c: float) -> float:
    return float(Fraction(a) * Fraction(b) + Fraction(c))  # one rounding, to nearest even


def words(t: float):
    bits = struct.unpack("<Q", struct.pack("<d", t))[0]
    return bits >> 32, bits & 0xFFFFFFFF


def reference_cells(px, py, c, s, tx, ty, inv):
    x = (px * c - py * s) + tx  # likelihood_field_model.hpp:82-83, every operation rounded
    y = (px * s + py * c) + ty
    return math.floor(x * inv), math.floor(y * inv)  # regular_grid.hpp:75-78


def kernel_words(px, py, c, s, tx, ty, inv, guard=(GUARD_X, GUARD_Y)):
    """-> (cell x, cell y, x fraction word, y fraction word) as fixed_lookup computes them (before clamping to the border)."""
    cx, sx = c * inv, s * inv
    # the magic constants ride in the FMAs' addend: (offset + 1 border cell) + (magic + guard), each sum rounded once
    ox, oy = (tx * inv + 1.0) + (MAGIC_X + guard[0]), (ty * inv + 1.0) + (MAGIC_Y + guard[1])
    gx = fma(px, cx, fma(-py, sx, ox))
    gy = fma(px, sx, fma(py, cx, oy))
    hx, lx = words(gx)
    hy, ly = words(gy)
    ux = (hx - BIAS_X) & 0xFFFFFFFF  # 4 * padded x + 2 fraction bits (padded x = cell + 1, for cells >= -1)
    uy = (hy - BIAS_Y) & 0xFFFFFFFF  # padded y
    to_signed = lambda u: u - (1 << 32) if u >= (1 << 31) else u  # noqa: E731
    return (to_signed(ux) >> 2) - 1, to_signed(uy) - 1, lx, ly


def kernel_cells(px, py, c, s, tx, ty, inv, guard=(GUARD_X, GUARD_Y), ambiguous=AMBIGUOUS_BELOW):
    """-> (cell x, cell y, ambiguous) as fixed_lookup computes them (before clamping to the border)."""
    xk, yk, lx, ly = kernel_words(px, py, c, s, tx, ty, inv, guard)
    return xk, yk, (lx <= ambiguous or ly <= ambiguous)


# ---- the field frame: transform = world_to_field * state (se2_math.cuh: rot_make, rot_mul, pose_mul, pose_inverse) ----
def rot_make(re, im):
    n = math.hypot(re, im)
    return re / n, im / n


def rot_mul(a, b):
    re = a[0] * b[0] - a[1] * b[1]
    im = a[0] * b[1] + a[1] * b[0]
    sq = re * re + im * im
    if sq != 1.0:
        scale = 2.0 / (1.0 + sq)
        re, im = re * scale, im * scale
    return rot_make(re, im)


def pose_mul(a, b):
    """(c, s, x, y) of a * b.  Only the heading goes through hypot, which may differ from the device's by an ulp; the
    translation is plain + and *, bit for bit the device's and the oracle's."""
    c, s = rot_mul(a[:2], b[:2])
    rx = a[0] * b[2] - a[1] * b[3]
    ry = a[1] * b[2] + a[0] * b[3]
    return (c, s, a[2] + rx, a[3] + ry)


def pose_inverse(a):
    c, s = rot_make(a[0], -a[1])
    nx, ny = a[2] * -1.0, a[3] * -1.0
    return (c, s, c * nx - s * ny, s * nx + c * ny)


# ---- classification -----------------------------------------------------------------------------------------------
@dataclass
class EdgeMap:
    """What the generator needs of a likelihood field: its geometry and which cell edges separate different values."""
    inv: float  # 1 / resolution, as the map computes it
    width: int
    height: int
    world_to_field: tuple  # pose_inverse(origin), computed on the host like the map's
    sharp_x: np.ndarray  # [height, width + 1]: the edge at x = e of row `row` separates two different values
    sharp_y: np.ndarray  # [height + 1, width]: the edge at y = e of column `col`

    @staticmethod
    def from_values(values, resolution, origin=(1.0, 0.0, 0.0, 0.0), thresh=0.0):
        """`values`: per-cell table values [height, width]; an edge counts where they differ by more than `thresh`."""
        h, w = values.shape
        sx = np.zeros((h, w + 1), dtype=bool)
        sy = np.zeros((h + 1, w), dtype=bool)
        sx[:, 1:w] = np.abs(np.diff(values, axis=1)) > thresh
        sy[1:h, :] = np.abs(np.diff(values, axis=0)) > thresh
        return EdgeMap(1.0 / resolution, w, h, pose_inverse(tuple(float(v) for v in origin)), sx, sy)


@dataclass
class Lookups:
    """Every lookup of one particle: the reference's cells, the kernel's cells and fraction words (FAR: far from edges)."""
    ref_x: np.ndarray
    ref_y: np.ndarray
    ker_x: np.ndarray
    ker_y: np.ndarray
    lx: np.ndarray
    ly: np.ndarray


def lookups(points, pose, inv, guard=(GUARD_X, GUARD_Y), near=1 << 12):
    """Classify scan `points` for one field-frame pose (c, s, tx, ty).  Lookups within `near` words of a quarter-cell
    edge (x) or a cell edge (y) are replayed exactly; the others keep the reference's cells and the word FAR."""
    c, s, tx, ty = pose
    px, py = points[:, 0], points[:, 1]
    gx = ((px * c - py * s) + tx) * inv  # numpy rounds every operation, as the reference does
    gy = ((px * s + py * c) + ty) * inv
    ref_x, ref_y = np.floor(gx).astype(np.int64), np.floor(gy).astype(np.int64)
    ker_x, ker_y = ref_x.copy(), ref_y.copy()
    lx = np.full(len(px), FAR, dtype=np.int64)
    ly = lx.copy()
    dx = np.abs(4.0 * gx - np.round(4.0 * gx)) * 2.0 ** 32  # distance to the nearest quarter edge, in x words
    dy = np.abs(gy - np.round(gy)) * 2.0 ** 32
    for b in np.nonzero((dx < near) | (dy < near))[0]:
        ker_x[b], ker_y[b], lx[b], ly[b] = kernel_words(float(px[b]), float(py[b]), c, s, tx, ty, inv, guard)
    return Lookups(ref_x, ref_y, ker_x, ker_y, lx, ly)


@dataclass
class Bands:
    flagged: int = 0  # lookups with a word <= the ambiguity limit
    guard_x: int = 0  # decided lookups with the x word in 5..GUARD_BAND
    guard_y: int = 0
    decided_particles: int = 0  # particles no chunk of which is redone
    flagged_particles: int = 0  # particles with at least one chunk redone
    split_particles: int = 0  # flagged in one chunk, in the guard band of a decided one in another
    wrong: int = 0  # decided lookups whose kernel cell (inside the grid) is not the reference's

    def __iadd__(self, o):
        for k in self.__dict__:
            setattr(self, k, getattr(self, k) + getattr(o, k))
        return self


def particle_bands(lk: Lookups, width, height, ambiguous=AMBIGUOUS_BELOW) -> Bands:
    n = len(lk.lx)
    flag = (lk.lx <= ambiguous) | (lk.ly <= ambiguous)
    chunk_flag = np.repeat([flag[i:i + CHUNK].any() for i in range(0, n, CHUNK)], CHUNK)[:n]
    decided = ~chunk_flag
    gx = decided & (lk.lx > AMBIGUOUS_BELOW) & (lk.lx <= GUARD_BAND)
    gy = decided & (lk.ly > AMBIGUOUS_BELOW) & (lk.ly <= GUARD_BAND)

    def cell(x, y):  # out-of-grid end points all read the unknown-space value
        inside = (x >= 0) & (x < width) & (y >= 0) & (y < height)
        return np.where(inside, x, -1), np.where(inside, y, -1)

    rx, ry = cell(lk.ref_x, lk.ref_y)
    kx, ky = cell(lk.ker_x, lk.ker_y)
    return Bands(flagged=int(flag.sum()), guard_x=int(gx.sum()), guard_y=int(gy.sum()), decided_particles=int(not chunk_flag.any()),
                 flagged_particles=int(chunk_flag.any()), split_particles=int(chunk_flag.any() and (gx | gy).any()),
                 wrong=int((decided & ((rx != kx) | (ry != ky))).sum()))


def cloud_bands(emap: EdgeMap, points, field_poses, guard=(GUARD_X, GUARD_Y), ambiguous=AMBIGUOUS_BELOW) -> Bands:
    out = Bands()
    for pose in field_poses:
        out += particle_bands(lookups(points, tuple(pose), emap.inv, guard), emap.width, emap.height, ambiguous)
    return out


def in_grid(emap: EdgeMap, pose, points_radius) -> bool:
    """fixed_pose_setup's test: every end point of the particle lies inside the grid."""
    cells = points_radius * emap.inv + 2.0
    gx, gy = pose[2] * emap.inv, pose[3] * emap.inv
    return gx - cells >= 0.0 and gx + cells < emap.width and gy - cells >= 0.0 and gy + cells < emap.height


# ---- the generator ------------------------------------------------------------------------------------------------
def solve_offset(u: float, target: Fraction, inv: float) -> float:
    """The translation t, rounded once from the exact rational, for which (u + t) * inv = target cells."""
    return float(target / Fraction(inv) - Fraction(u))


def nudge_to(u: float, t: float, inv: float, want: float):
    """t moved by up to 64 ulps so that the reference's (u + t) * inv is exactly `want`, or None."""
    up, down = t, t
    for _ in range(65):
        for tt in (up, down):
            if (u + tt) * inv == want:
                return tt
        up, down = math.nextafter(up, math.inf), math.nextafter(down, -math.inf)
    return None


def place(u: float, edge: Fraction, off, inv: float):
    """The translation that puts the reference's (u + t) * inv at edge + off cells (off a float), or exactly on the edge
    ("on"), or one ulp above or below it ("up", "down"); None if no translation does."""
    if not isinstance(off, str):
        return solve_offset(u, edge + Fraction(off), inv)
    e = float(edge)
    want = {"on": e, "up": math.nextafter(e, math.inf), "down": math.nextafter(e, -math.inf)}[off]
    return nudge_to(u, solve_offset(u, edge, inv), inv, want)


def hair_particle(rng, emap: EdgeMap, points, box, quarter=False, guarded=False, tries=400):
    """One world-frame state whose field-frame pose lies in `box` ((x lo, x hi), (y lo, y hi), in cells) and puts the end
    point of a scan point k a hair from an x edge (an integer one, or one time in four a quarter-cell edge) and that of a
    point k' (one time in four k itself: a corner) a hair from a y edge, both inside the grid.  Integer edges are only
    taken where they separate different table values.  No other lookup of the particle is flagged.  `quarter`:
    quarter-turn headings (identity map origin only), where the rotation is exact, and offsets of 0 and +-1 ulp of the
    reference's value join EPS.  `guarded`: offsets from GUARDED_X / GUARDED_Y only, so that the particle is decided by
    the fast path in the guard band.  -> (state, field-frame pose), or None after `tries` draws."""
    inv, w2f = emap.inv, emap.world_to_field
    identity = w2f == (1.0, 0.0, 0.0, 0.0)
    assert identity or not quarter
    radius = float(np.abs(points).sum(axis=1).max())
    offsets_x = GUARDED_X if guarded else EPS + (("on", "up", "down") if quarter else ())
    offsets_y = GUARDED_Y if guarded else offsets_x
    for _ in range(tries):
        if quarter:
            rot = ((1.0, 0.0), (0.0, 1.0), (-1.0, 0.0), (0.0, -1.0))[int(rng.integers(0, 4))]
        else:
            th = float(rng.uniform(-math.pi, math.pi))
            rot = (math.cos(th), math.sin(th))
        c, s = rot_mul(w2f[:2], rot)
        x0, y0 = float(rng.uniform(*box[0])) / inv, float(rng.uniform(*box[1])) / inv
        k = int(rng.integers(0, len(points)))
        k2 = k if rng.random() < 0.25 else int(rng.integers(0, len(points)))
        px, py, qx, qy = float(points[k, 0]), float(points[k, 1]), float(points[k2, 0]), float(points[k2, 1])
        u = px * c - py * s  # the x of point k before the offset, rounded as the reference rounds it
        v = qx * s + qy * c  # the y of point k'
        quarter_edge = rng.random() < 0.25
        gx = (u + x0) * inv
        ex = Fraction(round(4.0 * gx), 4) if quarter_edge else Fraction(round(gx))
        if quarter_edge and ex.denominator == 1:
            continue
        ey = Fraction(round((v + y0) * inv))
        ox = FINE if not guarded and rng.random() < 0.3 else offsets_x
        oy = FINE if not guarded and rng.random() < 0.3 else offsets_y
        tx = place(u, ex, ox[int(rng.integers(0, len(ox)))], inv)
        ty = place(v, ey, oy[int(rng.integers(0, len(oy)))], inv)
        if tx is None or ty is None:
            continue
        # the state whose field-frame translation is (tx, ty), and the field-frame pose the map computes from it
        state = (rot[0], rot[1], tx, ty) if identity else (rot[0], rot[1]) + pose_mul(pose_inverse(w2f), (c, s, tx, ty))[2:]
        pose = pose_mul(w2f, state)
        if not (box[0][0] <= pose[2] * inv <= box[0][1] and box[1][0] <= pose[3] * inv <= box[1][1]):
            continue
        if (radius + max(abs(pose[2]), abs(pose[3]))) * inv + 2.0 >= REACH_LIMIT:
            continue
        c1, s1 = pose[0], pose[1]  # the reference's end points of k and k', in cells
        xk, yk = ((px * c1 - py * s1) + pose[2]) * inv, ((px * s1 + py * c1) + pose[3]) * inv
        xk2, yk2 = ((qx * c1 - qy * s1) + pose[2]) * inv, ((qx * s1 + qy * c1) + pose[3]) * inv
        row, col, xe, ye = math.floor(yk), math.floor(xk2), round(xk), round(yk2)  # the x target's row, the y target's column
        if not (0 <= row < emap.height and 0 <= math.floor(xk) < emap.width and 0 <= col < emap.width and 0 < ye < emap.height):
            continue
        if not emap.sharp_y[ye, col] or not (quarter_edge or (0 < xe < emap.width and emap.sharp_x[row, xe])):
            continue
        everything = lookups(points, pose, inv)
        flag = (everything.lx <= AMBIGUOUS_BELOW) | (everything.ly <= AMBIGUOUS_BELOW)
        flag[[k, k2]] = False
        if flag.any():
            continue
        return np.array(state), np.array(pose)
    return None


def hair_cloud(rng, emap: EdgeMap, points, box, n, quarter_share=0.0, guarded_share=0.5):
    """n hair particles (hair_particle) -> (states [n, 4], field-frame poses [n, 4])."""
    states, poses = [], []
    while len(states) < n:
        got = hair_particle(rng, emap, points, box, quarter=rng.random() < quarter_share, guarded=rng.random() < guarded_share)
        if got is not None:
            states.append(got[0])
            poses.append(got[1])
    return np.array(states), np.array(poses)
