"""The fixed-point likelihood-field lookup against the oracle on the device, at end points a hair from a cell edge.

reweight_lfm.cuh finds each end point's cell from two FMAs per coordinate with a magic number in the addend, trusts it
when the fraction word is at least 5 and redoes the particle with the reference's operation sequence otherwise.  Random
poses land near enough to an edge to test that argument about once in 10^8 lookups; here every particle is built by
tests/_cell_edges.py so that two of its end points lie 2^-38 .. 2^-28 cells either side of an x edge (integer or quarter
cell) and of a y edge that separate different field values, at arbitrary headings, and exactly on or one ulp from an
edge at quarter turns.  Each case asserts that it reaches the bands it is there for: guard-band words (5..64) decided by
the fast path, for x and for y, and flagged words redone exactly.

Every kernel form of launch_reweight_lfm is run: reweight_lfm_fixed_param_kernel<1> (scans of 181 and 2048 points),
<2> (n at the pair threshold and above; distinct hair poses tiled, so they sit as first and as second particle of a
lane), the chunked reweight_lfm_fixed_kernel (2049 and 4097 points: the margin restarts per 2048-point chunk) and the
general reweight_lfm_kernel (a map wider than 7998 cells), each through fixed_lookup<true> (64-slot blocks of particles
that keep every end point inside the grid) and fixed_lookup<false> (blocks with one particle near the border, and maps too
narrow for the in-grid test).  Maps: the 200 x 200 synthetic map with a rotated and translated origin, a 7998 x 96 strip
whose particles sit up to 7550 cells along it with a 500-cell scan radius (every term close to the 2^13 cells the error
bound allows), and grids at 1/3 m (an inexact inverse) and 0.025 m.  The likelihood (sum of pz^3) is compared bit for bit
on every scan, the prob model's exp(sum of log pz), which underflows over long scans, on the 181-point ones.  Finally a
whole Amcl step over a hair cloud, and the same filter restored into a batch, whose reweight is
reweight_lfm_fixed_block at every scan length."""
import math
import zlib

import numpy as np
import pytest

import _cell_edges as ce

pytestmark = pytest.mark.gpu

PI = math.pi
# z_random / max_laser_distance = 0.25 keeps every log pz in [-1.4, -0.2]: exp(sum log pz) over a 181-point scan stays a
# normal double, where a wrong cell shows.  Over 2048 points and more it underflows, so longer scans are checked with pz^3.
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=2.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
PAIR_FILL, PAIR_CTAS_PER_SM, WARPS_PER_CTA, TASK = 6, 2, 8, 64  # kRwPairFill, kRwPairBlocksPerSm, kRwThreads / 32, 2 * 32
N_HAIR = 1280  # hair particles per cloud: 20 blocks of 64 slots
MIN_BAND = 300  # guard-band x lookups, guard-band y lookups and flagged lookups each cloud must reach


@pytest.fixture(scope="module")
def bb():
    import beluga_b200 as bb
    from beluga_b200 import build as bb_build

    bb_build.build()
    if bb.device_count() == 0:
        pytest.fail("no CUDA device: -m gpu tests must run on the GPU box")
    return bb


@pytest.fixture(scope="module")
def pair_min(bb):
    """The smallest particle count that runs reweight_lfm_fixed_param_kernel<2>."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return TASK * (PAIR_FILL * sms * PAIR_CTAS_PER_SM * WARPS_PER_CTA - 1) + 1


@pytest.fixture(scope="module")
def scene():
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=2)


def sparse_cells(shape, seed):
    """Single occupied cells at 4 % density: the distance field, and so the table, changes across almost every edge."""
    rng = np.random.default_rng(seed)
    return np.where(rng.random(shape) < 0.04, 100, 0).astype(np.int8)


# name -> (cells, resolution, origin (x, y, theta) or None, scan radius in metres, inner pose box, border pose box; cells)
def map_spec(name, scene):
    if name == "synthetic":  # 30-cell radius: poses 32 cells from every edge keep their end points in the grid
        return scene.cells, scene.resolution, (0.3, -0.2, 0.1), 1.5, ((33, 166), (33, 166)), ((6, 30), (33, 166))
    if name == "strip":  # terms near 2^13 cells: reach = 500 + 7550 + 2 < 8100; the strip is too narrow for the in-grid test
        return sparse_cells((96, 7998), 1), 0.05, None, 25.0, ((500, 7550), (-300, 400)), None
    if name == "third":
        return sparse_cells((300, 300), 2), 1.0 / 3.0, None, 20.0, ((63, 237), (63, 237)), ((20, 60), (63, 237))
    if name == "fine":
        return sparse_cells((400, 400), 3), 0.025, None, 3.0, ((123, 277), (123, 277)), ((40, 120), (123, 277))
    assert name == "wide"  # 8100 + 2 cells > kFixedMaxSide: the general kernel
    return sparse_cells((48, 8100), 4), 0.05, None, 25.0, ((500, 7550), (-300, 300)), None


class Cloud:
    """A map, a scan and N_HAIR hair particles on it, in blocks of 64 slots; every other block (when the map has room for
    the in-grid test) holds one particle near the border, at a lane that moves from block to block."""

    def __init__(self, bb, orc, scene, name, n_points):
        cells, res, origin, radius, inner, border = map_spec(name, scene)
        self.cells, self.res = cells, res
        self.origin = orc.IDENTITY.copy() if origin is None else orc.se2(*origin)
        rng = np.random.default_rng(zlib.crc32(f"{name}-{n_points}".encode()))
        r = radius * np.sqrt(rng.uniform(0.0, 1.0, n_points))
        a = rng.uniform(-PI, PI, n_points)
        pts = np.stack([r * np.cos(a), r * np.sin(a)], axis=1)
        self.points = pts * np.minimum(1.0, radius / np.maximum(np.abs(pts).sum(axis=1), 1e-300))[:, None]  # |x| + |y| <= radius
        grid = orc.Grid(cells, res, self.origin)
        pz = orc.likelihood_field(orc.LfmParam(**LFM), grid).astype(np.float64)
        # a wrong cell must move the weight: both tables differ across the edge by more than 1e-9 of any particle's sum
        sharp = None
        for f in (pz ** 3, np.log(pz)):
            e = ce.EdgeMap.from_values(f, res, thresh=1e-9 * n_points * np.abs(f).max())
            sharp = e if sharp is None else ce.EdgeMap(e.inv, e.width, e.height, e.world_to_field, sharp.sharp_x & e.sharp_x, sharp.sharp_y & e.sharp_y)
        w2f = orc.se2_inverse(self.origin)  # the map's world_to_field, from the host's libm as on the device
        self.emap = ce.EdgeMap(1.0 / res, cells.shape[1], cells.shape[0], tuple(float(v) for v in w2f), sharp.sharp_x, sharp.sharp_y)
        quarter = 0.3 if origin is None else 0.0
        blocks = N_HAIR // TASK
        n_border = blocks // 2 if border is not None else 0
        states, poses = ce.hair_cloud(rng, self.emap, self.points, inner, N_HAIR - n_border, quarter_share=quarter)
        if n_border:
            bs, bp = ce.hair_cloud(rng, self.emap, self.points, border, n_border, quarter_share=quarter)
            states, poses = list(states), list(poses)
            for j in range(n_border):  # block 2j + 1 gets a border particle at lane (7 j) mod 64
                at = (2 * j + 1) * TASK + (7 * j) % TASK
                states.insert(at, bs[j])
                poses.insert(at, bp[j])
            states, poses = np.array(states), np.array(poses)
        self.states, self.poses = states, poses
        self.radius = float(np.abs(self.points).sum(axis=1).max())
        self.inside = np.array([ce.in_grid(self.emap, p, self.radius) for p in poses])
        self.grid_bb = bb.OccupancyGrid(cells, res, self.origin)
        self.grid_orc = grid

    def oracle(self, orc, sensor, states=None):
        return orc.sensor_weights(sensor, orc.LfmParam(**LFM), self.grid_orc, self.points, self.states if states is None else states)

    def bands(self, poses=None):
        return ce.cloud_bands(self.emap, self.points, self.poses if poses is None else poses)


_clouds = {}


def cloud(bb, orc, scene, name, n_points):
    key = (name, n_points)
    if key not in _clouds:
        _clouds[key] = Cloud(bb, orc, scene, name, n_points)
    return _clouds[key]


def assert_weights(sensor, got, exp):
    """test_reweight_lfm_bit_exact's rule: bit for bit for pz^3, rtol 1e-13 (one exp() per particle) for log pz."""
    if sensor == 0:
        bad = np.nonzero(got != exp)[0]
        assert len(bad) == 0, f"{len(bad)} weights differ, first at {bad[:8]}"
    else:
        normal = exp > 1e-290
        assert np.allclose(got[normal], exp[normal], rtol=1e-13, atol=0.0)
        assert np.allclose(got[~normal], exp[~normal], rtol=1e-6, atol=1e-320)


def reweigh(bb, c, sensor, idx):
    f = bb.Filter(capacity=len(idx))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), c.grid_bb, prob=(sensor == 1))
    f.set_particles(c.states[idx])
    f.reweight(c.points)
    return f.particles()[1]


# form, map, scan points: every kernel launch_reweight_lfm can pick, on the maps that reach its lookup paths; the
# likelihood (pz^3) with every scan, the log likelihood with the short ones (LFM)
CASES = [("param1", "synthetic", 181), ("param1", "synthetic", 2048), ("param1", "strip", 181), ("param1", "third", 181),
         ("param1", "fine", 181), ("pair", "synthetic", 181), ("pair", "strip", 181), ("chunked", "synthetic", 2049),
         ("chunked", "strip", 4097), ("general", "wide", 181)]
CASES = [case + (sensor,) for case in CASES for sensor in (0, 1) if sensor == 0 or case[2] <= 181]


@pytest.mark.parametrize("form, name, n_points, sensor", CASES, ids=[f"{f}-{m}-{p}-{s}" for f, m, p, s in CASES])
def test_hair_clouds_match_the_oracle(bb, orc, scene, pair_min, form, name, n_points, sensor):
    c = cloud(bb, orc, scene, name, n_points)
    b = c.bands()
    assert b.wrong == 0  # the model's own claim on these cases
    if form != "general":
        assert min(b.guard_x, b.guard_y, b.flagged) >= MIN_BAND, b
        assert b.decided_particles >= 300 and b.flagged_particles >= 300, b
    if form == "chunked" and n_points > 2 * ce.CHUNK:
        assert b.split_particles >= 10, b  # flagged in one chunk, decided in the guard band in another
    # which lookup path each 32-slot warp takes (fixed_lookup<true> needs every particle of the warp inside)
    warps = c.inside.reshape(-1, 32).all(axis=1)
    if name in ("synthetic", "third", "fine"):
        assert warps.sum() >= 10 and (~warps).sum() >= 10
    exp = c.oracle(orc, sensor)
    assert sensor == 0 or (exp > 1e-290).all()  # no weight underflows: every wrong cell would show
    if form == "pair":
        n = pair_min + 37
        idx = np.arange(n) % len(c.states)  # a multiple of 64: every tile repeats the same 64-slot blocks
        assert_weights(sensor, reweigh(bb, c, sensor, idx), exp[idx])
    else:
        assert form != "param1" or n_points <= 2048
        assert form != "chunked" or n_points > 2048
        assert form != "general" or c.cells.shape[1] + 2 > 8000
        assert_weights(sensor, reweigh(bb, c, sensor, np.arange(len(c.states))), exp)


def test_field_frame_replay_is_the_oracles(orc, bb, scene):
    """The generator's pose_mul(world_to_field, state): the translation bit for bit the oracle's, the heading within an ulp
    (only hypot differs between libms), so the edges it aims at are the oracle's."""
    c = cloud(bb, orc, scene, "synthetic", 181)
    w2f = orc.se2_inverse(c.origin)
    for st, pose in zip(c.states[:200], c.poses[:200]):
        want = orc.se2_compose(w2f, st)
        assert pose[2] == want[2] and pose[3] == want[3]
        assert abs(pose[0] - want[0]) <= 2.3e-16 and abs(pose[1] - want[1]) <= 2.3e-16


def test_amcl_step_and_batch_over_a_hair_cloud(bb, orc, scene):
    """A normalising Amcl step with zero motion noise over a hair cloud, and the same filter restored into a batch (whose
    reweight is reweight_lfm_fixed_block for a 181-point scan too): byte for byte the same, and the weights the oracle's
    on the read-back states, normalised as the fixed-point CDF does it."""
    c = cloud(bb, orc, scene, "synthetic", 181)
    n = len(c.states)
    rng = np.random.default_rng(5)
    w0 = rng.uniform(0.5, 1.0, n)
    ap = bb.AmclParams(min_particles=n, max_particles=n, resample_interval=1000, seed=9)
    lfm = bb.LikelihoodFieldModelParam(**LFM)
    solo = bb.Amcl(bb.DifferentialDriveModelParam(0.0, 0.0, 0.0, 0.0), ap)
    solo.update_map(bb.SENSOR_LIKELIHOOD_FIELD, lfm, c.grid_bb)
    solo.initialize_states(c.states, w0)
    batch = bb.AmclBatch.from_states([solo.export_state()])
    batch.update_map(0, batch.add_likelihood_field_map(lfm, c.grid_bb))
    pose = orc.se2(1.0, 2.0, 0.3)
    rs = solo.update(pose, c.points)
    (rb,) = batch.update([pose], [c.points])
    assert rs.updated == rb.updated == 1 and rs.resampled == rb.resampled == 0
    ss, sw = solo.particles()
    bs, bw = batch.particles(0)
    assert ss.tobytes() == bs[:n].tobytes() and sw.tobytes() == bw[:n].tobytes()
    raw = w0 * c.oracle(orc, 0, ss)
    _, cdf, ex = orc.resample_indices(raw, orc.MULTINOMIAL, seed=9, step=1)
    assert sw.tobytes() == (raw / math.ldexp(float(int(cdf[-1])), -ex)).tobytes()
    # zero-noise motion moves the states by ulps at most: the cloud still sits in the bands
    assert np.abs(ss - c.states).max() < 1e-12
    field = np.array([orc.se2_compose(orc.se2_inverse(c.origin), st) for st in ss])
    b = c.bands(field)
    assert min(b.guard_x, b.guard_y, b.flagged) >= MIN_BAND, b
