"""The two-particle variant of the persistent likelihood-field kernel against the CPU oracle, bit for bit.

reweight_lfm_fixed_param_kernel<2> gives lane l of a 64-slot task the schedule slots l and l + 32.  The launcher runs it
when the pair tasks fill every resident warp PAIR_FILL times over (PAIR_FILL x SMs x PAIR_CTAS_PER_SM CTAs x 8 warps,
811 008 particles on a 132-SM H100); below that the one-particle kernel reweight_lfm_fixed_param_kernel<1> runs.
Filter.reweight uses no schedule, so slot j holds particle j.  Every case below uses more particles than the threshold
and reaches the pair kernel, except the `below` cases of test_pair_threshold_counts, which reach the one-particle kernel.
Scans of up to 1920 points are kernel parameters; all scans here are.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PAIR_FILL, PAIR_CTAS_PER_SM, WARPS_PER_CTA, TASK = 6, 2, 8, 64  # kRwPairFill, kRwPairBlocksPerSm, kRwThreads / 32, 2 * 32
PI = np.pi
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)


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
    """The smallest particle count that runs the pair kernel."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return TASK * (PAIR_FILL * sms * PAIR_CTAS_PER_SM * WARPS_PER_CTA - 1) + 1


@pytest.fixture(scope="module")
def scene():
    from beluga_b200 import synthetic

    # 254 + 2 border cells = 64 whole tiles per row: the bordered table has no padding columns, so a cell past the right
    # edge read without the clamp would be a cell of the next tile row, not another copy of the border value
    return synthetic.make_scenario(grid_size=254, n_beams=181, steps=2)


def poses(orc, xs, ys, ths):
    return np.array([orc.se2(x, y, t) for x, y, t in zip(xs, ys, ths)])


def weigh(bb, orc, scene, pts, distinct, idx, times=1):
    """GPU weights of the particles distinct[idx] after `times` launches, and the oracle's (computed once per distinct pose)."""
    f = bb.Filter(capacity=len(idx))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution, orc.IDENTITY), prob=False)
    f.set_particles(distinct[idx])
    for _ in range(times):
        f.reweight(pts)
    once = orc.sensor_weights(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution), pts, distinct)[idx]
    exp = once
    for _ in range(times - 1):
        exp = exp * once
    return f.particles()[1], exp


def mixed_poses(orc, scene, rng, n):
    """Poses all over the grid and up to a metre outside it: most warps clamp, a few run the in-grid loop."""
    extent = scene.cells.shape[0] * scene.resolution
    return poses(orc, rng.uniform(-1.0, extent + 1.0, n), rng.uniform(-1.0, extent + 1.0, n), rng.uniform(-PI, PI, n))


TAILS = [1, 2, 63, 64, 65, 127, 129]
COUNTS = [("below", 7), ("below", 1920)] + [(f"tail{k}", 7) for k in TAILS] + [("tail1", 1920)]


@pytest.mark.parametrize("count, n_points", COUNTS, ids=[f"{c}-{p}pts" for c, p in COUNTS])
def test_pair_threshold_counts(bb, orc, scene, pair_min, count, n_points):
    """The largest count that still runs the one-particle kernel ("below"), and counts that run the pair kernel with 1,
    2, 63, 64, 1, 63 and 1 slots of the last 64-slot task filled ("tail1" is the smallest pair count): the idle slots of
    the last task take the dummy pose and are not written, and one lane can have its first slot active and its second
    idle."""
    n = pair_min - 1 if count == "below" else pair_min - 1 + int(count[4:])
    rng = np.random.default_rng(n + n_points)
    distinct = mixed_poses(orc, scene, rng, 2048)
    pts = rng.uniform(-4.0, 4.0, (n_points, 2))
    got, exp = weigh(bb, orc, scene, pts, distinct, rng.integers(0, len(distinct), n))
    assert np.array_equal(got, exp)


def test_pair_kernel_rewinds_its_ticket_counter(bb, orc, scene, pair_min):
    """Two launches in a row on one filter, n not a multiple of 64: the last warp out must rewind the ticket counter."""
    rng = np.random.default_rng(8)
    n = pair_min + 37
    assert n % TASK != 0
    distinct = mixed_poses(orc, scene, rng, 2048)
    pts = rng.uniform(-4.0, 4.0, (64, 2))
    got, exp = weigh(bb, orc, scene, pts, distinct, rng.integers(0, len(distinct), n), times=2)
    assert np.array_equal(got, exp)


def test_exact_fallback_for_one_particle_of_a_pair(bb, orc, scene, pair_min):
    """Poses on exact cell multiples, with end points on cell multiples and one ulp either side, must be redone with the
    reference's operation sequence.  Each one shares its lane with a generic pose, as the first particle of the pair in
    some lanes and as the second in others, and every pose stays far enough inside the grid for its warp to run the
    in-grid loop."""
    res = scene.resolution
    rng = np.random.default_rng(17)
    m = rng.integers(-20, 21, (64, 2)).astype(np.float64) * res
    pts = np.concatenate([m, np.nextafter(m, np.inf), np.nextafter(m, -np.inf)])  # 192 points, |x| + |y| <= 2 m = 40 cells
    k = rng.integers(60, 195, (200, 2)).astype(np.float64)  # the in-grid test needs 42 cells to every edge
    edge = np.concatenate([poses(orc, k[:, 0] * res, k[:, 1] * res, np.zeros(200)),
                           poses(orc, k[:100, 0] * res, k[:100, 1] * res, np.full(100, PI / 2))])
    generic = poses(orc, rng.uniform(60.0, 195.0, 512) * res, rng.uniform(60.0, 195.0, 512) * res, rng.uniform(-PI, PI, 512))
    distinct = np.concatenate([generic, edge])
    n = pair_min + 100
    idx = rng.integers(0, len(generic), n)
    # one edge pose in every 16th task, in a lane that moves with the task, as its first particle (slot l) or its second (l + 32)
    tasks = np.arange(0, n // TASK, 16)
    for j, t in enumerate(tasks):
        idx[t * TASK + j % 32 + 32 * ((j // 32) % 2)] = len(generic) + j % len(edge)
    got, exp = weigh(bb, orc, scene, pts, distinct, idx)
    assert np.array_equal(got, exp)


def edge_group(orc, rng, res, side, radius_cells, edge, d, size=TASK):
    """`size` poses at distance d (cells) from one edge and well inside the others, at quarter-turn headings, so that an
    axis end point (radius_cells away) points square at that edge."""
    reach = radius_cells + 2.0
    out = []
    for _ in range(size):
        along = rng.uniform(reach + 1.0, side - reach - 1.0)
        x, y = [(d, along), (side - d, along), (along, d), (along, side - d)][edge]
        theta = rng.integers(-1, 3) * PI / 2 + rng.uniform(-1e-6, 1e-6)
        out.append(orc.se2(x * res, y * res, theta))
    return np.array(out)


def test_in_grid_test_over_both_particles_of_every_lane(bb, orc, scene, pair_min):
    """64-particle tasks on either side of the in-grid test (which asks for d >= radius + 2 cells), tasks whose end points
    reach the last cell or cross the edge, and tasks where a single particle of a single pair -- the first of its lane
    in some, the second in others -- has end points five cells past the edge, so the whole warp must clamp."""
    res = scene.resolution
    side = scene.cells.shape[0]
    r = 1.5  # |x| + |y| of the farthest end point, in metres
    rc = r / res
    ring = np.array([[r, 0.0], [-r, 0.0], [0.0, r], [0.0, -r], [0.75, 0.75], [-0.75, 0.75], [0.75, -0.75], [-0.75, -0.75]])
    rng = np.random.default_rng(23)
    groups = []
    for edge in range(4):
        for d in (rc + 3.0, rc + 1.0, rc + 0.5, rc - 0.5, rc - 4.5):
            groups.append(edge_group(orc, rng, res, side, rc, edge, d))
    inner = edge_group(orc, rng, res, side, rc, 0, side / 2, size=TASK * 8)  # every pose clears every edge
    for edge in range(4):
        for slot in (17, 49, 0, 63):  # lane 17 first / second, lane 0 first, lane 31 second
            g = inner[rng.integers(0, len(inner), TASK)]
            g[slot] = edge_group(orc, rng, res, side, rc, edge, rc - 4.5, size=1)[0]
            groups.append(g)
    special = np.concatenate(groups)
    distinct = np.concatenate([inner, special])
    n = pair_min + 5
    idx = rng.integers(0, len(inner), n)
    # the special groups fill whole tasks, spread over the launch
    starts = np.linspace(0, n // TASK - 1, len(groups)).astype(int) * TASK
    for g, s in enumerate(starts):
        idx[s:s + TASK] = len(inner) + g * TASK + np.arange(TASK)
    got, exp = weigh(bb, orc, scene, ring, distinct, idx)
    assert np.array_equal(got, exp)
