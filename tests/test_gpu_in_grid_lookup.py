"""The fixed-point reweight kernels skip the border clamp for warps whose particles' end points all lie inside the grid.
Whole warps on either side of that test, and warps whose end points reach the last cell of the grid or cross its edge by
one cell and by several, must weigh exactly what the CPU oracle weighs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

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
def scene():
    from beluga_b200 import synthetic

    # 254 + 2 border cells = 64 whole tiles per row: the bordered table has no padding columns, so a cell past the right
    # edge read without the clamp would be a cell of the next tile row, not another copy of the border value
    return synthetic.make_scenario(grid_size=254, n_beams=181, steps=2)


def edge_warps(orc, res, side, radius_cells):
    """Warps of 32 particles, each warp at one distance d (cells) from one edge and well inside the others, at
    quarter-turn headings so that an axis end point (radius_cells away) points square at that edge.  The in-grid test
    asks for d >= radius_cells + 2: one warp clears it by a cell and one misses it by a cell, and three take the clamped
    loop with end points in the last cell before the edge, one cell past it, and five cells past it."""
    rng = np.random.default_rng(23)
    reach = radius_cells + 2.0
    states = []
    for edge in range(4):
        for d in (reach + 1.0, reach - 1.0, radius_cells + 0.5, radius_cells - 0.5, radius_cells - 4.5):
            for _ in range(32):
                along = rng.uniform(reach + 1.0, side - reach - 1.0)
                x, y = [(d, along), (side - d, along), (along, d), (along, side - d)][edge]
                theta = rng.integers(-1, 3) * np.pi / 2 + rng.uniform(-1e-6, 1e-6)
                states.append(orc.se2(x * res, y * res, theta))
    return np.array(states)


@pytest.mark.parametrize("n_points", [8, 2504])  # scan as kernel parameters / staged through shared memory
def test_reweight_warps_either_side_of_the_in_grid_test(bb, orc, scene, n_points):
    res = scene.resolution
    side = scene.cells.shape[0]
    r = 1.5  # |x| + |y| of the farthest end point, in metres
    ring = np.array([[r, 0.0], [-r, 0.0], [0.0, r], [0.0, -r], [0.75, 0.75], [-0.75, 0.75], [0.75, -0.75], [-0.75, -0.75]])
    pts = np.tile(ring, (n_points // len(ring), 1))
    states = edge_warps(orc, res, side, r / res)
    f = bb.Filter(capacity=len(states))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, res, orc.IDENTITY), prob=False)
    f.set_particles(states)
    f.reweight(pts)
    got = f.particles()[1]
    exp = orc.sensor_weights(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, res), pts, states)
    assert np.array_equal(got, exp)
