"""The persistent likelihood-field reweight kernel stages the whole scan into shared memory once per CTA, up to
kChunkBeams = 2048 points; longer scans go through the chunked kernel.  Both sides of that limit, and an empty scan,
against the CPU oracle, bit for bit, with the one-particle kernel (small filters) and the two-particle kernel
(filters of 811 009 particles and more on a 132-SM H100)."""
import math

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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=2)


def weights(bb, orc, scene, states, pts):
    f = bb.Filter(capacity=len(states))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution, orc.IDENTITY))
    f.set_particles(states)
    f.reweight(pts)
    got = f.particles()[1]
    exp = orc.sensor_weights(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution), pts, states)
    return got, exp


@pytest.mark.parametrize("n_points", [0, 2047, 2048, 2049])
def test_one_particle_kernel_around_the_staging_limit(bb, orc, scene, n_points):
    rng = np.random.default_rng(n_points)
    extent = scene.cells.shape[0] * scene.resolution
    n = 3001
    xs, ys, th = rng.uniform(-1.0, extent + 1.0, n), rng.uniform(-1.0, extent + 1.0, n), rng.uniform(-math.pi, math.pi, n)
    states = np.array([orc.se2(x, y, t) for x, y, t in zip(xs, ys, th)])
    pts = rng.uniform(-6.0, 6.0, (n_points, 2))
    got, exp = weights(bb, orc, scene, states, pts)
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("n_points", [2048, 2049])
def test_two_particle_kernel_around_the_staging_limit(bb, orc, scene, n_points):
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 64 * (6 * sms * 2 * 8) + 37  # above the pair threshold (kRwPairFill x SMs x 2 CTAs x 8 warps pair tasks), ragged last task
    rng = np.random.default_rng(10 + n_points)
    extent = scene.cells.shape[0] * scene.resolution
    m = 2048  # distinct poses, repeated: the oracle weighs each once
    distinct = np.array([orc.se2(x, y, t) for x, y, t in zip(rng.uniform(-1.0, extent + 1.0, m), rng.uniform(-1.0, extent + 1.0, m),
                                                                rng.uniform(-math.pi, math.pi, m))])
    idx = rng.integers(0, m, n)
    pts = rng.uniform(-6.0, 6.0, (n_points, 2))
    f = bb.Filter(capacity=n)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution, orc.IDENTITY))
    f.set_particles(distinct[idx])
    f.reweight(pts)
    exp = orc.sensor_weights(0, orc.LfmParam(**LFM), orc.Grid(scene.cells, scene.resolution), pts, distinct)[idx]
    assert np.array_equal(f.particles()[1], exp)
