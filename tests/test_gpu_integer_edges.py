"""Where a kernel turns a coordinate into an integer -- a spatial-hash bucket or a grid cell -- against the oracle, with
particle states at the edges of the double range: NaN, +-inf, beyond +-2^63, far off the map, NaN headings.

The rules (DESIGN.md section 1): floor(v) becomes INT64_MIN when it is NaN or outside [-2^63, 2^63), so +1e300, -1e300,
+-inf and NaN share one bucket per axis and NaN never shares bucket 0 with a particle in [0, r).  A beam whose source or far
end is not finite is a miss.  A ray whose span stays below 2^29 cells walks the reference's line; beyond that its far end
is pulled back, per axis, to 2^29 - 1 cells from the source.

Consumers covered: the particle histogram, the clusterizer and KLD (single filter and batch), the beam model in every
kernel form and in a batch step, and the likelihood field's general path and its fixed / general split."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
RES = (0.5, 0.5, 0.17453292519943295)  # spatial_resolution of the KLD tests
# x (or y) values whose bucket the device's saturating conversion would put elsewhere than the reference's rule
EDGE = [NAN, 1e300, -1e300, INF, -INF, 2.0**63, -(2.0**63) * 1.5, 9.3e18, -9.3e18]


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=4)


def pose(x, y, c=1.0, s=0.0):
    return [c, s, x, y]


def edge_cloud(rng, n, kinds, ordinary_buckets=1):
    """n states: ordinary particles in `ordinary_buckets` buckets of RES (the first one holding x, y in [0, 0.5) and a
    heading in [0, 0.17)), and edge states of the given kinds at scattered positions.  The edge states keep the first
    bucket's y and heading, so that only their x decides whether they join it (NaN under a saturating conversion) or
    share one bucket with each other (the reference's rule)."""
    th = rng.uniform(0.01, 0.15, n)
    b = rng.integers(0, ordinary_buckets, n).astype(np.float64)
    states = np.stack([np.cos(th), np.sin(th), rng.uniform(0.05, 0.45, n) + 2.0 * b, rng.uniform(0.05, 0.45, n)], axis=1)
    edges = []
    for kind in kinds:
        if kind == "nan":
            edges += [pose(NAN, 0.2, 0.999, 0.05), pose(NAN, NAN, 0.999, 0.05)]
        elif kind == "overflow":
            edges += [pose(1e300, 0.2, 0.999, 0.05), pose(-1e300, 0.2, 0.999, 0.05), pose(2.0**63, 0.2, 0.999, 0.05),
                      pose(-(2.0**64), 0.2, 0.999, 0.05)]
        elif kind == "inf":
            edges += [pose(INF, 0.2, 0.999, 0.05), pose(-INF, 0.2, 0.999, 0.05)]
        elif kind == "heading_nan":
            edges += [pose(0.2, 0.2, NAN, NAN), pose(0.2, 0.2, 1.0, NAN)]
        elif kind == "y":
            edges += [pose(0.2, v, 0.999, 0.05) for v in EDGE]
    pos = rng.permutation(n)[: 4 * len(edges)]
    for j, p in enumerate(pos):
        states[p] = edges[j % len(edges)]
    return states


def same_bytes(a, b):
    return np.asarray(a, dtype=np.float64).tobytes() == np.asarray(b, dtype=np.float64).tobytes()


def host_histogram(orc, states, weights, linear, angular):
    seen, order = {}, []
    for i, st in enumerate(states):
        h = orc.spatial_hash(st, linear, linear, angular)
        if h not in seen:
            seen[h] = [i, 0.0, 0]
            order.append(h)
        seen[h][1] += weights[i]
        seen[h][2] += 1
    return seen, order


def check_histogram(orc, got, states, weights, linear, angular):
    rep, w, count, first, top = got
    seen, order = host_histogram(orc, states, weights, linear, angular)
    assert len(rep) == len(order)
    assert np.array_equal(first, [seen[h][0] for h in order])
    assert same_bytes(rep, states[first])  # NaN states bit for bit
    assert np.array_equal(w, [seen[h][1] for h in order])
    assert np.array_equal(count, [seen[h][2] for h in order])
    assert top == max(linear, max(seen[h][1] for h in order))


def check_cluster(orc, got, states, weights, linear, angular, percentile):
    mean, cov, ids, cells, clusters = got
    want_ids = orc.cluster_ids(states, weights, linear, angular, percentile)
    assert np.array_equal(ids.astype(np.uint64), want_ids)
    assert clusters == int(want_ids.max()) + 1
    assert cells == len({orc.spatial_hash(s, linear, linear, angular) for s in states})
    want_mean, want_cov = orc.cluster_based_estimate(states, weights, linear, angular, percentile)
    for g, e in ((mean, want_mean), (cov, want_cov)):
        g, e = np.asarray(g), np.asarray(e)
        assert np.array_equal(np.isnan(g), np.isnan(e)) and np.array_equal(np.isinf(g), np.isinf(e))
        fin = np.isfinite(e)
        assert np.allclose(g[fin], e[fin], rtol=1e-9, atol=1e-9)


KINDS = [["nan"], ["overflow"], ["inf"], ["heading_nan"], ["y"], ["nan", "overflow", "inf", "heading_nan", "y"]]


@pytest.mark.parametrize("kinds", KINDS, ids=["+".join(k) for k in KINDS])
def test_histogram_and_clusters_of_edge_clouds(bb, orc, kinds):
    """Bins and cluster ids bit-exact against the oracle; the edge states are light, so the heaviest cluster (and its
    estimate) stays finite, and heavy, so that it is made of them."""
    rng = np.random.default_rng(len(kinds) * 7 + len(kinds[0]))
    states = edge_cloud(rng, 3000, kinds, ordinary_buckets=3)
    finite = np.isfinite(states).all(axis=1)
    for heavy in (False, True):
        weights = rng.uniform(0.5, 1.5, len(states))
        weights[~finite] = 40.0 if heavy else 1e-3
        f = bb.Filter(capacity=len(states))
        f.set_particles(states, weights)
        for linear, angular in ((1e-3, 1e-3), RES[1:]):
            check_histogram(orc, f.particle_histogram(linear, angular), states, weights, linear, angular)
        check_cluster(orc, f.cluster_estimate(linear=0.5, angular=0.524, percentile=0.9, with_ids=True), states, weights, 0.5, 0.524, 0.9)


def test_nan_and_overflow_do_not_join_or_split_buckets(bb, orc):
    """The counts the two rules disagree on, stated outright: one ordinary bucket, a NaN x in it under a saturating
    conversion, and +-1e300 in two buckets under it; the reference's rule makes those three one bucket of their own."""
    states = np.array([pose(0.2, 0.2, 0.999, 0.05), pose(NAN, 0.2, 0.999, 0.05), pose(1e300, 0.2, 0.999, 0.05), pose(-1e300, 0.2, 0.999, 0.05)])
    f = bb.Filter(capacity=4)
    f.set_particles(states, np.ones(4))
    rep, w, count, first, _ = f.particle_histogram(*RES[1:])
    assert list(first) == [0, 1] and list(count) == [1, 3]


@pytest.mark.parametrize("kinds", KINDS, ids=["+".join(k) for k in KINDS])
@pytest.mark.parametrize("ordinary_buckets", [1, 2])
def test_kld_count_and_ancestors_on_edge_clouds(bb, orc, kinds, ordinary_buckets):
    """take_while_kld over the systematic comb: the count depends on the number of distinct buckets k, and with k of 2
    to 4 one bucket more or less moves the cutoff (k <= 2: no cutoff at all)."""
    n = 2048
    rng = np.random.default_rng(100 + 10 * len(kinds) + ordinary_buckets)
    states = edge_cloud(rng, n, kinds, ordinary_buckets)
    w = np.ones(n)
    seed = 77
    f = bb.Filter(capacity=n, seed=seed, record_ancestors=True)
    f.set_particles(states, w)
    got = f.resample(bb.RESAMPLE_SYSTEMATIC, step=8, max_particles=n, min_particles=4, spatial_resolution=RES)
    idx, _, _ = orc.resample_indices(w, bb.RESAMPLE_SYSTEMATIC, seed=seed, step=8, m=n)
    hashes = [orc.spatial_hash(states[i], *RES) for i in idx]
    assert got == orc.kld_take_count(hashes, 4, n, 0.05, 3.0)
    assert np.array_equal(f.ancestors(), idx[:got])


def test_batch_members_on_edge_clouds(bb, orc):
    """cluster_estimates and particle_histograms of batch members holding edge clouds equal a standalone filter's, byte for
    byte, and the oracle's bins."""
    rng = np.random.default_rng(5)
    clouds = [edge_cloud(rng, n, kinds, 3) for n, kinds in ((500, ["nan"]), (2000, ["overflow", "inf"]), (33, ["heading_nan"]), (1200, KINDS[-1]))]
    weights = [rng.uniform(0.5, 1.5, len(s)) for s in clouds]
    params = [bb.AmclParams(min_particles=len(s), max_particles=len(s), seed=m) for m, s in enumerate(clouds)]
    batch = bb.AmclBatch([bb.StationaryModelParam() for _ in clouds], params)
    for m, (s, w) in enumerate(zip(clouds, weights)):
        batch.initialize_states(m, s, w)
    ests = batch.cluster_estimates(linear=0.5, angular=0.524, percentile=0.9, with_counts=True)
    hists = batch.particle_histograms(None, *RES[1:])
    for m, (s, w) in enumerate(zip(clouds, weights)):
        f = bb.Filter(capacity=len(s))
        f.set_particles(s, w)
        one = f.cluster_estimate(linear=0.5, angular=0.524, percentile=0.9, with_ids=True)
        mean, cov, cells, clusters = ests[m]
        assert same_bytes(mean, one[0]) and same_bytes(cov, one[1]) and (cells, clusters) == one[3:], m
        check_cluster(orc, one, s, w, 0.5, 0.524, 0.9)
        bins, top = hists[m]
        rep, hw, count, first, t_top = f.particle_histogram(*RES[1:])
        assert same_bytes(bins["rep"].reshape(-1, 4), rep) and np.array_equal(bins["first"], first) and np.array_equal(bins["count"], count)
        assert same_bytes(bins["weight"], hw) and top == t_top, m
        check_histogram(orc, (rep, hw, count, first, t_top), s, w, *RES[1:])


# ---- beam model ------------------------------------------------------------------------------------------------------
def walled(cells):
    cells = cells.copy()
    cells[0, :] = cells[-1, :] = cells[:, 0] = cells[:, -1] = 100
    return cells


def beam_edge_states(rng, n, width_m, height_m):
    """Ordinary states on the map, and the edge states: NaN, +-inf and far-away coordinates, NaN headings on the map,
    states just off the map and beyond the int range of cells."""
    th = rng.uniform(-math.pi, math.pi, n)
    states = np.stack([np.cos(th), np.sin(th), rng.uniform(0.0, width_m, n), rng.uniform(0.0, height_m, n)], axis=1)
    cx, cy = 0.5 * width_m, 0.5 * height_m
    edges = [pose(NAN, cy), pose(cx, NAN), pose(NAN, NAN), pose(INF, cy), pose(-INF, cy), pose(cx, INF), pose(cx, -INF),
             pose(1e300, cy), pose(-1e300, -1e300), pose(1e12, -3e11), pose(-5e9, cy), pose(cx, 3e9),
             pose(cx, cy, NAN, NAN), pose(cx, cy, 1.0, NAN), pose(cx, cy, NAN, 0.0), pose(0.1 * width_m, 0.3 * height_m, NAN, NAN),
             pose(-1e-9, cy), pose(width_m + 1e-9, cy), pose(cx, -1e-9, 0.0, 1.0)]
    pos = rng.permutation(n)[: 2 * len(edges)]
    for j, p in enumerate(pos):
        states[p] = edges[j % len(edges)]
    return states


@pytest.mark.parametrize("shape, launches", [("two_pass", 3), ("fused", 2), ("fine_cells", 3)])
def test_beam_edge_states_match_oracle(bb, orc, scene, shape, launches):
    """The three kernel forms on a walled map: the two-pass walk with the normaliser table, the fused kernel (a grid wider
    than 65534 cells) and the two-pass walk with per-beam normalisers (fine cells).  A NaN source or end point must not
    become cell 0 -- an occupied wall cell."""
    rng = np.random.default_rng(31)
    cells, res, max_range = walled(scene.cells), scene.resolution, 20.0
    if shape == "fused":
        cells = walled(np.pad(scene.cells, ((0, 0), (0, 70_000 - scene.cells.shape[1])), constant_values=0))
    elif shape == "fine_cells":
        res, max_range = 0.01, 30.0
    scale = res / scene.resolution
    height, width = cells.shape
    states = beam_edge_states(rng, 400, min(width, 400) * res, height * res)
    pts = scene.scans[0][::3] * scale
    bp = dict(sigma_hit=0.2 * scale, lambda_short=0.1 / scale, beam_max_range=max_range)
    f = bb.Filter(capacity=len(states))
    f.set_beam_map(bb.BeamModelParam(**bp), bb.OccupancyGrid(cells, res))
    f.set_particles(states)
    before = f.launch_count()
    f.reweight(pts)
    assert f.launch_count() - before == launches
    exp = orc.sensor_weights(orc.BEAM, orc.BeamParam(**bp), orc.Grid(cells, res), pts, states)
    assert np.allclose(f.particles()[1], exp, rtol=1e-11, atol=1e-300)


@pytest.mark.parametrize("max_range", [4000.0, 5000.0, 6000.0, 1e6])
def test_beam_reach_past_2_to_the_28_cells(bb, orc, scene, max_range):
    """1e-5 m cells: a 4000 m and a 5000 m range reach 4e8 and 5e8 cells, between 2^28 and 2^29, where the reference's
    int arithmetic is still exact and every far end must be the reference's cell.  6000 m and 1e6 m reach past 2^29, where
    both sides pull the far end back to 2^29 - 1 cells per axis.  Edge states included."""
    rng = np.random.default_rng(int(max_range))
    res = 1e-5
    scale = res / scene.resolution
    cells = walled(scene.cells)
    height, width = cells.shape
    states = beam_edge_states(rng, 300, width * res, height * res)
    pts = scene.scans[0][::3] * scale
    bp = dict(sigma_hit=0.2 * scale, lambda_short=0.1 / scale, beam_max_range=max_range)
    f = bb.Filter(capacity=len(states))
    f.set_beam_map(bb.BeamModelParam(**bp), bb.OccupancyGrid(cells, res))
    f.set_particles(states)
    f.reweight(pts)
    exp = orc.sensor_weights(orc.BEAM, orc.BeamParam(**bp), orc.Grid(cells, res), pts, states)
    assert np.allclose(f.particles()[1], exp, rtol=1e-11, atol=1e-300)


@pytest.mark.parametrize("sensor", ["beam_two_pass", "beam_fused", "lfm_general"])
def test_batch_step_over_edge_states_equals_standalone_twins(bb, scene, sensor):
    """One KLD-free batch step over members holding edge states equals a standalone Amcl's, byte for byte: states,
    weights and estimate.  The batch's beam kernels (two-pass and fused) and its general likelihood-field kernel
    (a map wider than kFixedMaxSide) run the same block bodies as the single filter's."""
    rng = np.random.default_rng(3)
    cells = walled(scene.cells)
    if sensor == "beam_fused":
        cells = walled(np.pad(scene.cells, ((0, 0), (0, 70_000 - scene.cells.shape[1])), constant_values=0))
    elif sensor == "lfm_general":
        cells = np.pad(scene.cells, ((0, 0), (0, 8200 - scene.cells.shape[1])), constant_values=0)
    grid = bb.OccupancyGrid(cells, scene.resolution)
    extent = scene.cells.shape[0] * scene.resolution
    sizes = (300, 33, 1000)
    clouds = [beam_edge_states(rng, n, extent, extent) for n in sizes]
    params = [bb.AmclParams(min_particles=n, max_particles=n, seed=10 + m) for m, n in enumerate(sizes)]
    motions = [bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05) for _ in sizes]
    batch = bb.AmclBatch(motions, params)
    if sensor == "lfm_general":
        kind, sp = bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM)
        batch.set_likelihood_field_map(sp, grid)
    else:
        kind, sp = bb.SENSOR_BEAM, bb.BeamModelParam(beam_max_range=20.0)
        batch.set_beam_map(sp, grid)
    twins = []
    for m, s in enumerate(clouds):
        batch.initialize_states(m, s)
        batch.force_update(m)
        t = bb.Amcl(motions[m], params[m])
        t.update_map(kind, sp, grid)
        t.initialize_states(s)
        t.force_update()
        twins.append(t)
    pose = bb.se2(*scene.poses[0])
    got = batch.update([pose] * len(sizes), [scene.scans[0]] * len(sizes))
    for m, t in enumerate(twins):
        r = t.update(pose, scene.scans[0])
        assert got[m].updated == r.updated == 1
        bs, bw = batch.particles(m)
        ts, tw = t.particles()
        assert same_bytes(bs, ts) and same_bytes(bw, tw), m
        assert same_bytes(got[m].estimate.mean, r.estimate.mean) and same_bytes(got[m].estimate.cov, r.estimate.cov), m


# ---- likelihood field ------------------------------------------------------------------------------------------------
def test_lfm_general_path_with_edge_states(bb, orc, scene):
    """An 8200-wide map takes the general kernel; NaN states, NaN headings and far-away states land outside the grid on
    both sides, bit for bit."""
    cells = np.pad(scene.cells, ((0, 0), (0, 8200 - scene.cells.shape[1])), constant_values=0)
    rng = np.random.default_rng(9)
    extent = scene.cells.shape[0] * scene.resolution
    states = beam_edge_states(rng, 500, extent, extent)
    pts = rng.uniform(-8.0, 8.0, (181, 2))
    f = bb.Filter(capacity=len(states))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(cells, scene.resolution))
    f.set_particles(states)
    f.reweight(pts)
    exp = orc.sensor_weights(0, orc.LfmParam(**LFM), orc.Grid(cells, scene.resolution), pts, states)
    assert np.array_equal(f.particles()[1], exp)


@pytest.mark.parametrize("width", [7998, 7999])
def test_lfm_either_side_of_the_fixed_point_split(bb, orc, scene, width):
    """width + 2 <= kFixedMaxSide selects the fixed-point kernel: 7998 is its widest map, 7999 the narrowest general one.
    Ordinary states spread along the whole width, plus the edge states; bit-exact."""
    cells = np.pad(scene.cells, ((0, 0), (0, width - scene.cells.shape[1])), constant_values=0)
    cells[:, width - 40:width - 30] = 100
    res = scene.resolution
    rng = np.random.default_rng(width)
    states = beam_edge_states(rng, 2000, width * res, cells.shape[0] * res)
    pts = rng.uniform(-8.0, 8.0, (181, 2))
    f = bb.Filter(capacity=len(states))
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(cells, res))
    f.set_particles(states)
    f.reweight(pts)
    exp = orc.sensor_weights(0, orc.LfmParam(**LFM), orc.Grid(cells, res), pts, states)
    assert np.array_equal(f.particles()[1], exp)
