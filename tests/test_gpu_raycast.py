"""Ray casts on the device (bb200_filter_cast_rays, bb200_amcl_batch_cast_rays) against the CPU oracle's Ray2d::cast with the
same raw {cos, sin} bearings (tests/_raycast_oracle.py), compared with == on doubles, inf for a miss: the reference's
known answers, a sweep over poses, bearings and maximum ranges on the 2000^2 synthetic map, every map form, and a batch of
members on several maps that must equal the standalone filter and leave every member as it was."""
import ctypes as C
import math
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _raycast_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

PI = math.pi
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
INVALID, STATE = -1, -4


@pytest.fixture(scope="module")
def bb():
    import beluga_b200

    if beluga_b200.device_count() == 0:
        pytest.skip("no CUDA device")
    return beluga_b200


def se2(x, y, theta):
    return np.array([math.cos(theta), math.sin(theta), x, y])


def bearing(theta):
    return np.array([math.cos(theta), math.sin(theta)])


def same(a, b) -> bool:
    """== on doubles with inf for a miss (NaN never occurs: a miss is inf)."""
    return a.shape == b.shape and bool(np.all(a == b))


def oracle(grid, poses, bearings, max_range):
    return _raycast_oracle.cast_rays(grid.cells, grid.resolution, grid.origin, poses, bearings, max_range)


def filter_on(bb, sensor, grid):
    f = bb.Filter(capacity=64)
    if sensor == bb.SENSOR_BEAM:
        f.set_beam_map(bb.BeamModelParam(), grid)
    else:
        f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid, prob=sensor == bb.SENSOR_LIKELIHOOD_FIELD_PROB)
    return f


SENSORS = ["beam", "lfm", "lfm_prob"]


def sensor_of(bb, name):
    return {"beam": bb.SENSOR_BEAM, "lfm": bb.SENSOR_LIKELIHOOD_FIELD, "lfm_prob": bb.SENSOR_LIKELIHOOD_FIELD_PROB}[name]


# ---- algorithm/test_raycasting.cpp:31-131 (tests/test_oracle_golden.py restates them for the oracle) ------------------------
def grid5(bb, occupied, resolution=0.5, origin=None):
    cells = np.zeros((5, 5), dtype=np.int8)
    for (r, c) in occupied:
        cells[r, c] = 100
    return bb.OccupancyGrid(cells, resolution, np.array([1.0, 0.0, 0.0, 0.0]) if origin is None else origin)


NOMINAL = [((0.5, 0.0, 0.0), 5.0, 0.0, None), ((0.0, 1.0, 0.0), 5.0, 0.0, 1.0), ((0.0, 1.0, 0.0), 5.0, PI / 2, None),
           ((1.0, 1.0, 0.0), 5.0, PI / 2, 0.0), ((0.0, 0.0, PI / 2), 1.0, 0.0, None), ((1.0, 0.0, 0.0), 5.0, PI / 2, 1.0),
           ((0.0, 0.0, 0.0), 5.0, PI / 4, math.sqrt(2))]


@pytest.mark.parametrize("sensor", SENSORS)
def test_reference_known_answers(bb, sensor):
    cases = [(grid5(bb, [(2, 2)]), NOMINAL),
             (grid5(bb, [(2, 2)], 0.5, se2(0.5, 0.0, -PI / 4)), [((0.5, 0.0, 0.0), 5.0, 0.0, math.sqrt(2))])]
    for grid, answers in cases:
        f = filter_on(bb, sensor_of(bb, sensor), grid)
        batch = bb.AmclBatch([bb.DifferentialDriveModelParam()], [bb.AmclParams(min_particles=64, max_particles=64)])
        if sensor == "beam":
            batch.set_beam_map(bb.BeamModelParam(), grid)
        else:
            batch.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grid, prob=sensor == "lfm_prob")
        for pose, max_range, theta, expected in answers:
            p, b = se2(*pose)[None], bearing(theta)[None]
            want = np.array([[math.inf if expected is None else expected]])
            assert same(oracle(grid, p, b, max_range), want)
            assert same(f.cast_rays(p, b, max_range), want), (pose, theta)
            assert same(batch.cast_rays([p], b, max_range)[0], want), (pose, theta)


# ---- sweep on the 2000^2 synthetic map ---------------------------------------------------------------------------------------
def sweep_poses(rng, n, size_m, resolution):
    inside = np.stack([se2(x, y, t) for x, y, t in zip(rng.uniform(0, size_m, n), rng.uniform(0, size_m, n), rng.uniform(-PI, PI, n))])
    # exactly on cell edges, and on the grid's own edges
    k = rng.integers(0, int(size_m / resolution) + 1, (n // 8, 2))
    edges = np.stack([se2(a * resolution, b * resolution, t) for (a, b), t in zip(k, rng.uniform(-PI, PI, len(k)))])
    corners = np.stack([se2(x, y, t) for x in (0.0, size_m, -1e-12) for y in (0.0, size_m) for t in (0.0, PI / 2, -PI / 4)])
    outside = np.stack([se2(x, y, t) for x, y, t in zip(rng.uniform(-30, size_m + 30, n // 8), rng.choice([-5.0, size_m + 5.0, 1e12, -1e12], n // 8),
                                                        rng.uniform(-PI, PI, n // 8))])
    special = []
    for v in (math.nan, math.inf, -math.inf):
        for comp in range(4):
            p = se2(size_m / 2, size_m / 3, 0.7)
            p[comp] = v
            special.append(p)
    unnormalised = inside[: n // 8].copy()
    unnormalised[:, :2] *= rng.uniform(0.5, 2.0, (n // 8, 1))
    return np.concatenate([inside, edges, corners, outside, np.stack(special), unnormalised])


def sweep_bearings(rng):
    axes = [(1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0)]
    h = math.sqrt(0.5)
    diagonal = [(h, h), (-h, h), (h, -h), (-h, -h), (1.0, 1.0), (-2.0, 2.0)]
    special = [(0.0, 0.0), (math.nan, 0.0), (0.5, 0.0), (0.0, 3.0)]
    unit = [tuple(bearing(t)) for t in rng.uniform(-PI, PI, 34)]
    other = [tuple(bearing(t) * s) for t, s in zip(rng.uniform(-PI, PI, 16), rng.uniform(0.25, 4.0, 16))]
    b = np.array(axes + diagonal + special + unit + other)
    assert len(b) == 64
    return b


MAX_RANGES = [0.0, 0.02, 60.0, 1e9, math.nan, -3.0]


@pytest.fixture(scope="module")
def sweep(bb):
    from beluga_b200 import synthetic

    cells = synthetic.make_map(2000)
    grid = bb.OccupancyGrid(cells, 0.05)
    rng = np.random.default_rng(7)
    poses = sweep_poses(rng, 15000, 100.0, 0.05)
    assert 19000 < len(poses) < 22000
    return grid, poses, sweep_bearings(rng)


@pytest.mark.parametrize("sensor", SENSORS)
def test_sweep_on_the_2000_map(bb, sweep, sensor):
    grid, poses, bearings = sweep
    f = filter_on(bb, sensor_of(bb, sensor), grid)
    hits = 0
    for max_range in MAX_RANGES:
        before = f.launch_count()
        got = f.cast_rays(poses, bearings, max_range)
        assert f.launch_count() - before == 1
        want = oracle(grid, poses, bearings, max_range)
        bad = np.argwhere(~(got == want))
        assert len(bad) == 0, (max_range, bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])
        if math.isnan(max_range):
            assert np.isinf(got).all()
        hits += int(np.isfinite(got).sum())
    assert hits > len(poses) * len(bearings)  # the sweep is not all misses


def test_rotated_translated_origin(bb):
    from beluga_b200 import synthetic

    cells = synthetic.make_map(500, seed=3)
    origin = se2(-7.25, 3.5, 0.7)
    grid = bb.OccupancyGrid(cells, 0.05, origin)
    rng = np.random.default_rng(11)
    local = np.stack([se2(x, y, t) for x, y, t in zip(rng.uniform(-2, 27, 3000), rng.uniform(-2, 27, 3000), rng.uniform(-PI, PI, 3000))])
    # world-frame sensor poses: origin * local (Sophus SE2 product)
    c, s = origin[0], origin[1]
    poses = np.stack([np.array([c * p[0] - s * p[1], s * p[0] + c * p[1], (c * p[2] - s * p[3]) + origin[2], (s * p[2] + c * p[3]) + origin[3]])
                      for p in local])
    bearings = sweep_bearings(rng)
    for sensor in SENSORS:
        f = filter_on(bb, sensor_of(bb, sensor), grid)
        for max_range in (0.5, 30.0, 1e9):
            assert same(f.cast_rays(poses, bearings, max_range), oracle(grid, poses, bearings, max_range)), (sensor, max_range)


def test_grid_wider_than_65534_cells(bb):
    # The beam model's two-pass walk has no padded free-distance copy of this map; the cast walks the plain one.
    width, height = 70000, 6
    cells = np.zeros((height, width), dtype=np.int8)
    cells[:, [0, 100, 65535, 65536, width - 1]] = 100
    cells[3, 40000] = 100
    grid = bb.OccupancyGrid(cells, 0.1)
    rng = np.random.default_rng(5)
    poses = np.stack([se2(x, y, t) for x, y, t in zip(rng.uniform(0, width * 0.1, 400), rng.uniform(0, height * 0.1, 400),
                                                      rng.choice([0.0, PI, 0.01, PI - 0.003], 400))])
    bearings = np.array([(1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), bearing(0.002), bearing(PI - 0.001), bearing(1.0)])
    for sensor in SENSORS:
        f = filter_on(bb, sensor_of(bb, sensor), grid)
        for max_range in (10.0, 7000.0, 1e9):
            assert same(f.cast_rays(poses, bearings, max_range), oracle(grid, poses, bearings, max_range)), (sensor, max_range)


def test_likelihood_field_map_uploads_on_the_first_cast_only(bb):
    from beluga_b200 import synthetic

    sc = synthetic.make_scenario(grid_size=4000, n_beams=60, steps=4)
    grid = bb.OccupancyGrid(sc.cells, sc.resolution)
    motion = bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05)
    params = bb.AmclParams(min_particles=2000, max_particles=2000, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=3)
    a, twin = bb.Amcl(motion, params), bb.Amcl(motion, params)
    counts = {}
    for g in (a, twin):
        before = g.filter.launch_count()
        g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), grid)
        g.initialize(sc.initial_mean, sc.initial_cov)
        counts.setdefault("map_and_initialize", []).append(g.filter.launch_count() - before)
    pose = bb.se2(*sc.poses[0])[None]
    bearings = bb.scan_bearings(-PI, 2 * PI / 360, 360)
    elapsed = []
    for _ in range(2):
        before = a.filter.launch_count()
        t0 = time.perf_counter()
        got = a.cast_rays(pose, bearings, 30.0)
        elapsed.append(time.perf_counter() - t0)
        assert a.filter.launch_count() - before == 1
        assert same(got, oracle(grid, pose, bearings, 30.0))
    # The first cast builds the 16M-cell free-distance map on the host (about half a second); the second reuses it.
    assert elapsed[0] > 0.05 and elapsed[1] < elapsed[0] / 5, elapsed
    for k in range(1, 4):
        step = []
        for g in (a, twin):
            before = g.filter.launch_count()
            r = g.update(bb.se2(*sc.poses[k]), sc.scans[k])
            step.append((g.filter.launch_count() - before, bytes(r)))
        assert step[0] == step[1]
    assert counts["map_and_initialize"][0] == counts["map_and_initialize"][1]
    s0, w0 = a.particles()
    s1, w1 = twin.particles()
    assert s0.tobytes() == s1.tobytes() and w0.tobytes() == w1.tobytes()


# ---- batches -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fleet(bb):
    """Three maps: a beam map of the 2000^2 synthetic grid, a likelihood field of a 500^2 grid and a likelihood-field-prob map
    of a rotated 400^2 grid."""
    from beluga_b200 import synthetic

    grids = [bb.OccupancyGrid(synthetic.make_map(2000, seed=4), 0.05), bb.OccupancyGrid(synthetic.make_map(500, seed=5), 0.05),
             bb.OccupancyGrid(synthetic.make_map(400, seed=6), 0.05, se2(1.5, -2.0, 0.4))]
    return grids


def make_batch(bb, grids, k=8):
    params = [bb.AmclParams(min_particles=1000 + 100 * m, max_particles=1000 + 100 * m, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=20 + m)
              for m in range(k)]
    batch = bb.AmclBatch([bb.DifferentialDriveModelParam(0.1, 0.05, 0.1, 0.05) for _ in range(k)], params)
    ids = [batch.add_beam_map(bb.BeamModelParam(), grids[0]),
           batch.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grids[1]),
           batch.add_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), grids[2], prob=True)]
    for m in range(k):
        batch.update_map(m, ids[m % 3])
        batch.initialize(m, (10.0 + m, 12.0, 0.3 * m), np.diag([0.05, 0.05, 0.02]))
    return batch, ids


def member_rays(bb, rng, k):
    counts = [(5, 64), (0, 16), (3, 0), (40, 360), (1, 1), (17, 7), (0, 0), (9, 100)][:k]
    poses = [np.stack([se2(x, y, t) for x, y, t in zip(rng.uniform(-1, 22, n), rng.uniform(-1, 22, n), rng.uniform(-PI, PI, n))])
             if n else np.zeros((0, 4)) for n, _ in counts]
    bearings = [np.stack([bearing(t) for t in rng.uniform(-PI, PI, nb)]) if nb else np.zeros((0, 2)) for _, nb in counts]
    return poses, bearings


def test_batch_members_equal_the_filter_and_the_oracle(bb, fleet):
    grids = fleet
    batch, ids = make_batch(bb, grids)
    vacant = 6
    batch.remove_member(vacant)
    rng = np.random.default_rng(9)
    poses, bearings = member_rays(bb, rng, 8)
    max_range = [25.0, 3.0, 60.0, 12.5, 1e9, 0.0, 4.0, 30.0]
    filters = [filter_on(bb, s, g) for s, g in zip((bb.SENSOR_BEAM, bb.SENSOR_LIKELIHOOD_FIELD, bb.SENSOR_LIKELIHOOD_FIELD_PROB), grids)]
    present_sets = [None, [m != 2 and m != vacant for m in range(8)], [m == 3 for m in range(8)]]
    map_sets = [None, [-1, ids[0], -1, ids[2], ids[1], -1, -1, ids[0]]]
    for present in present_sets:
        for map_ids in map_sets:
            before = batch.launch_count()
            out = batch.cast_rays(poses, bearings, max_range, present=present, map_ids=map_ids)
            assert batch.launch_count() - before == 1  # whatever K, the maps and the ray counts
            for m in range(8):
                selected = m != vacant and (present is None or present[m])
                if not selected:
                    assert out[m] is None
                    continue
                which = (m % 3) if map_ids is None or map_ids[m] == -1 else ids.index(map_ids[m])
                want = oracle(grids[which], poses[m], bearings[m], max_range[m])
                assert same(out[m], want), (m, which)
                assert same(filters[which].cast_rays(poses[m], bearings[m], max_range[m]), want)
    # a shared bearing array and one maximum range for every member
    shared = bearings[3]
    out = batch.cast_rays(poses, shared, 20.0)
    for m in range(8):
        if m != vacant:
            assert same(out[m], oracle(grids[m % 3], poses[m], shared, 20.0))
    # no rays at all: no launch
    before = batch.launch_count()
    empty = batch.cast_rays([np.zeros((0, 4))] * 8, np.zeros((0, 2)), 5.0)
    assert batch.launch_count() == before and all(o is None or o.shape[0] == 0 for o in empty)


def test_batch_launches_do_not_depend_on_k(bb, fleet):
    grids = fleet
    rng = np.random.default_rng(21)
    for k in (1, 3, 8):
        batch, _ = make_batch(bb, grids, k)
        poses, bearings = member_rays(bb, rng, k)
        before = batch.launch_count()
        batch.cast_rays(poses, [b if len(b) else bearing(0.0)[None] for b in bearings], 10.0)
        assert batch.launch_count() - before == 1


def test_casting_changes_no_member(bb, fleet):
    from beluga_b200 import synthetic

    grids = fleet
    a, ids = make_batch(bb, grids)
    twin, _ = make_batch(bb, grids)
    rng = np.random.default_rng(13)
    poses, bearings = member_rays(bb, rng, 8)
    scans = [synthetic.raycast_ranges(grids[m % 3].cells, 0.05, (10.0 + m, 12.0, 0.3 * m), 60, 20.0) for m in range(8)]
    points = [np.stack([r * np.cos(t), r * np.sin(t)], 1) for r, t in ((s, np.linspace(-PI, PI, len(s), endpoint=False)) for s in scans)]
    points = [p[np.isfinite(p).all(1)] for p in points]
    controls = [[bb.se2(10.0 + m + 0.3 * k, 12.0, 0.3 * m) for m in range(8)] for k in range(3)]
    results = []
    for b, cast in ((a, True), (twin, False)):
        r0 = b.update(controls[0], points)
        r1 = b.update(controls[1], points)
        if cast:
            b.cast_rays(poses, bearings, 15.0, map_ids=[ids[(m + 1) % 3] for m in range(8)])
        r2 = b.update(controls[2], points)
        results.append(([bytes(x) for x in r0 + r1 + r2], [b.particles(m) for m in range(8)], [b.export_member(m) for m in range(8)]))
    (ra, pa, ea), (rb, pb, eb) = results
    assert ra == rb
    for m in range(8):
        assert pa[m][0].tobytes() == pb[m][0].tobytes() and pa[m][1].tobytes() == pb[m][1].tobytes()
    assert ea == eb


def test_refusals_leave_the_batch_unchanged(bb, fleet):
    grids = fleet
    batch, ids = make_batch(bb, grids)
    batch.remove_member(5)
    joined = batch.add_member(bb.DifferentialDriveModelParam(), bb.AmclParams(min_particles=500, max_particles=500))  # no map
    assert joined == 5
    batch.remove_member(6)
    removed = batch.add_beam_map(bb.BeamModelParam(), grids[1])
    batch.remove_map(removed)
    rng = np.random.default_rng(17)
    poses, bearings = member_rays(bb, rng, 8)
    blobs = batch.export_members()
    launches = batch.launch_count()

    def refused(status, **kw):
        with pytest.raises(bb.BelugaB200Error) as e:
            batch.cast_rays(poses, bearings, 10.0, **kw)
        assert e.value.status == status

    refused(STATE)  # member 5 joined without a map
    refused(INVALID, map_ids=[-1] * 5 + [removed] + [-1] * 2)  # a removed map id
    refused(INVALID, map_ids=[-1] * 5 + [ids[0]] + [-1, 99])  # an unknown one
    refused(INVALID, present=[True] * 8, map_ids=[-1] * 5 + [ids[0]] + [-1] * 2)  # a vacant slot
    # n_poses * n_bearings overflows (caught before any array is read)
    lib, k = batch._lib, 8
    d = C.POINTER(C.c_double)
    buf = np.zeros(8)
    ptrs = (d * k)(*[buf.ctypes.data_as(d)] * k)
    n_poses = (C.c_uint64 * k)(*([1] * 7 + [1 << 62]))
    n_bearings = (C.c_uint64 * k)(*([1] * 7 + [8]))
    mask = (C.c_uint8 * k)(*[1, 1, 1, 1, 1, 0, 0, 1])
    assert lib.bb200_amcl_batch_cast_rays(batch._h, mask, None, ptrs, n_poses, ptrs, n_bearings, (C.c_double * k)(*[1.0] * k), ptrs) == INVALID
    n_bearings[7] = 1
    nulls = (d * k)(*([buf.ctypes.data_as(d)] * 7 + [None]))
    assert lib.bb200_amcl_batch_cast_rays(batch._h, mask, None, nulls, n_bearings, ptrs, n_bearings, (C.c_double * k)(*[1.0] * k), ptrs) == INVALID
    assert batch.launch_count() == launches
    after = batch.export_members()
    assert [after[m] for m in range(8) if m not in (5, 6)] == [blobs[m] for m in range(8) if m not in (5, 6)]


def test_filter_refusals(bb):
    f = bb.Filter(capacity=16)
    with pytest.raises(bb.BelugaB200Error) as e:
        f.cast_rays(se2(0, 0, 0)[None], bearing(0.0)[None], 1.0)
    assert e.value.status == STATE
    f.set_beam_map(bb.BeamModelParam(), grid5(bb, [(2, 2)]))
    d = C.POINTER(C.c_double)
    buf = np.zeros(8)
    p = buf.ctypes.data_as(d)
    assert f._lib.bb200_filter_cast_rays(f._h, p, 1 << 62, p, 8, 1.0, p) == INVALID
    assert f._lib.bb200_filter_cast_rays(f._h, None, 1, p, 1, 1.0, p) == INVALID
    assert f._lib.bb200_filter_cast_rays(f._h, p, 1, p, 1, 1.0, None) == INVALID
    before = f.launch_count()
    assert f.cast_rays(np.zeros((0, 4)), bearing(0.0)[None], 1.0).shape == (0, 1)
    assert f.launch_count() == before
