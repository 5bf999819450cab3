"""A sharded filter through the whole beluga_ros node cycle (bb200_sharded_amcl_update_scan / _update_point_cloud /
_particle_histogram / _sample_states / _cast_rays), with all shards on ONE device as in tests/test_gpu_sharded_local.py.  Each
case runs twins: a single Amcl with the same parameters and seed, and where it applies the host conversion followed by
bb200_sharded_amcl_update.  Particle sets, histogram bins, pose samples and ray casts are compared byte for byte, and so are
the update results of the two sharded filters.  Two things add per shard and are compared to rounding: the estimate of a
step (against the single filter, whose decisions, counts and normalisation factor are still equal bit for bit) and the
raw moments of a histogram cell whose particles lie in several shards."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _raycast_oracle  # noqa: E402
from test_cluster_scale_cpu import histogram, spatial_hash  # noqa: E402

pytestmark = pytest.mark.gpu

MOTION = (0.1, 0.05, 0.1, 0.05)
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
INVALID, STATE, CAPACITY = -1, -4, -5
N = 12_000  # divisible by 1, 2, 3, 4 and 8
SHARDS = [1, 2, 3, 4, 8]
STEPPING = [2, 3, 4, 8]  # a filter of one shard refuses to step (bb200_sharded_amcl_update: "this shard has not joined its peers")
SENSORS = {"likelihood-field": 0, "beam": 2}
CELL = np.dtype([("rep", "<f8", 4), ("hash", "<u8"), ("first", "<u4"), ("count", "<u4"), ("weight", "<f8"), ("m", "<f8", 9)])


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

    return synthetic.make_scenario(grid_size=200, n_beams=181, steps=12)


def sensor_params(bb, sensor):
    return bb.BeamModelParam(beam_max_range=20.0) if sensor == bb.SENSOR_BEAM else bb.LikelihoodFieldModelParam(**LFM)


def make_twins(bb, scene, shards, sensor=0, n=N, init="normal", **kw):
    """(sharded filter, single Amcl) with the same parameters, map and initial particles."""
    ap = dict(min_particles=n, max_particles=n, seed=41, **kw)
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap), devices=[0] * shards)
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    for f in (single, group):
        f.update_map(sensor, sensor_params(bb, sensor), grid)
        if init == "normal":
            f.initialize(scene.initial_mean, scene.initial_cov)
        else:
            f.initialize_from_map()
    return group, single


def same_bytes(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def same_result(a, b):
    return bytes(a) == bytes(b)


def same_step(a, b):
    """Sharded and single results: the same decisions, count and normalisation factor, bit for bit (the estimates sum the
    same terms grouped per shard, see tests/test_gpu_sharded_local.py)."""
    return (a.updated, a.resampled, a.n_particles, a.weight_sum) == (b.updated, b.resampled, b.n_particles, b.weight_sum)


def same_particles(x, y):
    (sx, wx), (sy, wy) = x.particles(), y.particles()
    return same_bytes(sx, sy) and same_bytes(wx, wy)


# ---- measurements -------------------------------------------------------------------------------------------------------
ORIGIN = np.array([0.0, -1.0, 0.0, 0.12, 1.0, 0.0, 0.0, -0.05, 0.0, 0.0, 1.0, 0.3])  # yaw 90 deg, shifted, lifted


def scan_of(scene, k):
    """The scenario's step-k scan as a laser scan, with NaN and out-of-range readings."""
    pts = scene.scans[k]
    ranges = np.hypot(pts[:, 0], pts[:, 1]).astype(np.float32)
    ranges[5::17] = np.nan
    ranges[7::23] = 100.0  # beyond max_range
    ranges[11::29] = 0.01  # below min_range
    n = len(ranges)
    return ranges, float(np.float32(-math.pi)), float(np.float32(2 * math.pi / n))


def cloud_of(scene, k, dtype):
    """The scenario's step-k points as a padded PointCloud2 buffer (x at byte 4, one pad scalar after z)."""
    pts = scene.scans[k]
    rec = np.zeros((len(pts), 5), dtype=dtype)
    rec[:, 1:3] = pts
    rec[:, 3] = 0.25
    rec[3::31, 1] = np.nan
    return rec, rec.itemsize * 5, rec.itemsize


def measurement(bb, scene, k):
    """Step k's measurement: scans and clouds alternate, with max_beams, a laser origin and both point types."""
    if k % 2 == 0:
        ranges, amin, ainc = scan_of(scene, k)
        kw = dict(min_range=0.05, max_range=18.0, max_beams=60 if k % 4 == 2 else 0, laser_origin=ORIGIN if k % 4 == 2 else None)
        return "scan", (ranges, amin, ainc), kw, bb.scan_to_points(ranges, amin, ainc, **kw)
    data, step, xoff = cloud_of(scene, k, np.float32 if k % 4 == 1 else np.float64)
    kw = dict(origin=ORIGIN if k % 4 == 3 else None)
    return "cloud", (data, step, xoff, data.dtype), kw, bb.point_cloud_to_points(data, step, xoff, data.dtype, **kw)


def step(f, kind, args, kw, control):
    return f.update_scan(control, *args, **kw) if kind == "scan" else f.update_point_cloud(control, *args, **kw)


@pytest.mark.parametrize("sensor", sorted(SENSORS))
@pytest.mark.parametrize("shards", STEPPING)
def test_scans_and_clouds_follow_the_twins(bb, scene, shards, sensor):
    """Ten steps of update_scan / update_point_cloud equal, byte for byte, the host conversion + update on another sharded
    filter and the single filter's update_scan / update_point_cloud."""
    group, single = make_twins(bb, scene, shards, SENSORS[sensor], resample_scheme=0)
    points, _ = make_twins(bb, scene, shards, SENSORS[sensor], resample_scheme=0)
    for k in range(10):
        control = bb.se2(*scene.poses[k])
        kind, args, kw, pts = measurement(bb, scene, k)
        rg, rs, rp = step(group, kind, args, kw, control), step(single, kind, args, kw, control), points.update(control, pts)
        assert rg.updated == 1
        assert same_result(rg, rp), f"step {k} ({kind}): the sharded conversion differs from the host conversion"
        assert same_step(rg, rs)
        assert same_particles(group, points) and same_particles(group, single), f"step {k} ({kind})"


def test_one_shard_refuses_scans_and_clouds_as_it_refuses_points(bb, scene):
    group, _ = make_twins(bb, scene, 1)
    before = group.particles()
    control = bb.se2(*scene.poses[0])
    statuses = set()
    for k in range(2):
        kind, args, kw, pts = measurement(bb, scene, k)
        for call in (lambda: step(group, kind, args, kw, control), lambda: group.update(control, pts)):
            with pytest.raises(bb.BelugaB200Error) as e:
                call()
            statuses.add(e.value.status)
    assert statuses == {STATE}
    assert same_bytes(group.particles()[0], before[0])


def test_refusals_leave_the_filter_unchanged(bb, scene):
    from beluga_b200 import _capi

    group, single = make_twins(bb, scene, 4)
    lib = _capi.load()
    d = C.POINTER(C.c_double)
    control = bb.se2(*scene.poses[0])
    pose = control.ctypes.data_as(d)
    res = _capi.UpdateResult()
    before = group.particles()
    ranges = np.ones(10, np.float32)
    good_scan = _capi.LaserScan(ranges.ctypes.data_as(C.POINTER(C.c_float)), 10, 0.0, 0.1, 0.0, 10.0, 0, None)
    no_ranges = _capi.LaserScan(None, 10, 0.0, 0.1, 0.0, 10.0, 0, None)
    data = np.zeros((4, 3), np.float32)
    clouds = [_capi.PointCloud(data.ctypes.data, 4, 12, 0, 2, None),     # not FLOAT32 / FLOAT64
              _capi.PointCloud(data.ctypes.data, 4, 8, 0, 7, None),      # z does not fit in point_step
              _capi.PointCloud(data.ctypes.data, 4, 12, 4, 7, None),     # x_offset pushes z out
              _capi.PointCloud(None, 4, 12, 0, 7, None)]                 # no data
    h, a = group._h, single._h
    cases = [(lib.bb200_sharded_amcl_update_scan, lib.bb200_amcl_update_scan, (pose, C.byref(no_ranges), C.byref(res))),
             (lib.bb200_sharded_amcl_update_scan, lib.bb200_amcl_update_scan, (None, C.byref(good_scan), C.byref(res))),
             (lib.bb200_sharded_amcl_update_scan, lib.bb200_amcl_update_scan, (pose, None, C.byref(res))),
             (lib.bb200_sharded_amcl_update_scan, lib.bb200_amcl_update_scan, (pose, C.byref(good_scan), None)),
             (lib.bb200_sharded_amcl_update_point_cloud, lib.bb200_amcl_update_point_cloud, (pose, None, C.byref(res)))]
    cases += [(lib.bb200_sharded_amcl_update_point_cloud, lib.bb200_amcl_update_point_cloud, (pose, C.byref(c), C.byref(res))) for c in clouds]
    for sharded_call, single_call, args in cases:
        st_single, st_sharded = single_call(a, *args), sharded_call(h, *args)
        assert st_single == st_sharded == INVALID
        assert same_bytes(group.particles()[0], before[0]) and same_bytes(group.particles()[1], before[1])
    # neither the particles nor the policies moved: the next step still equals the twin's
    kind, args, kw, _ = measurement(bb, scene, 2)
    assert same_step(step(group, kind, args, kw, control), step(single, kind, args, kw, control))
    assert same_particles(group, single)


# ---- histogram ------------------------------------------------------------------------------------------------------------
def cells_ptr(arr):
    from beluga_b200 import _capi

    return arr.ctypes.data_as(C.POINTER(_capi.ClusterCell))


def raw_bins(call, handle, linear, angular):
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert call(handle, linear, angular, None, 0, C.byref(n), C.byref(top)) == 0
    arr = np.zeros(max(n.value, 1), CELL)
    assert call(handle, linear, angular, cells_ptr(arr), n.value, C.byref(n), C.byref(top)) == 0
    return arr[: n.value], top.value


def sharded_bins(group, linear, angular):
    from beluga_b200 import _capi

    return raw_bins(_capi.load().bb200_sharded_amcl_particle_histogram, group._h, linear, angular)


def single_bins(single, linear, angular):
    from beluga_b200 import _capi

    return raw_bins(_capi.load().bb200_filter_particle_histogram, single.filter._h, linear, angular)


def spanning_hashes(group, linear, angular):
    """Hashes of the cells whose particles lie in more than one shard."""
    seen = {}
    for f in group.shards:
        states, _ = f.particles()
        for h in np.unique(spatial_hash(states, linear, linear, angular)):
            seen[int(h)] = seen.get(int(h), 0) + 1
    return {h for h, c in seen.items() if c > 1}


def check_cells(got, want, unit):
    for field in ("rep", "hash", "first", "count"):
        assert same_bytes(got[field], want[field]), field
    if unit:
        assert same_bytes(got["weight"], want["weight"])
    scale = np.maximum(1.0, np.abs(want["m"])).max()
    assert np.abs(got["m"] - want["m"]).max() <= 1e-12 * scale * max(1, int(want["count"].max()))


@pytest.mark.parametrize("sensor", sorted(SENSORS))
@pytest.mark.parametrize("shards", SHARDS)
def test_histogram_equals_the_single_filter(bb, scene, shards, sensor):
    """After initialize_from_map and after a resampling step (unit weights) the bins equal the single filter's: every field
    byte for byte, and the raw moments of a cell inside one shard too (both filters accumulate about the map centre after
    initialize_from_map); a cell across shards adds its moments shard by shard."""
    group, single = make_twins(bb, scene, shards, SENSORS[sensor], init="map", resample_scheme=1)
    for phase in ("initialized", "resampled") if shards in STEPPING else ("initialized",):
        if phase == "resampled":
            control = bb.se2(*scene.poses[0])
            assert group.update(control, scene.scans[0]).resampled == single.update(control, scene.scans[0]).resampled == 1
        for linear, angular in ((1e-3, 1e-3), (0.2, 0.524)):
            got, top_g = sharded_bins(group, linear, angular)
            want, top_s = single_bins(single, linear, angular)
            assert len(got) == len(want) and top_g == top_s
            check_cells(got, want, unit=True)
            if phase == "initialized":
                inside = ~np.isin(want["hash"], np.array(sorted(spanning_hashes(group, linear, angular)), dtype=np.uint64))
                assert same_bytes(got["m"][inside], want["m"][inside])
            rep, w, count, first, top = group.particle_histogram(linear, angular)
            assert same_bytes(rep, got["rep"]) and same_bytes(w, got["weight"]) and same_bytes(count, got["count"]) and top == top_g


@pytest.mark.parametrize("shards", [2, 3, 8])
def test_histogram_of_normalised_weights_sums_shard_by_shard(bb, scene, shards):
    """After a step that normalises without resampling, cells, counts and representatives equal the single filter's; a
    cell's weight is each shard's sequential sum, added in rank order."""
    group, single = make_twins(bb, scene, shards, resample_interval=2, resample_scheme=1)
    control = bb.se2(*scene.poses[0])
    assert group.update(control, scene.scans[0]).resampled == single.update(control, scene.scans[0]).resampled == 0
    linear, angular = 0.2, 0.524
    got, top = sharded_bins(group, linear, angular)
    want, _ = single_bins(single, linear, angular)
    check_cells(got, want, unit=False)
    expected = {}
    for f in group.shards:  # rank order
        states, weights = f.particles()
        first, _, weight, _ = histogram(states, weights, linear, angular)
        for h, w in zip(spatial_hash(states[first], linear, linear, angular), weight):
            expected[int(h)] = expected[int(h)] + w if int(h) in expected else w
    assert same_bytes(got["weight"], np.array([expected[int(h)] for h in got["hash"]]))
    assert top == max(1e-3, got["weight"].max())


def test_histogram_capacity_and_count_query(bb, scene):
    from beluga_b200 import _capi

    lib = _capi.load()
    group, _ = make_twins(bb, scene, 4)
    n, top = C.c_uint64(0), C.c_double(0.0)
    assert lib.bb200_sharded_amcl_particle_histogram(group._h, 0.2, 0.524, None, 0, C.byref(n), C.byref(top)) == 0
    assert n.value > 1 and top.value >= 1e-3
    small = np.zeros(n.value - 1, CELL)
    m = C.c_uint64(0)
    assert lib.bb200_sharded_amcl_particle_histogram(group._h, 0.2, 0.524, cells_ptr(small), len(small), C.byref(m), None) == CAPACITY
    assert m.value == n.value
    assert lib.bb200_sharded_amcl_particle_histogram(group._h, 0.0, 0.524, None, 0, C.byref(m), None) == INVALID
    empty = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=N, max_particles=N), devices=[0, 0])
    assert lib.bb200_sharded_amcl_particle_histogram(empty._h, 0.2, 0.524, None, 0, C.byref(m), None) == STATE


# ---- pose samples ---------------------------------------------------------------------------------------------------------
COUNTS = (1, N // 2 + 1, N)  # N // 2 + 1 is not a multiple of 2, 3, 4 or 8


def check_samples(group, single, tag):
    before = group.particles()
    for count, stp in zip(COUNTS, (0xFFFFFFFF, 0xFFFFFFF0, 77)):
        got = group.sample_states(count, step=stp)
        assert same_bytes(got, single.filter.sample_states(count, step=stp)), (tag, count)
        after = group.particles()
        assert same_bytes(after[0], before[0]) and same_bytes(after[1], before[1]), (tag, count)


@pytest.mark.parametrize("sensor", sorted(SENSORS))
@pytest.mark.parametrize("shards", SHARDS)
def test_samples_equal_the_single_filter(bb, scene, shards, sensor):
    """After initialisation, after a resampling step and after a step that keeps its particles (current CDF); a following
    update still equals the twin's."""
    group, single = make_twins(bb, scene, shards, SENSORS[sensor], resample_interval=2, resample_scheme=0)
    check_samples(group, single, "initialized")
    if shards not in STEPPING:
        return
    for k, tag in ((0, "normalized"), (1, "resampled")):
        control = bb.se2(*scene.poses[k])
        rg, rs = group.update(control, scene.scans[k]), single.update(control, scene.scans[k])
        assert same_step(rg, rs) and rg.resampled == (tag == "resampled")
        check_samples(group, single, tag)
    control = bb.se2(*scene.poses[2])
    assert same_step(group.update(control, scene.scans[2]), single.update(control, scene.scans[2]))
    assert same_particles(group, single)


@pytest.mark.parametrize("shards", [2, 3, 4, 8])
def test_samples_use_the_global_exponent(bb, orc, scene, shards):
    """Weights whose largest value sits in the last shard: a CDF quantised with each shard's own exponent would draw other
    particles.  The draws are the oracle's multinomial indices over the global weights."""
    rng = np.random.default_rng(shards)
    th = rng.uniform(-math.pi, math.pi, N)
    states = np.stack([np.cos(th), np.sin(th), rng.uniform(2.0, 8.0, N), rng.uniform(2.0, 8.0, N)], axis=1)
    weights = rng.uniform(0.0, 1.0, N) ** 6 * 1e-3
    weights[N - 5] = 0.75  # the heaviest particle, in the last shard
    group, single = make_twins(bb, scene, shards)
    single.initialize_states(states, weights)
    shard = N // shards
    for r, f in enumerate(group.shards):
        f.set_particles(states[r * shard:(r + 1) * shard], weights[r * shard:(r + 1) * shard])
    for count, stp in zip(COUNTS, (5, 0xFFFFFFFE, 9)):
        got = group.sample_states(count, step=stp)
        assert same_bytes(got, single.filter.sample_states(count, step=stp)), count
        idx, _, _ = orc.resample_indices(weights, orc.MULTINOMIAL, seed=41, step=stp, m=count)
        assert same_bytes(got, states[idx]), count


@pytest.mark.parametrize("shards", [4, 8])
def test_samples_over_more_slots_than_a_shard_holds(bb, scene, shards):
    """count = max_particles = 400 000 over shards of 100 000 or 50 000: every shard's draw walks all 400 000 global slots,
    more resample blocks than a launch over its own capacity has, after initialisation and after a step that keeps its
    particles (current CDF)."""
    n = 400_000
    group, single = make_twins(bb, scene, shards, n=n, resample_interval=2, resample_scheme=0)
    for phase in ("initialized", "normalized"):
        if phase == "normalized":
            control = bb.se2(*scene.poses[0])
            assert same_step(group.update(control, scene.scans[0]), single.update(control, scene.scans[0]))
        before = group.particles()
        for count, stp in ((n, 0xFFFFFFFF), (n - 1, 3)):
            assert same_bytes(group.sample_states(count, step=stp), single.filter.sample_states(count, step=stp)), (phase, count)
        after = group.particles()
        assert same_bytes(after[0], before[0]) and same_bytes(after[1], before[1])


@pytest.mark.parametrize("shards", [2, 4])
def test_samples_rebuild_cdfs_built_shard_by_shard(bb, scene, shards):
    """CDFs that each shard built with its own exponent (bb200_filter_build_cdf on the shard's handle) are current but are no
    global CDF: the sharded call rebuilds it and still draws the single filter's samples."""
    rng = np.random.default_rng(10 + shards)
    th = rng.uniform(-math.pi, math.pi, N)
    states = np.stack([np.cos(th), np.sin(th), rng.uniform(2.0, 8.0, N), rng.uniform(2.0, 8.0, N)], axis=1)
    weights = rng.uniform(0.0, 1.0, N) ** 6 * 1e-4
    weights[N - 3] = 0.9  # the last shard's largest weight is far above the others'
    group, single = make_twins(bb, scene, shards)
    single.initialize_states(states, weights)
    shard = N // shards
    exponents = set()
    for r, f in enumerate(group.shards):
        f.set_particles(states[r * shard:(r + 1) * shard], weights[r * shard:(r + 1) * shard])
        exponents.add(f.build_cdf()[1])  # this shard's own exponent
    assert len(exponents) > 1
    for count, stp in ((N, 21), (N // 2 + 1, 22)):
        assert same_bytes(group.sample_states(count, step=stp), single.filter.sample_states(count, step=stp)), count


def test_sample_refusals(bb, scene):
    from beluga_b200 import _capi

    lib = _capi.load()
    empty = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=N, max_particles=N), devices=[0, 0, 0])
    out = np.zeros((N + 1, 4))
    d = out.ctypes.data_as(C.POINTER(C.c_double))
    assert lib.bb200_sharded_amcl_sample_states(empty._h, 1, 0, d) == STATE
    group, _ = make_twins(bb, scene, 3)
    assert lib.bb200_sharded_amcl_sample_states(group._h, N + 1, 0, d) == CAPACITY
    assert lib.bb200_sharded_amcl_sample_states(group._h, 1, 0, None) == INVALID
    assert lib.bb200_sharded_amcl_sample_states(group._h, 0, 0, None) == 0


# ---- ray casts ------------------------------------------------------------------------------------------------------------
def rays(scene, n_poses, n_bearings, seed):
    rng = np.random.default_rng(seed)
    extent = scene.cells.shape[1] * scene.resolution
    th = rng.uniform(-math.pi, math.pi, n_poses)
    poses = np.stack([np.cos(th), np.sin(th), rng.uniform(-2.0, extent + 2.0, n_poses), rng.uniform(-2.0, extent + 2.0, n_poses)], axis=1)
    poses[::13, 2] = -7.5  # outside the grid
    a = np.linspace(-math.pi, math.pi, n_bearings, endpoint=False)
    return poses, np.stack([np.cos(a), np.sin(a)], axis=1)


@pytest.mark.parametrize("sensor", sorted(SENSORS))
@pytest.mark.parametrize("shards", SHARDS)
def test_ray_casts_equal_the_filter_and_the_oracle(bb, scene, shards, sensor):
    group, single = make_twins(bb, scene, shards, SENSORS[sensor])
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    poses, bearings = rays(scene, 97, 37, shards)
    before = group.particles()
    for max_range in (4.0, 30.0, float("nan")):
        got = group.cast_rays(poses, bearings, max_range)
        assert np.array_equal(got, single.cast_rays(poses, bearings, max_range))
        assert np.array_equal(got, _raycast_oracle.cast_rays(grid.cells, grid.resolution, grid.origin, poses, bearings, max_range))
    # fewer poses than shards, and no rays at all
    assert np.array_equal(group.cast_rays(poses[:1], bearings, 9.0), single.cast_rays(poses[:1], bearings, 9.0))
    assert group.cast_rays(poses[:0], bearings, 9.0).shape == (0, len(bearings))
    assert group.cast_rays(poses, bearings[:0], 9.0).shape == (len(poses), 0)
    assert same_particles(group, single) and same_bytes(group.particles()[0], before[0])


def test_ray_cast_refusals(bb, scene):
    from beluga_b200 import _capi

    lib = _capi.load()
    d = C.POINTER(C.c_double)
    buf = np.zeros(8)
    p = buf.ctypes.data_as(d)
    nomap = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(min_particles=N, max_particles=N), devices=[0, 0])
    assert lib.bb200_sharded_amcl_cast_rays(nomap._h, p, 1, p, 1, 1.0, p) == STATE
    group, single = make_twins(bb, scene, 2)
    for args in ((None, 1, p, 1, 1.0, p), (p, 1, None, 1, 1.0, p), (p, 1, p, 1, 1.0, None), (p, 1 << 40, p, 1 << 40, 1.0, p)):
        assert lib.bb200_sharded_amcl_cast_rays(group._h, *args) == lib.bb200_filter_cast_rays(single.filter._h, *args) == INVALID
    assert lib.bb200_sharded_amcl_cast_rays(group._h, p, 1 << 30, p, 1 << 20, 1.0, p) == CAPACITY
    assert lib.bb200_sharded_amcl_cast_rays(group._h, None, 0, None, 0, 1.0, None) == 0


# ---- two devices ----------------------------------------------------------------------------------------------------------
def test_two_devices(bb, scene):
    """One scan step, one histogram, one sample and one cast on shards spread over two GPUs."""
    if bb.device_count() < 2:
        pytest.skip("needs two devices")
    n = 4000
    ap = dict(min_particles=n, max_particles=n, seed=3, resample_scheme=0)
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap), devices=[0, 1])
    grid = bb.OccupancyGrid(scene.cells, scene.resolution)
    for f in (single, group):
        f.update_map(0, bb.LikelihoodFieldModelParam(**LFM), grid)
        f.initialize(scene.initial_mean, scene.initial_cov)
    kind, args, kw, _ = measurement(bb, scene, 0)
    control = bb.se2(*scene.poses[0])
    assert same_step(step(group, kind, args, kw, control), step(single, kind, args, kw, control))
    assert same_particles(group, single)
    got, _ = sharded_bins(group, 0.2, 0.524)
    want, _ = single_bins(single, 0.2, 0.524)
    check_cells(got, want, unit=True)
    assert same_bytes(group.sample_states(n, step=11), single.filter.sample_states(n, step=11))
    poses, bearings = rays(scene, 33, 19, 2)
    assert np.array_equal(group.cast_rays(poses, bearings, 12.0), single.cast_rays(poses, bearings, 12.0))
