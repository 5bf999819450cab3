"""The standalone clusterizer (cluster.cu, cluster_host.cpp) at the sizes a 1M-particle filter produces, against the
oracle and against the NumPy histogram of tests/test_cluster_scale_cpu.py.

The device path changes with the size of its input: the stable LSD radix sort runs max(1, ceil(bits(cells) / 8)) passes
(1 up to 256 cells, 2 up to 65 536, 3 up to 2^24, 4 above) and leaves its result in one of two buffer pairs by the parity
of that count; cell_record_warp keeps four gathers in flight per lane while 128 or more particles remain and finishes in a
remainder loop, and adds non-unit weights in one sequential chain; the host's cluster map rehashes while it fills when
there are more cells than n / 5, and is kept between calls on one thread.  Every one of those paths is taken here.

Histograms are compared bit for bit (first index, count, representative bytes, sequential weight sum, max_bin_weight);
cluster ids, cell and cluster counts exactly; mean and covariance within the rounding bound of estimate_tolerance."""
import math
import threading

import numpy as np
import pytest

from test_cluster_scale_cpu import histogram, spatial_hash

pytestmark = pytest.mark.gpu

N = 1_000_000
EPS = np.finfo(np.float64).eps
MOTION = (0.1, 0.05, 0.1, 0.05)
LFM = dict(max_obstacle_distance=2.0, max_laser_distance=100.0, z_hit=0.5, z_random=0.5, sigma_hit=0.2)
CLUSTER = dict(linear=0.2, angular=0.524, percentile=0.9)  # the clusterizer's defaults


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
    """bench.py's workload: the 2000 x 2000 map at 0.05 m (100 m x 100 m) and its 1080-beam scans."""
    from beluga_b200 import synthetic

    return synthetic.make_scenario(grid_size=2000, n_beams=1080, steps=100)


def same_bytes(a, b):
    return np.asarray(a, dtype=np.float64).tobytes() == np.asarray(b, dtype=np.float64).tobytes()


def sort_passes(cells):
    return max(1, -(-(cells - 1).bit_length() // 8))


def histogram_launches(passes):
    """Clusterizer::cell_records: cluster_cells_begin (3), cluster_sort (2 + 3 per pass), cluster_records (1).
    Filter.particle_histogram calls the C function twice: once for the bin count, once for the bins."""
    return 2 * (3 + (2 + 3 * passes) + 1)


def lattice_cloud(rng, counts, linear, angular, unit=False):
    """len(counts) occupied cells of spatial_hash{linear, linear, angular}, cell k holding counts[k] particles spread
    inside it, in shuffled particle order.  Cell k is (k mod 4096, k / 4096 mod 4096, k / 2^24) in x, y and heading, so
    neighbouring cells are adjacent and the first 2^24 cells share one heading bucket."""
    counts = np.asarray(counts, dtype=np.int64)
    cell = np.repeat(np.arange(len(counts)), counts)[rng.permutation(int(counts.sum()))]
    u = rng.uniform(0.05, 0.95, (len(cell), 3))
    th = ((cell >> 24) - 1 + u[:, 2]) * angular
    states = np.stack([np.cos(th), np.sin(th), ((cell & 4095) - 2048 + u[:, 0]) * linear, (((cell >> 12) & 4095) - 2048 + u[:, 1]) * linear], axis=1)
    weights = np.ones(len(cell)) if unit else rng.uniform(0.25, 4.0, len(cell))
    return states, weights


def check_histogram(f, states, weights, linear, angular):
    """Filter.particle_histogram against the NumPy histogram, bit for bit -> (bins, launches of the call)."""
    before = f.launch_count()
    rep, w, count, first, top = f.particle_histogram(linear, angular)
    launches = f.launch_count() - before
    want_first, want_count, want_w, _ = histogram(states, weights, linear, angular)
    assert np.array_equal(first, want_first)
    assert np.array_equal(count, want_count)
    assert same_bytes(rep, states[want_first])
    assert w.tobytes() == want_w.tobytes()
    assert top == max(1e-3, float(want_w.max()))  # beluga_ros/particle_cloud.hpp:197
    return len(first), launches


def estimate_tolerance(states, weights, ids):
    """How far two correct computations of the cluster estimate may lie apart.

    The oracle sums the selected cluster's terms one after another (mean of w/S * (cos, sin, x, y), then w/S * centred
    products); the device adds raw moments about a pivot in warp trees, per cell and then cell by cell on the host.
    Either way a sum of N terms carries at most (N + 2) eps sum|terms| of rounding (N - 1 additions, plus the products and
    the division by S), so the two results may differ by twice that.  The pivot is some point of the cloud's bounding
    box, so |x - pivot| <= |x| + max|x|.  The covariance is E[d d] - E[d] E[d] on the device and E[(x - m)(x - m)] in the
    oracle: both bounds are added, plus the error of E[d] times 2 |E[d]|.  The heading is (mc, ms) / |(mc, ms)|, whose
    error is that of (mc, ms) over the norm, which the oracle's cov[2, 2] = -2 log(norm) gives back.
    At 10^6 particles 50 m from the origin the bound on the position is about 1e-7 m (the 1e-9 of tests/test_gpu_cluster.py
    is not a bound there), and still a thousand times finer than one particle more or less in a cluster of 10^5."""
    ids = np.asarray(ids, dtype=np.int64)
    mass = np.bincount(ids, weights=weights)
    size = np.bincount(ids)
    eligible = np.where(size > 1, mass, -np.inf)
    sel = ids == int(np.argmax(eligible)) if np.isfinite(eligible.max()) else np.ones(len(ids), dtype=bool)
    w, s = weights[sel], states[sel]
    n, total = len(w), w.sum()
    g = 2.0 * (n + 3) * EPS  # two sides, each (n + 2) eps plus the subtraction's rounding
    x, y = s[:, 2], s[:, 3]
    ax, ay = np.abs(x) + np.abs(x).max(), np.abs(y) + np.abs(y).max()  # bounds of |x - pivot|, |y - pivot|
    mx, my = np.dot(w, x) / total, np.dot(w, y) / total
    cx, cy = np.abs(x - mx), np.abs(y - my)
    dmx, dmy = np.dot(w, ax) / total, np.dot(w, ay) / total
    corr = 1.0 - np.dot(w, w) / total**2
    mc, ms = np.dot(w, s[:, 0]) / total, np.dot(w, s[:, 1]) / total
    norm = max(math.hypot(mc, ms), EPS)
    tol_mean = np.array([2 * g / norm, 2 * g / norm, g * dmx, g * dmy])

    def tol_cov(a, b, ca, cb, da, db):
        return g * (np.dot(w, a * b) / total + np.dot(w, ca * cb) / total + 2 * da * db) / corr

    tol = np.zeros((3, 3))
    tol[0, 0] = tol_cov(ax, ax, cx, cx, dmx, dmx)
    tol[0, 1] = tol[1, 0] = tol_cov(ax, ay, cx, cy, dmx, dmy)
    tol[1, 1] = tol_cov(ay, ay, cy, cy, dmy, dmy)
    tol[2, 2] = 4 * g / norm
    return tol_mean, tol


def check_cluster(orc, got, states, weights, linear=0.2, angular=0.524, percentile=0.9):
    """Filter.cluster_estimate(with_ids=True) against orc.cluster_ids / orc.cluster_based_estimate."""
    mean, cov, ids, cells, clusters = got
    want_ids = orc.cluster_ids(states, weights, linear, angular, percentile)
    assert np.array_equal(ids.astype(np.uint64), want_ids)
    assert clusters == int(want_ids.max()) + 1
    assert cells == len(np.unique(spatial_hash(states, linear, linear, angular)))
    want_mean, want_cov = orc.cluster_based_estimate(states, weights, linear, angular, percentile)
    tol_mean, tol_cov = estimate_tolerance(states, weights, want_ids)
    assert np.all(np.abs(mean - want_mean) <= tol_mean), (mean - want_mean, tol_mean)
    finite = np.isfinite(want_cov)
    assert np.array_equal(np.isfinite(cov), finite)
    assert np.all(np.abs(cov - want_cov)[finite] <= tol_cov[finite]), (cov - want_cov, tol_cov)
    return cells, clusters


def fresh_thread(fn):
    """fn() on a new thread: select_cluster's per-thread map starts empty there, as on a filter's first call."""
    out = {}

    def run():
        try:
            out["value"] = fn()
        except BaseException as e:  # noqa: BLE001 -- re-raised on the caller's thread
            out["error"] = e

    t = threading.Thread(target=run)
    t.start()
    t.join()
    if "error" in out:
        raise out["error"]
    return out["value"]


# ---- 2. every radix pass count -------------------------------------------------------------------------------------
PASS_CELLS = [256, 257, 65_536, 65_537, 2**24, 2**24 + 1]


@pytest.mark.parametrize("cells", PASS_CELLS)
def test_histogram_at_every_radix_pass_boundary(bb, cells):
    """Exactly 256, 257, 65 536, 65 537, 2^24 and 2^24 + 1 occupied cells: 1, 2, 2, 3, 3 and 4 sort passes, so the sorted
    order is read from either buffer pair and every pass after the first reads the previous pass's indices.  Most cells
    hold one particle, 64 hold many, the weights are not unit."""
    rng = np.random.default_rng(cells)
    counts = np.ones(cells, dtype=np.int64)
    heavy = rng.choice(cells, size=min(cells, 64), replace=False)
    counts[heavy] += rng.multinomial(min(4 * cells, 2**20), np.full(len(heavy), 1.0 / len(heavy)))
    linear, angular = 0.05, 0.25
    states, weights = lattice_cloud(rng, counts, linear, angular)
    f = bb.Filter(capacity=len(states))
    f.set_particles(states, weights)
    bins, launches = check_histogram(f, states, weights, linear, angular)
    assert bins == cells
    assert sort_passes(cells) == {256: 1, 257: 2, 65_536: 2, 65_537: 3, 2**24: 3, 2**24 + 1: 4}[cells]
    assert launches == histogram_launches(sort_passes(cells))
    f.close()


# ---- 3. cell occupancy extremes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("unit", [True, False], ids=["unit", "weighted"])
def test_one_cell_holds_every_particle(bb, orc, unit):
    """10^6 particles in one cell: one warp gathers them all, four at a time, and with non-unit weights adds 10^6 weights
    in one chain that must be the reference's `entry.weight += weight` bit for bit."""
    rng = np.random.default_rng(1 + unit)
    states, weights = lattice_cloud(rng, [N], CLUSTER["linear"], CLUSTER["angular"], unit=unit)
    f = bb.Filter(capacity=N)
    f.set_particles(states, weights)
    bins, launches = check_histogram(f, states, weights, CLUSTER["linear"], CLUSTER["angular"])
    assert bins == 1 and launches == histogram_launches(1)
    assert check_cluster(orc, f.cluster_estimate(with_ids=True, **CLUSTER), states, weights) == (1, 1)


@pytest.mark.parametrize("unit", [True, False], ids=["unit", "weighted"])
def test_cells_either_side_of_the_four_gather_loop(bb, orc, unit):
    """Cells of 95, 96, 127, 128 and 129 particles (the four-gather loop runs while p + 96 < end: none, one or two rounds
    with a remainder of up to 32 per lane), and of 1, 31, 32, 33, 63, 64, 65 and 160, 161 for the remainder loop's edges."""
    rng = np.random.default_rng(7 + unit)
    sizes = np.array([95, 96, 127, 128, 129, 1, 31, 32, 33, 63, 64, 65, 160, 161])
    counts = np.repeat(sizes, 40)[rng.permutation(40 * len(sizes))]
    states, weights = lattice_cloud(rng, counts, CLUSTER["linear"], CLUSTER["angular"], unit=unit)
    f = bb.Filter(capacity=len(states))
    f.set_particles(states, weights)
    bins, _ = check_histogram(f, states, weights, CLUSTER["linear"], CLUSTER["angular"])
    assert bins == len(counts)
    check_cluster(orc, f.cluster_estimate(with_ids=True, **CLUSTER), states, weights)


@pytest.mark.parametrize("unit", [True, False], ids=["unit", "weighted"])
def test_one_huge_cell_among_singletons(bb, orc, unit):
    """9 x 10^5 particles in one cell and 10^5 cells of one particle each: one warp works through the huge cell while
    the others finish single particles."""
    rng = np.random.default_rng(11 + unit)
    counts = np.ones(100_001, dtype=np.int64)
    counts[rng.integers(0, len(counts))] = 900_000
    states, weights = lattice_cloud(rng, counts, CLUSTER["linear"], CLUSTER["angular"], unit=unit)
    f = bb.Filter(capacity=len(states))
    f.set_particles(states, weights)
    bins, launches = check_histogram(f, states, weights, CLUSTER["linear"], CLUSTER["angular"])
    assert bins == len(counts) and launches == histogram_launches(3)
    check_cluster(orc, f.cluster_estimate(with_ids=True, **CLUSTER), states, weights)


# ---- 4. the cluster estimate at 10^6 particles -----------------------------------------------------------------------
def test_cluster_estimate_of_a_global_localisation_cloud(bb, orc, scene):
    """initialize_uniform over the bench map's free cells: nearly every particle in a cell of its own, far more cells than
    n / 5, so the host map rehashes while it fills (as the reference's does)."""
    f = bb.Filter(capacity=N, seed=5)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    f.initialize_uniform(N)
    states, weights = f.particles()
    cells, clusters = check_cluster(orc, f.cluster_estimate(with_ids=True, **CLUSTER), states, weights)
    assert cells > N // 5 and clusters > 1000


def test_cluster_estimate_of_the_bench_posterior(bb, orc, scene):
    """bench.py's filter (10^6 particles, systematic resampling, seed 1) after three updates on its scans."""
    g = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION),
                bb.AmclParams(min_particles=N, max_particles=N, resample_scheme=bb.RESAMPLE_SYSTEMATIC, seed=1))
    g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    g.initialize(scene.initial_mean, scene.initial_cov)
    for k in range(3):
        assert g.update(bb.se2(*scene.poses[k]), scene.scans[k]).updated == 1
    states, weights = g.particles()
    assert np.all(weights == 1.0)
    check_cluster(orc, g.filter.cluster_estimate(with_ids=True, **CLUSTER), states, weights)


def test_cluster_estimate_of_a_lattice_of_65537_cells(bb, orc):
    """65 537 cells (three sort passes) filled to 10^6 particles, non-unit weights: neighbouring cells of different mean
    weight, so the flood stops at many borders."""
    rng = np.random.default_rng(65537)
    counts = 1 + rng.multinomial(N - 65_537, np.full(65_537, 1.0 / 65_537))
    states, weights = lattice_cloud(rng, counts, CLUSTER["linear"], CLUSTER["angular"])
    f = bb.Filter(capacity=N)
    f.set_particles(states, weights)
    cells, clusters = check_cluster(orc, f.cluster_estimate(with_ids=True, **CLUSTER), states, weights)
    assert cells == 65_537 and clusters > 1


# ---- 5. repeated calls on one filter ---------------------------------------------------------------------------------
def test_repeated_calls_on_one_filter_equal_a_fresh_filter(bb, orc):
    """Few cells, about 10^6 cells, few, many again, on one filter and one thread, unit weights (every cell weight ties,
    so the map's iteration order decides the heap order and with it the cluster ids).  The map kept between calls must
    behave as a fresh one: after the rehashing call it has more buckets than a freshly reserved map and has to be
    replaced.  Each call equals a fresh filter's on a fresh thread, byte for byte, and the oracle."""
    def few(seed):
        r = np.random.default_rng(seed)
        return lattice_cloud(r, 1 + r.multinomial(N - 40, np.full(40, 1.0 / 40)), CLUSTER["linear"], CLUSTER["angular"], unit=True)

    def many(seed):
        r = np.random.default_rng(seed)
        th = r.uniform(-math.pi, math.pi, N)
        return np.stack([np.cos(th), np.sin(th), r.uniform(0.0, 100.0, N), r.uniform(0.0, 100.0, N)], axis=1), np.ones(N)

    f = bb.Filter(capacity=N)
    for k, (states, weights) in enumerate([few(1), many(2), few(3), many(4)]):
        f.set_particles(states, weights)
        got_hist = f.particle_histogram(CLUSTER["linear"], CLUSTER["angular"])
        got = f.cluster_estimate(with_ids=True, **CLUSTER)

        def fresh(states=states, weights=weights):
            g = bb.Filter(capacity=N)
            g.set_particles(states, weights)
            return g.particle_histogram(CLUSTER["linear"], CLUSTER["angular"]), g.cluster_estimate(with_ids=True, **CLUSTER)

        want_hist, want = fresh_thread(fresh)
        for a, b in zip(got_hist, want_hist):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), k
        assert same_bytes(got[0], want[0]) and same_bytes(got[1], want[1]), k
        assert np.array_equal(got[2], want[2]) and got[3:] == want[3:], k
        cells, _ = check_cluster(orc, got, states, weights)
        assert (cells > N // 5) == (k % 2 == 1), (k, cells)


# ---- 6. pose samples at 10^6 -----------------------------------------------------------------------------------------
def test_sample_states_at_full_capacity(bb, orc, scene):
    """sample_states(1) and sample_states(capacity) draw the oracle's multinomial indices of that step, from the CDF the
    call builds, and again after a reweight has left the CDF stale; the particle set stays as it was."""
    rng = np.random.default_rng(6)
    seed = 13
    f = bb.Filter(capacity=N, seed=seed)
    f.set_likelihood_field_map(bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
    th = rng.uniform(-math.pi, math.pi, N)
    states = np.stack([np.cos(th), np.sin(th), rng.uniform(2.0, 98.0, N), rng.uniform(2.0, 98.0, N)], axis=1)
    weights = rng.uniform(0.0, 1.0, N) ** 4
    f.set_particles(states, weights)
    for phase in ("set", "reweighted"):
        if phase == "reweighted":
            f.reweight(scene.scans[0])
            st_now, weights = f.particles()
            assert np.array_equal(st_now, states) and not np.array_equal(weights, np.ones(N))
        for count, step in ((1, 0xFFFFFFFF), (N, 0xFFFFFFFE)):
            got = f.sample_states(count, step=step)
            idx, _, _ = orc.resample_indices(weights, orc.MULTINOMIAL, seed=seed, step=step, m=count)
            assert same_bytes(got, states[idx]), (phase, count)
            st_after, w_after = f.particles()
            assert same_bytes(st_after, states) and same_bytes(w_after, weights), (phase, count)


# ---- 7. shards -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shards", [2, 4])
def test_sharded_cluster_estimate_of_a_global_localisation_cloud(bb, scene, shards):
    """initialize_from_map on the bench map, one filter over 2 or 4 shards on one device and a single Amcl with the same
    seed: the global-index RNG makes the two sets identical.  Far more than 65 537 cells, and tens of thousands of them
    hold particles from both sides of a shard boundary, so their records are merged from per-shard parts.  Straight after
    initialisation and after one update, cells, clusters and estimate equal the single filter's."""
    ap = dict(min_particles=N, max_particles=N, seed=23, resample_scheme=bb.RESAMPLE_SYSTEMATIC)
    single = bb.Amcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap))
    group = bb.ShardedAmcl(bb.DifferentialDriveModelParam(*MOTION), bb.AmclParams(**ap), devices=[0] * shards)
    for g in (single, group):
        g.update_map(bb.SENSOR_LIKELIHOOD_FIELD, bb.LikelihoodFieldModelParam(**LFM), bb.OccupancyGrid(scene.cells, scene.resolution))
        g.initialize_from_map()
    for stage in ("initialised", "updated"):
        if stage == "updated":
            pose = bb.se2(*scene.poses[0])
            assert single.update(pose, scene.scans[0]).updated == 1 and group.update(pose, scene.scans[0]).updated == 1
        ss, sw = single.particles()
        gs, gw = group.particles()
        assert same_bytes(ss, gs) and same_bytes(sw, gw) and np.all(sw == 1.0), stage
        hashes = spatial_hash(ss, CLUSTER["linear"], CLUSTER["linear"], CLUSTER["angular"])
        shard_of = np.arange(N) // (N // shards)
        _, inverse = np.unique(hashes, return_inverse=True)
        lo = np.full(inverse.max() + 1, shards)
        hi = np.full(inverse.max() + 1, -1)
        np.minimum.at(lo, inverse, shard_of)
        np.maximum.at(hi, inverse, shard_of)
        straddling, multi = (lo != hi).sum(), (np.bincount(inverse) > 1).sum()
        if stage == "initialised":  # independent draws by global index: about half or more of the shared cells straddle
            assert len(lo) > N // 5 and straddling > 0.4 * multi
        else:  # the resample keeps an ancestor's copies at adjacent indices: fewer, but still tens of thousands
            assert straddling > 20_000
        for kw in (CLUSTER, dict(linear=0.05, angular=0.1, percentile=0.5)):
            ms, cs, _, cells_s, clusters_s = single.filter.cluster_estimate(with_ids=True, **kw)
            mg, cg, cells_g, clusters_g = group.cluster_estimate(**kw)
            assert (cells_g, clusters_g) == (cells_s, clusters_s), (stage, kw)
            assert np.abs(ms - mg).max() < 1e-12 and np.abs(cs - cg).max() < 1e-12, (stage, kw, ms - mg, cs - cg)
